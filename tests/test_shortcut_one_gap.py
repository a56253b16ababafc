"""CPU: the one-gap check of the exact extension shortcut (gapless_job_shortcut, pipeline_core.cuh).  A job whose seed-diagonal segment T
lies within min(2 o, o + match - mismatch) of match * M (o = the smaller gap-open magnitude) is claimed only when no pair of band
diagonals can carry a one-gap alignment reaching T.  Every claimed job must have the (score, sink) of the oracle's banded DP (and of the
reference's own aln::banded_alignment_score<BAND> where oracle/_ref is built, bands 31 and 15); the rule without the check must claim a
subset of it with the same results.  The host build (tests/host/shortcut_harness.cu) runs the routine with the check on and off.

Cases built to break the bound: two substitutions at every spacing, three or four with some in the clip rows, a 1-2 base indel a few
rows from either end (the gapless diagonal then shows one or two differences and a one-gap alignment is perfect) with the seed's diagonal
on either side of it, indels and substitutions inside homopolymers and period-2 / 3 / 7 repeats, ragged and short reads, windows longer
than needed and too short; bands 31, 15 and 8, four schemes."""
import ctypes as C
import os
import subprocess
import numpy as np
import pytest
from oracle import orc
from nvbio_b200.strings import pack_symbols

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "host", "libshortcut_harness.so")
SRC = os.path.join(HERE, "host", "shortcut_harness.cu")
SCHEMES = ((2, -2, -5, -3), (1, -4, -6, -1), (2, -6, -8, -3), (3, -1, -2, -2))
STRIDE = 160


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


@pytest.fixture(scope="module")
def H():
    deps = [SRC] + [os.path.join(HERE, "..", "nvbio_b200", "csrc", f) for f in ("fm_core.cuh", "pipeline_core.cuh", "common.cuh")]
    if not os.path.exists(SO) or any(os.path.getmtime(d) > os.path.getmtime(SO) for d in deps):
        from nvbio_b200.build import NVCC
        subprocess.check_call([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17",
                               "-Wno-deprecated-declarations", "-Xcompiler", "-fPIC", "-shared", "-o", SO, SRC])
    return C.CDLL(SO)


@pytest.fixture(scope="module")
def O():
    return orc.Oracle()


@pytest.fixture(scope="module")
def R():
    return orc.Ref() if orc.Ref.available() else None


def one_gap_limit(scheme):
    """delta = match * M - T below which the rule with the check claims (and below o without it)"""
    m, s, go = scheme[0], scheme[1], scheme[2]
    o = -go
    return min(2 * o, o + m - s), o


def mutate(r, q, rng):
    r[q] = (r[q] + 1 + rng.integers(0, 3, np.size(q))) % 4


class Jobs:
    """reads with the seed's diagonal at text position pos (window begins band // 2 earlier), windows `extra` symbols longer than the band
    needs (negative: too short)"""

    def __init__(self, text, band):
        self.text, self.band = text, band
        self.reads, self.pos, self.extra, self.label = [], [], [], []

    def add(self, read, pos, label, extra=0):
        assert pos >= 32 and pos + len(read) + self.band + 16 < len(self.text)
        self.reads.append(np.asarray(read, np.uint8)); self.pos.append(pos); self.extra.append(extra); self.label.append(label)

    def arrays(self):
        n = len(self.reads)
        M = np.array([len(r) for r in self.reads], np.uint32)
        flat = np.zeros((n, STRIDE), np.uint8)
        for a, r in enumerate(self.reads):
            flat[a, :len(r)] = r
        to = (np.array(self.pos) - self.band // 2).astype(np.uint32)
        N = (M.astype(np.int64) + self.band - 1 + np.array(self.extra)).astype(np.uint32)
        po = (np.arange(n) * STRIDE).astype(np.uint32)
        return flat.reshape(-1), po, M, to, N


def shortcut(H, J, scheme, one_gap):
    flat, po, M, to, N = J.arrays()
    n = len(po)
    sw = np.concatenate([pack_symbols(flat, 2, True), np.zeros(2, np.uint32)])
    gw = np.concatenate([pack_symbols(np.concatenate([J.text, np.zeros(64, np.uint8)]), 2, True), np.zeros(2, np.uint32)])
    solved = np.zeros(n, np.uint8); score = np.zeros(n, np.int32); sink = np.zeros((n, 2), np.uint32)
    H.hs_gapless_job_shortcut(_p(sw), _p(gw), _p(po), _p(M), _p(to), _p(N), C.c_uint32(n), C.c_uint32(J.band), C.c_int32(scheme[0]),
                              C.c_int32(scheme[1]), C.c_int32(scheme[2]), C.c_int(1 if one_gap else 0), _p(solved), _p(score), _p(sink))
    return solved.astype(bool), score, sink


def check(H, O, R, J, scheme):
    """both rules against the DP; returns (claimed with the check, claimed without it)"""
    flat, po, M, to, N = J.arrays()
    ws, wx, wy, _ = O.banded_gotoh(J.band, 1, scheme, flat, po, M, J.text, to, N)
    new, sc, sk = shortcut(H, J, scheme, True)
    old, osc, osk = shortcut(H, J, scheme, False)
    bad = np.flatnonzero(new & ((sc != ws) | (sk[:, 0] != wx) | (sk[:, 1] != wy)))
    assert len(bad) == 0, [(J.label[a], int(sc[a]), int(ws[a]), tuple(sk[a]), (int(wx[a]), int(wy[a]))) for a in bad[:5]]
    assert not new[N < M + J.band - 1].any()
    assert not (old & ~new).any(), "the rule without the check claims a job the rule with it does not"
    assert np.array_equal(sc[old], osc[old]) and np.array_equal(sk[old], osk[old])
    if R is not None and J.band in (31, 15):
        full = N >= M + J.band - 1
        rs, rx, ry, _ = R.banded_gotoh(J.band, 1, scheme, flat, po, M, J.text, to, N)
        assert np.array_equal(rs[full], ws[full]) and np.array_equal(rx[full], wx[full]) and np.array_equal(ry[full], wy[full])
    return new, old


def random_text(rng, n=400_000, repeats=False):
    text = rng.integers(0, 4, n).astype(np.uint8)
    if repeats:
        for st, period in ((20_000, 1), (40_000, 2), (60_000, 3), (80_000, 7)):
            text[st:st + 3_000] = np.tile(text[st:st + period], 3_000 // period + 1)[:3_000]
    return text


def indel_read(text, p, M, cut, L, insert, rng):
    """the M symbols at text position p with L symbols deleted after read row cut - 1 (insert: L random symbols inserted there instead)"""
    if insert:
        return np.concatenate([text[p:p + cut], rng.integers(0, 4, L).astype(np.uint8), text[p + cut:p + M - L]])
    return np.concatenate([text[p:p + cut], text[p + cut + L:p + M + L]])


@pytest.mark.parametrize("band", [31, 15, 8])
@pytest.mark.parametrize("scheme", SCHEMES)
def test_two_substitutions_every_spacing(H, O, R, band, scheme):
    """every pair of rows (adjacent, at and next to both ends); reads with exactly two interior substitutions on random text are all
    claimed whenever their delta lies in the claimed region"""
    rng = np.random.default_rng(band * 7 + scheme[0])
    text = random_text(rng)
    M = 150
    J = Jobs(text, band)
    pairs = [(p, q) for p in range(M) for q in range(p + 1, M)]
    for p, q in pairs:
        pos = int(rng.integers(64, len(text) - 400))
        r = text[pos:pos + M].copy()
        mutate(r, np.array([p, q]), rng)
        J.add(r, pos, (p, q))
    new, old = check(H, O, R, J, scheme)
    lim, o = one_gap_limit(scheme)
    m, s = scheme[0], scheme[1]
    interior = np.array([16 <= p and q <= M - 17 for p, q in pairs])
    if 2 * (m - s) < lim:
        assert new[interior].all(), [pairs[a] for a in np.flatnonzero(interior & ~new)[:5]]
    if 2 * (m - s) >= o:
        assert not old[interior].any()
    print("band %d scheme %s: two substitutions, %d of %d claimed (without the check %d)" % (band, scheme, new.sum(), len(pairs), old.sum()))


def crafted(rng, text, band):
    J = Jobs(text, band)
    M = 150

    def place(lo=64, hi=None):
        return int(rng.integers(lo, (hi or len(text) - 400)))
    # three or four substitutions, at least one in the first or last five rows
    for _ in range(1500):
        pos = place(); r = text[pos:pos + M].copy()
        k = int(rng.integers(3, 5))
        q = rng.choice(M, k, replace=False)
        q[0] = rng.integers(0, 5) if rng.integers(0, 2) else M - 1 - rng.integers(0, 5)
        mutate(r, np.unique(q), rng)
        J.add(r, pos, "clip")
    # a 1-2 base indel 1..8 rows from either end, the seed's diagonal on either side, sometimes with a substitution elsewhere
    for L in (1, 2):
        for insert in (False, True):
            for k in range(1, 9):
                for at_end in (False, True):
                    for seed_on_long in (False, True):
                        for _ in range(12):
                            p = place()
                            cut = M - k if at_end else k
                            r = indel_read(text, p, M, cut, L, insert, rng)
                            if rng.integers(0, 3) == 0:
                                mutate(r, np.array([int(rng.integers(20, M - 20))]), rng)
                            # rows >= cut lie on the diagonal p + L (deletion) / p - L (insertion)
                            after = p + (-L if insert else L)
                            on_after = (not at_end) == seed_on_long
                            J.add(r, after if on_after else p, ("indel", L, insert, k, at_end, seed_on_long))
    # inside and across homopolymers and period-2 / 3 / 7 repeats: substitutions and indels anywhere
    for _ in range(2500):
        st = int(rng.choice([20_000, 40_000, 60_000, 80_000]))
        p = place(st - 200, st + 3_000)
        kind = int(rng.integers(0, 3))
        if kind == 0:
            r = text[p:p + M].copy(); mutate(r, rng.choice(M, int(rng.integers(1, 4)), replace=False), rng); pos = p
        else:
            L = int(rng.integers(1, 3)); insert = bool(rng.integers(0, 2)); cut = int(rng.integers(1, M))
            r = indel_read(text, p, M, cut, L, insert, rng)
            pos = p if rng.integers(0, 2) else p + (-L if insert else L)
        J.add(r, pos, "repeat")
    # ragged and short reads with 0-4 substitutions; windows longer than needed and too short
    for a in range(1500):
        m = int(rng.integers(1, 151)) if a % 3 else int(rng.integers(1, 24))
        pos = place(); r = text[pos:pos + m].copy()
        mutate(r, rng.choice(m, min(m, int(rng.integers(0, 5))), replace=False), rng)
        J.add(r, pos, "ragged", extra=int(rng.choice([0, 0, 5, 10, -1, -3])))
    return J


@pytest.mark.parametrize("band", [31, 15, 8])
@pytest.mark.parametrize("scheme", SCHEMES)
def test_crafted_cases(H, O, R, band, scheme):
    rng = np.random.default_rng(1000 + band * 10 + scheme[0])
    J = crafted(rng, random_text(rng, repeats=True), band)
    new, old = check(H, O, R, J, scheme)
    print("band %d scheme %s: crafted, %d of %d claimed (without the check %d)" % (band, scheme, new.sum(), len(new), old.sum()))


def c3_jobs(rng, text, n_reads, band=31, M=150):
    """bench.py's read model: 1 % substitutions and 0.1 % indels (1-3 bases) per base; a read with an indel gives a job on either side"""
    J = Jobs(text, band)
    for _ in range(n_reads):
        p = int(rng.integers(64, len(text) - 400))
        ind = np.flatnonzero(rng.random(M) < 0.001)
        if len(ind):
            cut = int(ind[0]) if ind[0] > 0 else 1
            L = int(rng.integers(1, 4)); insert = bool(rng.integers(0, 2))
            r = indel_read(text, p, M, cut, L, insert, rng)
            pos2 = p + (-L if insert else L)
        else:
            r = text[p:p + M].copy(); pos2 = None
        sub = np.flatnonzero(rng.random(M) < 0.01)
        if len(sub):
            mutate(r, sub, rng)
        J.add(r, p, "c3")
        if pos2 is not None:
            J.add(r, pos2, "c3 indel")
    return J


def test_c3_claimed_fraction(H, O, R):
    """on the headline read model the claimed share of jobs rises from about 0.42 to about 0.61"""
    rng = np.random.default_rng(31)
    J = c3_jobs(rng, random_text(rng, 2_000_000), 20_000)
    new, old = check(H, O, R, J, (2, -2, -5, -3))
    print("C3 sample: %d jobs, claimed %.3f without the check, %.3f with it" % (len(new), old.mean(), new.mean()))
    assert 0.39 < old.mean() < 0.45 and 0.58 < new.mean() < 0.64
