"""The 16-bit packed Gotoh kernels (gotoh_pair_kernel, gotoh_full_pair_kernel, gotoh_full_warp_kernel) at the edges of their admission
rules (pair_path_ok, full_pair_path_ok, the selector-row cap of banded_impl).  Every case runs just inside a limit, where the packed kernel
must take the whole batch and match the int32 oracle exactly, and outside it, where the batch must go to the int32 kernels and still be
exact; the route is read back through nvb_debug_gotoh_last_route.  The batches are shaped so that the packed path can take them at all:
equal lengths within each pair, full text windows, no N.

The unmarked tests at the end run the same edges through the host build of the very same per-thread routines (tests/host)."""
import ctypes as C
import zlib
import numpy as np
import pytest
import torch
from oracle import orc
import nvbio_b200 as nb
from nvbio_b200 import aln
from nvbio_b200._lib import GotohSchemeStruct
from nvbio_b200.strings import PackedStringSet, pack_symbols
from tests.gpu_util import require_gpu, host_u32
from tests.test_host_core import H, _p, _gotoh_pair, fixed_problems   # noqa: F401  (H: the host-harness fixture)

BANDS = (7, 15, 31)
GLOBAL, LOCAL, SEMI = 0, 1, 2


@pytest.fixture(scope="module")
def O():
    return orc.Oracle()


# --------------------------------------------------------------------------------------------------------------------------------------
# problems and schemes
# --------------------------------------------------------------------------------------------------------------------------------------
def cat(*prs):
    """one batch out of several (pattern, p_off, p_len, text, t_off, t_len) tuples"""
    pats, po, pl, txts, to, tl = [], [], [], [], [], []
    a = b = 0
    for pat, p_off, p_len, txt, t_off, t_len in prs:
        pats.append(pat); txts.append(txt)
        po.append(np.asarray(p_off, np.uint32) + a); pl.append(np.asarray(p_len, np.uint32)); a += len(pat)
        to.append(np.asarray(t_off, np.uint32) + b); tl.append(np.asarray(t_len, np.uint32)); b += len(txt)
    return (np.concatenate(pats), np.concatenate(po), np.concatenate(pl), np.concatenate(txts), np.concatenate(to), np.concatenate(tl))


def window_problems(rng, n, band, m, kind):
    """n patterns of m symbols against full windows of m + band - 1 text symbols: 'exact' = a substring of the window (H grows by the
    match score every row), 'mismatch' = a homopolymer against a homopolymer of another symbol (H, E and F go deep negative)"""
    N = m + band - 1
    pats, txts = [], []
    for _ in range(n):
        if kind == "mismatch":
            a = int(rng.integers(0, 4))
            p, t = np.full(m, a, np.uint8), np.full(N, (a + 1 + int(rng.integers(0, 3))) % 4, np.uint8)
        else:
            t = rng.integers(0, 4, N).astype(np.uint8)
            j = int(rng.integers(0, band))
            p = t[j:j + m].copy()
        pats.append(p); txts.append(t)
    return (np.concatenate(pats), np.arange(n, dtype=np.uint32) * m, np.full(n, m, np.uint32),
            np.concatenate(txts), np.arange(n, dtype=np.uint32) * N, np.full(n, N, np.uint32))


def banded_batch(rng, band, m, n=61):
    """reads with substitutions and indels (fixed_problems), exact reads and all-mismatch homopolymers, every pattern m symbols long;
    an odd count leaves a tail alignment alone in its pair"""
    k = n // 3
    return cat(fixed_problems(rng, n - 2 * k, band, m), window_problems(rng, k, band, m, "exact"), window_problems(rng, k, band, m, "mismatch"))


def full_batch(rng, n_pairs, m, n):
    """pairs of equal (m, n): patterns that are substrings of their text (with a few substitutions), random patterns, homopolymers"""
    pats, txts = [], []
    for i in range(2 * n_pairs):
        t = rng.integers(0, 4, n).astype(np.uint8)
        kind = i % 3
        if kind == 0 and n >= m:
            st = int(rng.integers(0, n - m + 1)); p = t[st:st + m].copy()
            for _k in range(int(rng.integers(0, 4))):
                p[int(rng.integers(0, m))] = rng.integers(0, 4)
        elif kind == 1:
            p = rng.integers(0, 4, m).astype(np.uint8)
        else:
            p = np.full(m, int(rng.integers(0, 4)), np.uint8); t = np.full(n, (int(p[0]) + 1) % 4, np.uint8)
        pats.append(p); txts.append(t)
    c = 2 * n_pairs
    return (np.concatenate(pats), np.arange(c, dtype=np.uint32) * m, np.full(c, m, np.uint32),
            np.concatenate(txts), np.arange(c, dtype=np.uint32) * n, np.full(c, n, np.uint32))


def edge_table(lo, hi):
    """a 256 x 2 quality table (substitution on a match, on a mismatch) that reaches both bounds: match scores in [hi // 2, hi], mismatch
    scores in [lo, lo // 2]"""
    q = np.arange(256)
    tab = np.stack([hi - (q % 7) * (hi - hi // 2) // 6, lo - (q % 5) * (lo - lo // 2) // 4], axis=1).astype(np.int32)
    tab[0] = (hi, lo)
    return np.ascontiguousarray(tab)


class Scheme6:
    """(match, mismatch, pattern gap open / ext, text gap open / ext) through the C struct, optionally with a quality table (its
    bounds declared as its true minimum and maximum)"""

    def __init__(self, s6, qtab=None):
        self.s6 = tuple(s6) if len(s6) == 6 else tuple(s6) + (s6[2], s6[3])
        self.qtab = qtab
        self.bounds = (int(qtab.min()), int(qtab.max())) if qtab is not None else (0, 0)
        self.table = None

    def struct(self):
        s = GotohSchemeStruct()
        s.match, s.mismatch, s.pattern_gap_open, s.pattern_gap_ext, s.text_gap_open, s.text_gap_ext = self.s6
        if self.qtab is not None and self.table is None:
            self.table = torch.from_numpy(self.qtab).cuda()
        s.d_qual_table = self.table.data_ptr() if self.qtab is not None else None
        s.qual_table_min, s.qual_table_max = self.bounds
        return s


# --------------------------------------------------------------------------------------------------------------------------------------
# the banded edge cases: (name, band, type, scheme, pattern length, admitted, quality table or None)
# --------------------------------------------------------------------------------------------------------------------------------------
def banded_cases(band):
    cap = 801 - band                       # round16(cap + band - 1) x 128 threads x 2 B = 200 KB of selector rows
    out = []
    for typ in (GLOBAL, LOCAL, SEMI):
        # selector rows; LOCAL: exact reads reach H = 2 * cap >= 1024, the top bit of the u16 key (H << 5) | j
        out += [("cap", band, typ, (2, -2, -5, -3), cap, True), ("cap+1", band, typ, (2, -2, -5, -3), cap + 1, False)]
        # max_m * max|s| + (B + 3) * max|gap| == 30000 exactly, far enough past it to wrap 16 bits, one row past it (gaps
        # cost more per symbol than a mismatch, so the all-mismatch homopolymers score -max_m * s)
        s, m = {7: (58, 500), 15: (60, 470), 31: (50, 532)}[band]
        deep = {7: 640, 15: 600, 31: 700}[band]
        assert m * s + (band + 3) * 100 == 30000
        out += [("bound", band, typ, (2, -s, -100, -100), m, True), ("bound-wrap", band, typ, (2, -s, -100, -100), deep, False),
                ("bound+1", band, typ, (2, -s, -100, -100), m + 1, False)]
        # F's infimum raised so that INF + Ge cannot wrap (|Ge| above the least gap cost)
        out += [("inf", band, typ, (2, -2, -5, -3, -9, -1), 300, True), ("inf", band, typ, (1, -3, -12, -6, -4, -1), 300, True)]
    # LOCAL: max_m * match = 2047 is the last key that fits, 3910 and 2070 are refused (both would overflow the key)
    out += [("key", band, LOCAL, (23, -2, -5, -3), 89, True), ("key-wrap", band, LOCAL, (23, -2, -5, -3), 170, False),
            ("key+1", band, LOCAL, (23, -2, -5, -3), 90, False)]
    # int8 substitution bytes: s_hi - Go = 127 and s_lo - Go = -128 exactly, one past either edge
    for typ in (GLOBAL, SEMI):
        out += [("int8", band, typ, (122, -133, -5, -3), 200, True), ("int8-hi", band, typ, (123, -133, -5, -3), 200, False),
                ("int8-lo", band, typ, (122, -134, -5, -3), 200, False)]
    return [c + (None,) for c in out] + banded_table_cases(band)


def banded_table_cases(band):
    """quality tables whose bounds sit on the int8 edge (Go = -8: [-136, 119]) or one past it, and LOCAL tables on the key edge"""
    s6 = (0, 0, -8, -3, -7, -2)
    out = []
    for typ in (GLOBAL, SEMI):
        out += [("qtab", band, typ, s6, 200, True, edge_table(-136, 119)), ("qtab-hi", band, typ, s6, 200, False, edge_table(-136, 120)),
                ("qtab-lo", band, typ, s6, 200, False, edge_table(-137, 119))]
    out += [("qtab-key", band, LOCAL, s6, 204, True, edge_table(-136, 10)), ("qtab-key+1", band, LOCAL, s6, 205, False, edge_table(-136, 10))]
    return out


def case_id(c):
    return "%s-B%d-t%d-%s-m%d" % (c[0], c[1], c[2], ",".join(str(v) for v in c[3]), c[4])


def case_problems(c, n=61):
    name, band, typ, s6, m, ok, qtab = c
    rng = np.random.default_rng(zlib.crc32(case_id(c).encode()))
    pr = banded_batch(rng, band, m, n)
    qual = rng.integers(0, 8, len(pr[0])).astype(np.uint8) if qtab is not None else None      # quality 0: the table's bounds
    return pr, qual


def oracle_banded(O, c, pr, qual):
    name, band, typ, s6, m, ok, qtab = c
    return O.banded_gotoh(band, typ, s6, *pr, qual=qual, qtab=qtab)


# --------------------------------------------------------------------------------------------------------------------------------------
# device helpers
# --------------------------------------------------------------------------------------------------------------------------------------
def last_route():
    packed, n = C.c_int(-1), C.c_uint32(0xFFFFFFFF)
    assert nb.lib().nvb_debug_gotoh_last_route(C.byref(packed), C.byref(n)) == 0
    return packed.value, n.value


def gpu_banded(band, typ, scheme, pr, max_m, pbits=2, qual=None):
    pat, p_off, p_len, txt, t_off, t_len = pr
    P = PackedStringSet.from_symbols(pat, p_off, p_len, bits=pbits, big_endian=True)
    P.length = max_m
    T = PackedStringSet.from_symbols(txt, t_off, t_len, bits=2, big_endian=True)
    q = torch.from_numpy(qual).cuda() if qual is not None else None
    s, k = aln.batch_banded_alignment_score(band, aln.make_gotoh_aligner(typ, scheme), P, T, quals=q)
    route = last_route()
    k = host_u32(k)
    return (s.cpu().numpy(), k[:, 0].copy(), k[:, 1].copy()), route


def debug_knobs(**kw):
    """set nvbio_b200_debug.h knobs for a block, restoring their defaults afterwards"""
    defaults = dict(force_gotoh_path=0, pair_format=1, pair_rows2=1, full_warp=0, full_minb=0, traceback_fast=1, full_traceback_warp=0)

    class _Ctx:
        def __enter__(self):
            for k, v in kw.items():
                getattr(nb.lib(), "nvb_debug_" + k)(C.c_int(v))

        def __exit__(self, *a):
            for k in kw:
                getattr(nb.lib(), "nvb_debug_" + k)(C.c_int(defaults[k]))
    return _Ctx()


def assert_same(got, want, what):
    for g, w, f in zip(got, want[:3], ("score", "sink.x", "sink.y")):
        bad = np.flatnonzero(np.asarray(g, np.int64) != np.asarray(w, np.int64))
        assert len(bad) == 0, "%s: %s differs at %d alignments, first %d: got %d want %d" % (what, f, len(bad), bad[0], g[bad[0]], w[bad[0]])


def assert_route(route, admitted, what):
    packed, n_int32 = route
    if admitted:
        assert packed != 0 and n_int32 == 0, "%s: the packed kernel must take the whole batch, route %s" % (what, route)
    else:
        assert packed == 0, "%s: the batch must go to the int32 kernels, route %s" % (what, route)


# --------------------------------------------------------------------------------------------------------------------------------------
# banded pair kernel
# --------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("band", BANDS)
def test_banded_pair_kernel_at_its_limits(O, band):
    """every kernel variant (2-bit / 4-bit big-endian compile-time pattern readers, run-time format; two rows in flight or one) and
    the int32 kernel equal the oracle at every edge; the route says which side of the edge the batch was on"""
    require_gpu()
    for c in banded_cases(band):
        name, band_, typ, s6, m, ok, qtab = c
        pr, qual = case_problems(c)
        want = oracle_banded(O, c, pr, qual)
        assert want[3].all()
        sch = Scheme6(s6, qtab)
        variants = [(2, 1, 1), (2, 1, 0), (4, 1, 1), (4, 1, 0), (4, 0, 1), (4, 0, 0)] if qtab is None else [(4, 1, 1), (4, 1, 0)]
        for pbits, fmt, rows2 in variants:
            with debug_knobs(pair_format=fmt, pair_rows2=rows2):
                got, route = gpu_banded(band, typ, sch, pr, m, pbits=pbits, qual=qual)
            what = "%s pbits=%d fmt=%d rows2=%d" % (case_id(c), pbits, fmt, rows2)
            assert_same(got, want, what)
            assert_route(route, ok, what)
        with debug_knobs(force_gotoh_path=1):
            got, route = gpu_banded(band, typ, sch, pr, m, pbits=4, qual=qual)
        assert_same(got, want, case_id(c) + " int32")
        assert route == (0, 0)


def test_banded_edges_reach_their_values(O):
    """the edge batches really take the values the rules bound: LOCAL keys with the top bit set, GLOBAL scores past -29,000 at the
    30000 bound, scores that would wrap 16 bits one step outside"""
    for band in BANDS:
        cs = {(c[0], c[2]): c for c in banded_cases(band)}
        for key, test in ((("cap", LOCAL), lambda s: s.max() >= 1024 * 1.5), (("bound", GLOBAL), lambda s: s.min() <= -26000),
                          (("bound-wrap", GLOBAL), lambda s: s.min() < -32768), (("key", LOCAL), lambda s: s.max() == 2047),
                          (("key-wrap", LOCAL), lambda s: s.max() >= 2048), (("int8", GLOBAL), lambda s: s.max() >= 20000)):
            c = cs[key]
            pr, qual = case_problems(c)
            assert test(oracle_banded(O, c, pr, qual)[0].astype(np.int64)), case_id(c)


@pytest.mark.gpu
def test_banded_edges_vs_reference_templates(O):
    """the oracle at these edges == the reference's own aln::banded_alignment_score (where oracle/_ref is built)"""
    if not orc.Ref.available():
        pytest.skip("oracle/_ref/libnvbio_ref.so not present")
    R = orc.Ref()
    for band in BANDS:
        for c in banded_cases(band):
            if c[6] is not None or len(c[3]) != 4:
                continue
            pr, qual = case_problems(c, n=21)
            assert_same(R.banded_gotoh(band, c[2], c[3], *pr)[:3], oracle_banded(O, c, pr, qual), case_id(c) + " ref")


@pytest.mark.gpu
@pytest.mark.parametrize("band", BANDS)
def test_banded_traceback_at_the_selector_cap(O, band):
    """nvb_banded_gotoh_traceback at the longest patterns the packed score pass admits (and one longer), through the gapless fast path
    and with every alignment through the direction matrix: score, sink, source and ops == the oracle"""
    require_gpu()
    cap = 801 - band
    for m in (cap, cap + 1):
        rng = np.random.default_rng(band * 1000 + m)
        pr = banded_batch(rng, band, m, n=31)
        pat, p_off, p_len, txt, t_off, t_len = pr
        P = PackedStringSet.from_symbols(pat, p_off, p_len, bits=4, big_endian=True)
        T = PackedStringSet.from_symbols(txt, t_off, t_len, bits=2, big_endian=True)
        max_ops = m + band + 1
        for typ in (GLOBAL, LOCAL, SEMI):
            want = O.banded_traceback(band, typ, (2, -2, -5, -3), *pr, max_ops=max_ops)
            for fast in (1, 0):
                with debug_knobs(traceback_fast=fast):
                    tb = aln.batch_banded_alignment_traceback(band, aln.make_gotoh_aligner(typ, aln.SimpleGotohScheme(2, -2, -5, -3)), P, T,
                                                              max_ops=max_ops)
                    route = last_route()
                what = "B%d m%d t%d fast=%d" % (band, m, typ, fast)
                n_ops = tb["n_ops"].cpu().numpy(); ops = tb["ops"].cpu().numpy()
                assert np.array_equal(tb["score"].cpu().numpy(), want["score"]), what
                assert np.array_equal(host_u32(tb["sink"]), want["sink"]) and np.array_equal(host_u32(tb["source"]), want["source"]), what
                assert np.array_equal(n_ops.astype(np.uint32), want["n_ops"]), what
                for i in range(len(n_ops)):
                    assert np.array_equal(ops[i, :n_ops[i]], want["ops"][i, :n_ops[i]]), (what, i)
                # the score pass of the fast path is the packed kernel exactly when the selector rows fit
                assert_route(route, fast == 1 and typ != GLOBAL and m == cap, what)


# --------------------------------------------------------------------------------------------------------------------------------------
# full-matrix kernels
# --------------------------------------------------------------------------------------------------------------------------------------
FULL_S = (2, -3, -5, -5)                  # max |value| 5: (m + n + 4) * 5 <= 30000 <=> m + n <= 5996


def full_cases():
    """(name, type, scheme, m, n, admitted): the 16-bit bound exactly, far enough past it to wrap, one text row more"""
    out = []
    for typ in (GLOBAL, LOCAL, SEMI):
        out += [("bound", typ, FULL_S, 200, 5796, True), ("bound-wrap", typ, FULL_S, 200, 7000, False), ("bound+1", typ, FULL_S, 200, 5797, False)]
    # LOCAL keys: min(m, n) * match = 2040, then 2048
    out += [("key", LOCAL, (8, -3, -5, -5), 255, 600, True), ("key+1", LOCAL, (8, -3, -5, -5), 256, 600, False)]
    return out


def gpu_full(typ, scheme, pr, qual=None):
    pat, p_off, p_len, txt, t_off, t_len = pr
    P = PackedStringSet.from_symbols(pat, p_off, p_len, bits=2, big_endian=True)
    T = PackedStringSet.from_symbols(txt, t_off, t_len, bits=2, big_endian=True)
    q = torch.from_numpy(qual).cuda() if qual is not None else None
    s, k = aln.batch_alignment_score(aln.make_gotoh_aligner(typ, scheme), P, T, quals=q)
    route = last_route()
    k = host_u32(k)
    return (s.cpu().numpy(), k[:, 0].copy(), k[:, 1].copy()), route


@pytest.mark.gpu
def test_full_pair_kernel_at_its_limits(O):
    """gotoh_full_pair_kernel at minb 2 / 3 / 4 and its quality-table form: (m + n + 4) * max|value| = 30000 exactly (GLOBAL scores
    near -28,000), one text row more, and LOCAL keys at 2040 / 2048 == the oracle; the int32 kernel == the oracle"""
    require_gpu()
    for name, typ, s4, m, n, ok in full_cases():
        rng = np.random.default_rng(7000 + 10 * typ + m + n)
        pr = full_batch(rng, 4, m, n)
        want = O.gotoh_full(typ, s4, *pr)
        if name == "bound" and typ == GLOBAL:
            assert want[0].min() < -27000
        what = "%s t%d m%d n%d" % (name, typ, m, n)
        for minb in (2, 3, 4):
            with debug_knobs(full_warp=2, full_minb=minb):
                got, route = gpu_full(typ, Scheme6(s4), pr)
            assert_same(got, want, what + " minb=%d" % minb)
            assert_route(route, ok, what)
            assert not ok or route[0] == 1
        with debug_knobs(force_gotoh_path=1):
            got, route = gpu_full(typ, Scheme6(s4), pr)
        assert_same(got, want, what + " int32")
        # quality-dependent scores with the same bounds (the per-column-profile kernel): mismatch -3 .. -2, gaps -5, match up to s4[0]
        qtab = edge_table(-3, s4[0])
        qual = rng.integers(0, 8, len(pr[0])).astype(np.uint8)
        s6 = (0, 0, -5, -5, -5, -5)
        want_q = O.gotoh_full(typ, s6, *pr, qual=qual, qtab=qtab)
        got, route = gpu_full(typ, Scheme6(s6, qtab), pr, qual=qual)
        assert_same(got, want_q, what + " qtab")
        assert_route(route, ok, what + " qtab")


@pytest.mark.gpu
@pytest.mark.parametrize("W", range(1, 9))
def test_full_warp_kernel_at_its_limits(O, W):
    """gotoh_full_warp_kernel<TYPE, W>: pattern lengths filling W columns per lane (the last lane partly empty below W = 8), texts
    at the 16-bit bound, far past it and one row past it; LOCAL keys at 2040 with 255 columns"""
    require_gpu()
    m = 256 if W == 8 else 32 * W - 3
    # (GLOBAL at m + n = 7400 scores below -32768: refused, and it would wrap)
    cases = [(typ, FULL_S, m, 5996 - m, True) for typ in (GLOBAL, LOCAL, SEMI)] + [(GLOBAL, FULL_S, m, 7400 - m, False)] + \
        [(typ, FULL_S, m, 5997 - m, False) for typ in (GLOBAL, LOCAL, SEMI)]
    if W == 8:
        cases += [(LOCAL, (8, -3, -5, -5), 255, 600, True), (LOCAL, (8, -3, -5, -5), 256, 600, False)]
    for typ, s4, mm, n, ok in cases:
        rng = np.random.default_rng(8000 + 10 * W + typ + n)
        pr = full_batch(rng, 3, mm, n)
        want = O.gotoh_full(typ, s4, *pr)
        with debug_knobs(full_warp=1):
            got, route = gpu_full(typ, Scheme6(s4), pr)
        what = "W%d t%d m%d n%d" % (W, typ, mm, n)
        assert_same(got, want, what)
        assert_route(route, ok, what)
        assert not ok or route[0] == 2


@pytest.mark.gpu
@pytest.mark.parametrize("typ", [GLOBAL, LOCAL, SEMI])
def test_full_traceback_on_long_texts(O, typ):
    """nvb_gotoh_traceback at the 16-bit bound (200 x 5796), by the direction-matrix kernel and by the packed score pass + warp
    traceback: score, sink, source and every op == the oracle"""
    require_gpu()
    rng = np.random.default_rng(9000 + typ)
    pr = full_batch(rng, 2, 200, 5796)
    pat, p_off, p_len, txt, t_off, t_len = pr
    max_ops = 200 + 5796 + 1
    want = O.gotoh_full_traceback(typ, FULL_S, *pr, max_ops=max_ops)
    P = PackedStringSet.from_symbols(pat, p_off, p_len, bits=4, big_endian=True)
    T = PackedStringSet.from_symbols(txt, t_off, t_len, bits=2, big_endian=True)
    for warp in (0, 1):
        with debug_knobs(full_traceback_warp=warp):
            tb = aln.batch_alignment_traceback(aln.make_gotoh_aligner(typ, Scheme6(FULL_S)), P, T, max_ops=max_ops)
            route = last_route()
        n_ops = tb["n_ops"].cpu().numpy(); ops = tb["ops"].cpu().numpy()
        assert np.array_equal(tb["score"].cpu().numpy(), want["score"]), warp
        assert np.array_equal(host_u32(tb["sink"]), want["sink"]) and np.array_equal(host_u32(tb["source"]), want["source"]), warp
        assert np.array_equal(n_ops.astype(np.uint32), want["n_ops"]), warp
        for i in range(len(n_ops)):
            assert np.array_equal(ops[i, :n_ops[i]], want["ops"][i, :n_ops[i]]), (warp, i)
        assert_route(route, warp == 1, "traceback warp=%d" % warp)


# --------------------------------------------------------------------------------------------------------------------------------------
# windowed scoring past the short2 checkpoints
# --------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("typ", [GLOBAL, LOCAL, SEMI])
def test_windowed_score_past_the_checkpoint_range(O, typ):
    """(300, -200, -500, -300) on 150 bp reads: H passes 32767, so a checkpoint stored between windows wraps as the reference's short2
    does; every pass still equals the oracle (state, sinks, alive flags, checkpoints), one window over the whole pattern equals
    nvb_banded_gotoh_score, and the exact LOCAL reads show the windows part from the one-pass score"""
    require_gpu()
    band, scheme, m = 31, (300, -200, -500, -300), 150
    rng = np.random.default_rng(9500 + typ)
    pr = cat(fixed_problems(rng, 40, band, m), window_problems(rng, 24, band, m, "exact"))
    pat, p_off, p_len, txt, t_off, t_len = pr
    n = len(p_off)
    P = PackedStringSet.from_symbols(pat, p_off, p_len, bits=4, big_endian=True)
    T = PackedStringSet.from_symbols(txt, t_off, t_len, bits=2, big_endian=True)
    al = aln.make_gotoh_aligner(typ, aln.SimpleGotohScheme(*scheme))
    whole = O.banded_gotoh(band, typ, scheme, *pr)
    for W in (32, m):
        so = orc.window_state(n, band)
        st = aln.BandedWindowState(n, band, "cuda")
        for wb in range(0, m, W):
            O.banded_gotoh_window(band, typ, scheme, *pr, wb, wb + W, so)
            aln.batch_banded_alignment_score_window(band, al, P, T, wb, wb + W, st)
            torch.cuda.synchronize()
            k = host_u32(st.sink)
            assert np.array_equal(st.alive.cpu().numpy(), so["alive"]), (typ, W, wb)
            assert np.array_equal(st.score.cpu().numpy(), so["score"]) and np.array_equal(k[:, 0], so["sx"]) and np.array_equal(k[:, 1], so["sy"]), (typ, W, wb)
            alive = so["alive"].astype(bool)
            assert np.array_equal(st.ckpt.cpu().numpy()[alive], so["ckpt"][alive]), (typ, W, wb)
        if W == m:
            assert np.array_equal(so["score"], whole[0]) and np.array_equal(so["sx"], whole[1]) and np.array_equal(so["sy"], whole[2])
        elif typ == LOCAL:
            assert whole[0].max() > 32767 and (so["score"] != whole[0]).any()


# --------------------------------------------------------------------------------------------------------------------------------------
# host mirror: the same edges through the host build of gotoh_pair / gotoh_full_pair (runs without a GPU)
# --------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("band", BANDS)
def test_host_banded_pair_at_its_limits(H, O, band):
    """gotoh_pair (host build, both row schedules) at every banded edge: where pair_path_ok admits the batch the packed routine equals
    the oracle with no fallback; the rule admits exactly the cases inside the edge (the selector cap is a device launch limit: the host
    routine has no such cap and must be exact there too)"""
    for c in banded_cases(band):
        name, band_, typ, s6, m, ok, qtab = c
        pr, qual = case_problems(c, n=9)
        want = oracle_banded(O, c, pr, qual)
        s6x = s6 if len(s6) == 6 else s6 + (s6[2], s6[3])
        for rows2 in (1, 0):
            H.hh_set_pair_rows2(C.c_int(rows2))
            try:
                r, got, nf = _gotoh_pair(H, band, typ, s6x, pr, m, pbits=4 if qtab is not None else 2, qtab=qtab, qual=qual)
            finally:
                H.hh_set_pair_rows2(C.c_int(1))
            if r == 0:
                assert_same(got, want, "%s rows2=%d" % (case_id(c), rows2))
                assert nf == 0, case_id(c)
            assert (r == 0) == (ok or name == "cap+1"), (case_id(c), r)


def host_full_pair(H, typ, s6, pr):
    pat, p_off, p_len, txt, t_off, t_len = pr
    pw, tw = pack_symbols(pat, 2, True), pack_symbols(txt, 2, True)
    n = len(p_off)
    score = np.zeros(n, np.int32); sx = np.zeros(n, np.uint32); sy = np.zeros(n, np.uint32)
    s6 = np.array(s6, np.int32)
    packed = H.hh_gotoh_full_pair(C.c_int(typ), _p(s6), _p(pw), C.c_uint32(2), C.c_uint32(1), _p(p_off), _p(p_len),
                                  _p(tw), C.c_uint32(2), C.c_uint32(1), _p(t_off), _p(t_len), C.c_uint32(n), _p(score), _p(sx), _p(sy))
    return packed, (score, sx, sy)


def test_host_full_pair_at_its_limits(H, O):
    """gotoh_full_pair (host build) at the full-matrix edges: whenever full_pair_path_ok admits a batch the packed routine equals the
    oracle; the rule admits exactly the cases inside the edge"""
    for name, typ, s4, m, n, ok in full_cases():
        rng = np.random.default_rng(7500 + 10 * typ + m + n)
        pr = full_batch(rng, 1, m, n)
        s6 = s4 + (s4[2], s4[3])
        admitted = H.hh_full_pair_path_ok(C.c_int(typ), _p(np.array(s6, np.int32)), C.c_uint32(m), C.c_uint32(n))
        if admitted:
            want = O.gotoh_full(typ, s4, *pr)
            packed, got = host_full_pair(H, typ, s6, pr)
            assert packed == len(pr[1])
            assert_same(got, want, "%s t%d m%d n%d" % (name, typ, m, n))
        assert bool(admitted) == ok, (name, typ, m, n)
