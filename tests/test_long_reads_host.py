"""CPU: the exact extension shortcut (gapless_job_shortcut, pipeline_core.cuh, through the host harness of test_shortcut_one_gap.py) on
reads of 151 to 2000 bp.  Its proof -- an alignment with g gaps, q mismatches and u unaligned rows scores at most
m * M - m * u - (m - s) * q - g * o, so it reaches the seed diagonal's best T only if m * u + (m - s) * q + g * o <= delta -- is written
for any read length M, but the bound's U = (delta - o) / m, the rows [U, M - 1 - U] it scans and the per-diagonal spans were only run on
reads of at most 150 bp.  Here: exact reads, one or two substitutions anywhere, and one-gap cases (a 1-2 base indel 1 to 8 rows from
either end, the seed's diagonal on either side of it) at M in {151, 255, 256, 257, 511, 512, 1024, 2000} and bands 7, 15 and 31.  Every
claimed job has the oracle's banded LOCAL (score, sink); the rule without the one-gap check claims a subset with the same results; exact
reads and reads with two interior substitutions are claimed."""
import numpy as np
import pytest
from tests.test_shortcut_one_gap import H, O, R, Jobs, check, indel_read, mutate, one_gap_limit, random_text  # noqa: F401  (fixtures)

LENGTHS = (151, 255, 256, 257, 511, 512, 1024, 2000)
SCHEMES = ((2, -2, -5, -3), (1, -4, -6, -1))


class LongJobs(Jobs):
    """Jobs with a read stride wide enough for the longest read (a multiple of 16 symbols, as the pipeline's strings are)"""

    def arrays(self):
        stride = (max(len(r) for r in self.reads) + 15) // 16 * 16
        n = len(self.reads)
        M = np.array([len(r) for r in self.reads], np.uint32)
        flat = np.zeros((n, stride), np.uint8)
        for a, r in enumerate(self.reads):
            flat[a, :len(r)] = r
        to = (np.array(self.pos) - self.band // 2).astype(np.uint32)
        N = (M.astype(np.int64) + self.band - 1 + np.array(self.extra)).astype(np.uint32)
        po = (np.arange(n) * stride).astype(np.uint32)
        return flat.reshape(-1), po, M, to, N


def long_jobs(rng, text, band, M):
    J = LongJobs(text, band)

    def place():
        return int(rng.integers(64, len(text) - M - 400))
    for _ in range(24):                                                    # exact
        p = place(); J.add(text[p:p + M].copy(), p, "exact")
    for _ in range(40):                                                    # one substitution, anywhere (the clip rows included)
        p = place(); r = text[p:p + M].copy(); mutate(r, np.array([int(rng.integers(0, M))]), rng); J.add(r, p, "sub1")
    for k in range(60):                                                    # two substitutions: interior, then one near an end
        p = place(); r = text[p:p + M].copy()
        q = np.sort(rng.choice(np.arange(16, M - 16), 2, replace=False)) if k < 40 else \
            np.array([int(rng.integers(0, 6)) if k % 2 else M - 1 - int(rng.integers(0, 6)), int(rng.integers(20, M - 20))])
        mutate(r, np.unique(q), rng)
        J.add(r, p, ("sub2", k < 40))
    for L in (1, 2):                                                       # one gap a few rows from either end, seed on either side
        for insert in (False, True):
            for k in (1, 2, 3, 5, 8):
                for at_end in (False, True):
                    for seed_on_long in (False, True):
                        p = place()
                        cut = M - k if at_end else k
                        r = indel_read(text, p, M, cut, L, insert, rng)
                        after = p + (-L if insert else L)
                        on_after = (not at_end) == seed_on_long
                        J.add(r, after if on_after else p, ("indel", L, insert, k, at_end, seed_on_long))
    return J


@pytest.mark.parametrize("band", [7, 15, 31])
@pytest.mark.parametrize("scheme", SCHEMES)
def test_long_reads(H, O, R, band, scheme):
    rng = np.random.default_rng(band * 13 + scheme[0])
    text = random_text(rng)
    lim, _ = one_gap_limit(scheme)
    m, s = scheme[0], scheme[1]
    for M in LENGTHS:
        J = long_jobs(rng, text, band, M)
        new, old = check(H, O, R, J, scheme)
        exact = np.array([lb == "exact" for lb in J.label])
        interior2 = np.array([isinstance(lb, tuple) and lb[0] == "sub2" and lb[1] for lb in J.label])
        assert new[exact].all(), (M, band, scheme)
        if 2 * (m - s) < lim:
            assert new[interior2].all(), (M, band, scheme, np.flatnonzero(interior2 & ~new)[:5])
        assert new.mean() > 0.3, (M, band, scheme, new.mean())
        print("M %d band %d scheme %s: %d of %d claimed (without the check %d)" % (M, band, scheme, new.sum(), len(new), old.sum()))
