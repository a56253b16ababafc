"""CPU: the first seed-match pass locates the lone surviving row of a k-mer with 5 to 8 occurrences on the wide k-mer table
(nvb_fm_index.ktab_located = 4 / 5): the 8-symbol contexts in the entry pick the row and its position comes from the full suffix array.
The host build (tests/host/wide_harness.cu) gives the same (status, x, y) for every seed at levels 2 to 5, one and two passes, and the
second pass is left only the seeds the entry cannot decide."""
import numpy as np
import pytest
from tests.test_located_rows import make_index
from tests.test_wide_ktab import H, O, build_wide, check_same, ktab8_of  # noqa: F401  (H, O: fixtures)


@pytest.mark.parametrize("bits", [2, 4])
def test_wide_lone_row_below_rem(H, O, bits):  # noqa: F811
    """a 6-row k-mer whose only row matching the unread symbols (compared without the position test) lies at text position 2: the
    context's missing symbols read as A, so an all-A prefix makes it the lone survivor although fewer than rem symbols precede it.  Its SA
    is below rem and the seed is empty; with rem = 2 the same row is located"""
    rng = np.random.default_rng(58 + bits)
    n, k = 400, 6
    text = rng.integers(0, 4, n).astype(np.uint8)
    kmer = np.array([0, 1, 2, 3, 3, 0], np.uint8)
    text[0:2] = [1, 2]
    starts = [2, 60, 130, 200, 270, 340]
    for st in starts:
        text[st:st + k] = kmer
    for st in starts[1:]:
        text[st - 8:st] = rng.integers(0, 3, 8)         # every other row's nearest preceding symbol differs from text[1] = 2
        text[st - 1] = int(rng.integers(0, 2))
    occ = [i for i in range(n - k + 1) if np.array_equal(text[i:i + k], kmer)]
    assert occ == starts
    idx, full_sa, gw, ctx, rows = make_index(H, O, text, k)
    k8 = ktab8_of(H, idx, n, k)
    wide = build_wide(H, k8, full_sa, gw, n, k)

    def queries(parts):
        lens = np.array([len(p) for p in parts], np.uint32)
        return np.concatenate(parts).astype(np.uint8), np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint32), lens

    # the row at position 2: rem = 3..8 (text[0:2] padded with A) -> empty, rem = 2 -> located at 0
    lone = [np.concatenate([np.zeros(rem - 2, np.uint8), text[0:2], kmer]) for rem in range(3, 9)] + [text[0:2 + k]]
    ref, nd2, nd4 = check_same(H, idx, full_sa, gw, ctx, wide, k, rows, *queries(lone), bits)
    assert (ref[:6, 0] == 0).all() and list(ref[6]) == [2, 0, 0xFFFFFFFF]
    assert nd2 == len(lone) and nd4 == 0                 # the entry decides every one of them in the first pass
    # the other rows, rem = 1..8: whatever the walk gives
    check_same(H, idx, full_sa, gw, ctx, wide, k, rows, *queries([text[st - rem:st + k] for st in starts[1:] for rem in range(1, 9)]), bits)


def test_deferred_fraction_lone_row_headline(H, O):  # noqa: F811
    """the scaled analogue of bench.py's index and seeds of test_wide_ktab.py (k = 10 over 1.86 Mbp, n / 4^k = 1.77, seeds of k + 5
    symbols): with the lone survivor of a 5- to 8-row k-mer located in the first pass, the wide table hands on below 0.02 of the
    genome-sampled seeds (about 0.11 when only 3- and 4-row k-mers are located there) and almost none of the random ones"""
    rng = np.random.default_rng(1771)
    k, L, nq = 10, 15, 20000
    n = int(1.77 * 4 ** k)
    text = rng.integers(0, 4, n).astype(np.uint8)
    idx, full_sa, gw, ctx, rows = make_index(H, O, text, k)
    k8 = ktab8_of(H, idx, n, k)
    wide = build_wide(H, k8, full_sa, gw, n, k)
    lens = np.full(nq, L, np.uint32)
    offs = (np.arange(nq) * L).astype(np.uint32)
    sampled = np.concatenate([text[s:s + L] for s in rng.integers(0, n - L, nq)]).astype(np.uint8)
    random = rng.integers(0, 4, nq * L).astype(np.uint8)
    after = []
    for q in (sampled, random):
        _, _, nd4 = check_same(H, idx, full_sa, gw, ctx, wide, k, rows, q, offs, lens, 2)
        after.append(nd4 / nq)
    assert after[0] < 0.02 and after[1] < 0.002, after
