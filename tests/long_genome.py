"""FM-indices of genomes longer than 2^31 bases, known in closed form: T = A^F . R for a random R (R[0] != A, R[-1] != A).

No suffix sort reaches such a length in a test, but SA(T) follows from SA(R) alone.  Row 0 is `$`.  Then come the suffixes that start
with A, each A^t . X with X a non-empty suffix of R that starts with a non-A symbol: the run suffix at i < F has t = F - i and X = R, the
R suffix at F + j with R[j] = A has t = the A-run length at j and X = R[j + t:].  They sort by t descending, then by X's rank among R's
suffixes.  With m = the longest A-run of R, every t > m belongs to a run suffix alone, so rows 1 .. F - m hold SA = row - 1 (the "head");
the rest (the "tail": about r / 4 + m A-suffixes, then R's non-A suffixes in SA(R) order, offset by F) is sorted on the host in O(r).

Two such genomes A^F . R and A^F' . R with F, F' > m have the same rows after the head: row rho >= 1 of the shorter one is row
rho + (F - F') of the longer one, at text position + (F - F').  So any result on a 2-3 Gbp T can be predicted from a few-Mbp partner
T' = A^F' . R that the device builds and the suite already pins against the oracle.  Queries of A's alone are the exception: their ranges
start at row 1 on both, and their sizes are `a_run_range_size`.

`LongGenome` holds the O(r) part; `device_genome` / `device_index` make the O(n) arrays on the device (host memory stays O(r))."""
import numpy as np
import torch

from nvbio_b200.fmindex import FMIndexDevice
from nvbio_b200.strings import pack_symbols

CHUNK = 1 << 27            # rows per device arange chunk (1 GiB of int64)


def a_runs(R: np.ndarray) -> np.ndarray:
    """run[j] = the number of A's (symbol 0) starting at R[j] (0 where R[j] != A)"""
    r = len(R)
    idx = np.where(R != 0, np.arange(r, dtype=np.int64), r)
    nxt = np.minimum.accumulate(idx[::-1])[::-1]        # the first non-A at or after j
    return nxt - np.arange(r, dtype=np.int64)


class LongGenome:
    """the suffix array, BWT and range sizes of T = A^F . R from SA(R) (sa_R: R's suffix array with its `$` row, n_R + 1 entries)"""

    def __init__(self, R: np.ndarray, F: int, sa_R: np.ndarray):
        R = np.ascontiguousarray(R, dtype=np.uint8)
        r = len(R)
        assert r >= 2 and R[0] != 0 and R[-1] != 0 and F >= 1
        sa_R = np.asarray(sa_R, dtype=np.int64)[1:]                      # R's suffixes, `$` row dropped
        assert len(sa_R) == r
        self.R, self.F, self.r, self.n = R, int(F), r, int(F) + r
        self.runs = a_runs(R)
        self.m = int(self.runs.max())
        isa = np.empty(r + 1, np.int64)
        isa[sa_R] = np.arange(r, dtype=np.int64)
        isa[r] = -1
        self.h = max(self.F - self.m, 0)                                   # head rows 1 .. h: SA = row - 1
        # A-suffixes of the tail: run suffixes with t <= min(F, m), R suffixes at A's; key (t descending, rank of X)
        t_run = np.arange(1, min(self.F, self.m) + 1, dtype=np.int64)
        ja = np.nonzero(self.runs)[0]
        t_all = np.concatenate([t_run, self.runs[ja]])
        x_rank = np.concatenate([np.full(len(t_run), isa[0]), isa[ja + self.runs[ja]]])
        pos = np.concatenate([self.F - t_run, self.F + ja])
        order = np.lexsort((x_rank, -t_all))
        non_a = sa_R[R[sa_R] != 0]
        self.tail = np.concatenate([pos[order], self.F + non_a]).astype(np.int64)     # SA of rows h + 1 .. n
        assert len(self.tail) == self.n - self.h
        self.primary = 1 if self.h >= 1 else self.h + 1 + int(np.nonzero(self.tail == 0)[0][0])
        # stored BWT (the `$` row removed): R[-1] for row 0, then A for rows 2 .. h, then the tail rows' T[SA - 1]
        tp = self.tail[self.tail != 0] - 1
        self.tail_bwt = np.where(tp < self.F, 0, R[np.maximum(tp - self.F, 0)]).astype(np.uint8)
        self.tail_start = max(self.h, 1)                                   # first stored-BWT symbol of the tail

    # -- host views (tests at small n) ------------------------------------------------------
    def text(self) -> np.ndarray:
        return np.concatenate([np.zeros(self.F, np.uint8), self.R])

    def sa(self) -> np.ndarray:
        """the whole suffix array with SA[0] = n (the oracle's convention); O(n) -- small n only"""
        return np.concatenate([[self.n], np.arange(self.h, dtype=np.int64), self.tail]).astype(np.int64)

    def bwt(self) -> np.ndarray:
        """the stored BWT symbols; O(n) -- small n only"""
        out = np.zeros(self.n, np.uint8)
        out[0] = self.R[-1]
        out[self.tail_start:] = self.tail_bwt
        return out

    # -- row map and closed-form ranges -------------------------------------------------------
    def shift(self, partner: "LongGenome") -> int:
        """rows >= 1 and text positions of `partner` (the same R, F' > m) move by this much on self"""
        assert partner.m < min(self.F, partner.F) and np.array_equal(partner.R, self.R)
        return self.F - partner.F

    def a_run_range_size(self, s: int) -> int:
        """rows of the query A^s (rows 1 .. size): run positions 0 .. F - s and R positions with an A-run of s or more"""
        return max(self.F - s + 1, 0) + int((self.runs >= s).sum())

    def boundary_range_size(self, s: int, q: int) -> int:
        """rows of the query A^s . R[:q] (1 <= q): the run end at F - s (s <= F) and R positions whose A-run is exactly s and that
        are followed by R[:q]"""
        assert q >= 1
        j = np.nonzero(self.runs == s)[0]
        j = j[j + s + q <= self.r]
        hit = np.ones(len(j), bool)
        for i in range(q):
            hit &= self.R[j + s + i] == self.R[i]
        return int(s <= self.F) + int(hit.sum())


# -- device arrays -------------------------------------------------------------------------------
def splice_symbols(words: torch.Tensor, at: int, sym: np.ndarray):
    """OR the 2-bit big-endian symbols `sym` into int32 `words` from symbol `at` on (the words there hold A's = zero bits)"""
    lead = at % 16
    packed = pack_symbols(np.concatenate([np.zeros(lead, np.uint8), sym]), pad_words=0)
    w0 = at // 16
    words[w0:w0 + len(packed)] |= torch.from_numpy(packed.view(np.int32)).to(words.device)


def device_genome(lg: LongGenome, device="cuda") -> torch.Tensor:
    """T's 2-bit big-endian words, readable 2 words past the end (the seed + extend and context kernels over-read)"""
    gw = torch.zeros((lg.n + 15) // 16 + 4, dtype=torch.int32, device=device)
    splice_symbols(gw, lg.F, lg.R)
    return gw


def device_bwt(lg: LongGenome, device="cuda") -> torch.Tensor:
    """the stored BWT words (ceil(n / 64) * 4) that from_bwt takes"""
    bw = torch.zeros(((lg.n + 63) // 64) * 4, dtype=torch.int32, device=device)
    splice_symbols(bw, lg.tail_start, lg.tail_bwt)
    splice_symbols(bw, 0, lg.R[-1:])
    return bw


def wrap_i32(t: torch.Tensor) -> torch.Tensor:
    """int64 values in [0, 2^32) -> their uint32 bit patterns as int32"""
    return torch.where(t >= 1 << 31, t - (1 << 32), t).to(torch.int32)


def device_sa(lg: LongGenome, device="cuda") -> torch.Tensor:
    """the full suffix array in the index's format (n + 1 int32 words, SA[0] = 0xFFFFFFFF), the head made in chunks on the device"""
    sa = torch.empty(lg.n + 1, dtype=torch.int32, device=device)
    sa[0] = -1
    for lo in range(0, lg.h, CHUNK):
        hi = min(lg.h, lo + CHUNK)
        sa[1 + lo:1 + hi] = wrap_i32(torch.arange(lo, hi, dtype=torch.int64, device=device))
    sa[lg.h + 1:] = wrap_i32(torch.from_numpy(lg.tail).to(device))
    return sa


def device_index(lg: LongGenome, sa: torch.Tensor, sa_interval: int = 1) -> FMIndexDevice:
    """T's index from its stored BWT (from_bwt), with the full suffix array `sa` (sa_interval 1) or every sa_interval-th row of it"""
    bw = device_bwt(lg, sa.device)
    ssa = sa if sa_interval == 1 else sa[::sa_interval].clone()
    idx = FMIndexDevice.from_bwt(bw, lg.n, lg.primary, ssa, sa_interval=sa_interval)
    del bw
    return idx
