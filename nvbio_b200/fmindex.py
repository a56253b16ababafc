"""Host-side mirror of nvbio's FM-index interface for the hot path (nvbio/fmindex/fmindex.h,
nvbio/fmindex/filter.h, nvbio/io/fmindex/fmindex.h) over the C ABI.  torch = device memory + streams."""
import ctypes as C
from typing import Optional
import numpy as np
import torch
from ._lib import lib, check, FmIndexStruct, NvbError
from .strings import PackedStringSet

MATCH_FORWARD_ORDER = 1
MATCH_COMPLEMENT = 2
MAX_LENGTH = 0xFFFFFFFE     # NVB_FM_MAX_LENGTH: the longest text an index may have


# device memory that build_ktab leaves free after the per-row array (a seed + extend call's temp buffers); without that room the
# array is left out
ROWS_HEADROOM = 4 << 30


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _np_u32(t: torch.Tensor) -> np.ndarray:
    return t.detach().cpu().numpy().view(np.uint32)


def _dev_u32(a: np.ndarray, device) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint32).view(np.int32)).to(device)


class FMIndexDevice:
    """Device-resident FM-index in the reference's production layout: interleaved 32-byte
    {bwt,occ} blocks + SA sampled every 16 rows (io::FMIndexDataDevice, nvbio/io/fmindex/fmindex.h:294-352)."""

    def __init__(self, bwt_occ: torch.Tensor, ssa: Optional[torch.Tensor], L2, length: int, primary: int,
                 sa_interval: int = 16, ktab: Optional[torch.Tensor] = None, ktab_k: int = 0):
        assert bwt_occ.is_cuda and bwt_occ.data_ptr() % 32 == 0
        self.bwt_occ, self.ssa = bwt_occ, ssa
        self.L2 = [int(v) for v in L2]
        self.length, self.primary = int(length), int(primary)
        self.sa_interval = int(sa_interval)        # 16 = the reference's SA_INT; 1 = full suffix array
        self.ktab, self.ktab_k = ktab, int(ktab_k)  # optional k-mer range table (an extension)
        self.ktab_located = 0                       # 1: 16-byte entries {x, y, SA[x], SA[y]} (build_ktab(k, located=True)); 2: + text context (text=...)
        self.ktab_wide = False                      # with ktab_located == 2: 32-byte entries (nvb_fm_build_ktab_wide)
        self.rows = None                            # with a context table: {SA[r], 16 symbols before SA[r]} per row (nvb_fm_build_rows)

    # -- views ------------------------------------------------------------------------------
    def struct(self) -> FmIndexStruct:
        s = FmIndexStruct()
        s.d_bwt_occ = self.bwt_occ.data_ptr()
        s.d_ssa = self.ssa.data_ptr() if self.ssa is not None else None
        s.length, s.primary = self.length, self.primary
        for i in range(5):
            s.L2[i] = self.L2[i]
        s.sa_interval = self.sa_interval
        s.d_ktab = self.ktab.data_ptr() if self.ktab is not None else None
        s.ktab_k = self.ktab_k if self.ktab is not None else 0
        s.ktab_located = int(self.ktab_located) if self.ktab is not None else 0
        if s.ktab_located == 2 and self.ktab_wide:
            s.ktab_located = 4
        if s.ktab_located in (2, 4) and self.rows is not None:
            s.ktab_located, s.d_rows = s.ktab_located + 1, self.rows.data_ptr()
        return s

    @property
    def device(self):
        return self.bwt_occ.device

    def nbytes(self):
        return (self.bwt_occ.numel() * 4 + (self.ssa.numel() * 4 if self.ssa is not None else 0) +
                (self.ktab.numel() * 4 if self.ktab is not None else 0) + (self.rows.numel() * 4 if self.rows is not None else 0))

    def build_ktab(self, k: int = 12, located: bool = False, text: Optional[torch.Tensor] = None):
        """k-mer range table (4^k x uint2): replaces the first k LF steps of every match().  located=True builds 16-byte entries
        {x, y, SA[x], SA[y]} instead (needs the full suffix array): a seed whose k-mer occurs once or twice is located by the look-up
        itself.  With text (the 2-bit big-endian words the index was built from) one-row entries also carry the 16 symbols before
        SA[x] (nvb_fm_build_ktab_context): such a seed needs no read of the text at all.  With the full suffix array and text, the
        per-row array `rows` (nvb_fm_build_rows, (n + 1) x 8 bytes) is built as well when it fits the device's free memory: seeds whose
        k-mer occurs 3 to 8 times are then resolved by one gather of their rows.  Results are the same with and without it.
        With the full suffix array and text, when a 16-byte table would not fit the device's L2 cache (so that every look-up is a DRAM
        request) and a 32-byte one leaves ROWS_HEADROOM free, the table gets 32-byte entries instead (nvb_fm_build_ktab_wide,
        ktab_wide): the look-up then also carries the contexts of k-mers with 3 to 8 occurrences, and most such seeds need no further
        gather."""
        self.ktab = None                                   # release a previous table (and rows) before allocating the new one
        self.rows = None
        self.ktab_wide = False
        full_text = located and text is not None and self.sa_interval == 1 and self.ssa is not None
        wide = False
        if full_text:
            l2 = torch.cuda.get_device_properties(self.device).L2_cache_size
            free, _ = torch.cuda.mem_get_info(self.device)
            wide = 4 ** k * 16 > l2 and 4 ** k * 32 + ROWS_HEADROOM <= free
        tab = torch.empty((4 ** k, 8 if wide else (4 if located else 2)), dtype=torch.int32, device=self.device)
        s = self.struct()
        if wide:
            assert text.is_cuda and text.dtype == torch.int32
            check(lib().nvb_fm_build_ktab_wide(C.byref(s), C.c_uint32(k), C.c_void_p(text.data_ptr()), C.c_void_p(tab.data_ptr()), _stream()),
                  "nvb_fm_build_ktab_wide")
        elif located and text is not None:
            assert text.is_cuda and text.dtype == torch.int32
            check(lib().nvb_fm_build_ktab_context(C.byref(s), C.c_uint32(k), C.c_void_p(text.data_ptr()), C.c_void_p(tab.data_ptr()), _stream()),
                  "nvb_fm_build_ktab_context")
        elif located:
            check(lib().nvb_fm_build_ktab_located(C.byref(s), C.c_uint32(k), C.c_void_p(tab.data_ptr()), _stream()), "nvb_fm_build_ktab_located")
        else:
            check(lib().nvb_fm_build_ktab(C.byref(s), C.c_uint32(k), C.c_void_p(tab.data_ptr()), _stream()), "nvb_fm_build_ktab")
        self.ktab, self.ktab_k, self.ktab_located = tab, k, (2 if (located and text is not None) else (1 if located else 0))
        self.ktab_wide = wide
        if full_text:
            need = (self.length + 1) * 8
            free, _ = torch.cuda.mem_get_info(self.device)
            if need + ROWS_HEADROOM <= free:
                rows = torch.empty((self.length + 1, 2), dtype=torch.int32, device=self.device)
                check(lib().nvb_fm_build_rows(C.byref(self.struct()), C.c_void_p(text.data_ptr()), C.c_void_p(rows.data_ptr()), _stream()),
                      "nvb_fm_build_rows")
                self.rows = rows
        return self

    # -- construction -----------------------------------------------------------------------
    @staticmethod
    def from_host(bwt_occ: np.ndarray, ssa: Optional[np.ndarray], L2, length, primary, device="cuda", sa_interval=16):
        """upload host arrays laid out as the reference's loader produces them
        (nvbio/io/fmindex/fmindex_impl.cu:263-331)"""
        return FMIndexDevice(_dev_u32(bwt_occ, device), None if ssa is None else _dev_u32(ssa, device), L2, length, primary,
                             sa_interval=sa_interval)

    @staticmethod
    def from_bwt(bwt_words: torch.Tensor, n: int, primary: int, ssa: Optional[torch.Tensor], sa_interval: int = 16):
        """occ table + interleave on the device (replaces build_occurrence_table + the interleave loop)"""
        L = lib()
        n_blocks = (n + 63) // 64
        bwt_occ = torch.empty(n_blocks * 8, dtype=torch.int32, device=bwt_words.device)
        L2 = (C.c_uint32 * 5)()
        tb = C.c_size_t(0)
        r = L.nvb_fm_build_occ(C.c_void_p(bwt_words.data_ptr()), C.c_uint32(n), C.c_void_p(bwt_occ.data_ptr()), L2,
                               None, C.byref(tb), _stream())
        if r != -2:
            check(r, "nvb_fm_build_occ(size query)")
        temp = torch.empty(max(tb.value, 1), dtype=torch.uint8, device=bwt_words.device)
        check(L.nvb_fm_build_occ(C.c_void_p(bwt_words.data_ptr()), C.c_uint32(n), C.c_void_p(bwt_occ.data_ptr()), L2,
                                 C.c_void_p(temp.data_ptr()), C.byref(tb), _stream()), "nvb_fm_build_occ")
        return FMIndexDevice(bwt_occ, ssa, list(L2), n, primary, sa_interval=sa_interval)

    @staticmethod
    def from_text(text_words: torch.Tensor, n: int, want_sa: bool = False, sa_interval: int = 16):
        """suffix-sort a 2-bit big-endian packed text on the device and build the whole index.
        text_words must be readable 2 words past ceil(n/16).  Returns (index, sa or None).
        sa_interval: 16 = the reference's format; smaller powers of two (down to 1) trade HBM for locate steps."""
        L = lib()
        dev = text_words.device
        bwt = torch.empty(((n + 63) // 64) * 4, dtype=torch.int32, device=dev)
        ssa = torch.empty((n + sa_interval) // sa_interval, dtype=torch.int32, device=dev)
        sa = torch.empty(n + 1, dtype=torch.int32, device=dev) if want_sa else None
        primary = C.c_uint32(0)
        tb = C.c_size_t(0)
        args = (C.c_void_p(text_words.data_ptr()), C.c_uint32(n), C.c_void_p(bwt.data_ptr()), C.byref(primary),
                C.c_void_p(ssa.data_ptr()), C.c_uint32(sa_interval), C.c_void_p(sa.data_ptr()) if sa is not None else None)
        r = L.nvb_fm_build_bwt(*args, None, C.byref(tb), _stream())
        if r != -2:
            check(r, "nvb_fm_build_bwt(size query)")
        temp = torch.empty(tb.value, dtype=torch.uint8, device=dev)
        check(L.nvb_fm_build_bwt(*args, C.c_void_p(temp.data_ptr()), C.byref(tb), _stream()), "nvb_fm_build_bwt")
        del temp
        idx = FMIndexDevice.from_bwt(bwt, n, int(primary.value), ssa, sa_interval=sa_interval)
        return idx, sa

    def to_host(self):
        return dict(bwt_occ=_np_u32(self.bwt_occ), ssa=None if self.ssa is None else _np_u32(self.ssa),
                    L2=np.array(self.L2, dtype=np.uint32), n=self.length, primary=self.primary, sa_interval=self.sa_interval)


def rank(fmi: FMIndexDevice, k: torch.Tensor, c: torch.Tensor) -> torch.Tensor:
    """nvbio::rank(fm_index, k, c) for arrays of (k, c); k int32 (uint32 bit pattern), c uint8"""
    n = k.numel()
    out = torch.empty(n, dtype=torch.int32, device=k.device)
    s = fmi.struct()
    check(lib().nvb_fm_rank(C.byref(s), C.c_void_p(k.data_ptr()), C.c_void_p(c.data_ptr()), C.c_uint32(n),
                            C.c_void_p(out.data_ptr()), _stream()), "nvb_fm_rank")
    return out


def rank4(fmi: FMIndexDevice, k: torch.Tensor) -> torch.Tensor:
    """nvbio::rank4(fm_index, k): int32 [n,4] = occurrences of A,C,G,T in rows [0,k]"""
    n = k.numel()
    out = torch.empty((n, 4), dtype=torch.int32, device=k.device)
    s = fmi.struct()
    check(lib().nvb_fm_rank4(C.byref(s), C.c_void_p(k.data_ptr()), C.c_uint32(n), C.c_void_p(out.data_ptr()), _stream()), "nvb_fm_rank4")
    return out


def match(fmi: FMIndexDevice, queries: PackedStringSet, flags: int = 0, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """nvbio::match(fm_index, pattern, len) for a string set -> int32 [n,2] inclusive SA ranges (uint32 bits)"""
    n = queries.count
    if out is None:
        out = torch.empty((n, 2), dtype=torch.int32, device=fmi.device)
    s, q = fmi.struct(), queries.struct()
    check(lib().nvb_fm_match(C.byref(s), C.byref(q), C.c_uint32(n), C.c_uint32(flags),
                             C.c_void_p(out.data_ptr()), _stream()), "nvb_fm_match")
    return out


def match_approx(fmi: FMIndexDevice, queries: PackedStringSet, exact_len: int, find_exact: bool = True, max_out: int = 64, flags: int = 0):
    """nvBowtie's map<find_exact> (one substitution after the first exact_len consumed symbols) for a string set.
    Returns (ranges int32[n,max_out,2], counts int32[n], range_sums int32[n])."""
    n = queries.count
    dev = fmi.device
    ranges = torch.zeros((n, max_out, 2), dtype=torch.int32, device=dev)
    counts = torch.empty(n, dtype=torch.int32, device=dev)
    sums = torch.empty(n, dtype=torch.int32, device=dev)
    s, q = fmi.struct(), queries.struct()
    check(lib().nvb_fm_match_approx(C.byref(s), C.byref(q), C.c_uint32(n), C.c_uint32(flags), C.c_uint32(exact_len),
                                    C.c_int(1 if find_exact else 0), C.c_uint32(max_out), C.c_void_p(ranges.data_ptr()),
                                    C.c_void_p(counts.data_ptr()), C.c_void_p(sums.data_ptr()), _stream()), "nvb_fm_match_approx")
    return ranges, counts, sums


def locate(fmi: FMIndexDevice, rows: torch.Tensor) -> torch.Tensor:
    """nvbio::locate(fm_index, row) for an array of SA rows"""
    n = rows.numel()
    out = torch.empty(n, dtype=torch.int32, device=rows.device)
    s = fmi.struct()
    check(lib().nvb_fm_locate(C.byref(s), C.c_void_p(rows.data_ptr()), C.c_uint32(n), C.c_void_p(out.data_ptr()), _stream()),
          "nvb_fm_locate")
    return out


def dict_rank(text_words: torch.Tensor, occ: torch.Tensor, K: int, i: torch.Tensor, c: Optional[torch.Tensor] = None) -> torch.Tensor:
    """generic rank dictionary (rank_dictionary_inl.h:243-422): text_words / occ / i are int32 or int64 tensors (32- or 64-bit words and
    counters, bit patterns of the unsigned values); returns rank(i, c) [n], or all four symbols [n, 4] when c is None"""
    wb = 32 if text_words.dtype == torch.int32 else 64
    ib = 32 if occ.dtype == torch.int32 else 64
    assert i.dtype == occ.dtype
    n = i.numel()
    if c is None:
        out = torch.empty((n, 4), dtype=occ.dtype, device=i.device)
        check(lib().nvb_dict_rank4(C.c_void_p(text_words.data_ptr()), C.c_uint32(wb), C.c_void_p(occ.data_ptr()), C.c_uint32(ib), C.c_uint32(K),
                                   C.c_void_p(i.data_ptr()), C.c_uint32(n), C.c_void_p(out.data_ptr()), _stream()), "nvb_dict_rank4")
        return out
    out = torch.empty(n, dtype=occ.dtype, device=i.device)
    check(lib().nvb_dict_rank(C.c_void_p(text_words.data_ptr()), C.c_uint32(wb), C.c_void_p(occ.data_ptr()), C.c_uint32(ib), C.c_uint32(K),
                              C.c_void_p(i.data_ptr()), C.c_void_p(c.data_ptr()), C.c_uint32(n), C.c_void_p(out.data_ptr()), _stream()), "nvb_dict_rank")
    return out


def dict_build_occ(text_words: torch.Tensor, n_symbols: int, K: int, index_bits: int = 32):
    """build_occurrence_table<2,K> on the device (rank_dictionary_inl.h:42-77): returns (occ, [count A, C, G, T])"""
    wb = 32 if text_words.dtype == torch.int32 else 64
    n_blocks = (n_symbols + K - 1) // K
    occ = torch.empty(n_blocks * 4, dtype=torch.int32 if index_bits == 32 else torch.int64, device=text_words.device)
    counts = (C.c_uint64 * 4)()
    tb = C.c_size_t(0)
    r = lib().nvb_dict_build_occ(C.c_void_p(text_words.data_ptr()), C.c_uint32(wb), C.c_uint64(n_symbols), C.c_uint32(K), C.c_uint32(index_bits),
                                 C.c_void_p(occ.data_ptr()), counts, None, C.byref(tb), _stream())
    if r != -2:
        check(r, "nvb_dict_build_occ(size query)")
    temp = torch.empty(max(tb.value, 1), dtype=torch.uint8, device=text_words.device)
    check(lib().nvb_dict_build_occ(C.c_void_p(text_words.data_ptr()), C.c_uint32(wb), C.c_uint64(n_symbols), C.c_uint32(K), C.c_uint32(index_bits),
                                   C.c_void_p(occ.data_ptr()), counts, C.c_void_p(temp.data_ptr()), C.byref(tb), _stream()), "nvb_dict_build_occ")
    return occ, [int(v) for v in counts]


MAP_EXACT, MAP_APPROX = 0, 1


class MapParamsStruct(C.Structure):         # nvb_map_params
    _fields_ = [(k, C.c_uint32) for k in ("algorithm", "seed_len", "seed_freq", "max_hits", "max_reseed", "rep_seeds", "subseed_len",
                                          "min_read_len", "fw", "rc")]


def map_seeds(fmi: FMIndexDevice, reads: PackedStringSet, algorithm: int = MAP_EXACT, seed_len: int = 22, seed_freq: int = 10, max_hits: int = 100,
              max_reseed: int = 2, rep_seeds: int = 1000, subseed_len: int = 0, min_read_len: int = 12, fw: bool = True, rc: bool = True,
              queue: Optional[torch.Tensor] = None, retry: int = 0, seed_freq_per_read: Optional[torch.Tensor] = None):
    """nvBowtie's seed mapping stage (map_queues_kernel<EXACT|APPROX>, mapping_inl.h:229-366,539-591) for a read batch.
    Returns (hits int32 [n_reads, max_hits, 2] = (range_begin, packed bits) sorted by range size, counts [n_reads],
    reseed uint8 [n_queue], stats int32 [n_queue, 2] = (range_sum, range_count))."""
    n_reads = reads.count
    n_queue = n_reads if queue is None else queue.numel()
    dev = fmi.device
    hits = torch.zeros((n_reads, max_hits, 2), dtype=torch.int32, device=dev)
    counts = torch.zeros(n_reads, dtype=torch.int32, device=dev)
    reseed = torch.full((n_queue,), 7, dtype=torch.uint8, device=dev)
    stats = torch.zeros((n_queue, 2), dtype=torch.int32, device=dev)
    p = MapParamsStruct(algorithm, seed_len, seed_freq, max_hits, max_reseed, rep_seeds, subseed_len, min_read_len, int(fw), int(rc))
    s, q = fmi.struct(), reads.struct()
    check(lib().nvb_map_seeds(C.byref(s), C.byref(q), C.c_void_p(queue.data_ptr()) if queue is not None else None, C.c_uint32(n_queue), C.c_uint32(retry),
                              C.byref(p), C.c_void_p(seed_freq_per_read.data_ptr()) if seed_freq_per_read is not None else None,
                              C.c_void_p(hits.data_ptr()), C.c_void_p(counts.data_ptr()), C.c_void_p(reseed.data_ptr()), C.c_void_p(stats.data_ptr()),
                              _stream()), "nvb_map_seeds")
    return hits, counts, reseed, stats


def locate_init(fmi: FMIndexDevice, rows: torch.Tensor, idx: Optional[torch.Tensor] = None):
    """first pass of nvBowtie's two-pass locate (locate_inl.h:122-166): (sampled SA row, LF steps) per queued row"""
    n = rows.numel()
    r = torch.empty(n, dtype=torch.int32, device=rows.device); t = torch.empty(n, dtype=torch.int32, device=rows.device)
    s = fmi.struct()
    check(lib().nvb_fm_locate_init(C.byref(s), C.c_void_p(rows.data_ptr()), C.c_void_p(idx.data_ptr()) if idx is not None else None, C.c_uint32(n),
                                   C.c_void_p(r.data_ptr()), C.c_void_p(t.data_ptr()), _stream()), "nvb_fm_locate_init")
    return r, t


def locate_lookup(fmi: FMIndexDevice, sampled_rows: torch.Tensor, steps: torch.Tensor, idx: Optional[torch.Tensor] = None) -> torch.Tensor:
    """second pass (locate_inl.h:168-210): ssa[row / SA_INT] + steps"""
    n = sampled_rows.numel()
    out = torch.empty(n, dtype=torch.int32, device=sampled_rows.device)
    s = fmi.struct()
    check(lib().nvb_fm_locate_lookup(C.byref(s), C.c_void_p(sampled_rows.data_ptr()), C.c_void_p(steps.data_ptr()),
                                     C.c_void_p(idx.data_ptr()) if idx is not None else None, C.c_uint32(n), C.c_void_p(out.data_ptr()), _stream()),
          "nvb_fm_locate_lookup")
    return out


def locate_sorted(fmi: FMIndexDevice, rows: torch.Tensor) -> torch.Tensor:
    """locate() with the SA rows radix-sorted first to gather locality (aligner_best_approx.h:737-756); positions in input order"""
    n = rows.numel()
    out = torch.empty(n, dtype=torch.int32, device=rows.device)
    s = fmi.struct()
    tb = C.c_size_t(0)
    r = lib().nvb_fm_locate_sorted(C.byref(s), C.c_void_p(rows.data_ptr()), C.c_uint32(n), C.c_void_p(out.data_ptr()), None, C.byref(tb), _stream())
    if r != -2:
        check(r, "nvb_fm_locate_sorted(size query)")
    temp = torch.empty(max(tb.value, 1), dtype=torch.uint8, device=rows.device)
    check(lib().nvb_fm_locate_sorted(C.byref(s), C.c_void_p(rows.data_ptr()), C.c_uint32(n), C.c_void_p(out.data_ptr()), C.c_void_p(temp.data_ptr()),
                                     C.byref(tb), _stream()), "nvb_fm_locate_sorted")
    return out


class FMIndexFilterDevice:
    """nvbio::FMIndexFilter<device_tag, fm_index_type> (nvbio/fmindex/filter.h:145-214):
    rank() -> n_hits, then ranges()/slots()/n_hits() and locate(begin, end) -> (text pos, query id) hits."""

    def __init__(self):
        self._fmi = None
        self._ranges = None
        self._slots = None
        self._n_hits = 0
        self._n_queries = 0

    def rank(self, fm_index: FMIndexDevice, string_set: PackedStringSet, flags: int = 0) -> int:
        L = lib()
        n = string_set.count
        dev = fm_index.device
        self._fmi, self._n_queries = fm_index, n
        self._ranges = torch.empty((n, 2), dtype=torch.int32, device=dev)
        self._slots = torch.empty(n, dtype=torch.int64, device=dev)
        n_hits = C.c_uint64(0)
        tb = C.c_size_t(0)
        s, q = fm_index.struct(), string_set.struct()
        r = L.nvb_fm_filter_rank(C.byref(s), C.byref(q), C.c_uint32(n), C.c_uint32(flags), C.c_void_p(self._ranges.data_ptr()),
                                 C.c_void_p(self._slots.data_ptr()), C.byref(n_hits), None, C.byref(tb), _stream())
        if r != -2:
            check(r, "nvb_fm_filter_rank(size query)")
        temp = torch.empty(max(tb.value, 1), dtype=torch.uint8, device=dev)
        check(L.nvb_fm_filter_rank(C.byref(s), C.byref(q), C.c_uint32(n), C.c_uint32(flags), C.c_void_p(self._ranges.data_ptr()),
                                   C.c_void_p(self._slots.data_ptr()), C.byref(n_hits), C.c_void_p(temp.data_ptr()),
                                   C.byref(tb), _stream()), "nvb_fm_filter_rank")
        self._n_hits = int(n_hits.value)
        return self._n_hits

    def n_hits(self):
        return self._n_hits

    def ranges(self):
        return self._ranges

    def slots(self):
        return self._slots

    def locate(self, begin: int, end: int, hits: Optional[torch.Tensor] = None) -> torch.Tensor:
        if self._fmi is None:
            raise NvbError("FMIndexFilterDevice.locate() before rank()")
        if not (0 <= begin <= end <= self._n_hits):
            raise NvbError("FMIndexFilterDevice.locate: [begin, end) must lie inside [0, n_hits()]")
        if hits is None:
            hits = torch.empty((end - begin, 2), dtype=torch.int32, device=self._fmi.device)
        s = self._fmi.struct()
        check(lib().nvb_fm_filter_locate(C.byref(s), C.c_void_p(self._ranges.data_ptr()), C.c_void_p(self._slots.data_ptr()),
                                         C.c_uint32(self._n_queries), C.c_uint64(begin), C.c_uint64(end),
                                         C.c_void_p(hits.data_ptr()), _stream()), "nvb_fm_filter_locate")
        return hits
