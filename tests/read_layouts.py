"""Read layouts of the C ABI's string sets (include/nvbio_b200.h, nvb_string_set), for tests of every entry point that reads caller
strings.  String i = symbols [off_i, off_i + len_i) of one packed stream, off_i = offsets[i] or i * stride, len_i = lengths[i] or length,
2- or 4-bit symbols of either endianness; base qualities are indexed like the symbols (quals[off_i + p]).

build(reads, quals, bits, big_endian, layout) stores the same reads in one of LAYOUTS:
  concat             PackedStringSet.from_symbols: big-endian or not, tightly concatenated, zero words after the last read
  stride_odd         no offsets; an odd stride a few symbols above the longest read; lengths only for a ragged batch
  fixed              no offsets, no lengths, an odd stride above the length (equal-length reads only)
  offsets_only       offsets, no lengths (equal-length reads only)
  sparse             offsets in a permuted storage order with gaps of 0-40 symbols
  aliased            as sparse, but a read whose symbols and qualities already lie in the stream (a copy or an infix of an earlier read)
                     is pointed there instead of stored again
  mates_interleaved  paired batches: index order stays mate 1 of every pair, then mate 2; storage puts the two mates of a pair side by side
  high               offsets at or above 2^31, the last read's last symbol at 2^32 - 1
  slack              concat's offsets with `length` one word above the longest read
Every layout but concat is poisoned: each symbol and quality byte that belongs to no read is random, 4-bit nibbles 5-15 included, and
so are the words after the last read.  Every layout with offsets or a stride starts its reads at every phase modulo the symbols per word
(given at least that many reads).  high fills 2^32 symbols and a 4 GiB quality buffer with torch.randint on the device and writes each
read's few words in place (patch_words)."""
from dataclasses import dataclass
from typing import List, Optional
import numpy as np
import torch
from nvbio_b200.strings import PackedStringSet, pack_symbols

LAYOUTS = ("concat", "stride_odd", "fixed", "offsets_only", "sparse", "aliased", "mates_interleaved", "high", "slack")
FIXED_ONLY = ("fixed", "offsets_only")          # layouts without a lengths array
PAD_WORDS = 4                                   # words after the last read (pack_symbols' padding), poisoned
TOP = 1 << 32                                   # high: the stream's symbol count


@dataclass
class Placement:
    """where a layout puts every read: off[i] (symbol offset), and the set's fields"""
    off: np.ndarray                  # int64, per read
    offsets: bool
    lengths: bool
    stride: int
    length: int
    n_symbols: int                   # symbols of the stream before the padding words


@dataclass
class HostLayout:
    """a layout on the host: words (uint32, padding included) and quals (uint8, one per stream symbol), with the set's fields"""
    words: np.ndarray
    quals: np.ndarray
    place: Placement
    lens: np.ndarray
    bits: int
    big_endian: bool

    def set_fields(self):
        p = self.place
        return (p.off.astype(np.uint32) if p.offsets else None, self.lens.astype(np.uint32) if p.lengths else None, p.stride, p.length)


def _spw(bits):
    return 32 // bits


def odd_stride(L, extra=3):
    s = L + extra
    return s + 1 if s % 2 == 0 else s


def _phase_gaps(rng, n, spw):
    """gap(cur, k): the 0-40 symbols to skip at stream position cur so that the k-th of n strings starts at phase targets[k] mod spw,
    the targets a shuffle of k mod spw"""
    targets = rng.permutation(np.arange(n) % spw)
    return lambda cur, k: ((int(targets[k]) - cur) % spw) + spw * int(rng.integers(0, (40 - spw) // spw + 1))


def _packed_run(rng, lens_in_order, spw, start=0):
    """symbol offsets of strings of the given lengths stored in this order, every start phase mod spw present"""
    gap = _phase_gaps(rng, len(lens_in_order), spw)
    out, cur = [], start
    for k, L in enumerate(lens_in_order):
        cur += gap(cur, k)
        out.append(cur)
        cur += int(L)
    return np.array(out, np.int64), cur


def with_aliases(reads: List[np.ndarray], quals: List[np.ndarray], rng, every=9, min_len=40):
    """copies of the reads with some of them replaced by a copy of an earlier read or by an infix of one (qualities alike), so that the
    aliased layout has strings to share: every `every`-th read from read 4 on, copies and infixes alternating"""
    reads, quals = [r.copy() for r in reads], [q.copy() for q in quals]
    for k, i in enumerate(range(4, len(reads), every)):
        j = int(rng.integers(0, i))
        if k % 2 == 0 or len(reads[j]) <= min_len:
            reads[i], quals[i] = reads[j].copy(), quals[j].copy()
        else:
            L = int(rng.integers(min_len, len(reads[j])))
            a = int(rng.integers(0, len(reads[j]) - L + 1))
            reads[i], quals[i] = reads[j][a:a + L].copy(), quals[j][a:a + L].copy()
    return reads, quals


def place(reads, quals, layout, bits, rng, top=TOP) -> Placement:
    """the placement of `layout` (every layout but high's fill; aliased needs the reads and qualities to find its shared strings)"""
    lens = np.array([len(r) for r in reads], np.int64)
    n, spw, L = len(reads), _spw(bits), int(lens.max()) if len(reads) else 0
    ragged = bool(len(reads)) and bool((lens != lens[0]).any())
    if layout in ("concat", "slack"):
        off = np.cumsum(lens) - lens
        return Placement(off, True, True, 0, L + (spw if layout == "slack" else 0), int(lens.sum()))
    if layout in ("stride_odd", "fixed"):
        if layout == "fixed" and ragged:
            raise ValueError("the fixed layout takes equal-length reads")
        s = odd_stride(L, 3 if layout == "stride_odd" else 8)
        return Placement(np.arange(n, dtype=np.int64) * s, False, layout == "stride_odd" and ragged, s, L, n * s)
    if layout in ("offsets_only", "sparse"):
        if layout == "offsets_only" and ragged:
            raise ValueError("the offsets_only layout takes equal-length reads")
        order = rng.permutation(n)
        o, end = _packed_run(rng, lens[order], spw)
        off = np.empty(n, np.int64); off[order] = o
        return Placement(off, True, layout == "sparse", 0, L, end)
    if layout == "mates_interleaved":
        if n % 2:
            raise ValueError("the mates_interleaved layout takes paired batches")
        h = n // 2
        order = np.stack([np.arange(h), h + np.arange(h)], axis=1).reshape(-1)        # pair p: mate 1, then mate 2
        o, end = _packed_run(rng, lens[order], spw)
        off = np.empty(n, np.int64); off[order] = o
        return Placement(off, True, True, 0, L, end)
    if layout == "aliased":
        # place reads in index order after a phase-targeted gap, unless their symbols (and qualities) already lie in the stream; gaps
        # hold 255 here, so that no match runs across one (the stream's gaps are random)
        sym = np.full(int(lens.sum()) + 41 * n + 1, 255, np.uint8)
        qb = np.zeros_like(sym)
        gap = _phase_gaps(rng, n, spw)
        off, cur, k = np.zeros(n, np.int64), 0, 0
        for i, r in enumerate(reads):
            hay, needle, at, found = sym[:cur].tobytes(), r.tobytes(), 0, -1
            while len(r):
                at = hay.find(needle, at)
                if at < 0:
                    break
                if quals is None or np.array_equal(qb[at:at + len(r)], quals[i]):
                    found = at
                    break
                at += 1
            if found >= 0:
                off[i] = found
                continue
            cur += gap(cur, k); k += 1
            off[i] = cur
            sym[cur:cur + len(r)] = r
            if quals is not None:
                qb[cur:cur + len(r)] = quals[i]
            cur += len(r)
        return Placement(off, True, True, 0, L, cur)
    if layout == "high":
        # two clusters: one just above 2^31, one ending at the top of the stream
        order = rng.permutation(n)
        a, b = order[:n // 2], order[n // 2:]
        o1, _ = _packed_run(rng, lens[a], spw, start=top // 2 + 5)
        o2, end2 = _packed_run(rng, lens[b], spw)
        off = np.empty(n, np.int64); off[a] = o1; off[b] = o2 + (top - end2)
        return Placement(off, True, True, 0, L, top)
    raise ValueError("unknown layout %r" % (layout,))


def patch_words(idx: np.ndarray, vals: np.ndarray, off: np.ndarray, reads, bits, big_endian) -> np.ndarray:
    """the words idx (sorted, unique) with values vals after writing read i's symbols at symbol off[i], for every read: high's in-place
    write of a few words of a stream too large to pack on the host"""
    spw = _spw(bits)
    mask = (1 << bits) - 1
    vals = vals.astype(np.uint32).copy()
    if not len(reads):
        return vals
    p = np.concatenate([int(o) + np.arange(len(r), dtype=np.int64) for o, r in zip(off, reads)])
    c = np.concatenate([np.asarray(r, np.uint32) for r in reads]) & np.uint32(mask)
    w = np.searchsorted(idx, p // spw)
    assert np.array_equal(idx[np.minimum(w, len(idx) - 1)], p // spw), "patch_words: a read's word is missing from idx"
    k = (p % spw).astype(np.uint32)
    sh = (32 - bits - bits * k) if big_endian else (bits * k)
    np.bitwise_and.at(vals, w, ~(np.uint32(mask) << sh))
    np.bitwise_or.at(vals, w, c << sh)
    return vals


def touched_words(off, lens, bits):
    spw = _spw(bits)
    return np.unique(np.concatenate([np.arange(int(o) // spw, (int(o) + int(L) - 1) // spw + 1, dtype=np.int64)
                                     for o, L in zip(off, lens) if L] or [np.zeros(0, np.int64)]))


def build_host(reads, quals, bits, big_endian, layout, rng, top=None) -> HostLayout:
    """the layout on the host.  high only with a small `top` (the stream's symbol count): the routine that writes the reads into the
    device's random words, on a host array"""
    lens = np.array([len(r) for r in reads], np.int64)
    if layout == "high":
        if top is None:
            raise ValueError("build_host: high needs a small top; build() fills the device")
        p = place(reads, quals, "high", bits, rng, top=top)
    else:
        p = place(reads, quals, layout, bits, rng)
    spw = _spw(bits)
    nw = -(-p.n_symbols // spw) + PAD_WORDS
    if layout == "concat":
        sym = np.zeros(nw * spw, np.uint8)
        q = np.zeros(nw * spw, np.uint8)
    else:
        sym = rng.integers(0, 1 << bits, nw * spw).astype(np.uint8)
        q = rng.integers(0, 256, nw * spw).astype(np.uint8)
    if layout == "high":
        words = pack_symbols(sym, bits, big_endian, pad_words=0)
        idx = touched_words(p.off, lens, bits)
        words[idx] = patch_words(idx, words[idx], p.off, reads, bits, big_endian)
    else:
        for o, r in zip(p.off, reads):
            sym[o:o + len(r)] = r
        words = pack_symbols(sym, bits, big_endian, pad_words=0)
    for o, qq in zip(p.off, quals if quals is not None else []):
        q[o:o + len(qq)] = qq
    return HostLayout(words=words, quals=q, place=p, lens=lens, bits=bits, big_endian=big_endian)


@dataclass
class DeviceLayout:
    reads: PackedStringSet
    quals: Optional[torch.Tensor]
    off: np.ndarray                  # int64 symbol offset of every read
    name: str


def _set(words, p: Placement, lens, bits, big_endian, dev):
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.uint32).view(np.int32)).to(dev)     # noqa: E731
    return PackedStringSet(words=words, bits=bits, big_endian=big_endian, offsets=t(p.off) if p.offsets else None,
                           lengths=t(lens) if p.lengths else None, stride=p.stride, length=p.length, count=len(lens))


def build(reads, quals, bits, big_endian, layout, seed=0, device="cuda") -> DeviceLayout:
    """the reads (and qualities, or None) stored in `layout` on the device"""
    rng = np.random.default_rng(seed)
    lens = np.array([len(r) for r in reads], np.int64)
    if layout != "high":
        h = build_host(reads, quals, bits, big_endian, layout, rng)
        words = torch.from_numpy(h.words.view(np.int32)).to(device)
        q = torch.from_numpy(h.quals).to(device) if quals is not None else None
        return DeviceLayout(_set(words, h.place, lens, bits, big_endian, device), q, h.place.off, layout)
    p = place(reads, quals, "high", bits, rng)
    gen = torch.Generator(device=device)
    gen.manual_seed(seed)
    nw = TOP // _spw(bits) + PAD_WORDS
    words = torch.randint(0, 256, (4 * nw,), dtype=torch.uint8, device=device, generator=gen).view(torch.int32)
    idx = touched_words(p.off, lens, bits)
    it = torch.from_numpy(idx).to(device)
    vals = words[it].cpu().numpy().view(np.uint32)
    words[it] = torch.from_numpy(patch_words(idx, vals, p.off, reads, bits, big_endian).view(np.int32)).to(device)
    q = None
    if quals is not None:
        q = torch.randint(0, 256, (TOP,), dtype=torch.uint8, device=device, generator=gen)
        qi = np.concatenate([int(o) + np.arange(len(qq), dtype=np.int64) for o, qq in zip(p.off, quals)])
        q[torch.from_numpy(qi).to(device)] = torch.from_numpy(np.concatenate(quals)).to(device)
    return DeviceLayout(_set(words, p, lens, bits, big_endian, device), q, p.off, layout)


def layouts_for(paired: bool, fixed_len: bool):
    """the layouts a batch can take: the fixed-length ones need equal lengths, mates_interleaved a paired batch"""
    return tuple(l for l in LAYOUTS if (fixed_len or l not in FIXED_ONLY) and (paired or l != "mates_interleaved"))
