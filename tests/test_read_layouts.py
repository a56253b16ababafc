"""CPU: the read layouts of tests/read_layouts.py decode back, through the header's string-set rule, to the reads and qualities they were
built from, and poison everything else; the map_seeds entry point refuses little-endian reads before any CUDA call."""
import ctypes as C
import numpy as np
import pytest
from nvbio_b200.strings import unpack_symbols
from tests import read_layouts as rl


def reads_of(rng, n, lo, hi, bits):
    reads = [rng.integers(0, 4, int(rng.integers(lo, hi + 1))).astype(np.uint8) for _ in range(n)]
    if bits == 4:
        for r in reads[::5]:
            r[rng.integers(0, len(r), 2)] = 4
    quals = [rng.integers(2, 41, len(r)).astype(np.uint8) for r in reads]
    return reads, quals


def decode(h: rl.HostLayout):
    """every string of the set by the header's rule: off_i = offsets ? offsets[i] : i * stride, len_i = lengths ? lengths[i] : length
    (uint32 arithmetic), as symbols and as quals[off_i + p]"""
    offsets, lengths, stride, length = h.set_fields()
    n, spw = len(h.lens), 32 // h.bits
    sym = unpack_symbols(h.words, len(h.words) * spw, h.bits, h.big_endian)
    out = []
    for i in range(n):
        off = int(offsets[i]) if offsets is not None else (i * stride) & 0xFFFFFFFF
        ln = int(lengths[i]) if lengths is not None else length
        out.append((off, sym[off:off + ln], h.quals[off:off + ln]))
    return sym, out


def check_layout(h: rl.HostLayout, reads, quals, layout):
    sym, got = decode(h)
    spw = 32 // h.bits
    inside = np.zeros(len(sym), bool)
    for i, (off, s, q) in enumerate(got):
        assert np.array_equal(s, reads[i]) and np.array_equal(q, quals[i]), (layout, i)
        inside[off:off + len(s)] = True
    out_s, out_q = sym[~inside], h.quals[~inside]
    if layout == "concat":
        assert not out_s.any()                                              # from_symbols' zero padding
        return
    # outside the reads: random symbols (every value, 4-bit nibbles 5-15 included) and random quality bytes, the padding words too
    vals = np.unique(out_s)
    assert vals.max() < 1 << h.bits and len(vals) >= min(1 << h.bits, len(out_s) // 4), layout
    assert (out_s == 0).mean() < 2.0 / (1 << h.bits), layout
    assert len(np.unique(out_q)) >= min(200, len(out_q) // 2) and (out_q == 0).sum() <= max(2, len(out_q) // 20), layout
    last = max(off + len(s) for off, s, _ in got)
    tail = sym[last:]
    assert len(tail) >= rl.PAD_WORDS * spw and (tail != 0).mean() > 0.5, layout
    if layout not in ("concat", "slack"):
        phases = {off % spw for off, _, _ in got}
        assert phases == set(range(spw)), (layout, sorted(phases))


@pytest.mark.parametrize("bits", [2, 4])
@pytest.mark.parametrize("be", [True, False])
@pytest.mark.parametrize("layout", [l for l in rl.LAYOUTS if l != "high"])
def test_layout_decodes_to_its_reads(bits, be, layout):
    rng = np.random.default_rng(bits * 10 + be)
    fixed = layout in rl.FIXED_ONLY
    reads, quals = reads_of(rng, 120, 60 if fixed else 20, 60, bits)
    if layout == "aliased":
        reads, quals = rl.with_aliases(reads, quals, rng, every=5, min_len=10)
    h = rl.build_host(reads, quals, bits, be, layout, np.random.default_rng(3))
    check_layout(h, reads, quals, layout)
    p = h.place
    if layout == "aliased":
        # copies share their source's offset and length; infixes start inside another read's span
        spans = list(zip(p.off.tolist(), h.lens.tolist()))
        copies = sum(spans[i] in spans[:i] for i in range(len(spans)))
        infixes = sum(any(o < oi < o + ln and oi + li <= o + ln for o, ln in spans) for oi, li in spans)
        assert copies >= 5 and infixes >= 5, (copies, infixes)
    if layout == "slack":
        assert p.length == max(len(r) for r in reads) + 32 // bits
    if layout == "stride_odd":
        assert p.stride % 2 == 1 and p.stride > p.length and p.lengths
    if layout == "fixed":
        assert not p.offsets and not p.lengths and p.stride > p.length
    if layout == "offsets_only":
        assert p.offsets and not p.lengths
        assert not np.all(np.diff(p.off) > 0)                               # a permuted storage order
    if layout == "sparse":
        gaps = np.diff(np.sort(p.off)) - h.lens[np.argsort(p.off)][:-1]
        assert gaps.min() >= 0 and gaps.max() <= 40
        assert not np.all(np.diff(p.off) > 0)
    if layout == "mates_interleaved":
        n = len(reads) // 2
        order = np.argsort(p.off)                                           # storage: mate 1 of pair p, then its mate 2
        assert np.array_equal(order[0::2], np.arange(n)) and np.array_equal(order[1::2], np.arange(n) + n)


@pytest.mark.parametrize("bits", [2, 4])
@pytest.mark.parametrize("be", [True, False])
def test_high_patch_routine_at_a_small_base(bits, be):
    """high's fill at a 2^16-symbol stream: random words, each read's words patched in place; reads in two clusters, one just above half
    the stream and one ending on its last symbol"""
    rng = np.random.default_rng(bits + 2 * be)
    reads, quals = reads_of(rng, 80, 20, 60, bits)
    top = 1 << 16
    h = rl.build_host(reads, quals, bits, be, "high", np.random.default_rng(5), top=top)
    check_layout(h, reads, quals, "high")
    off = h.place.off
    assert off.min() >= top // 2 and (off + h.lens).max() == top
    # the patch leaves every symbol outside the reads as it was
    spw = 32 // bits
    poison = rl.pack_symbols(np.random.default_rng(0).integers(0, 1 << bits, top).astype(np.uint8), bits, be, pad_words=0)
    idx = rl.touched_words(off, h.lens, bits)
    patched = poison.copy()
    patched[idx] = rl.patch_words(idx, poison[idx], off, reads, bits, be)
    sym0, sym1 = unpack_symbols(poison, top, bits, be), unpack_symbols(patched, top, bits, be)
    inside = np.zeros(top, bool)
    for o, r in zip(off, reads):
        inside[o:o + len(r)] = True
        assert np.array_equal(sym1[o:o + len(r)], r)
    assert np.array_equal(sym0[~inside], sym1[~inside])
    assert len(idx) <= sum(len(r) // spw + 2 for r in reads)


def test_high_offsets_reach_the_top_of_uint32():
    rng = np.random.default_rng(1)
    reads, quals = reads_of(rng, 64, 80, 150, 2)
    p = rl.place(reads, quals, "high", 2, rng)
    lens = np.array([len(r) for r in reads])
    assert p.off.min() >= 1 << 31 and (p.off + lens).max() == 1 << 32
    assert np.all(p.off.astype(np.uint32).view(np.int32) < 0)               # the sign bit of the int32 offsets tensor


def test_map_seeds_refuses_little_endian_reads():
    """nvb_map_seeds reads big-endian strings only: little-endian 2- and 4-bit reads (and 8-bit ones) are NVB_E_UNSUPPORTED, answered
    before any CUDA call; big-endian reads pass the checks (an empty queue then returns NVB_OK without a launch)"""
    from nvbio_b200 import _lib
    from nvbio_b200._lib import StringSetStruct, FmIndexStruct
    from nvbio_b200.fmindex import MapParamsStruct
    L = _lib.lib()
    fm = FmIndexStruct(); fm.d_bwt_occ = 32; fm.d_ssa = 32; fm.length = 1000; fm.primary = 5; fm.sa_interval = 16
    mp = MapParamsStruct(); mp.algorithm = 0; mp.seed_len = 20; mp.seed_freq = 10; mp.max_hits = 100; mp.fw = mp.rc = 1

    def call(bits, be, n_queue):
        s = StringSetStruct(); s.d_words = 16; s.bits = bits; s.big_endian = 1 if be else 0; s.stride = 160; s.length = 150
        return L.nvb_map_seeds(C.byref(fm), C.byref(s), None, C.c_uint32(n_queue), C.c_uint32(0), C.byref(mp), None, C.c_void_p(16),
                               C.c_void_p(16), None, None, None)
    for bits in (2, 4):
        assert call(bits, False, 8) == -4 and call(bits, False, 0) == -4, bits
        assert call(bits, True, 0) == 0, bits
    assert call(8, True, 8) == -4 and call(8, False, 0) == -4
