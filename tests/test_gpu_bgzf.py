"""-m gpu: nvb_bgzf_compress on the device.  Round trips at sizes around the block and match-length edges on zero, 0xFF, random, periodic,
3-byte-match, Fibonacci-skewed, single-byte and match-free inputs: every member's header, BSIZE, CRC32, ISIZE and size bound, gzip of the
whole stream, and every member byte-equal to the host build of the same routines (tests/host/bgzf_harness.cu).  Determinism across calls,
streams and grid sizes.  BAM: seed_extend(_paired) -> finish_alignments -> bam_records -> bgzf_compress -> write_bam reads back through
gzip to the host path's bytes and through htslib (where oracle/_ref is built) to its SAM text, at >= 0.9x zlib level 1's ratio.  A capacity
that cuts mid-stream; n = 0."""
import ctypes as C
import gzip
import zlib
import numpy as np
import pytest
import torch
import nvbio_b200 as nb
from nvbio_b200 import aln
from nvbio_b200.pipeline import MapqParams
from oracle.ref_bam import RefBam
from tests.gpu_util import require_gpu
from tests.test_bgzf_host import H, BLOCK, EOF_BLOCK, check_member, find_matches, member, fib  # noqa: F401  (H: the host harness fixture)
from tests.test_gpu_finish import se_world, read_set  # noqa: F401  (the single-end world fixture)
from tests.test_gpu_paired_traceback import world, run as run_paired  # noqa: F401  (the paired world fixture)

SIZES = [0, 1, 2, 3, 257, 258, 259, 0xFEFF, 0xFF00, 0xFF01, 2 * 0xFF00, 2 * 0xFF00 + 1, 10_000_000]
KINDS = ["zeros", "ff", "random"] + ["period_%d" % p for p in (1, 2, 3, 4, 7, 258, 259, 32768, 32769)] + \
        ["three_byte_matches", "fibonacci", "single_byte", "no_match"]


def make(kind, n, seed=0):
    rng = np.random.default_rng(seed + n)
    if kind == "zeros":
        return bytes(n)
    if kind == "ff":
        return b"\xff" * n
    if kind == "random":
        return rng.integers(0, 256, n, dtype=np.uint8).tobytes()
    if kind.startswith("period_"):
        p = int(kind[7:])
        return np.resize(rng.integers(0, 256, p, dtype=np.uint8), n).tobytes()
    if kind == "three_byte_matches":
        tri = rng.integers(0, 256, (4, 3), dtype=np.uint8)
        k = -(-n // 6)
        fresh = rng.integers(0, 256, (k, 3), dtype=np.uint8)
        return np.concatenate([tri[rng.integers(0, 4, k)], fresh], axis=1).reshape(-1)[:n].tobytes()
    if kind == "fibonacci":
        w = np.array(fib(20), np.float64)
        return (rng.choice(20, n, p=w / w.sum()).astype(np.uint8) * 13).tobytes()
    if kind == "single_byte":
        return b"\x2a" * n
    if kind == "no_match":                                       # the 16-bit counter: hardly a 3-byte window repeats within a block
        i = np.arange(-(-n // 2))
        return np.stack([(i >> 8) & 0xFF, i & 0xFF], axis=1).reshape(-1)[:n].astype(np.uint8).tobytes()
    raise ValueError(kind)


def dev(data: bytes) -> torch.Tensor:
    return torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda() if data else torch.empty(0, dtype=torch.uint8, device="cuda")


def check_stream(b, data, H=None):
    torch.cuda.synchronize()
    nbk = -(-len(data) // BLOCK)
    off = b.offsets.cpu().numpy()
    assert b.n_blocks == nbk and b.stored() == nbk and off[0] == 0 and (np.diff(off) > 0).all()
    z = b.to_bytes()
    assert len(z) == off[-1]
    for i in range(nbk):
        blk = data[i * BLOCK:(i + 1) * BLOCK]
        m = z[off[i]:off[i + 1]]
        check_member(m, blk)
        if H is not None:
            want, _ = member(H, blk, find_matches(H, blk), 0)
            assert m == want, i
    assert gzip.decompress(z + EOF_BLOCK) == data
    return z


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_round_trip(H, kind):
    require_gpu()
    for n in SIZES:
        if n > 3 * BLOCK and kind not in ("random", "zeros", "period_3", "fibonacci", "period_32769"):
            continue
        data = make(kind, n)
        b = nb.bgzf_compress(dev(data))
        z = check_stream(b, data, H if n <= 3 * BLOCK else None)
        off = b.offsets.cpu().numpy()
        if kind == "random":                                     # the stored fallback
            assert (np.diff(off) == np.minimum(BLOCK, n - BLOCK * np.arange(len(off) - 1)) + 31).all()
        if kind in ("zeros", "ff", "single_byte", "period_1") and n >= BLOCK:
            assert off[1] < 1000
        if kind == "period_32769" and n >= BLOCK:                # distance 32769 is out of the window: no gain on the first repeat
            assert len(z) > 0.4 * n


@pytest.mark.gpu
def test_determinism():
    require_gpu()
    from nvbio_b200._lib import lib
    rng = np.random.default_rng(9)
    parts = [make(k, int(rng.integers(1, 200_000)), int(s)) for s, k in enumerate(KINDS * 3)]
    data = b"".join(parts)
    x = dev(data)
    call = nb.BgzfCall(x)
    a = call.run().to_bytes()
    assert call.run().to_bytes() == a
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        c = nb.bgzf_compress(x, stream=side)
    side.synchronize()
    assert c.to_bytes() == a
    try:
        lib().nvb_debug_bgzf_grid(C.c_uint32(3))
        d = nb.BgzfCall(x).run().to_bytes()
    finally:
        lib().nvb_debug_bgzf_grid(C.c_uint32(0))
    assert d == a
    assert gzip.decompress(a + EOF_BLOCK) == data


@pytest.mark.gpu
def test_capacity_and_empty():
    require_gpu()
    data = make("fibonacci", 5 * BLOCK + 100)
    x = dev(data)
    full = nb.bgzf_compress(x)
    off = full.offsets.cpu().numpy()
    for cap in (0, int(off[1]) - 1, int(off[3]) + 7, int(off[-1]) - 1, int(off[-1])):
        cut = nb.BgzfCall(x, capacity=cap).run()
        torch.cuda.synchronize()
        k = int(np.searchsorted(off[1:], cap, side="right"))
        assert torch.equal(cut.offsets, full.offsets) and cut.stored() == k
        assert cut.to_bytes() == full.to_bytes()[:int(off[k])]
    with pytest.raises(ValueError):
        nb.write_bam("/dev/null", b"", [nb.BgzfCall(x, capacity=int(off[2])).run()])
    e = nb.bgzf_compress(torch.empty(0, dtype=torch.uint8, device="cuda"))
    torch.cuda.synchronize()
    assert e.n_blocks == 0 and e.offsets.cpu().tolist() == [0] and e.to_bytes() == b""


def zlib1_size(data):
    s = 0
    for i in range(0, len(data), BLOCK):
        c = zlib.compressobj(1, zlib.DEFLATED, -15)
        s += len(c.compress(data[i:i + BLOCK]) + c.flush()) + 26
    return s


def check_bam(recs, contigs, tmp_path, tag):
    """the device-compressed file against the host path's: same content through gzip and htslib; ratio >= 0.9 x zlib level 1's"""
    header = nb.bam_header(contigs)
    ph, pd = str(tmp_path / (tag + "_host.bam")), str(tmp_path / (tag + "_dev.bam"))
    nb.write_bam(ph, header, [recs])
    blocks = nb.bgzf_compress(recs)
    nb.write_bam(pd, header, [blocks])
    raw = recs.to_bytes()
    assert gzip.decompress(open(pd, "rb").read()) == gzip.decompress(open(ph, "rb").read())
    if RefBam.available():
        assert RefBam().format(pd) == RefBam().format(ph)
    assert blocks.n_input == len(raw)
    assert int(blocks.offsets[-1]) <= zlib1_size(raw) / 0.9, (int(blocks.offsets[-1]), zlib1_size(raw))


@pytest.mark.gpu
@pytest.mark.parametrize("bits", [2, 4])
@pytest.mark.parametrize("qual", [False, True])
def test_bam_single_end(se_world, bits, qual, tmp_path):
    require_gpu()
    w = se_world
    rng = np.random.default_rng(41 + bits)
    reads = [r.copy() for r in w["reads"]]
    if bits == 4:
        for r in reads:
            r[rng.random(len(r)) < 0.005] = 4
    rs = read_set(reads, bits)
    q = torch.from_numpy(np.concatenate(w["quals"])).cuda() if qual else None
    scheme = aln.SimpleGotohScheme(2, -2, -5, -3)
    params = nb.SeedExtendParams(seed_len=20, seed_interval=10, band_len=31, type=aln.LOCAL, both_strands=True, max_seed_hits=50, scheme=scheme)
    ws = nb.seed_extend(w["fmi"], w["gw"], rs, params, traceback=True, mapq=MapqParams.local(160), hit_capacity=64 * len(reads))
    f = nb.finish_alignments(w["gw"], rs, ws.best_ops, ws.best_n_ops, ws.best_begin, ws.best_strand, genome_len=w["G"])
    contigs = nb.ContigTable(["c0", "c1", "c2"], [w["G"] // 3, w["G"] // 3, w["G"] - 2 * (w["G"] // 3)])
    recs = nb.bam_records(ws, f, rs, contigs, nb.numbered_names(len(reads), "se"), quals=q)
    check_bam(recs, contigs, tmp_path, "se%d%d" % (bits, qual))


@pytest.mark.gpu
@pytest.mark.parametrize("qual", [False, True])
def test_bam_paired(world, qual, tmp_path):
    require_gpu()
    w = world
    pair = nb.PairParams(min_frag=0, max_frag=420, min_mate_score=50)
    _, ws = run_paired(w, pair, qual=qual, mapq=MapqParams.local(120))
    lens = np.array([len(r) for r in w["reads"]], np.uint32)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint32)
    rs = nb.PackedStringSet.from_symbols(np.concatenate(w["reads"]), offs, lens, bits=2, big_endian=True)
    G = int(w["idx"].n)
    f = nb.finish_alignments(w["gw"], rs, ws.mate_ops, ws.mate_n_ops, ws.mate_begin, ws.mate_strand, genome_len=G)
    contigs = nb.ContigTable(["c0", "c1"], [G // 2, G - G // 2])
    q = torch.from_numpy(np.concatenate(w["quals"])).cuda() if qual else None
    recs = nb.bam_records(ws, f, rs, contigs, nb.numbered_names(w["n_pairs"], "pair"), quals=q)
    check_bam(recs, contigs, tmp_path, "pe%d" % qual)
