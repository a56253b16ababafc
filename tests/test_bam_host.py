"""CPU: nvb_bam_records' per-record routines (bam_core.cuh), compiled for the host by tests/host/bam_harness.cu, against the restatement in
tests/bam_oracle.py and against htslib's encoding of the restatement's SAM lines (live where oracle/_ref is built, else tests/golden/bam.npz):
records of alignments traced by the oracle and finished by the host build of finish_alignment on a genome cut into contigs (some shorter
than a read), single end and paired, 2- and 4-bit reads with N, both strands, with and without qualities, MAPQ and XS; hand-built inputs at
every tag-type edge; reg2bin at the bin-level edges; the .ann reader against nvbio's save_bns; write_bam read back by htslib and gzip."""
import ctypes as C
import gzip
import os
import subprocess
import numpy as np
import pytest
from oracle import orc
from oracle.ref_bam import RefBam
from nvbio_b200 import bam as nbam
from nvbio_b200.io import read_ann
from nvbio_b200.strings import pack_symbols
from nvbio_b200._lib import BamInStruct
from tests import bam_oracle as bo
from tests.golden.make_bam_golden import fixture_inputs, reg2bin_points, ann_fixtures, TAG_EDGES, name
from tests.test_finish_host import traced_batch, run_host as finish_host, SCHEMES

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "bam.npz")
LIVE = RefBam.available()


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _compile(tmp_path_factory, src, so_name):
    so = str(tmp_path_factory.mktemp(so_name) / ("lib%s.so" % so_name))
    from nvbio_b200.build import NVCC
    subprocess.check_call([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "-Wno-deprecated-declarations",
                           "-Xcompiler", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "host", src)])
    return C.CDLL(so)


@pytest.fixture(scope="module")
def H(tmp_path_factory):
    h = _compile(tmp_path_factory, "bam_harness.cu", "bam_harness")
    h.hh_reg2bin.restype = C.c_uint32
    return h


@pytest.fixture(scope="module")
def HF(tmp_path_factory):
    return _compile(tmp_path_factory, "finish_harness.cu", "finish_harness_bam")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def run_host(H, inp, bits=2, big_endian=True, capacity=None):
    """the harness on inputs in bam_oracle's layout: (list of record bytes that were stored, offsets, counts)"""
    n = len(inp["n_ops"])
    lens = np.array([len(r) for r in inp["reads"]], np.uint32)
    offs = (np.concatenate([[0], np.cumsum(lens)[:-1]]) + 5).astype(np.uint32)
    sym = np.concatenate([np.zeros(5, np.uint8)] + list(inp["reads"]) + [np.zeros(1, np.uint8)])
    keep = []
    words = pack_symbols(sym, bits, big_endian); keep.append(words)
    a = BamInStruct()
    a.reads.d_words, a.reads.bits, a.reads.big_endian = words.ctypes.data, bits, int(big_endian)
    a.reads.d_offsets, a.reads.d_lengths = offs.ctypes.data, lens.ctypes.data
    keep += [offs, lens]
    if inp["quals"] is not None:
        q = np.concatenate([np.zeros(5, np.uint8)] + [np.asarray(x, np.uint8) for x in inp["quals"]] + [np.zeros(1, np.uint8)])
        keep.append(q); a.d_read_quals = q.ctypes.data

    def arr(x, dt):
        if x is None:
            return None
        y = np.ascontiguousarray(np.asarray(x).astype(dt) if np.asarray(x).dtype != dt else x)
        keep.append(y)
        return y.ctypes.data
    a.d_n_ops = arr(inp["n_ops"], np.uint32); a.d_begin = arr(inp["begin"], np.uint32); a.d_strand = arr(inp["strand"], np.uint8)
    f = a.finish
    f.d_cigar, f.max_cigar, f.d_n_cigar = arr(inp["cigar"], np.uint32), inp["cigar"].shape[1], arr(inp["n_cigar"], np.uint32)
    f.d_md, f.max_md, f.d_md_len, f.d_edits = arr(inp["md"], np.uint8), inp["md"].shape[1], arr(inp["md_len"], np.uint32), arr(inp["edits"], np.uint32)
    a.d_score = arr(inp["score"], np.int32); a.d_mapq = arr(inp["mapq"], np.uint8); a.d_second_score = arr(inp["second"], np.int32)
    a.d_pair_flags = arr(inp["pair_flags"], np.uint32)
    a.d_contig_begin = arr(inp["contig_begin"], np.uint32); a.n_contigs = len(inp["contig_begin"]) - 1
    nb = [nm.encode() for nm in inp["names"]]
    a.d_names = arr(np.frombuffer(b"".join(nb) + b"\0", np.uint8), np.uint8)
    a.d_name_offsets = arr(np.concatenate([[0], np.cumsum([len(x) for x in nb])]), np.uint32)
    total_bound = sum(36 + 256 + 4 * inp["cigar"].shape[1] + len(r) * 2 + 50 + inp["md"].shape[1] for r in inp["reads"])
    cap = total_bound if capacity is None else capacity
    buf = np.full(max(cap, 1) + 16, 0xA5, np.uint8)
    o = np.zeros(n + 1, np.uint64); cnt = np.zeros(4, np.uint32)
    H.hh_bam(C.byref(a), C.c_uint32(n), _p(buf), C.c_uint64(cap), _p(o), _p(cnt))
    recs = [buf[int(o[k]):int(o[k + 1])].tobytes() for k in range(n) if int(o[k + 1]) <= cap]
    return recs, o, cnt, buf


def check_against_oracle(H, inp, bits=2):
    want, cnt = bo.records(inp)
    got, o, gcnt, _ = run_host(H, inp, bits)
    assert list(gcnt) == cnt
    assert len(got) == len(want)
    for k, (g, (w, sam)) in enumerate(zip(got, want)):
        assert g == w, (k, sam)
    return want, cnt


# ---- records of traced and finished alignments ----------------------------------------------------------------------------------------

def traced_inputs(HF, rng, genome, bits, paired, n_reads=200, band=31, typ=1, scheme=SCHEMES[0], quals=True, mapq=True):
    O = orc.Oracle()
    b = traced_batch(O, rng, genome, band, typ, scheme, bits, n_reads)
    if paired:
        h = n_reads // 2
        for p in range(0, h, 7):                                 # equal begins
            for f in ("reads", "strand", "ops", "n_ops", "begin"):
                getattr(b, f)[h + p] = getattr(b, f)[p]
        for p in range(2, h, 13):                                # both mates unaligned
            b.n_ops[p] = b.n_ops[h + p] = 0
    fo = finish_host(HF, b, bits)
    n = len(b)
    G = len(genome)
    # contigs: some shorter than a read, plus boundaries planted exactly at and one base before the end of traced alignments
    cuts = set(int(x) for x in rng.integers(1, G, 12)) | {40, 75, 130}
    ends = []
    for a in range(0, n, 9):
        nc = int(fo["n_cigar"][a]); row = fo["cigar"][a * fo["max_cigar"]:a * fo["max_cigar"] + nc]
        rl = sum(int(c) >> 4 for c in row if int(c) & 15 in (0, 2))
        if b.n_ops[a] and fo["edits"][a][0] != 0xFFFFFFFF and int(b.begin[a][0]) + rl < G:
            ends.append(int(b.begin[a][0]) + rl - (a // 9) % 2)
    cuts |= set(e for e in ends if 0 < e < G)
    cb = np.array([0] + sorted(cuts) + [G], np.int64)
    rl = np.array([len(r) for r in b.reads])
    inp = dict(reads=b.reads, quals=[rng.integers(0, 42, L).astype(np.uint8) for L in rl] if quals else None,
               n_ops=np.array(b.n_ops, np.uint32), begin=np.array(b.begin, np.uint32).reshape(-1, 2), strand=np.array(b.strand, np.uint8),
               cigar=fo["cigar"][:n * fo["max_cigar"]].reshape(n, -1), n_cigar=fo["n_cigar"],
               md=fo["md"][:n * fo["max_md"]].reshape(n, -1), md_len=fo["md_len"], edits=fo["edits"],
               score=rng.integers(-300, 300, n).astype(np.int32), mapq=rng.integers(0, 61, n).astype(np.uint8) if mapq else None,
               second=np.where(rng.random(n) < 0.3, -(1 << 31), rng.integers(-300, 300, n)).astype(np.int32) if mapq else None,
               pair_flags=rng.choice([0, 1, 2, 4], n // 2).astype(np.uint32) if paired else None,
               contig_begin=cb, contig_names=["ctg%d" % i for i in range(len(cb) - 1)], contig_lengths=list(np.diff(cb)),
               names=[name(rng, int(rng.integers(1, 40))) for _ in range(n // 2 if paired else n)])
    return inp


@pytest.fixture(scope="module")
def genome():
    rng = np.random.default_rng(77)
    return rng.integers(0, 4, 20_000).astype(np.uint8)


@pytest.mark.parametrize("bits", [2, 4])
@pytest.mark.parametrize("paired", [False, True])
def test_traced_records(H, HF, genome, bits, paired):
    rng = np.random.default_rng(10 * bits + paired)
    R = RefBam() if LIVE else None
    total = np.zeros(4, np.int64)
    pair_cases = np.zeros(4, np.int64)
    for i, (typ, band, scheme) in enumerate([(1, 31, SCHEMES[0]), (2, 15, SCHEMES[2]), (1, 7, SCHEMES[1]), (0, 63, SCHEMES[3]), (2, 31, SCHEMES[0])]):
        inp = traced_inputs(HF, rng, genome, bits, paired, band=band, typ=typ, scheme=scheme, quals=i % 2 == 0, mapq=i % 3 != 2)
        want, cnt = check_against_oracle(H, inp, bits)
        total += cnt
        # the generic (little-endian) gather gives the same bytes
        assert run_host(H, inp, bits, big_endian=False)[0] == [w for w, _ in want]
        if R is not None:
            hdr = bo.header_text(inp["contig_names"], inp["contig_lengths"])
            assert R.encode(hdr, [s for _, s in want]) == [w for w, _ in want]
        if paired:
            for p in range(len(want) // 2):
                f0, f1 = [int.from_bytes(want[2 * p + m][0][18:20], "little") for m in (0, 1)]
                t0 = int.from_bytes(want[2 * p][0][32:36], "little", signed=True)
                r0, r1 = [int.from_bytes(want[2 * p + m][0][4:8], "little", signed=True) for m in (0, 1)]
                pair_cases += (f0 & 4 and f1 & 4, (f0 & 4) != (f1 & 4), not (f0 & 4 or f1 & 4) and r0 != r1 and t0 == 0,
                               not (f0 & 4 or f1 & 4) and want[2 * p][0][8:12] == want[2 * p + 1][0][8:12] and t0 > 0)
    assert total[0] >= 600 and total[1] > 200 and total[2] > 10, total
    if paired:
        assert (pair_cases > 0).all(), pair_cases


def test_unmapped_by_contig_rule_drops_proper_pair():
    """a pair whose mate 2 crosses a contig boundary: mate 1 loses 0x2 and gets 0x8; mate 2 is unmapped at mate 1's placement"""
    inp = fixture_inputs(True, 5, n=4)
    h = 2
    for a in range(4):
        inp["n_ops"][a] = 10; inp["edits"][a] = (1, 1, 0, 0); inp["n_cigar"][a] = 1; inp["cigar"][a, 0] = 10 << 4
        inp["md_len"][a] = 2; inp["md"][a, :2] = np.frombuffer(b"10", np.uint8); inp["reads"][a] = np.zeros(10, np.uint8)
        inp["begin"][a] = (100 + 30 * a, 0); inp["strand"][a] = a >= h
    inp["quals"] = None
    inp["pair_flags"][:] = 1
    inp["begin"][h] = (int(inp["contig_begin"][1]) - 5, 0)   # mate 2 of pair 0 ends 5 bases past chr1
    out, cnt = bo.records(inp)
    assert cnt == [4, 3, 1, 0]
    f = [int.from_bytes(r[18:20], "little") for r, _ in out]
    assert f[0] == 0x1 | 0x40 | 0x8 and f[1] == 0x1 | 0x80 | 0x4
    assert out[1][0][4:12] == out[0][0][4:12] and out[1][0][24:32] == out[0][0][4:12]
    assert f[2] == 0x1 | 0x2 | 0x40 | 0x20 and f[3] == 0x1 | 0x2 | 0x80 | 0x10


def test_fixture_matches_htslib(H, golden):
    """hand-built inputs: the restatement gives the fixture's SAM lines, htslib's bytes of them (stored in the fixture) equal the
    restatement's bytes, and so do the shipped routine's; every tag-type edge occurs"""
    lines = str(golden["lines"]).split("\n")
    sizes = golden["record_sizes"]; raw = golden["records"].tobytes()
    recs = [raw[o - s:o] for o, s in zip(np.cumsum(sizes), sizes)]
    i = 0
    types = set()
    for paired in (False, True):
        for seed in (5, 6):
            inp = fixture_inputs(paired, seed)
            want, _ = check_against_oracle(H, inp, 4)
            for w, sam in want:
                assert sam == lines[i] and w == recs[i], (i, sam)
                i += 1
            for w, sam in want:
                for t in sam.split("\t")[11:]:
                    if ":i:" in t:
                        types.add(int(t.split(":")[2]))
    assert i == len(lines)
    assert set(TAG_EDGES) <= types
    names = [ln.split("\t")[0] for ln in lines]
    assert min(map(len, names)) == 1 and max(map(len, names)) == 254


@pytest.mark.skipif(not LIVE, reason="oracle/_ref/libnvbio_ref_bam.so (htslib) is not built here")
def test_fixture_equals_live_htslib(golden):
    R = RefBam()
    lines = str(golden["lines"]).split("\n")
    hdrs = str(golden["headers"]).split("\x00")
    sizes = golden["batch_sizes"]
    got, o = [], 0
    for hdr, k in zip(hdrs, sizes):
        got += R.encode(hdr, lines[o:o + k]); o += k
    assert b"".join(got) == golden["records"].tobytes()
    assert [[R.reg2bin(b, e) for e in (b + 1, b + 2, b + 16384, b + 131072)] for b in golden["reg2bin_points"]] == golden["reg2bin"].tolist()


def test_reg2bin(H, golden):
    pts = reg2bin_points()
    assert pts == golden["reg2bin_points"].tolist()
    for b, row in zip(pts, golden["reg2bin"].tolist()):
        for e, want in zip((b + 1, b + 2, b + 16384, b + 131072), row):
            assert H.hh_reg2bin(C.c_int64(b), C.c_int64(e)) == want == bo.reg2bin(b, e), (b, e)
    assert H.hh_reg2bin(C.c_int64(-1), C.c_int64(0)) == 4680 == bo.reg2bin(-1, 0)


def test_capacity_stores_whole_records(H):
    inp = fixture_inputs(False, 5, n=60)
    full, o, cnt, _ = run_host(H, inp, 2)
    cap = int(o[37]) + 5                                     # cuts record 37
    got, o2, cnt2, buf = run_host(H, inp, 2, capacity=cap)
    assert np.array_equal(o, o2) and np.array_equal(cnt, cnt2)
    assert got == full[:37] and (buf[int(o[37]):] == 0xA5).all()


def test_ann_reader(tmp_path, golden):
    """read_ann equals what nvbio's save_bns wrote (the fixture's files; live where oracle/_ref is built)"""
    anns = str(golden["ann"]).split("\x00")
    for i, (names, annos, lengths) in enumerate(ann_fixtures()):
        p = tmp_path / ("g%d.ann" % i)
        p.write_text(anns[i])
        a = read_ann(str(p))
        assert a["names"] == names and a["lengths"].tolist() == lengths and a["l_pac"] == sum(lengths)
        assert a["offsets"].tolist() == np.concatenate([[0], np.cumsum(lengths)[:-1]]).tolist()
        t = nbam.ContigTable.from_ann(str(p))
        assert t.names == names and t.genome_len == sum(lengths)
    if LIVE:
        from oracle.ref_bam import save_bns
        names, annos, lengths = ann_fixtures()[0]
        save_bns(str(tmp_path / "live"), names, annos, [0, 1000, 1077], lengths, [0, 1, 2], sum(lengths))
        assert (tmp_path / "live.ann").read_text() == anns[0]


def test_write_bam_round_trip(H, tmp_path):
    """write_bam's file: gzip gives header + records back; htslib (where built) reads every record back as the restatement's SAM line"""
    inp = fixture_inputs(True, 5)
    recs, _, _, _ = run_host(H, inp, 4)
    want, _ = bo.records(inp)
    t = nbam.ContigTable(inp["contig_names"], inp["contig_lengths"])
    hdr = nbam.bam_header(t, program="test")
    p = str(tmp_path / "out.bam")
    nbam.write_bam(p, hdr, [b"".join(recs[:100]), b"".join(recs[100:])])
    assert gzip.open(p).read() == hdr + b"".join(recs)
    raw = open(p, "rb").read()
    assert raw.endswith(bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000"))
    if LIVE:
        assert RefBam().format(p) == "".join(s + "\n" for _, s in want)


def test_argument_validation_without_gpu():
    """nvb_bam_records rejects NULL required pointers, n_contigs = 0, 8-bit reads, an odd paired n and a misaligned d_records with
    NVB_E_INVALID (-1) before any CUDA call"""
    from nvbio_b200 import _lib
    from nvbio_b200._lib import BamOutStruct
    L = _lib.lib()

    def good():
        a = BamInStruct()
        a.reads.d_words, a.reads.bits, a.reads.big_endian, a.reads.stride, a.reads.length = 16, 2, 1, 160, 150
        a.d_n_ops = a.d_begin = a.d_strand = a.d_score = a.d_contig_begin = a.d_names = a.d_name_offsets = 16
        a.n_contigs = 3
        f = a.finish
        f.d_cigar, f.max_cigar, f.d_n_cigar, f.d_md, f.max_md, f.d_md_len, f.d_edits = 16, 184, 16, 16, 547, 16, 16
        o = BamOutStruct(); o.d_records, o.capacity, o.d_offsets, o.d_counts = 256, 1 << 20, 16, 16
        return a, o

    def call(a, o, n=8, tb=True):
        t = C.c_size_t(0)
        return L.nvb_bam_records(C.byref(a) if a is not None else None, C.c_uint32(n), C.byref(o) if o is not None else None, None,
                                 C.byref(t) if tb else None, None)

    a, o = good()
    assert call(None, o) == -1 and call(a, None) == -1 and call(a, o, tb=False) == -1
    for f in ("d_n_ops", "d_begin", "d_strand", "d_score", "d_contig_begin", "d_names", "d_name_offsets", "n_contigs"):
        a, o = good(); setattr(a, f, 0 if f == "n_contigs" else None); assert call(a, o) == -1, f
    for f in ("d_cigar", "d_n_cigar", "d_md", "d_md_len", "d_edits", "max_cigar", "max_md"):
        a, o = good(); setattr(a.finish, f, 0 if f.startswith("max") else None); assert call(a, o) == -1, f
    for f in ("d_offsets", "d_counts", "d_records"):
        a, o = good(); setattr(o, f, None); assert call(a, o) == -1, f
    a, o = good(); o.d_records = 257; assert call(a, o) == -1
    a, o = good(); a.reads.bits = 8; assert call(a, o) == -1
    a, o = good(); a.reads.d_words = None; assert call(a, o) == -1
    a, o = good(); a.d_pair_flags = 16; assert call(a, o, n=7) == -1
