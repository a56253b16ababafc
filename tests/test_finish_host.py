"""CPU: nvb_finish_alignments' per-alignment routine (finish_alignment, finish_core.cuh), compiled for the host by tests/host/finish_harness.cu,
against the restatement in tests/finish_oracle.py on alignments traced by the oracle's banded (bands 3 to 63) and full-matrix tracebacks
(all three types, several schemes, 2- and 4-bit reads with N, both strands, genome ends) and on hand-built op streams; MD + CIGAR rebuild the
reference span, NM = XM + I + D; nvBowtie's own analyze_md_string / count_symbols / reference_cigar_length agree (tests/golden/finish.npz,
and live where oracle/_ref is built); and the entry point's argument validation."""
import ctypes as C
import os
import subprocess
import numpy as np
import pytest
from oracle import orc
from oracle.ref_finish import RefFinish
from nvbio_b200.strings import pack_symbols
from tests import finish_oracle as fo

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "host", "finish_harness.cu")
GOLDEN = os.path.join(HERE, "golden", "finish.npz")
NONE = 0xFFFFFFFF


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


@pytest.fixture(scope="module")
def H(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("finish_harness") / "libfinish_harness.so")
    from nvbio_b200.build import NVCC
    subprocess.check_call([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17",
                           "-Wno-deprecated-declarations", "-Xcompiler", "-fPIC", "-shared", "-o", so, SRC])
    return C.CDLL(so)


class Batch:
    """alignments over one genome: caller reads, strands, ops (END -> START), n_ops, begins"""

    def __init__(self, genome, genome_len=None, max_ops=1300):
        self.genome = np.asarray(genome, np.uint8)
        self.genome_len = len(self.genome) if genome_len is None else genome_len
        self.max_ops = max_ops
        self.reads, self.strand, self.ops, self.n_ops, self.begin = [], [], [], [], []

    def add(self, read, strand, ops, begin, n_ops=None):
        self.reads.append(np.asarray(read, np.uint8)); self.strand.append(strand)
        ops = np.asarray(ops, np.uint8)
        self.n_ops.append(len(ops) if n_ops is None else n_ops)
        row = np.zeros(self.max_ops, np.uint8); k = min(len(ops), self.max_ops); row[:k] = ops[:k]
        self.ops.append(row); self.begin.append(begin)

    def __len__(self):
        return len(self.reads)


def run_host(H, b, bits=2, big_endian=True, max_cigar=None, max_md=None, sentinel=False):
    n = len(b)
    lens = np.array([len(r) for r in b.reads], np.uint32)
    offs = (np.concatenate([[0], np.cumsum(lens)[:-1]]) + 3).astype(np.uint32)            # unaligned offsets
    sym = np.concatenate([np.zeros(3, np.uint8)] + b.reads + [np.zeros(1, np.uint8)])
    rw = pack_symbols(sym, bits, big_endian)
    gw = pack_symbols(b.genome[:b.genome_len], 2, True)
    max_cigar = b.max_ops + 2 if max_cigar is None else max_cigar
    max_md = 3 * b.max_ops + 1 if max_md is None else max_md
    pad = 1 if sentinel else 0
    o = dict(cigar=np.full((n, max_cigar + pad), 0xA5A5A5A5, np.uint32), n_cigar=np.zeros(n, np.uint32),
             md=np.full((n, max_md + pad), 0xA5, np.uint8), md_len=np.zeros(n, np.uint32), edits=np.zeros((n, 4), np.uint32))
    # the harness writes row a at a * max_cigar / a * max_md: with a sentinel column the rows are laid out by hand below
    cig = np.full(n * max_cigar + pad, 0xA5A5A5A5, np.uint32); md = np.full(n * max_md + pad, 0xA5, np.uint8)
    H.hh_finish(C.c_uint32(bits), C.c_uint32(int(big_endian)), _p(gw), C.c_uint32(b.genome_len), _p(rw), _p(offs), _p(lens), C.c_uint32(n),
                _p(np.array(b.strand, np.uint8)), _p(np.stack(b.ops) if n else np.zeros((0, b.max_ops), np.uint8)), C.c_uint32(b.max_ops),
                _p(np.array(b.n_ops, np.uint32)), _p(np.array(b.begin, np.uint32).reshape(-1, 2) if n else np.zeros((0, 2), np.uint32)),
                _p(cig), C.c_uint32(max_cigar), _p(o["n_cigar"]), _p(md), C.c_uint32(max_md), _p(o["md_len"]), _p(o["edits"]))
    o["cigar"], o["md"] = cig, md
    o["max_cigar"], o["max_md"] = max_cigar, max_md
    return o


def check(b, o):
    """every field == the restatement; MD + CIGAR rebuild the reference span; NM = XM + I + D.  Returns the number of finished alignments"""
    done = 0
    for a in range(len(b)):
        cigar, md, ed = fo.finish(b.ops[a], b.n_ops[a], b.max_ops, b.begin[a], b.strand[a], b.reads[a], b.genome, b.genome_len)
        nc, ml = int(o["n_cigar"][a]), int(o["md_len"][a])
        got_c = [(int(v) >> 4, int(v) & 15) for v in o["cigar"][a * o["max_cigar"]:a * o["max_cigar"] + nc]]
        got_md = bytes(o["md"][a * o["max_md"]:a * o["max_md"] + ml]).decode()
        assert (got_c, got_md, tuple(int(v) for v in o["edits"][a])) == (cigar, md, ed), (a, b.begin[a], b.strand[a], fo.cigar_text(cigar), md)
        if ed[0] == NONE or b.n_ops[a] == 0:
            continue
        x = int(b.begin[a][0]); M = sum(k for k, op in cigar if op == 0); D = sum(k for k, op in cigar if op == 2)
        want = "".join(fo.ref_char(b.genome, b.genome_len, x + c) for c in range(M + D))
        assert fo.rebuild_reference(cigar, md, b.reads[a], b.strand[a]) == want, (a, md)
        assert ed[0] == ed[1] + sum(k for k, op in cigar if op in (1, 2))
        assert sum(k for k, op in cigar if op != 2) == len(b.reads[a])
        done += 1
    return done


SCHEMES = [(2, -2, -5, -3), (1, -3, -4, -1), (0, -6, -5, -3), (2, -1, -1, -1)]


def traced_batch(O, rng, genome, band, typ, scheme, bits, n_reads, full=False):
    """reads drawn from the genome (substitutions, 1-3 bp indels, N for 4-bit reads; some at either end, some running past it), each traced
    against a window around its origin by the oracle; the window past the genome's end is padded"""
    G = len(genome)
    pats, txts, w0s, strands = [], [], [], []
    for _ in range(n_reads):
        M = int(rng.integers(20, 151))
        where = rng.random()
        x = int(rng.integers(0, 8)) if where < 0.15 else (G - M + int(rng.integers(-8, band // 2 + 2)) if where < 0.35 else int(rng.integers(0, G - M)))
        x = max(0, x)
        src = np.concatenate([genome[x:x + M], rng.integers(0, 4, max(0, x + M - G)).astype(np.uint8)])[:M]
        q = src.copy()
        mut = rng.random(M) < rng.choice([0.0, 0.02, 0.08])
        q[mut] = rng.integers(0, 4, int(mut.sum()))
        if M > 30 and rng.random() < 0.4:
            k, d = int(rng.integers(8, M - 12)), int(rng.integers(1, 4))
            q = np.concatenate([q[:k], q[k + d:]]) if rng.random() < 0.5 else np.concatenate([q[:k], rng.integers(0, 4, d).astype(np.uint8), q[k:]])
        if bits == 4:
            q[rng.random(len(q)) < 0.01] = 4
        w0 = max(0, x - band // 2)
        tl = len(q) + band + (60 if full else 0)
        t = np.concatenate([genome[w0:w0 + tl], np.zeros(max(0, w0 + tl - G), np.uint8)])[:tl]
        pats.append(q.astype(np.uint8)); txts.append(t); w0s.append(w0); strands.append(int(rng.integers(0, 2)))
    p_len = np.array([len(p) for p in pats], np.uint32); t_len = np.array([len(t) for t in txts], np.uint32)
    p_off = np.concatenate([[0], np.cumsum(p_len)[:-1]]).astype(np.uint32); t_off = np.concatenate([[0], np.cumsum(t_len)[:-1]]).astype(np.uint32)
    P, T = np.concatenate(pats + [np.zeros(8, np.uint8)]), np.concatenate(txts + [np.zeros(8, np.uint8)])
    if full:
        r = O.gotoh_full_traceback(typ, scheme, P, p_off, p_len, T, t_off, t_len, max_ops=512)
    else:
        r = O.banded_traceback(band, typ, scheme, P, p_off, p_len, T, t_off, t_len, max_ops=512)
    b = Batch(genome, max_ops=512)
    for i in range(n_reads):
        k = int(r["n_ops"][i])
        b.add(fo.strand_read(pats[i], strands[i]), strands[i], r["ops"][i, :min(k, 512)],
              (w0s[i] + int(r["source"][i, 0]), int(r["source"][i, 1])), n_ops=k)
    return b


@pytest.fixture(scope="module")
def genome():
    rng = np.random.default_rng(31)
    g = rng.integers(0, 4, 20_000).astype(np.uint8)
    g[5000:5600] = np.tile(g[5000:5060], 10)                # a tandem repeat
    g[9000:9400] = g[12000:12400]                           # a planted repeat
    return g


@pytest.mark.parametrize("bits", [2, 4])
def test_oracle_traced_alignments(H, genome, bits):
    O = orc.Oracle()
    rng = np.random.default_rng(100 + bits)
    total = 0
    for band in (3, 5, 7, 15, 31, 63):
        for typ in (0, 1, 2):
            for scheme in SCHEMES[:2] if band in (3, 63) else SCHEMES:
                b = traced_batch(O, rng, genome, band, typ, scheme, bits, 100)
                o = run_host(H, b, bits)
                total += check(b, o)
                # the generic (little-endian) gather gives the same answer
                ol = run_host(H, b, bits, big_endian=False)
                for k in ("n_cigar", "md_len", "edits", "cigar", "md"):
                    assert np.array_equal(o[k], ol[k]), k
    for typ in (0, 1, 2):
        for scheme in SCHEMES:
            b = traced_batch(O, rng, genome, 31, typ, scheme, bits, 100, full=True)
            total += check(b, run_host(H, b, bits))
    assert total >= 5000


def build_case(rng, genome, G, x, script, strand, bits=2):
    """(caller read, ops END -> START, begin) of a script such as [('S', 3), ('M', 10), ('X', 1), ('D', 2), ('I', 1), ('N', 1)]:
    S clipped read symbols, M matching columns, X mismatching ones, N read Ns, I inserted read symbols, D deleted genome symbols"""
    read, ops, by, gx = [], [], 0, x
    for t, k in script:
        for _ in range(k):
            if t in "MXN":
                g = int(genome[gx]) if gx < G else int(rng.integers(0, 4))
                read.append(g if t == "M" else ((g + int(rng.integers(1, 4))) % 4 if t == "X" else 4)); ops.append(0); gx += 1
            elif t in "SI":
                read.append(int(rng.integers(0, 4)))
                if t == "I":
                    ops.append(1)
                elif not ops:
                    by += 1
            else:
                ops.append(2); gx += 1
    s = np.array(read, np.uint8)
    return fo.strand_read(s, strand), np.array(ops[::-1], np.uint8), (x, by)


HAND = [
    [("M", 255)], [("M", 256)], [("M", 1000)], [("M", 1100), ("X", 1), ("M", 99)],
    [("X", 2), ("M", 5), ("X", 1), ("X", 1), ("M", 3), ("X", 3)], [("X", 1)], [("M", 1)], [("I", 1)],
    [("M", 10), ("X", 1), ("D", 3), ("M", 10)], [("M", 10), ("D", 2), ("X", 1), ("M", 4)], [("M", 6), ("I", 2), ("D", 3), ("M", 6)],
    [("M", 6), ("D", 3), ("I", 2), ("M", 6)], [("M", 6), ("D", 1), ("I", 1), ("D", 1), ("M", 6)], [("I", 7)], [("D", 4)], [("D", 4), ("S", 3)],
    [("S", 4), ("M", 20), ("S", 6)], [("S", 4), ("X", 1), ("M", 20), ("X", 1), ("S", 6)], [("S", 1), ("I", 3), ("M", 5), ("I", 2), ("S", 2)],
    [("M", 300), ("D", 12), ("M", 300), ("I", 9), ("M", 40)], [("D", 2), ("M", 10), ("D", 1)], [("M", 17), ("D", 255), ("M", 3)],
]


@pytest.mark.parametrize("bits", [2, 4])
def test_hand_built_op_streams(H, genome, bits):
    rng = np.random.default_rng(7 + bits)
    G = len(genome)
    b = Batch(genome)
    for script in HAND + ([[("N", 1)], [("M", 3), ("N", 2), ("X", 1), ("N", 1), ("M", 2)], [("S", 2), ("N", 1), ("M", 9)]] if bits == 4 else []):
        for strand in (0, 1):
            for x in (0, 1234, G - 1300):
                r, ops, beg = build_case(rng, genome, G, x, script, strand, bits)
                b.add(r, strand, ops, beg)
    for strand in (0, 1):                                    # columns past the genome's end, in M runs, mismatches and deletions
        for script, x in (([("M", 40)], G - 10), ([("M", 20), ("X", 1), ("M", 20)], G - 30), ([("M", 5), ("D", 3), ("M", 5)], G - 6),
                          ([("M", 16)], G), ([("S", 3), ("M", 33), ("S", 2)], G - 17)):
            r, ops, beg = build_case(rng, genome, G, x, script, strand, bits)
            b.add(r, strand, ops, beg)
    for strand in (0, 1):                                    # reads of length 1
        for script in ([("M", 1)], [("X", 1)], [("I", 1)]):
            r, ops, beg = build_case(rng, genome, G, 77, script, strand, bits)
            b.add(r, strand, ops, beg)
    finished = len(b)
    r, ops, beg = build_case(rng, genome, G, 500, [("M", 30), ("I", 2), ("M", 10)], 0, bits)
    b.add(r, 0, ops, beg, n_ops=b.max_ops + 1)               # truncated by the traceback
    b.add(r, 0, ops, (NONE, 0))                              # begin.x unknown
    b.add(r, 0, ops, (500, 1))                               # one read symbol too many
    b.add(r, 1, ops, (500, len(r) + 1))                      # begin.y past the read
    b.add(r[:-1], 0, ops, (500, 0))                          # read too short
    bad = ops.copy(); bad[3] = 3
    b.add(r, 0, bad, (500, 0))                               # an op byte that is no op
    b.add(r, 0, ops[:0], (NONE, NONE))                       # unaligned
    o = run_host(H, b, bits)
    assert check(b, o) == finished
    assert (o["edits"][finished:-1, 0] == NONE).all() and not o["n_cigar"][finished:].any() and not o["md_len"][finished:].any()
    assert not o["edits"][-1].any()
    # the MD is spec-conformant and multi-digit numbers appear
    import re
    mds = [bytes(o["md"][a * o["max_md"]:a * o["max_md"] + int(o["md_len"][a])]).decode() for a in range(finished)]
    assert all(re.fullmatch(r"[0-9]+(([A-Z]|\^[A-Z]+)[0-9]+)*", m) for m in mds)
    assert "1000" in mds and "256" in mds and any(m.startswith("0") and m.endswith("0") for m in mds)


def test_capacity_truncation(H, genome):
    """runs and MD bytes beyond max_cigar / max_md are counted, not stored; the slot after them stays untouched"""
    rng = np.random.default_rng(3)
    b = Batch(genome, max_ops=200)
    for script in ([("S", 2), ("M", 10), ("X", 1), ("M", 3), ("D", 2), ("M", 4), ("I", 1), ("M", 9), ("S", 1)], [("X", 1)] * 1 + [("M", 150)]):
        r, ops, beg = build_case(rng, genome, len(genome), 900, script, 0)
        b.add(r, 0, ops, beg)
    full = run_host(H, b)
    check(b, full)
    for mc, mm in ((1, 1), (3, 5), (2, 200)):
        o = run_host(H, b, max_cigar=mc, max_md=mm, sentinel=True)
        assert np.array_equal(o["n_cigar"], full["n_cigar"]) and np.array_equal(o["md_len"], full["md_len"])
        assert np.array_equal(o["edits"], full["edits"])
        assert o["cigar"][-1] == 0xA5A5A5A5 and o["md"][-1] == 0xA5
        for a in range(len(b)):
            kc, km = min(mc, int(full["n_cigar"][a])), min(mm, int(full["md_len"][a]))
            assert np.array_equal(o["cigar"][a * mc:a * mc + kc], full["cigar"][a * full["max_cigar"]:a * full["max_cigar"] + kc])
            assert np.array_equal(o["md"][a * mm:a * mm + km], full["md"][a * full["max_md"]:a * full["max_md"] + km])


# ---- pin to nvBowtie's own output helpers ----------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def test_fixture_matches_restatement(golden):
    """the fixture was written from the restatement's MDS vectors; the restatement still writes them, and the reference's analyze_md_string /
    count_symbols / reference_cigar_length (stored in the fixture) equal our XM / XO / XG, I + D and genome span"""
    from tests.golden.make_finish_golden import fixture_alignments
    b, mds, cig, ours = fixture_alignments()
    assert np.array_equal(np.concatenate(mds), golden["mds"]) and np.array_equal(np.concatenate(cig).reshape(-1), golden["cigar"].reshape(-1))
    ref = golden["ref"]                                      # per alignment: n_mm, n_gapo, n_gape, I, D, reference length
    assert len(ref) == len(b) >= 1000
    assert np.array_equal(ref[:, 0:3], ours[:, 1:4])
    assert np.array_equal(ref[:, 3] + ref[:, 4], ours[:, 0] - ours[:, 1])
    assert np.array_equal(ref[:, 5], ours[:, 4])


@pytest.mark.skipif(not RefFinish.available(), reason="oracle/_ref/libnvbio_ref_finish.so (the reference's own code) is not built here")
def test_fixture_equals_live_reference(golden):
    R = RefFinish()
    got = R.analyze(golden["mds"], golden["mds_off"], golden["cigar"], golden["cigar_off"])
    assert np.array_equal(got, golden["ref"])


def test_shipped_routine_on_fixture(H):
    """the host build of the shipped routine gives the fixture's counts on the fixture's alignments"""
    from tests.golden.make_finish_golden import fixture_alignments
    b, _, _, ours = fixture_alignments()
    o = run_host(H, b)
    check(b, o)
    assert np.array_equal(o["edits"][:, 1:4].astype(np.int64), ours[:, 1:4])


def test_argument_validation_without_gpu():
    """nvb_finish_alignments rejects NULL inputs / outputs and zero capacities with NVB_E_INVALID (-1) and 8-bit reads with NVB_E_UNSUPPORTED
    (-4), before any CUDA call"""
    from nvbio_b200 import _lib
    from nvbio_b200._lib import StringSetStruct, BestAlignmentOutStruct, FinishOutStruct
    L = _lib.lib()

    def good():
        ss = StringSetStruct(); ss.d_words = 16; ss.bits = 2; ss.big_endian = 1; ss.stride = 160; ss.length = 150
        a = BestAlignmentOutStruct(); a.d_ops, a.max_ops, a.d_n_ops, a.d_begin, a.d_strand = 16, 182, 16, 16, 16
        o = FinishOutStruct(); o.d_cigar, o.max_cigar, o.d_n_cigar, o.d_md, o.max_md, o.d_md_len, o.d_edits = 16, 184, 16, 16, 547, 16, 16
        return ss, a, o

    def call(g=16, ss=None, a=None, o=None, n=8):
        return L.nvb_finish_alignments(C.c_void_p(g) if g else None, C.c_uint32(1000), C.byref(ss) if ss is not None else None, C.c_uint32(n),
                                       C.byref(a) if a is not None else None, C.byref(o) if o is not None else None, None)

    ss, a, o = good()
    assert call(0, ss, a, o) == -1 and call(16, None, a, o) == -1 and call(16, ss, None, o) == -1 and call(16, ss, a, None) == -1
    for f in ("d_ops", "d_n_ops", "d_begin", "d_strand", "max_ops"):
        ss, a, o = good(); setattr(a, f, 0 if f == "max_ops" else None); assert call(16, ss, a, o) == -1, f
    for f in ("d_cigar", "d_n_cigar", "d_md", "d_md_len", "d_edits", "max_cigar", "max_md"):
        ss, a, o = good(); setattr(o, f, 0 if f.startswith("max") else None); assert call(16, ss, a, o) == -1, f
    ss, a, o = good(); ss.d_words = None
    assert call(16, ss, a, o) == -1
    ss, a, o = good(); ss.bits = 8
    assert call(16, ss, a, o) == -4
    ss, a, o = good()
    assert call(16, ss, a, o, n=0) == 0                      # nothing to do: no CUDA call either
