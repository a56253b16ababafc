"""CPU: Gotoh tracebacks under a quality-table scheme (nvBowtie's QualityGotohScheme: substitution scores by the read base's quality from a
256 x 2 table).  Every CIGAR / MD / NM written for a quality-scored read comes from such a traceback, so the path it picks -- not only its
score -- must be the reference's:

- the oracle's quality tracebacks (banded and full matrix) == the reference's own templates run with a table-driven scheme: on seeded
  batches (live where oracle/_ref exports the quality tracebacks, else the reference's stored answers to the very same calls,
  tests/golden/ref_calls.pkl.gz) and on the committed fixture tests/golden/traceback_quality.npz;
- the product's per-thread routines compiled for the host (tests/host/host_harness.cu, full_tb_harness.cu) == the oracle: the direction-
  matrix traceback at bands 3 / 5 / 7 / 15 / 31, the gapless fast path, and the rescued-mate warp traceback's lanes."""
import ctypes as C
import os
import subprocess
import tempfile
import numpy as np
import pytest
from oracle import orc
from nvbio_b200.strings import pack_symbols
from tests.golden import make_traceback_quality_golden as G, ref_replay
from tests.golden.make_traceback_quality_golden import SCHEME6, banded_problems, full_problems, quality_table

HERE = os.path.dirname(os.path.abspath(__file__))
CORE = [os.path.join(HERE, "..", "nvbio_b200", "csrc", f) for f in
        ("fm_core.cuh", "gotoh_core.cuh", "gotoh_full_core.cuh", "pipeline_core.cuh", "common.cuh")]


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _u32(a):
    return np.ascontiguousarray(a, dtype=np.uint32)


def _harness(name):
    """tests/host/<name>.cu compiled for the host (the same library the other host tests load), rebuilt when a source is newer"""
    src, so = os.path.join(HERE, "host", name + ".cu"), os.path.join(HERE, "host", "lib" + name + ".so")
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in [src] + CORE):
        from nvbio_b200.build import NVCC
        subprocess.check_call([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17",
                               "-Wno-deprecated-declarations", "-Xcompiler", "-fPIC", "-shared", "-o", so, src])
    return C.CDLL(so)


@pytest.fixture(scope="module")
def H():
    return _harness("host_harness")


@pytest.fixture(scope="module")
def FT():
    return _harness("full_tb_harness")


@pytest.fixture(scope="module")
def O():
    return orc.Oracle()


QUALITY_TRACEBACKS = ("ref_banded_traceback_q", "ref_gotoh_full_traceback_q")


@pytest.fixture(scope="module")
def R():
    """the reference's quality tracebacks: live where oracle/_ref exports them, else their stored answers (tests/golden/ref_calls.pkl.gz)"""
    yield ref_replay.reference(QUALITY_TRACEBACKS)
    ref_replay.save_recordings()


@pytest.fixture(scope="module")
def live_ref():
    if not ref_replay.live_exports(QUALITY_TRACEBACKS):
        pytest.skip("regenerating the fixture needs oracle/_ref built with the quality tracebacks")
    return orc.Ref()


def assert_same_traceback(a, b, ctx):
    """every field of two traceback results; ops compared up to each alignment's op count (and the stored width)"""
    for k in ("score", "sink", "source", "n_ops", "clips"):
        if k in a and k in b:
            assert np.array_equal(np.asarray(a[k]).astype(np.int64), np.asarray(b[k]).astype(np.int64)), (ctx, k)
    for i in range(len(a["n_ops"])):
        k = min(int(a["n_ops"][i]), a["ops"].shape[1], b["ops"].shape[1])
        assert np.array_equal(a["ops"][i][:k], b["ops"][i][:k]), (ctx, i)


def gapped(o):
    """number of alignments whose path holds an insertion or a deletion"""
    return sum(int((o["ops"][i][:min(int(o["n_ops"][i]), o["ops"].shape[1])] != 0).any()) for i in range(len(o["n_ops"])))


# ---------------------------------------------------------------------------------------------------------------------------------
# 1. oracle == reference
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("typ", [0, 1, 2])
@pytest.mark.parametrize("band", [7, 15, 31])
def test_banded_quality_traceback_vs_reference(O, R, band, typ):
    """banded quality tracebacks: score, sink, source, n_ops, clips and every op, both tables, N's in patterns and texts, gap-rich reads
    with low-quality mismatches beside the gaps, every quality profile"""
    rng = np.random.default_rng(4000 + 10 * band + typ)
    n_gapped = 0
    for mb in (2, 0):
        qtab = quality_table(mb)
        for kw in (dict(n_pat=0.02, n_txt=0.02), dict(indel=0.02, tie=1.0), dict(profile="low", indel=0.01),
                   dict(profile="clamp"), dict(profile="high", sub=0.06), dict(profile="rand", ragged=False)):
            pr, qual = banded_problems(rng, 60, band, 150, **kw)
            a = O.banded_traceback(band, typ, SCHEME6, *pr, max_ops=2 * 150 + band, qual=qual, qtab=qtab)
            b = R.banded_traceback_q(band, typ, SCHEME6, *pr, qual, qtab, max_ops=2 * 150 + band)
            assert_same_traceback(a, b, (band, typ, mb, kw))
            n_gapped += gapped(b)
    assert n_gapped > 50


@pytest.mark.parametrize("typ", [0, 1, 2])
def test_full_quality_traceback_vs_reference(O, R, typ):
    """full-matrix quality tracebacks, patterns up to 256 and texts up to 512 symbols"""
    rng = np.random.default_rng(4100 + typ)
    n_gapped = 0
    for mb in (2, 0):
        qtab = quality_table(mb)
        for kw in (dict(n_pat=0.02, n_txt=0.01), dict(indel=0.02, tie=1.0), dict(profile="low"), dict(profile="clamp")):
            pr, qual = full_problems(rng, 30, 256, 512, **kw)
            a = O.gotoh_full_traceback(typ, SCHEME6, *pr, max_ops=256 + 512 + 1, qual=qual, qtab=qtab)
            b = R.gotoh_full_traceback_q(typ, SCHEME6, *pr, qual, qtab, max_ops=256 + 512 + 1)
            assert_same_traceback(a, b, (typ, mb, kw))
            n_gapped += gapped(b)
    assert n_gapped > 20


def test_null_table_keeps_the_simple_scheme(O):
    """qual / qtab left out (or a table that restates the constants) == today's simple-scheme traceback"""
    rng = np.random.default_rng(4200)
    pr, qual = banded_problems(rng, 50, 15, 120)
    flat = np.ascontiguousarray(np.tile(np.array([[2, -6]], np.int32), (256, 1)))
    for typ in (0, 1, 2):
        a = O.banded_traceback(15, typ, (2, -6, -8, -3, -7, -2), *pr)
        assert_same_traceback(a, O.banded_traceback(15, typ, SCHEME6, *pr, qual=qual, qtab=flat), ("banded", typ))
    pr, qual = full_problems(rng, 30, 120, 300)
    for typ in (0, 1, 2):
        a = O.gotoh_full_traceback(typ, (2, -6, -8, -3, -7, -2), *pr)
        assert_same_traceback(a, O.gotoh_full_traceback(typ, SCHEME6, *pr, qual=qual, qtab=flat), ("full", typ))


def _golden():
    return np.load(G.OUT)


def golden_cases():
    """(band, type, match bonus, problems, qual, expected traceback) of every case of the committed fixture"""
    g = _golden()
    for cid, band, typ, mb in g["cases"]:
        pr = tuple(g[f"c{cid}_{k}"] for k in ("pat", "p_off", "p_len", "txt", "t_off", "t_len"))
        res, flat = g[f"c{cid}_res"], g[f"c{cid}_ops"]
        n_ops = res[5]
        ops = np.zeros((len(n_ops), max(int(n_ops.max()), 1)), np.uint8)
        ends = np.cumsum(n_ops)
        for i in range(len(n_ops)):
            ops[i, :n_ops[i]] = flat[ends[i] - n_ops[i]:ends[i]]
        want = dict(score=res[0], sink=res[1:3].T, source=res[3:5].T, n_ops=n_ops, clips=res[6:8].T, ops=ops)
        yield int(band), int(typ), int(mb), pr, g[f"c{cid}_qual"], want, g["qtab%d" % mb], tuple(int(v) for v in g["scheme6"])


def test_quality_traceback_golden(O):
    """the committed quality tracebacks of the reference itself (tests/golden/traceback_quality.npz) == the oracle, with no oracle/_ref"""
    seen = set()
    for band, typ, mb, pr, qual, want, qtab, s6 in golden_cases():
        max_ops = want["ops"].shape[1]
        if band:
            got = O.banded_traceback(band, typ, s6, *pr, max_ops=max_ops, qual=qual, qtab=qtab)
        else:
            got = O.gotoh_full_traceback(typ, s6, *pr, max_ops=max_ops, qual=qual, qtab=qtab)
        assert_same_traceback(got, want, (band, typ, mb))
        seen.add((band, typ, mb))
    assert seen == {(b, t, m) for b in (0, 7, 15, 31) for t in (0, 1, 2) for m in (2, 0)}
    g = _golden()
    assert np.array_equal(g["qtab2"], quality_table(2)) and np.array_equal(g["qtab0"], quality_table(0))


def test_quality_golden_regenerates_byte_for_byte(live_ref):
    """the generator, run against the reference, reproduces the committed fixture exactly"""
    with tempfile.TemporaryDirectory() as d:
        path = G.main(os.path.join(d, "traceback_quality.npz"))
        with open(path, "rb") as f, open(G.OUT, "rb") as g:
            assert f.read() == g.read()


# ---------------------------------------------------------------------------------------------------------------------------------
# 2. the product's per-thread routines (host build) == the oracle
# ---------------------------------------------------------------------------------------------------------------------------------
def host_traceback(H, band, typ, scheme6, pr, qual, qtab, pbits, tbits, max_ops):
    """gotoh_generic_impl<B, TYPE, true> + gotoh_walk (what gotoh_traceback_kernel runs per thread) through hh_gotoh_traceback"""
    pat, p_off, p_len, txt, t_off, t_len = pr
    pw, tw = pack_symbols(pat, pbits, True), pack_symbols(txt, tbits, True)
    n = len(p_off)
    o = dict(score=np.zeros(n, np.int32), sink=np.zeros((n, 2), np.uint32), source=np.zeros((n, 2), np.uint32),
             ops=np.zeros((n, max_ops), np.uint8), n_ops=np.zeros(n, np.uint32))
    r = H.hh_gotoh_traceback(C.c_int(band), C.c_int(typ), _p(np.array(scheme6, np.int32)), _p(qtab), _p(pw), C.c_uint32(pbits), C.c_uint32(1),
                             _p(_u32(p_off)), _p(_u32(p_len)), _p(qual), _p(tw), C.c_uint32(tbits), C.c_uint32(1), _p(_u32(t_off)), _p(_u32(t_len)),
                             C.c_uint32(n), C.c_uint32(max_ops), _p(o["score"]), _p(o["sink"]), _p(o["source"]), _p(o["ops"]), _p(o["n_ops"]))
    assert r == 0
    return o


@pytest.mark.parametrize("typ", [0, 1, 2])
@pytest.mark.parametrize("band", [3, 5, 7, 15, 31])
def test_host_banded_traceback_quality(H, O, band, typ):
    """the direction-matrix traceback under quality tables == the oracle (bands 3 / 5 have no reference instantiation: there the oracle's
    generic-band restatement is the check): 2-bit patterns, 4-bit patterns and texts with N's, both tables, every quality profile"""
    rng = np.random.default_rng(4300 + 10 * band + typ)
    n_gapped = 0
    for mb in (2, 0):
        qtab = quality_table(mb)
        for kw, pbits, tbits in ((dict(), 2, 2), (dict(n_pat=0.02, n_txt=0.02), 4, 4), (dict(indel=0.02, tie=1.0), 2, 2),
                                 (dict(profile="low"), 2, 2), (dict(profile="clamp", n_pat=0.02), 4, 2), (dict(profile="rand"), 4, 4)):
            pr, qual = banded_problems(rng, 40, band, 150, **kw)
            want = O.banded_traceback(band, typ, SCHEME6, *pr, max_ops=400, qual=qual, qtab=qtab)
            got = host_traceback(H, band, typ, SCHEME6, pr, qual, qtab, pbits, tbits, 400)
            assert_same_traceback(got, want, (band, typ, mb, kw))
            n_gapped += gapped(want)
    assert n_gapped > 20


@pytest.mark.parametrize("typ", [0, 1, 2])
@pytest.mark.parametrize("band", [3, 5, 7, 15, 31])
def test_host_gapless_fast_path_quality(H, O, band, typ):
    """gapless_traceback with a quality table: whenever it claims an alignment from (score, sink) alone, the oracle's quality traceback is
    exactly that all-substitution suffix of the sink's diagonal.  LOCAL with match bonus 2, SEMI_GLOBAL / GLOBAL also with 0 (end-to-end);
    N's never claimed through; GLOBAL never claimed"""
    rng = np.random.default_rng(4400 + 10 * band + typ)
    claimed = refused = 0
    for mb in ((2,) if typ == 1 else (2, 0)):
        qtab = quality_table(mb)
        for kw in (dict(indel=0.003, sub=0.02), dict(indel=0.003, profile="low"), dict(indel=0.003, profile="clamp"),
                   dict(indel=0.02, tie=1.0), dict(n_pat=0.01, n_txt=0.01), dict(profile="high", sub=0.08)):
            pr, qual = banded_problems(rng, 80, band, 120, **kw)
            pat, p_off, p_len, txt, t_off, t_len = pr
            want = O.banded_traceback(band, typ, SCHEME6, *pr, max_ops=300, qual=qual, qtab=qtab)
            n = len(p_off)
            ln = np.zeros(n, np.uint32); ok = np.zeros(n, np.uint8)
            sink = np.ascontiguousarray(want["sink"].astype(np.uint32))
            H.hh_gapless_traceback(C.c_int(typ), _p(np.array(SCHEME6, np.int32)), _p(qtab), _p(qual),
                                   _p(pack_symbols(pat, 4, True)), C.c_uint32(4), C.c_uint32(1), _p(p_off), _p(p_len),
                                   _p(pack_symbols(txt, 4, True)), C.c_uint32(4), C.c_uint32(1), _p(t_off), _p(t_len), C.c_uint32(n),
                                   _p(np.ascontiguousarray(want["score"].astype(np.int32))), _p(sink), _p(ln), _p(ok))
            if typ == 0:
                assert not ok.any()
            for a in np.nonzero(ok)[0]:
                L = int(ln[a])
                assert int(want["n_ops"][a]) == L and not want["ops"][a][:L].any(), (band, typ, mb, kw, a)
                assert tuple(int(v) for v in want["source"][a]) == (int(sink[a, 0]) - L, int(sink[a, 1]) - L), (band, typ, mb, kw, a)
            claimed += int(ok.sum())
            # every all-substitution traceback of a read without N's on its diagonal is one the fast path should be able to claim
            refused += sum(1 for a in np.nonzero(ok == 0)[0] if typ != 0 and not want["ops"][a][:int(want["n_ops"][a])].any()
                           and int(want["n_ops"][a]) > 0 and want["score"][a] > (0 if typ == 1 else -10 ** 6)
                           and (typ == 1 or int(want["sink"][a][1]) == int(p_len[a]))
                           and not (pat[p_off[a]:p_off[a] + p_len[a]] > 3).any() and not (txt[t_off[a]:t_off[a] + t_len[a]] > 3).any())
    assert typ == 0 or claimed > 100
    assert refused == 0


def full_tb(FT, typ, scheme6, pr, qual, qtab, max_ops):
    """hh_full_tb: gotoh_full_impl2 + the row-major walk on the whole window, and the warp traceback's lanes (FullTbLane, emulated) + the
    step-major walk on the window cut by full_traceback_first_row"""
    pat, p_off, p_len, txt, t_off, t_len = pr
    pat = np.concatenate([pat, np.zeros(8, np.uint8)]); txt = np.concatenate([txt, np.zeros(8, np.uint8)])
    n = len(p_off)
    o = dict(score=np.zeros(n, np.int32), sink=np.zeros((n, 2), np.uint32), r0=np.zeros(n, np.uint32), src=np.zeros((n, 2), np.uint32),
             n_ops=np.zeros(n, np.uint32), ops=np.zeros((n, max_ops), np.uint8), src_cut=np.zeros((n, 2), np.uint32),
             n_ops_cut=np.zeros(n, np.uint32), ops_cut=np.zeros((n, max_ops), np.uint8))
    m, x, go, ge, tgo, tge = scheme6
    FT.hh_full_tb(C.c_int(typ), C.c_int32(m), C.c_int32(x), C.c_int32(go), C.c_int32(ge), C.c_int32(tgo), C.c_int32(tge), _p(qtab),
                  _p(pat), _p(_u32(p_off)), _p(_u32(p_len)), _p(qual), _p(txt), _p(_u32(t_off)), _p(_u32(t_len)), C.c_uint32(n), C.c_uint32(max_ops),
                  _p(o["score"]), _p(o["sink"]), _p(o["r0"]), _p(o["src"]), _p(o["n_ops"]), _p(o["ops"]),
                  _p(o["src_cut"]), _p(o["n_ops_cut"]), _p(o["ops_cut"]))
    return o


@pytest.mark.parametrize("typ", [0, 1, 2])
def test_host_full_traceback_quality(FT, O, typ):
    """the full-matrix traceback with a table, both as the direction-matrix kernel runs it and as the warp traceback's lanes do on their
    cut window == the oracle's quality traceback: score, sink, source, n_ops and every op; M up to 512 (every lane width), N up to 1000"""
    rng = np.random.default_rng(4500 + typ)
    n_cut = 0
    for mb in (2, 0):
        qtab = quality_table(mb)
        for max_m, max_n, kw in ((256, 512, dict()), (512, 1000, dict(indel=0.02, tie=1.0)), (100, 300, dict(profile="low")),
                                 (200, 400, dict(profile="clamp", n_pat=0.02))):
            pr, qual = full_problems(rng, 25, max_m, max_n, **kw)
            max_ops = max_m + max_n + 1
            want = O.gotoh_full_traceback(typ, SCHEME6, *pr, max_ops=max_ops, qual=qual, qtab=qtab)
            got = full_tb(FT, typ, SCHEME6, pr, qual, qtab, max_ops)
            assert_same_traceback(dict(score=got["score"], sink=got["sink"], source=got["src"], n_ops=got["n_ops"], ops=got["ops"]), want,
                                  (typ, mb, max_m, kw))
            assert_same_traceback(dict(source=got["src_cut"], n_ops=got["n_ops_cut"], ops=got["ops_cut"]), want, (typ, mb, max_m, kw, "cut"))
            n_cut += int((got["r0"] > 0).sum())
    assert typ != 1 or n_cut > 20
