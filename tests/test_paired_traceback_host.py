"""CPU: the window cuts of the rescued-mate traceback (full_traceback_first_row, pipeline_core.cuh) and the lanes of its warp kernel
(FullTbLane + the step-major walk, gotoh_full_core.cuh), compiled for the host by tests/host/full_tb_harness.cu.  On thousands of random
full-matrix problems the traceback of the cut window [r0, sink.x) -- LOCAL with the front and end cuts, SEMI_GLOBAL with the end cut,
GLOBAL uncut -- equals the traceback of the whole window in every field, and the cut never excludes the source.  Score and sink are
also checked against the oracle's full-matrix Gotoh, and the ops against the reference's traceback where oracle/_ref is built."""
import ctypes as C
import os
import subprocess
import numpy as np
import pytest
from oracle import orc
from nvbio_b200.aln import QualityGotohScheme

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "host", "libfull_tb_harness.so")
SRC = os.path.join(HERE, "host", "full_tb_harness.cu")


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


@pytest.fixture(scope="module")
def H():
    deps = [SRC] + [os.path.join(HERE, "..", "nvbio_b200", "csrc", f) for f in
                    ("gotoh_full_core.cuh", "gotoh_core.cuh", "pipeline_core.cuh", "fm_core.cuh", "common.cuh")]
    if not os.path.exists(SO) or any(os.path.getmtime(d) > os.path.getmtime(SO) for d in deps):
        from nvbio_b200.build import NVCC
        subprocess.check_call([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17",
                               "-Wno-deprecated-declarations", "-Xcompiler", "-fPIC", "-shared", "-o", SO, SRC])
    return C.CDLL(SO)


def problems(rng, n, max_m, max_n, tight=False):
    """patterns drawn from their text (mutated, with indels; some at either end of the window) or random; tandem repeats of period
    1 / 2 / 7; tight: long windows with the pattern near the end, where D_max decides the cut"""
    pats, txts = [], []
    for _ in range(n):
        M = int(rng.integers(1, max_m + 1)); N = int(rng.integers(1, max_n + 1))
        t = rng.integers(0, 4, N).astype(np.uint8)
        if rng.random() < 0.2:
            per = int(rng.choice([1, 2, 7])); t = np.tile(rng.integers(0, 4, per).astype(np.uint8), N)[:N]
        if rng.random() < 0.7 and N >= M:
            where = rng.random()
            s = 0 if where < 0.2 else (N - M if where < 0.5 or tight else int(rng.integers(0, N - M + 1)))
            q = t[s:s + M].copy()
            mut = rng.random(M) < rng.choice([0.0, 0.03, 0.1])
            q[mut] = rng.integers(0, 4, int(mut.sum()))
            if M > 12 and rng.random() < 0.5:
                k, d = int(rng.integers(3, M - 6)), int(rng.integers(1, 4))
                q = np.concatenate([q[:k], q[k + d:], rng.integers(0, 4, d).astype(np.uint8)]) if rng.random() < 0.5 else \
                    np.concatenate([q[:k], rng.integers(0, 4, d).astype(np.uint8), q[k:M - d]])
        else:
            q = rng.integers(0, 4, M).astype(np.uint8)
            if rng.random() < 0.3:
                q = np.tile(q[:int(rng.choice([1, 2, 7]))], M)[:M]
        pats.append(q[:M]); txts.append(t)
    p_len = np.array([len(q) for q in pats], np.uint32); t_len = np.array([len(t) for t in txts], np.uint32)
    p_off = np.concatenate([[0], np.cumsum(p_len)[:-1]]).astype(np.uint32); t_off = np.concatenate([[0], np.cumsum(t_len)[:-1]]).astype(np.uint32)
    pad = np.zeros(8, np.uint8)
    return np.concatenate(pats + [pad]), p_off, p_len, np.concatenate(txts + [pad]), t_off, t_len


def run(H, typ, scheme, pr, qtab=None, quals=None, max_ops=1200):
    pat, p_off, p_len, txt, t_off, t_len = pr
    n = len(p_off)
    o = dict(score=np.zeros(n, np.int32), sink=np.zeros((n, 2), np.uint32), r0=np.zeros(n, np.uint32), src=np.zeros((n, 2), np.uint32),
             n_ops=np.zeros(n, np.uint32), ops=np.zeros((n, max_ops), np.uint8), src_cut=np.zeros((n, 2), np.uint32),
             n_ops_cut=np.zeros(n, np.uint32), ops_cut=np.zeros((n, max_ops), np.uint8))
    m, x, go, ge, tgo, tge = scheme
    H.hh_full_tb(C.c_int(typ), C.c_int32(m), C.c_int32(x), C.c_int32(go), C.c_int32(ge), C.c_int32(tgo), C.c_int32(tge), _p(qtab),
                 _p(pat), _p(p_off), _p(p_len), _p(quals), _p(txt), _p(t_off), _p(t_len), C.c_uint32(n), C.c_uint32(max_ops),
                 _p(o["score"]), _p(o["sink"]), _p(o["r0"]), _p(o["src"]), _p(o["n_ops"]), _p(o["ops"]),
                 _p(o["src_cut"]), _p(o["n_ops_cut"]), _p(o["ops_cut"]))
    return o


SCHEMES = [(2, -2, -5, -3, -5, -3), (1, -3, -4, -1, -4, -1), (0, -5, -8, -3, -8, -3), (2, -1, -1, -1, -1, -1)]


@pytest.mark.parametrize("typ", [0, 1, 2])
def test_cut_window_traceback_equals_full_window(H, typ):
    rng = np.random.default_rng(600 + typ)
    O = orc.Oracle()
    R = orc.Ref() if orc.Ref.available() else None
    total = cut = 0
    for si, sch in enumerate(SCHEMES + ["qual"]):
        for max_m, max_n, tight in ((40, 120, False), (150, 500, False), (150, 500, True), (300, 400, False)):
            qtab = quals = None
            pr = problems(rng, 250, max_m, max_n, tight)
            scheme = sch
            if sch == "qual":
                q = QualityGotohScheme(2, 2, 6, 5, 3, 5, 3, device="cpu")
                qtab = np.ascontiguousarray(q.table_host, dtype=np.int32)
                quals = rng.integers(0, 45, len(pr[0])).astype(np.uint8)
                scheme = (2, -6, q.pgo, q.pge, q.tgo, q.tge)
            o = run(H, typ, scheme, pr, qtab, quals)
            for k, kc in (("src", "src_cut"), ("n_ops", "n_ops_cut")):
                assert np.array_equal(o[k], o[kc]), (typ, sch, max_m, k)
            for a in range(len(pr[1])):
                k = min(int(o["n_ops"][a]), o["ops"].shape[1])
                assert np.array_equal(o["ops"][a, :k], o["ops_cut"][a, :k]), (typ, sch, a)
            assert np.all(o["r0"] <= o["src"][:, 0])                           # the cut never excludes the source
            if typ != 1:
                assert not o["r0"].any()
            total += len(pr[1]); cut += int((o["r0"] > 0).sum())
            # score / sink of the shipped full-matrix routine == the oracle's
            if sch != "qual":
                s, sx, sy = O.gotoh_full(typ, scheme[:4], *pr)
                assert np.array_equal(o["score"], s) and np.array_equal(o["sink"][:, 0], sx) and np.array_equal(o["sink"][:, 1], sy)
                if R is not None and si == 0 and max_m <= 256 and max_n <= 512:
                    want = R.gotoh_full_traceback(typ, scheme[:4], *pr, max_ops=1200)
                    assert np.array_equal(o["n_ops_cut"], want["n_ops"].astype(np.uint32))
    assert total >= 5000
    if typ == 1:
        assert cut > 0.3 * total


def test_tight_d_max_cut_is_exact(H):
    """alignments at the far end of long LOCAL windows with deletions: the cut row sits close to the source"""
    rng = np.random.default_rng(77)
    pr = problems(rng, 600, 150, 500, tight=True)
    o = run(H, 1, (2, -2, -5, -3, -5, -3), pr)
    assert np.array_equal(o["src"], o["src_cut"]) and np.array_equal(o["n_ops"], o["n_ops_cut"])
    gap = o["src"][:, 0].astype(np.int64) - o["r0"].astype(np.int64)
    assert gap.min() >= 0 and (o["r0"] > 0).sum() > 300
