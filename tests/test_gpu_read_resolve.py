"""pipe_resolve_reads_kernel (the per-read path of nvb_seed_extend): hit slots by a single-pass look-back over tiles of 128 reads, the
six-window de-duplication per read, truncation at the hit capacity and jobs that overflow a CTA's shared-memory stage.  Every result is
compared with the per-hit path (nvb_debug_pipeline_path(1)); the job count with a restatement of the de-duplication rule applied to the
per-hit path's hits."""
import ctypes as C

import numpy as np
import pytest
import torch

import nvbio_b200 as nb
from nvbio_b200 import aln, synth
from nvbio_b200.strings import PackedStringSet, pack_symbols, unpack_symbols
from tests.gpu_util import require_gpu, host_u32

pytestmark = pytest.mark.gpu

L = 150
LOCAL_WINDOWS = 6             # RJ_LOCAL: distinct windows remembered per read


def params(seed_interval=10):
    return nb.SeedExtendParams(seed_len=20, seed_interval=seed_interval, band_len=31, type=aln.LOCAL, both_strands=True,
                               max_seed_hits=40, scheme=aln.SimpleGotohScheme(2, -2, -5, -3))


def _debug(name, v):
    getattr(nb.lib(), name)(C.c_int(v))


@pytest.fixture(scope="module")
def genome():
    require_gpu()
    n = 400_000
    gw = synth.random_genome_words(n, seed=211)
    gsym = unpack_symbols(host_u32(gw), n).copy()
    gsym[100_000:130_000] = np.tile(gsym[5000:5500], 60)               # a 500 bp unit 60 times: reads there have ~40 hits per seed
    gw = torch.from_numpy(pack_symbols(gsym, 2, True).view(np.int32)).cuda()
    fmi, _ = nb.FMIndexDevice.from_text(gw, n, sa_interval=1)
    fmi.build_ktab(10, located=True, text=gw)                          # the headline index format: located ranges, two-pass match
    return n, gw, fmi


def reads(gw, n, n_reads, seed, lo=0, hi=None):
    rw, _, _ = synth.sample_reads(gw, n, n_reads, L, sub_rate=0.01, indel_rate=0.001, seed=seed, mut_seed=seed + 1)
    if hi is not None:                                                 # every read from [lo, hi): resample positions inside it
        sym = unpack_symbols(host_u32(gw), n)
        pos = np.random.default_rng(seed).integers(lo, hi - L, n_reads)
        buf = np.stack([sym[p:p + L] for p in pos]).astype(np.uint8)
        words = pack_symbols(np.concatenate([buf, np.zeros((n_reads, 160 - L), np.uint8)], 1).reshape(-1), 2, True).view(np.int32)
        rw = torch.from_numpy(words[:n_reads * 10].copy()).cuda().reshape(n_reads, 10)     # 160 symbols = 10 words per read
    return PackedStringSet.fixed(rw.reshape(-1), n_reads, L, stride=rw.shape[1] * 16)


def per_read(fmi, gw, rs, p, cap, **kw):
    kw.setdefault("traceback", True)                                   # (for the best alignment's strand)
    ws = nb.seed_extend(fmi, gw, rs, p, hit_capacity=cap, **kw)
    torch.cuda.synchronize()
    return ws


def per_hit(fmi, gw, rs, p, cap, **kw):
    kw.setdefault("traceback", True)
    _debug("nvb_debug_pipeline_path", 1)
    try:
        ws = nb.seed_extend(fmi, gw, rs, p, hit_capacity=cap, keep_hits=True, **kw)
        torch.cuda.synchronize()
    finally:
        _debug("nvb_debug_pipeline_path", 0)
    return ws


def jobs_of(ws):
    """the per-read path's job count restated: per read, in hit order, a hit whose (string, window) is among the first
    LOCAL_WINDOWS distinct ones already seen makes no job; every other hit does"""
    k = int(ws.n_hits[0])
    hs = ws.hit_read[:k].cpu().numpy().tolist()
    hw = ws.hit_window[:k].cpu().numpy().tolist()
    jobs, cur, seen = 0, None, []
    for s, (b, e) in zip(hs, hw):
        if s // 2 != cur:
            cur, seen = s // 2, []
        key = (s, b, e)
        if key in seen:
            continue
        if len(seen) < LOCAL_WINDOWS:
            seen.append(key)
        jobs += 1
    return jobs


def assert_same(fast, slow, what):
    assert torch.equal(fast.n_hits[:2], slow.n_hits[:2]), (what, fast.n_hits, slow.n_hits)
    assert torch.equal(fast.best_score, slow.best_score), what
    assert torch.equal(fast.best_pos, slow.best_pos), what
    for k in ("best_strand", "best_n_ops", "best_begin", "best_ops"):
        assert torch.equal(getattr(fast, k), getattr(slow, k)), (what, k)
    assert int(fast.n_hits[2]) == jobs_of(slow), (what, int(fast.n_hits[2]), jobs_of(slow))


@pytest.mark.parametrize("n_reads,seed_interval", [(1, 10), (127, 10), (128, 10), (129, 10), (5000, 10), (5000, 4), (200_000, 10)])
def test_tile_boundaries(genome, n_reads, seed_interval):
    """1 to 200,000 reads (partial, exact and many tiles of 128); seed interval 4: 66 seeds per read instead of 28"""
    n, gw, fmi = genome
    rs = reads(gw, n, n_reads, seed=n_reads)
    p = params(seed_interval)
    cap = 400 * n_reads
    fast, slow = per_read(fmi, gw, rs, p, cap), per_hit(fmi, gw, rs, p, cap)
    assert int(slow.n_hits[1]) <= cap
    assert_same(fast, slow, n_reads)


def test_truncation(genome):
    """a hit capacity inside a read's hits, on a read boundary, on a tile boundary, 0 and >= the total"""
    n, gw, fmi = genome
    n_reads = 1000
    rs = reads(gw, n, n_reads, seed=77)
    p = params()
    full = per_hit(fmi, gw, rs, p, 400 * n_reads)
    total = int(full.n_hits[1])
    per = np.bincount(full.hit_read[:total].cpu().numpy() // 2, minlength=n_reads)
    excl = np.concatenate([[0], np.cumsum(per)])
    r = int(np.nonzero(per[300:] >= 2)[0][0]) + 300
    caps = {"inside a read": int(excl[r]) + 1, "read boundary": int(excl[r]), "tile boundary": int(excl[256]), "zero": 0,
            "total": total, "above": total + 17}
    for what, cap in caps.items():
        fast, slow = per_read(fmi, gw, rs, p, cap), per_hit(fmi, gw, rs, p, cap)
        assert int(fast.n_hits[0]) == min(cap, total) and int(fast.n_hits[1]) == total, what
        assert_same(fast, slow, what)


def test_stage_overflow(genome):
    """reads from the repeat: ~40 hits per seed, far more jobs per CTA than its stage holds.  Results equal the per-hit path's and the
    shortcut-off run's; MAPQ, traceback and paired outputs equal the per-hit path's"""
    n, gw, fmi = genome
    n_reads = 2048
    rs = reads(gw, n, n_reads, seed=5, lo=100_000, hi=130_000)
    p = params()
    cap = 800 * n_reads
    fast, slow = per_read(fmi, gw, rs, p, cap), per_hit(fmi, gw, rs, p, cap)
    assert int(fast.n_hits[2]) > 640 * (n_reads // 128)               # some CTA staged more than RJ_STAGE jobs
    assert_same(fast, slow, "overflow")
    _debug("nvb_debug_perfect_shortcut", 0)
    try:
        off = per_read(fmi, gw, rs, p, cap)
    finally:
        _debug("nvb_debug_perfect_shortcut", 1)
    assert torch.equal(fast.best_score, off.best_score) and torch.equal(fast.best_pos, off.best_pos) and torch.equal(fast.n_hits, off.n_hits)

    mq = nb.MapqParams.local(L)
    a = per_read(fmi, gw, rs, p, cap, mapq=mq, traceback=True)
    _debug("nvb_debug_pipeline_path", 1)
    try:
        b = nb.seed_extend(fmi, gw, rs, p, hit_capacity=cap, mapq=mq, traceback=True)
        torch.cuda.synchronize()
    finally:
        _debug("nvb_debug_pipeline_path", 0)
    for k in ("best_score", "best_pos", "second_score", "second_pos", "second_strand", "mapq", "best_strand", "best_n_ops", "best_begin", "best_ops"):
        assert torch.equal(getattr(a, k), getattr(b, k)), k

    pair = nb.PairParams(min_frag=0, max_frag=600)
    outs = []
    for path in (0, 1):
        _debug("nvb_debug_pipeline_path", path)
        try:
            w = nb.seed_extend_paired(fmi, gw, rs, p, pair, hit_capacity=cap, mapq=mq, traceback=True)
            torch.cuda.synchronize()
        finally:
            _debug("nvb_debug_pipeline_path", 0)
        outs.append(w)
    for k in ("pair_score", "pair_flags", "mate_score", "mate_pos", "mate_strand", "n_rescue", "second_pair_score", "mate_mapq",
              "mate_n_ops", "mate_begin", "mate_ops"):
        assert torch.equal(getattr(outs[0], k), getattr(outs[1], k)), k
