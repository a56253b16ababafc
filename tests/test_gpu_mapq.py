"""-m gpu: second-best distinct alignment and MAPQ of nvb_seed_extend_mapq against the oracle composition (tests/pipeline_oracle.py's
per-hit outputs + the second-best rule + BowtieMapq2, tests/mapq_oracle.py) on genomes with planted repeat families, and the same
outputs on every code path."""
import ctypes as C
import numpy as np
import pytest
import torch
from oracle import orc
import nvbio_b200 as nb
from nvbio_b200 import aln
from nvbio_b200.pipeline import MapqParams
from nvbio_b200.strings import PackedStringSet, pack_symbols
from tests.gpu_util import require_gpu, host_u32
from tests.pipeline_oracle import seed_extend_oracle
from tests.mapq_oracle import mapq_oracle, INT_MIN

pytestmark = pytest.mark.gpu

N_GENOME = 200_000


def rc(s):
    return np.where(s < 4, 3 - s, s)[::-1].astype(np.uint8)


def repeat_genome(seed=5):
    """random genome with repeat families for 100 bp reads: exact copies, copies with 1-3 substitutions per 100 bp, a reverse-complement
    copy, a period-40 tandem (neighbouring copies closer than len/2: not distinct) and a period-52 tandem (just beyond len/2)"""
    rng = np.random.default_rng(seed)
    g = rng.integers(0, 4, N_GENOME).astype(np.uint8)
    a = g[10_000:10_400].copy()
    g[30_000:30_400] = a; g[50_000:50_400] = a                                     # exact copies
    b = g[60_000:60_400].copy()
    for start, step in ((70_000, 100), (76_000, 50), (82_000, 33)):               # 1, 2 and 3 substitutions per 100 bp
        c = b.copy(); c[step // 2::step] = (c[step // 2::step] + 1) % 4
        g[start:start + 400] = c
    g[95_000:95_400] = rc(g[90_000:90_400])                                        # reverse-complement copy
    g[110_000:110_800] = np.tile(g[110_000:110_040], 20)                           # period 40 < 100 / 2
    g[120_000:120_832] = np.tile(g[120_000:120_052], 16)                           # period 52 > 100 / 2
    return g


def make_reads(g, n_reads=1200, L=100, ragged=False, seed=7):
    rng = np.random.default_rng(seed)
    regions = [(10_000, 300), (30_000, 300), (60_000, 300), (70_000, 300), (76_000, 300), (82_000, 300), (90_000, 300), (95_000, 300),
               (110_000, 700), (120_000, 730)]
    reads = []
    for i in range(n_reads):
        ln = int(rng.integers(L - 40, L + 1)) if ragged else L
        kind = i % 10
        if kind < 6:                                                                 # from a repeat family
            st, span = regions[int(rng.integers(0, len(regions)))]
            p = st + int(rng.integers(0, span - ln + 1))
        else:
            p = int(rng.integers(0, N_GENOME - ln))
        r = g[p:p + ln].copy()
        if kind == 6:
            r[rng.integers(0, ln, 2)] = rng.integers(0, 4, 2)
        elif kind == 7:                                                              # heavily mutated: some fall below the min score
            m = rng.random(ln) < 0.12
            r[m] = (r[m] + 1) % 4
        elif kind == 8 and i % 20 == 8:                                              # not from the genome: no hit
            r = rng.integers(0, 4, ln).astype(np.uint8)
        if rng.random() < 0.5:
            r = rc(r)
        reads.append(r)
    return reads


def packed(reads, bits=2, L=100):
    lens = np.array([len(r) for r in reads], np.uint32)
    offs = (np.cumsum(lens) - lens).astype(np.uint32)
    rs = PackedStringSet.from_symbols(np.concatenate(reads), offs, lens, bits=bits, big_endian=True)
    rs.length = L
    return rs


@pytest.fixture(scope="module")
def setup():
    require_gpu()
    O = orc.Oracle()
    g = repeat_genome()
    gw = torch.from_numpy(pack_symbols(g, 2, True).view(np.int32)).cuda()
    idx = O.build_index(g)
    fmi = nb.FMIndexDevice.from_host(idx.bwt_occ, idx.ssa, idx.L2, idx.n, idx.primary)
    return O, g, gw, idx, fmi


def run_mapq(fmi, gw, rs, params, mq, **kw):
    ws = nb.seed_extend(fmi, gw, rs, params, hit_capacity=1000 * rs.count, mapq=mq, **kw)
    torch.cuda.synchronize()
    return ws


def outputs(ws):
    return dict(best_score=ws.best_score.cpu().numpy().astype(np.int64), best_pos=host_u32(ws.best_pos).astype(np.int64),
                second_score=ws.second_score.cpu().numpy().astype(np.int64), second_pos=host_u32(ws.second_pos).astype(np.int64),
                second_strand=ws.second_strand.cpu().numpy().astype(np.int64), mapq=ws.mapq.cpu().numpy().astype(np.int64))


def check_vs_oracle(O, g, idx, fmi, gw, reads, rs, params, mq, quals=None):
    ws = run_mapq(fmi, gw, rs, params, mq)
    plain = nb.seed_extend(fmi, gw, rs, params, hit_capacity=1000 * rs.count)
    torch.cuda.synchronize()
    assert torch.equal(plain.best_score, ws.best_score) and torch.equal(plain.best_pos, ws.best_pos) and torch.equal(plain.n_hits, ws.n_hits)
    assert int(ws.n_hits[0]) == int(ws.n_hits[1])                                      # no hit dropped: the oracle keeps them all
    se = seed_extend_oracle(O, idx, g, reads, params, quals=quals)
    strands = 2 if params.both_strands else 1
    lens = np.array([len(r) for r in reads])
    want = mapq_oracle(se, lens, strands, mq.min_score.cpu().numpy(), mq.match_bonus)
    got = outputs(ws)
    for k in got:
        bad = np.nonzero(got[k] != want[k])[0]
        assert len(bad) == 0, (k, [(int(r), int(got[k][r]), int(want[k][r])) for r in bad[:5]])
    # the outputs cover the interesting cases
    has2 = want["second_score"] != INT_MIN
    aligned = want["best_score"] != INT_MIN
    min_s = mq.min_score.cpu().numpy()[lens]
    assert has2.sum() > 0.05 * len(reads) and (~has2 & aligned).sum() > 0.1 * len(reads)
    assert (has2 & (want["second_score"] == want["best_score"])).sum() > 20                  # equally good placements: low MAPQ
    if params.both_strands:
        assert (has2 & (want["second_strand"] != want["best_strand"])).sum() > 5                # the reverse-complement copy
    none = ~aligned
    assert none.sum() > 0 and (got["mapq"][none] == 0).all() and (got["second_pos"][none] == 0xFFFFFFFF).all()
    assert (got["second_strand"][~has2] == 0).all() and (got["second_pos"][~has2] == 0xFFFFFFFF).all()
    low = aligned & (want["best_score"] < min_s)
    assert (got["mapq"][low] == 0).all()
    return ws, want, low


@pytest.mark.parametrize("bits,ragged,both", [(2, False, True), (4, True, True), (2, True, False)])
def test_mapq_vs_oracle(setup, bits, ragged, both):
    O, g, gw, idx, fmi = setup
    reads = make_reads(g, ragged=ragged, seed=7 + bits)
    if bits == 4:
        rng = np.random.default_rng(3)
        for r in reads[::7]:
            r[rng.integers(0, len(r), 2)] = 4                                        # N
    rs = packed(reads, bits)
    params = nb.SeedExtendParams(seed_len=20, seed_interval=10, band_len=31, type=aln.LOCAL, both_strands=both, max_seed_hits=50,
                                 scheme=aln.SimpleGotohScheme(2, -2, -5, -3))
    check_vs_oracle(O, g, idx, fmi, gw, reads, rs, params, MapqParams.local(100))
    # a stricter min score (L,0,1.6: 160 of 200 for 100 bp) puts more reads below it: their MAPQ is 0
    _, _, low = check_vs_oracle(O, g, idx, fmi, gw, reads, rs, params, MapqParams.from_score_min("L", 0.0, 1.6, 100, 2))
    assert low.sum() > 3


def test_mapq_end_to_end(setup):
    """match bonus 0 (BowtieMapq2's monotone branch) with the end-to-end preset over SEMI_GLOBAL scores"""
    O, g, gw, idx, fmi = setup
    reads = make_reads(g, seed=21)
    rs = packed(reads)
    params = nb.SeedExtendParams(seed_len=22, seed_interval=10, band_len=31, type=aln.SEMI_GLOBAL, both_strands=True, max_seed_hits=50,
                                 scheme=aln.SimpleGotohScheme(0, -6, -5, -3))
    ws, want, low = check_vs_oracle(O, g, idx, fmi, gw, reads, rs, params, MapqParams.end_to_end(100))
    assert low.sum() > 5


def test_mapq_quality_scheme(setup):
    """nvBowtie's quality-dependent scoring (d_read_quals) through the new stage"""
    O, g, gw, idx, fmi = setup
    reads = make_reads(g, seed=33)
    rng = np.random.default_rng(9)
    quals = [rng.integers(0, 50, len(r)).astype(np.uint8) for r in reads]
    rs = packed(reads)
    sch = aln.QualityGotohScheme(match_bonus=2, mm_min=2, mm_max=6, read_gap_const=5, read_gap_coeff=3, ref_gap_const=5, ref_gap_coeff=3)
    params = nb.SeedExtendParams(seed_len=20, seed_interval=10, band_len=31, type=aln.LOCAL, both_strands=True, max_seed_hits=50, scheme=sch,
                                 read_quals=torch.from_numpy(np.concatenate(quals)).cuda())
    check_vs_oracle(O, g, idx, fmi, gw, reads, rs, params, MapqParams.local(100), quals=quals)


def test_mapq_same_on_every_path(setup):
    """per-read and per-hit paths, the exact shortcut on and off, job de-duplication on and off, the one- and two-pass seed match (full
    suffix array + located k-mer table), and with the traceback: identical second-best and MAPQ outputs; the traceback outputs equal
    nvb_seed_extend_traceback's"""
    O, g, gw, idx, fmi_s = setup
    L_ = nb.lib()
    reads = make_reads(g, n_reads=3000, ragged=True, seed=44)
    rs = packed(reads)
    params = nb.SeedExtendParams(seed_len=20, seed_interval=10, band_len=31, type=aln.LOCAL, both_strands=True, max_seed_hits=40,
                                 scheme=aln.SimpleGotohScheme(2, -2, -5, -3))
    mq = MapqParams.local(100)
    fmi = nb.FMIndexDevice.from_text(gw, N_GENOME, sa_interval=1)[0]
    fmi.build_ktab(8, located=True, text=gw)
    ref = outputs(run_mapq(fmi, gw, rs, params, mq))
    assert (ref["second_score"] != INT_MIN).sum() > 300

    def same(ws, what):
        got = outputs(ws)
        for k in got:
            assert np.array_equal(got[k], ref[k]), (what, k)

    same(run_mapq(fmi_s, gw, rs, params, mq), "sampled suffix array")
    for hook, off, on in ((L_.nvb_debug_pipeline_path, 1, 0), (L_.nvb_debug_perfect_shortcut, 0, 1), (L_.nvb_debug_seed_split, 0, 1)):
        hook(C.c_int(off))
        try:
            same(run_mapq(fmi, gw, rs, params, mq), hook.__name__)
        finally:
            hook(C.c_int(on))
    params.dedup_jobs = False
    same(run_mapq(fmi, gw, rs, params, mq), "dedup off")
    params.dedup_jobs = True
    same(run_mapq(fmi, gw, rs, params, mq, keep_hits=True), "per-hit outputs")
    tb = run_mapq(fmi, gw, rs, params, mq, traceback=True)
    same(tb, "traceback")
    plain = nb.seed_extend(fmi, gw, rs, params, hit_capacity=1000 * rs.count, traceback=True)
    torch.cuda.synchronize()
    for k in ("best_score", "best_pos", "best_ops", "best_n_ops", "best_begin", "best_strand"):
        assert torch.equal(getattr(tb, k), getattr(plain, k)), k


def test_debug_mapq_eval_equals_fixture():
    """the device build of the MAPQ function over the whole tests/golden/mapq.npz grid (nvBowtie's own BowtieMapq2)"""
    require_gpu()
    from tests.test_mapq import grid_points
    G = np.load(__file__.replace("test_gpu_mapq.py", "golden/mapq.npz"))
    cols, want = grid_points(G)
    d = [torch.from_numpy(np.ascontiguousarray(c).view(np.int32) if c.dtype == np.uint32 else np.ascontiguousarray(c)).cuda() for c in cols]
    out = torch.empty(len(want), dtype=torch.uint8, device="cuda")
    r = nb.lib().nvb_debug_mapq_eval(*[C.c_void_p(t.data_ptr()) for t in d], C.c_uint32(len(want)), C.c_void_p(out.data_ptr()),
                                     C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert r == 0
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy(), want)
