"""-m gpu: seed + extend on long and mixed-length reads, against the oracle composition (tests/pipeline_oracle.py, mapq_oracle.py,
pair_mapq_oracle.py, finish_oracle.py, bam_oracle.py).  The rest of the suite runs the whole chain on reads of at most 150 bp, while
several parts of it depend on the read length: the Gotoh route is chosen once per call from the batch's maximum length (the 16-bit packed
kernels' selector rows and LOCAL key rules), the rescue DP has its own LOCAL key rule, the per-hit leader look-back and the per-read
de-duplication remember a bounded number of hits / windows, and seeds per string, direction-matrix rows, max_ops, the MAPQ min-score table,
distinct_alignment's len / 2, the pairing's begin = end - len and the CIGAR / MD bounds all scale with it.

  1. single end, per-hit path, every hit (string, window, score, sink) and the best per read at 151 .. 2000 bp (fixed-length batches) and on
     a ragged 12 .. 2000 bp batch (2-bit, 4-bit with N, base qualities, and the reference-format index), LOCAL at bands 7 / 15 / 31 / 63 and
     every type at bands 7 / 15 / 31, schemes (2, -2, -5, -3) and (3, -1, -2, -2); a 150 bp batch with one 1024 bp read added;
  2. the packed kernels' length edges crossed through seed + extend, the route read back after each call: 682 / 683 at match 3 (LOCAL key
     rule), 770 / 771 at band 31 (selector rows), and through the paired rescue DP 511 / 512 at match 4 and 1023 / 1024 at match 2;
  3. the per-read path (shortcut on, without its one-gap check, off; seed split on and off) equal to the oracle and the per-hit path, its
     job count between the distinct (string, window) pairs and the kept hits, and a hit capacity that cuts a long read's hits;
  4. the traceback at bands 7 / 15 / 31 and every type equal to the oracle's banded traceback of the best job, and a max_ops that truncates;
  5. MAPQ on the ragged batch (LOCAL and end-to-end tables sized 2000), reads in a period-150 tandem repeat deciding distinctness by len / 2;
  6. paired end at 250 / 250, 300 / 150, 511 / 511, 511 / 512, 512 / 512 (traceback) and 600 / 600, 1023 / 1023, 1024 / 1024 (no
     traceback); 513 bp mates refused by the traceback;
  7. finish and BAM records of the long tracebacks, on contigs cut under some alignments;
  8. the streaming API at 300 bp (19 words per read), single end and paired.

The genome (400,003 symbols: not a multiple of 16) carries a repeat family (a 2,600 bp unit, longer than any read, copied four times, two
copies with a few substitutions), a period-7 tandem and a period-150 tandem.  The oracle's CPU DP is most of the run time: the band x type x
scheme product is spread over the lengths instead of run at each."""
import ctypes as C
import numpy as np
import pytest
import torch
from oracle import orc
from oracle.ref_bam import RefBam
import nvbio_b200 as nb
from nvbio_b200 import aln
from nvbio_b200._lib import NvbError
from nvbio_b200.pipeline import MapqParams, SeedExtendWorkspace
from nvbio_b200.strings import PackedStringSet, pack_symbols
from tests import bam_oracle as bo
from tests.gpu_util import require_gpu, host_u32
from tests.mapq_oracle import mapq_oracle
from tests.pair_mapq_oracle import pair_mapq_oracle
from tests.pipeline_oracle import seed_extend_oracle, _scheme_args
from tests.test_gpu_bam import planted_contigs, host_inputs, check_records
from tests.test_gpu_finish import check_device
from tests.test_gpu_paired_traceback import strand_string, PAIR_KEYS, TB_KEYS, MAPQ_KEYS
from tests.test_gpu_pipeline_matrix import assert_hits_equal, assert_best_equal, best_of, check_traceback, read_set, rc

pytestmark = pytest.mark.gpu

N_GENOME = 400_003
UNIT = 2_600                                    # repeat-family unit: longer than the longest read
FAMILY = (100_000, 140_000, 180_000, 220_000)   # copies of g[5000:7600]; the last two with a few substitutions
EXACT_COPIES = (5_000, 100_000, 140_000)
TANDEM7 = (300_000, 310_000)
TANDEM150 = (320_000, 326_000)
INT_MIN = -2**31
NONE = 0xFFFFFFFF
SEED_LEN, SEED_INTERVAL, MAX_SEED_HITS = 20, 10, 16

A = aln.SimpleGotohScheme(2, -2, -5, -3)
B = aln.SimpleGotohScheme(3, -1, -2, -2)
M4 = aln.SimpleGotohScheme(4, -4, -6, -2)
LO, SG, GL = aln.LOCAL, aln.SEMI_GLOBAL, aln.GLOBAL

# (band, type, scheme) per fixed length: every LOCAL band and every type at bands 7 / 15 / 31 appear; the first entry of an edge length is
# the configuration its route is asserted at
PLAN = {
    151:  [(7, LO, A), (15, SG, B)],
    250:  [(15, LO, B), (31, GL, A)],
    300:  [(31, LO, A), (7, SG, A)],
    511:  [(63, LO, B), (15, GL, B), (7, GL, A)],
    512:  [(7, LO, B), (31, SG, B)],
    513:  [(15, LO, A), (15, SG, A)],
    682:  [(15, LO, B), (31, GL, A)],
    683:  [(15, LO, B), (7, SG, B)],
    770:  [(31, LO, A), (63, LO, A)],
    771:  [(31, LO, A), (15, GL, A)],
    1023: [(31, LO, A), (31, SG, A)],
    1024: [(31, LO, A), (7, LO, A)],
    2000: [(31, LO, A), (15, SG, B)],
}
# route of the extension at an edge length under its first PLAN entry: 1 = the packed pair kernel, 0 = int32 only
#   682 / 683, match 3: LOCAL keys (h << 5) | j need max_m * match < 2048 (2046 / 2049)
#   770 / 771, band 31: the selector rows (max_m + band - 1, rounded up to 16) x 128 threads x 2 bytes must fit 200 KB
#   1023 / 1024: past the selector-row limit of every band, so int32 on both sides (the match-2 key edge is crossed by the rescue DP)
EDGE_ROUTES = {682: 1, 683: 0, 770: 1, 771: 0, 1023: 0, 1024: 0}
RAGGED_CONFIGS = [(7, LO, A), (15, LO, B), (31, LO, A), (63, LO, B), (15, SG, A), (31, SG, B), (15, GL, B), (31, GL, A)]


def _debug(name, v):
    getattr(nb.lib(), name)(C.c_int(v))


def last_route():
    packed, n = C.c_int(-1), C.c_uint32(0xFFFFFFFF)
    assert nb.lib().nvb_debug_gotoh_last_route(C.byref(packed), C.byref(n)) == 0
    return packed.value, n.value


def params(band, typ, scheme, **kw):
    return nb.SeedExtendParams(seed_len=SEED_LEN, seed_interval=SEED_INTERVAL, band_len=band, type=typ, both_strands=True,
                               max_seed_hits=MAX_SEED_HITS, scheme=scheme, **kw)


def capacity(reads):
    """every hit kept"""
    K = (max(len(r) for r in reads) - SEED_LEN) // SEED_INTERVAL + 1
    return 2 * K * MAX_SEED_HITS * len(reads) + 1024


def mutate(r, q, rng):
    r[q] = (r[q] + 1 + rng.integers(0, 3, np.size(q))) % 4


# ---------------------------------------------------------------------------------------------------------------------------------------
# world
# ---------------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def world():
    require_gpu()
    O = orc.Oracle()
    rng = np.random.default_rng(2000)
    n = N_GENOME
    g = rng.integers(0, 4, n).astype(np.uint8)
    unit = g[5_000:5_000 + UNIT].copy()
    for k, st in enumerate(FAMILY):
        u = unit.copy()
        if k >= 2:
            mutate(u, rng.choice(UNIT, 6, replace=False), rng)
        g[st:st + UNIT] = u
    g[TANDEM7[0]:TANDEM7[1]] = np.tile(g[TANDEM7[0]:TANDEM7[0] + 7], 2000)[:TANDEM7[1] - TANDEM7[0]]
    g[TANDEM150[0]:TANDEM150[1]] = np.tile(g[TANDEM150[0]:TANDEM150[0] + 150], 40)[:TANDEM150[1] - TANDEM150[0]]
    gw = torch.from_numpy(pack_symbols(np.concatenate([g, np.zeros(128, np.uint8)]), 2, True).view(np.int32)).cuda()
    idx = O.build_index(g)
    fmi, _ = nb.FMIndexDevice.from_text(gw, n, sa_interval=1)
    fmi.build_ktab(10, located=True, text=gw)
    ref_fmi = nb.FMIndexDevice.from_host(idx.bwt_occ, idx.ssa, idx.L2, idx.n, idx.primary)       # SA every 16, no k-mer table
    assert fmi.rows is not None
    return dict(O=O, g=g, gw=gw, idx=idx, fmi=fmi, ref_fmi=ref_fmi, n=n)


def sampled(g, L, rng):
    """L symbols from a random position with 1 % substitutions and 0.2 % indels (1-3 bp), either strand"""
    n = len(g)
    p = int(rng.integers(0, n - L - 100))
    r = g[p:p + L + 100].copy()
    m = rng.random(len(r)) < 0.01
    mutate(r, np.flatnonzero(m), rng)
    for q in sorted(np.flatnonzero(rng.random(L) < 0.002), reverse=True):
        k = int(rng.integers(1, 4))
        r = np.concatenate([r[:q], r[q + k:]]) if rng.random() < 0.5 else np.concatenate([r[:q], rng.integers(0, 4, k).astype(np.uint8), r[q:]])
    r = r[:L]
    return rc(r) if rng.random() < 0.5 else r


def kind_read(g, L, kind, rng):
    """one read of length L of a given kind (see fixed_reads)"""
    n = len(g)
    if kind == "sampled":
        return sampled(g, L, rng)
    if kind == "exact":
        p = int(rng.integers(0, n - L)); r = g[p:p + L].copy()
    elif kind == "sub2":
        p = int(rng.integers(0, n - L)); r = g[p:p + L].copy(); mutate(r, rng.choice(L, 2, replace=False), rng)
    elif kind == "indel":
        p = int(rng.integers(0, n - L - 8)); k = int(rng.integers(3, 7)); cut = L - k if rng.random() < 0.5 else k
        r = np.concatenate([g[p:p + cut], rng.integers(0, 4, int(rng.integers(1, 4))).astype(np.uint8), g[p + cut:p + L]])[:L] \
            if rng.random() < 0.5 else np.concatenate([g[p:p + cut], g[p + cut + int(rng.integers(1, 4)):p + L + 4]])[:L]
    elif kind == "start":
        r = g[:L].copy()
    elif kind == "end":
        r = g[n - L:].copy()
    elif kind == "past":
        k = int(rng.choice([3, 9, 40]))
        r = np.concatenate([g[n - L + k:], rng.integers(0, 4, k).astype(np.uint8)])
    elif kind == "family":
        st = int(rng.choice(FAMILY)); p = st + int(rng.integers(0, UNIT - L + 1)); r = g[p:p + L].copy()
    elif kind == "tandem7":
        p = int(rng.integers(TANDEM7[0], TANDEM7[1] - L)); r = g[p:p + L].copy()
    elif kind == "tandem150":
        p = int(rng.integers(TANDEM150[0], TANDEM150[1] - L)); r = g[p:p + L].copy()
    else:
        raise ValueError(kind)
    return rc(r) if rng.random() < 0.5 else r


FIXED_KINDS = ["sampled"] * 28 + ["exact"] * 6 + ["sub2"] * 4 + ["indel"] * 4 + ["start", "start", "end", "end", "past", "past", "past"] + \
              ["family"] * 8 + ["tandem7"] * 2 + ["tandem150"] * 2


def fixed_reads(w, L):
    rng = np.random.default_rng(L)
    return [kind_read(w["g"], L, k, rng).astype(np.uint8) for k in FIXED_KINDS]


RAGGED_LENGTHS = [12, 15, 19, 20, 31, 32, 33, 47, 48, 49, 100, 127, 128, 129, 150, 151, 255, 256, 257, 300, 511, 512, 513, 682, 683,
                  767, 768, 769, 1023, 1024, 1025, 1500, 1999, 2000]


@pytest.fixture(scope="module")
def ragged(world):
    """12 .. 2000 bp: shorter than a seed, lengths = 0, 1 and 15 mod 16, every kind of read; 4-bit copies with some N; base qualities"""
    rng = np.random.default_rng(77)
    kinds = ["sampled", "exact", "sub2", "indel", "family", "tandem150", "sampled", "past", "tandem7", "end", "start", "family"]
    reads = []
    for i, L in enumerate(RAGGED_LENGTHS + [int(v) for v in rng.integers(21, 2001, 46)]):
        k = kinds[i % len(kinds)]
        if L > 1990 and k in ("tandem7",):
            k = "sampled"
        reads.append(kind_read(world["g"], L, k, rng).astype(np.uint8))
    four = []
    for r in reads:
        r = r.copy(); r[rng.random(len(r)) < 0.004] = 4; four.append(r)
    quals = [rng.integers(2, 41, len(r)).astype(np.uint8) for r in reads]
    return dict(reads=reads, four=four, quals=quals)


# ---------------------------------------------------------------------------------------------------------------------------------------
# the checks of one (batch, configuration): per-hit path vs the oracle, per-read path, traceback
# ---------------------------------------------------------------------------------------------------------------------------------------
def per_hit(w, fmi, reads, p, bits=2, quals=None, what=()):
    """per-hit path: every hit and the best per read equal the oracle; returns (oracle result, per-hit best, route of the extension)"""
    want = seed_extend_oracle(w["O"], w["idx"], w["g"], reads, p, quals=quals)
    rs = read_set(reads, bits)
    ws = nb.seed_extend(fmi, w["gw"], rs, p, hit_capacity=capacity(reads), keep_hits=True)
    route = last_route()            # (no traceback, MAPQ or pairs: the extension is the call's only Gotoh call)
    assert_hits_equal(ws, want, what)
    got = best_of(ws)
    assert_best_equal(got, want, what + ("per hit",))
    return want, got, route


def per_read(w, fmi, reads, p, want, bits=2, what=()):
    """per-read path, shortcut on / without its one-gap check / off and seed split on / off: the best per read equals the oracle;
    distinct (string, window) pairs <= jobs <= kept hits"""
    rs = read_set(reads, bits)
    pairs = set(zip(want["hit_string"].tolist(), map(tuple, want["hit_window"].tolist())))
    eligible = p.type == LO and p.band_len <= 32 and bits == 2 and p.read_quals is None
    try:
        for split in (1, 0):
            _debug("nvb_debug_seed_split", split)
            for sc in ((1, 2, 0) if eligible else (1,)):
                _debug("nvb_debug_perfect_shortcut", sc)
                ws = nb.seed_extend(fmi, w["gw"], rs, p, hit_capacity=capacity(reads))
                got = best_of(ws)
                assert_best_equal(got, want, what + ("per read", split, sc))
                assert len(pairs) <= got["n_hits"][2] <= got["n_hits"][0], what + (split, sc, len(pairs), got["n_hits"])
    finally:
        _debug("nvb_debug_seed_split", 1); _debug("nvb_debug_perfect_shortcut", 1)


def traceback(w, fmi, reads, p, want, bits=2, what=()):
    """seed_extend(traceback=True) on the per-read path: the best per read equals the oracle, every alignment the oracle's banded traceback
    of the read's best job (strand included), replayed to its score and end"""
    rs = read_set(reads, bits)
    ws = nb.seed_extend(fmi, w["gw"], rs, p, hit_capacity=capacity(reads), traceback=True)
    best = best_of(ws)
    assert_best_equal(best, want, what + ("traceback",))
    ops, n_ops = ws.best_ops.cpu().numpy(), ws.best_n_ops.cpu().numpy()
    begin, strand = host_u32(ws.best_begin), ws.best_strand.cpu().numpy()
    checked = check_traceback(w, reads, p, best, ops, n_ops, begin, strand, want, what)
    assert checked > 0.8 * len(reads), what
    assert (n_ops <= ws.max_ops).all(), what
    # alignments pairing insertions with deletions: more ops than read length + band + 1 (a buffer of that size truncated them)
    return int(sum(n_ops[a] > len(r) + p.band_len + 1 for a, r in enumerate(reads)))


def run_config(w, reads, cfg, what):
    band, typ, scheme = cfg
    p = params(band, typ, scheme)
    want, _, route = per_hit(w, w["fmi"], reads, p, what=what)
    per_read(w, w["fmi"], reads, p, want, what=what)
    long_ops = traceback(w, w["fmi"], reads, p, want, what=what) if band <= 31 else 0
    return want, route, long_ops


# ---------------------------------------------------------------------------------------------------------------------------------------
# 1-4. fixed-length batches
# ---------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("L", sorted(PLAN))
def test_fixed_length(world, L):
    w = world
    reads = fixed_reads(w, L)
    long_ops = 0
    for i, cfg in enumerate(PLAN[L]):
        what = (L, cfg[0], cfg[1], repr(cfg[2]))
        want, route, k = run_config(w, reads, cfg, what)
        long_ops += k
        print("L %d band %d type %d %r: route %s, %d hits, %d alignments longer than L + band + 1 ops" % (L, cfg[0], cfg[1], cfg[2], route,
                                                                                                        want["n_hits"], k))
        if i == 0 and L in EDGE_ROUTES:
            assert route[0] == EDGE_ROUTES[L], (what, route)
        # more than 64 hits on the strings of the repeat-family reads (the per-hit leader look-back's limit)
        fam = [a for a, k in enumerate(FIXED_KINDS) if k == "family"]
        per_string = np.bincount(want["hit_string"], minlength=2 * len(reads))
        assert max(per_string[2 * a:2 * a + 2].max() for a in fam) > 64, what
        aligned = want["best_score"] != INT_MIN
        assert aligned.sum() > 0.8 * len(reads), what
    if L in (511, 2000):
        assert long_ops > 0, L


def test_packed_edge_both_sides(world):
    """each edge as a pair of calls on the same kind of reads, one below and one above it (the per-length test above pins each value)"""
    w = world
    for lo, hi, cfg in ((682, 683, (15, LO, B)), (770, 771, (31, LO, A))):
        routes = []
        for L in (lo, hi):
            reads = fixed_reads(w, L)[:20]
            rs = read_set(reads)
            nb.seed_extend(w["fmi"], w["gw"], rs, params(*cfg), hit_capacity=capacity(reads), keep_hits=True)
            routes.append(last_route()[0])
        print("edge %d / %d: routes %s" % (lo, hi, routes))
        assert routes == [1, 0], (lo, hi, routes)


def test_short_batch_with_one_long_read(world):
    """150 bp reads with one 1024 bp read added: the whole DP list leaves the packed kernel and the 150 bp reads' hits and results do not
    change"""
    w = world
    rng = np.random.default_rng(150)
    short = [kind_read(w["g"], 150, k, rng).astype(np.uint8) for k in FIXED_KINDS]
    long_ = fixed_reads(w, 1024)[0]
    p = params(31, LO, A)
    want_s, got_s, route_s = per_hit(w, w["fmi"], short, p, what=("short",))
    want_l, got_l, route_l = per_hit(w, w["fmi"], short + [long_], p, what=("short + 1024",))
    print("150 bp batch: route %s; with a 1024 bp read: route %s" % (route_s, route_l))
    assert route_s[0] == 1 and route_l[0] == 0
    n = len(short)
    for k in ("best_score", "best_pos"):
        assert np.array_equal(got_l[k][:n], got_s[k])
    hs = want_l["hit_string"] < 2 * n
    for k in ("hit_string", "hit_window", "hit_score", "hit_sink"):
        assert np.array_equal(want_l[k][hs], want_s[k])
    per_read(w, w["fmi"], short + [long_], p, want_l, what=("short + 1024",))


def test_truncated_hits_inside_a_long_read(world):
    """a hit capacity inside the hits of a 2000 bp repeat-family read: the per-read path equals the per-hit path with the same capacity"""
    w = world
    reads = fixed_reads(w, 2000)
    p = params(31, LO, A)
    rs = read_set(reads)
    full = nb.seed_extend(w["fmi"], w["gw"], rs, p, hit_capacity=capacity(reads), keep_hits=True)
    torch.cuda.synchronize()
    total = int(full.n_hits[1])
    per = np.bincount(full.hit_read[:total].cpu().numpy() // 2, minlength=len(reads))
    excl = np.concatenate([[0], np.cumsum(per)])
    fam = [a for a, k in enumerate(FIXED_KINDS) if k == "family"]
    r = max(fam, key=lambda a: per[a])
    assert per[r] > 128
    for cap in (int(excl[r]) + 1, int(excl[r]) + 65, int(excl[r + 1]) - 1):
        _debug("nvb_debug_pipeline_path", 1)
        try:
            slow = nb.seed_extend(w["fmi"], w["gw"], rs, p, hit_capacity=cap, keep_hits=True, traceback=True)
            torch.cuda.synchronize()
        finally:
            _debug("nvb_debug_pipeline_path", 0)
        fast = nb.seed_extend(w["fmi"], w["gw"], rs, p, hit_capacity=cap, traceback=True)
        torch.cuda.synchronize()
        assert int(fast.n_hits[0]) == cap and int(fast.n_hits[1]) == total, cap
        assert torch.equal(fast.n_hits[:2], slow.n_hits[:2]), cap
        for k in ("best_score", "best_pos", "best_strand", "best_n_ops", "best_begin", "best_ops"):
            assert torch.equal(getattr(fast, k), getattr(slow, k)), (cap, k)
        assert int(fast.n_hits[2]) <= cap


def test_traceback_max_ops_truncates(world):
    """a max_ops below what the alignments need: n_ops counts every op, only the first max_ops (END -> START) are stored"""
    w = world
    reads = fixed_reads(w, 511)
    p = params(15, LO, A)
    rs = read_set(reads)
    full = nb.seed_extend(w["fmi"], w["gw"], rs, p, hit_capacity=capacity(reads), traceback=True)
    ws = SeedExtendWorkspace(w["fmi"], w["gw"], rs, p, capacity(reads), traceback=True)
    small = 300
    ws.max_ops = small                      # the rows of best_ops are then small apart
    nb.seed_extend(w["fmi"], w["gw"], rs, p, workspace=ws)
    torch.cuda.synchronize()
    n = len(reads)
    n_full, n_small = full.best_n_ops.cpu().numpy(), ws.best_n_ops.cpu().numpy()
    assert np.array_equal(n_small, n_full) and (n_full > small).sum() > 0.5 * n
    ops = ws.best_ops.reshape(-1)[:n * small].reshape(n, small).cpu().numpy()
    fo = full.best_ops.cpu().numpy()
    for a in range(n):
        k = min(int(n_full[a]), small)
        assert np.array_equal(ops[a, :k], fo[a, :k]), a
    assert torch.equal(ws.best_begin, full.best_begin) and torch.equal(ws.best_score, full.best_score)


# ---------------------------------------------------------------------------------------------------------------------------------------
# 1, 3, 4. the ragged batch
# ---------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg", RAGGED_CONFIGS, ids=lambda c: "b%d_t%d_%r" % c)
def test_ragged(world, ragged, cfg):
    w = world
    reads = ragged["reads"]
    what = ("ragged",) + (cfg[0], cfg[1], repr(cfg[2]))
    want, route, _ = run_config(w, reads, cfg, what)
    assert route[0] == 0, what                                  # a 2000 bp read in the batch: int32 for every job
    short = [a for a, r in enumerate(reads) if len(r) < SEED_LEN]
    assert short and all(want["best_score"][a] == INT_MIN for a in short)


def test_ragged_4bit_quality_and_reference_index(world, ragged):
    w = world
    # 4-bit reads with N
    p = params(31, LO, A)
    want, _, _ = per_hit(w, w["fmi"], ragged["four"], p, bits=4, what=("4-bit",))
    per_read(w, w["fmi"], ragged["four"], p, want, bits=4, what=("4-bit",))
    traceback(w, w["fmi"], ragged["four"], p, want, bits=4, what=("4-bit",))
    # base qualities
    q = torch.from_numpy(np.concatenate(ragged["quals"])).cuda()
    pq = params(15, LO, aln.QualityGotohScheme(2, 2, 6, 5, 3, 5, 3), read_quals=q)
    want, _, _ = per_hit(w, w["fmi"], ragged["reads"], pq, quals=ragged["quals"], what=("quality",))
    per_read(w, w["fmi"], ragged["reads"], pq, want, what=("quality",))
    # the reference-format index (SA every 16, no k-mer table)
    want, _, _ = per_hit(w, w["ref_fmi"], ragged["reads"], p, what=("reference index",))
    per_read(w, w["ref_fmi"], ragged["reads"], p, want, what=("reference index",))


# ---------------------------------------------------------------------------------------------------------------------------------------
# 5. MAPQ on the ragged batch
# ---------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["local", "end_to_end"])
def test_ragged_mapq(world, ragged, mode):
    w = world
    reads = ragged["reads"]
    if mode == "local":
        p, mq = params(31, LO, A), MapqParams.local(2000)
    else:
        p, mq = params(31, SG, aln.SimpleGotohScheme(0, -6, -5, -3)), MapqParams.end_to_end(2000)
    rs = read_set(reads)
    ws = nb.seed_extend(w["fmi"], w["gw"], rs, p, hit_capacity=capacity(reads), mapq=mq)
    torch.cuda.synchronize()
    assert int(ws.n_hits[0]) == int(ws.n_hits[1])
    se = seed_extend_oracle(w["O"], w["idx"], w["g"], reads, p)
    lens = np.array([len(r) for r in reads])
    want = mapq_oracle(se, lens, 2, mq.min_score.cpu().numpy(), mq.match_bonus)
    got = dict(best_score=ws.best_score.cpu().numpy().astype(np.int64), best_pos=host_u32(ws.best_pos).astype(np.int64),
               second_score=ws.second_score.cpu().numpy().astype(np.int64), second_pos=host_u32(ws.second_pos).astype(np.int64),
               second_strand=ws.second_strand.cpu().numpy().astype(np.int64), mapq=ws.mapq.cpu().numpy().astype(np.int64))
    for k in got:
        bad = np.flatnonzero(got[k] != want[k])
        assert len(bad) == 0, (mode, k, [(int(r), len(reads[r]), int(got[k][r]), int(want[k][r])) for r in bad[:5]])
    # reads in the period-150 tandem longer than 300 bp: equally good placements 150 apart are not distinct, an equal second lies more than
    # len / 2 away
    tandem = [a for a, r in enumerate(reads) if len(r) > 300 and ragged_kind(a) == "tandem150" and want["second_score"][a] == want["best_score"][a]]
    assert tandem
    for a in tandem:
        assert abs(int(want["second_pos"][a]) - int(want["best_pos"][a])) > len(reads[a]) // 2, a
    # the path without per-hit outputs gives the same
    _debug("nvb_debug_pipeline_path", 1)
    try:
        slow = nb.seed_extend(w["fmi"], w["gw"], rs, p, hit_capacity=capacity(reads), mapq=mq)
        torch.cuda.synchronize()
    finally:
        _debug("nvb_debug_pipeline_path", 0)
    for k in ("best_score", "best_pos", "second_score", "second_pos", "second_strand", "mapq"):
        assert torch.equal(getattr(slow, k), getattr(ws, k)), k


def ragged_kind(a):
    kinds = ["sampled", "exact", "sub2", "indel", "family", "tandem150", "sampled", "past", "tandem7", "end", "start", "family"]
    return kinds[a % len(kinds)]


# ---------------------------------------------------------------------------------------------------------------------------------------
# 6. paired end
# ---------------------------------------------------------------------------------------------------------------------------------------
def pair_reads(w, L1, L2, n_pairs, max_frag, seed):
    """FR pairs: sampled fragments up to max_frag + 60 (some just beyond it), mate 1 forward or reverse, every fifth second mate heavily
    mutated; pairs at the genome's start and end; and, at each exact copy of the repeat family, mate 1 forward starting 400 bp before the
    copy and mate 2 (the same symbols at every copy) reverse inside it -- mate 2's single-end best is one of the copies, so the other pairs
    are rescued onto an exact copy (LOCAL score len * match)"""
    g, n = w["g"], w["n"]
    rng = np.random.default_rng(seed)
    m1, m2 = [], []
    for i in range(n_pairs):
        f = int(rng.integers(max(L1, L2) + 20, max_frag + 60))
        p = int(rng.integers(0, n - f))
        if i % 2 == 0:
            a, b = g[p:p + L1].copy(), rc(g[p + f - L2:p + f])
        else:                                                       # mate 1 reverse
            a, b = rc(g[p + f - L1:p + f]), g[p:p + L2].copy()
        mutate(a, np.flatnonzero(rng.random(L1) < 0.01), rng)
        mutate(b, np.flatnonzero(rng.random(L2) < (0.15 if i % 5 == 0 else 0.01)), rng)
        m1.append(a); m2.append(b)
    m1.append(g[:L1].copy()); m2.append(rc(g[max_frag - 100 - L2:max_frag - 100]))
    m1.append(g[n - max_frag + 50:n - max_frag + 50 + L1].copy()); m2.append(rc(g[n - L2:]))
    f = 400 + L2 + 26
    for c in EXACT_COPIES:
        m1.append(g[c - 400:c - 400 + L1].copy()); m2.append(rc(g[c - 400 + f - L2:c - 400 + f]))
    return m1 + m2, len(m1)


PAIRED = [  # (name, L1, L2, scheme, band, min_mate_score, traceback, route of the rescue DP: 1 packed pair kernel, 2 warp kernel, 0 int32)
    ("250/250", 250, 250, A, 31, 100, True, 2),
    ("300/150", 300, 150, A, 15, 100, True, 1),
    ("511/511", 511, 511, M4, 31, 400, True, 1),          # match 4: min(m, n) * 4 = 2044 < 2048
    ("511/512", 511, 512, M4, 31, 400, True, 0),          # the batch's maximum, 512: 2048
    ("512/512", 512, 512, M4, 15, 400, True, 0),
    ("600/600", 600, 600, A, 31, 150, False, 1),
    ("1023/1023", 1023, 1023, A, 31, 200, False, 1),      # match 2: 2046 < 2048
    ("1024/1024", 1024, 1024, A, 31, 200, False, 0),
]


def paired_oracle_checks(w, reads, n_pairs, p, pair, got, mq):
    want = pair_mapq_oracle(w["O"], w["idx"], w["g"], reads, p, pair, n_pairs, mq.min_score.cpu().numpy(), mq.match_bonus)
    assert tuple(int(v) for v in got["n_rescue"]) == tuple(want["n_rescue"])
    for k in ("pair_score", "pair_flags", "mate_score", "mate_pos", "mate_strand", "second_pair_score", "second_mate_pos",
              "second_mate_strand", "mate_second_score", "mate_mapq"):
        g = got[k].view(np.uint32).astype(np.int64) if k in ("mate_pos", "second_mate_pos") else got[k].astype(np.int64)
        assert np.array_equal(g, want[k]), (k, np.argwhere(g != want[k])[:6].tolist())
    return want


@pytest.mark.parametrize("case", PAIRED, ids=lambda c: c[0])
def test_paired(world, case):
    name, L1, L2, scheme, band, min_ms, tb, rescue_route = case
    w = world
    max_frag = 1500 if max(L1, L2) > 300 else 800
    reads, n_pairs = pair_reads(w, L1, L2, 36, max_frag, seed=L1 * 7 + L2)
    p = params(band, LO, scheme)
    pair = nb.PairParams(min_frag=0, max_frag=max_frag, min_mate_score=min_ms)
    mq = MapqParams.local(max(L1, L2))
    rs = read_set(reads)
    cap = capacity(reads)
    plain = nb.seed_extend_paired(w["fmi"], w["gw"], rs, p, pair, hit_capacity=cap)
    route = last_route()                    # (no traceback, no MAPQ: the rescue DP is the call's last Gotoh call)
    print("paired %s: rescue route %s" % (name, route))
    ws = nb.seed_extend_paired(w["fmi"], w["gw"], rs, p, pair, hit_capacity=cap, mapq=mq, traceback=tb)
    torch.cuda.synchronize()
    got = {k: getattr(ws, k).cpu().numpy().copy() for k in PAIR_KEYS + MAPQ_KEYS + (TB_KEYS if tb else ())}
    for k in PAIR_KEYS:
        assert np.array_equal(getattr(plain, k).cpu().numpy(), got[k]), (name, k)
    want = paired_oracle_checks(w, reads, n_pairs, p, pair, got, mq)
    fl = want["pair_flags"]
    assert (fl == 1).sum() > 0.3 * n_pairs and ((fl == 2) | (fl == 4)).sum() >= 3, (name, fl)
    # the pairs at the exact copies: rescued onto an exact copy at least once (H = len * match, the LOCAL key rule's edge)
    top = L2 * scheme.match
    copies = range(n_pairs - len(EXACT_COPIES), n_pairs)
    assert any(fl[q] == 4 and want["mate_score"][1, q] == top for q in copies), (name, [(int(fl[q]), int(want["mate_score"][1, q])) for q in copies])
    assert route[0] == rescue_route, (name, route)            # (after the values: a rule that admits too much fails on them first)
    if not tb:
        return
    # mates keeping their single-end best: nvb_seed_extend_traceback on the 2n reads; rescued mates: the oracle's full-matrix traceback
    single = nb.seed_extend(w["fmi"], w["gw"], rs, p, hit_capacity=cap, traceback=True)
    sbest = best_of(single)
    se = seed_extend_oracle(w["O"], w["idx"], w["g"], reads, p)
    assert_best_equal(sbest, se, name)
    s_ops, s_n, s_begin, s_strand = single.best_ops.cpu().numpy(), single.best_n_ops.cpu().numpy(), host_u32(single.best_begin), \
        single.best_strand.cpu().numpy()
    check_traceback(w, reads, p, sbest, s_ops, s_n, s_begin, s_strand, se, (name, "single end"))
    flags, mops, mn, mbeg = got["pair_flags"], got["mate_ops"], got["mate_n_ops"], got["mate_begin"].view(np.uint32)
    rescued = []
    for q in range(n_pairs):
        for m in range(2):
            r = m * n_pairs + q
            if flags[q] in (2, 4) and m == (0 if flags[q] == 2 else 1):
                rescued.append((q, m))
                continue
            assert mn[m, q] == s_n[r] and tuple(mbeg[m, q]) == tuple(s_begin[r]), (name, q, m)
            assert np.array_equal(mops[m, q, :mn[m, q]], s_ops[r, :s_n[r]]), (name, q, m)
    scheme6, _ = _scheme_args(p.scheme)
    pats, t_off, t_len = [], [], []
    for q, o in rescued:
        a = 1 - o
        ra = a * n_pairs + q
        end = int(sbest["best_pos"][ra]); beg = max(end - len(reads[ra]), 0)
        to, te = (beg, min(beg + pair.max_frag, w["n"])) if s_strand[ra] == 0 else (max(end - pair.max_frag, 0), end)
        pats.append(strand_string(reads[o * n_pairs + q], np.zeros(len(reads[o * n_pairs + q]), np.uint8), 1 - int(s_strand[ra]))[0])
        t_off.append(to); t_len.append(te - to)
    lens = np.array([len(x) for x in pats], np.uint32)
    o_ = w["O"].gotoh_full_traceback(p.type, scheme6, np.concatenate(pats), np.concatenate([[0], np.cumsum(lens)[:-1]]), lens, w["g"],
                                     np.array(t_off, np.uint32), np.array(t_len, np.uint32), max_ops=ws.max_ops)
    for i, (q, o) in enumerate(rescued):
        assert int(o_["score"][i]) == got["mate_score"][o, q] and t_off[i] + int(o_["sink"][i][0]) == int(got["mate_pos"][o, q].view(np.uint32)), (name, q, o)
        assert mn[o, q] == o_["n_ops"][i] and tuple(mbeg[o, q]) == (t_off[i] + int(o_["source"][i][0]), int(o_["source"][i][1])), (name, q, o)
        assert np.array_equal(mops[o, q, :mn[o, q]], o_["ops"][i, :mn[o, q]]), (name, q, o)
    # 7. finish and BAM records of both mates, on contigs cut under some alignments
    G = w["n"]
    f = nb.finish_alignments(w["gw"], rs, ws.mate_ops, ws.mate_n_ops, ws.mate_begin, ws.mate_strand, genome_len=G)
    n = 2 * n_pairs
    st = check_device(f, reads, got["mate_strand"].reshape(n), got["mate_ops"].reshape(n, -1), got["mate_n_ops"].reshape(n),
                      got["mate_begin"].reshape(n, 2).view(np.uint32), w["g"], G)
    assert st[0] > 0.8 * n, (name, st)
    rng = np.random.default_rng(L1 + L2)
    contigs = planted_contigs(got["mate_begin"].reshape(-1, 2).view(np.uint32), got["mate_n_ops"].reshape(-1), G, rng, short=False)
    names = nb.numbered_names(n_pairs, "p%d_" % L1)
    recs = nb.bam_records(ws, f, rs, contigs, names)
    inp = host_inputs(reads, None, ws.mate_n_ops, ws.mate_begin, ws.mate_strand, f, ws.mate_score, ws.mate_mapq, ws.mate_second_score,
                      ws.pair_flags, contigs, names)
    cnt = check_records(recs, inp)
    assert cnt[2] > 0 and cnt[1] > 0.6 * cnt[0], (name, cnt)


def test_paired_513_traceback_refused(world):
    """513 bp mates: the paired traceback is refused (NVB_E_UNSUPPORTED, nvBowtie's MAXIMUM_READ_LENGTH); without it the call matches the
    oracle"""
    w = world
    reads, n_pairs = pair_reads(w, 513, 513, 24, 1500, seed=513)
    p = params(31, LO, A)
    pair = nb.PairParams(min_frag=0, max_frag=1500, min_mate_score=150)
    rs = read_set(reads)
    with pytest.raises(NvbError, match=r"\(-4\)"):
        nb.seed_extend_paired(w["fmi"], w["gw"], rs, p, pair, hit_capacity=capacity(reads), traceback=True)
    mq = MapqParams.local(513)
    ws = nb.seed_extend_paired(w["fmi"], w["gw"], rs, p, pair, hit_capacity=capacity(reads), mapq=mq)
    torch.cuda.synchronize()
    got = {k: getattr(ws, k).cpu().numpy().copy() for k in PAIR_KEYS + MAPQ_KEYS}
    paired_oracle_checks(w, reads, n_pairs, p, pair, got, mq)


# ---------------------------------------------------------------------------------------------------------------------------------------
# 7. finish and BAM, single end
# ---------------------------------------------------------------------------------------------------------------------------------------
def test_ragged_finish_and_bam(world, ragged, tmp_path):
    w = world
    reads, G = ragged["reads"], w["n"]
    rs = read_set(reads)
    q = torch.from_numpy(np.concatenate(ragged["quals"])).cuda()
    names = nb.numbered_names(len(reads), "long")
    total = np.zeros(4, np.int64)
    for typ, scheme, mq in ((LO, A, MapqParams.local(2000)), (SG, aln.SimpleGotohScheme(0, -6, -5, -3), MapqParams.end_to_end(2000))):
        p = params(31, typ, scheme)
        ws = nb.seed_extend(w["fmi"], w["gw"], rs, p, hit_capacity=capacity(reads), traceback=True, mapq=mq)
        f = nb.finish_alignments(w["gw"], rs, ws.best_ops, ws.best_n_ops, ws.best_begin, ws.best_strand, genome_len=G)
        torch.cuda.synchronize()
        assert f.cigar.shape[1] == ws.max_ops + 2 and ws.max_ops == 2 * 2000 + 31
        ops, n_ops = ws.best_ops.cpu().numpy(), ws.best_n_ops.cpu().numpy()
        begin, strand = host_u32(ws.best_begin), ws.best_strand.cpu().numpy()
        st = check_device(f, reads, strand, ops, n_ops, begin, w["g"], G)
        assert st[0] > 0.8 * len(reads) and st[1] > 3, (typ, st)
        total += st
        contigs = planted_contigs(begin, n_ops, G, np.random.default_rng(typ))
        recs = nb.bam_records(ws, f, rs, contigs, names, quals=q)
        inp = host_inputs(reads, ragged["quals"], ws.best_n_ops, ws.best_begin, ws.best_strand, f, ws.best_score, ws.mapq, ws.second_score,
                          None, contigs, names)
        cnt = check_records(recs, inp)
        assert cnt[2] > 0 and cnt[1] > 0.4 * cnt[0] and cnt[3] == 0, (typ, cnt)
        if RefBam.available():                  # htslib's own reading of the written file (where oracle/_ref is built)
            path = str(tmp_path / ("long%d.bam" % typ))
            nb.write_bam(path, nb.bam_header(contigs), [recs])
            want, _ = bo.records(inp)
            assert RefBam().format(path) == "".join(s + "\n" for _, s in want)
    assert total[3] > 0, total                  # some alignments run past the genome's end


# ---------------------------------------------------------------------------------------------------------------------------------------
# 8. streaming API at 300 bp
# ---------------------------------------------------------------------------------------------------------------------------------------
def test_streaming_300(world):
    w = world
    L, wpr = 300, 19
    reads = fixed_reads(w, L) + [kind_read(w["g"], L, "sampled", np.random.default_rng(k)) for k in range(2)]
    n = len(reads) // 2 * 2
    reads = reads[:n]
    flat = np.zeros((n, wpr * 16), np.uint8)
    for a, r in enumerate(reads):
        flat[a, :L] = r
    words = torch.from_numpy(pack_symbols(flat.reshape(-1), 2, True).view(np.int32)[:n * wpr].copy()).reshape(n, wpr)
    rs = PackedStringSet.fixed(words.reshape(-1).cuda(), n, L, stride=wpr * 16)
    p = params(31, LO, A)
    cap = capacity(reads)
    plain = nb.seed_extend(w["fmi"], w["gw"], rs, p, hit_capacity=cap)
    torch.cuda.synchronize()
    host = words.pin_memory()
    st = nb.StreamingSeedExtend(w["fmi"], w["gw"], p, n, L, wpr, hit_capacity=cap, depth=2)
    try:
        sc, ps, nh = [v.clone() for v in st.result(st.submit(host))]
    finally:
        st.close()
    assert torch.equal(sc, plain.best_score.cpu()) and torch.equal(ps, plain.best_pos.cpu()) and torch.equal(nh, plain.n_hits.cpu())
    pair = nb.PairParams(min_frag=0, max_frag=800, min_mate_score=100)
    pw = nb.seed_extend_paired(w["fmi"], w["gw"], rs, p, pair, hit_capacity=cap)
    torch.cuda.synchronize()
    st = nb.StreamingSeedExtend(w["fmi"], w["gw"], p, n, L, wpr, hit_capacity=cap, depth=2, pair=pair)
    try:
        got = {k: v.clone() for k, v in st.result(st.submit(host)).items()}
    finally:
        st.close()
    for k in PAIR_KEYS:
        assert torch.equal(got[k].reshape(getattr(pw, k).shape), getattr(pw, k).cpu()), k
