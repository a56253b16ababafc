"""-m gpu: every entry point that reads caller strings gives bit-identical outputs on every read layout the C ABI accepts
(tests/read_layouts.py: concatenated, odd-stride, fixed, offsets-only, sparse, aliased, interleaved mates, offsets at and above 2^31 up to
the last uint32 symbol, and a slack `length`), 2- and 4-bit, big- and little-endian, with every symbol and quality byte outside the reads
poisoned.  The reference is the concat big-endian run of the same reads, anchored once against tests/pipeline_oracle.py.  Reads without N
give the same outputs at both widths, and reads that share an offset get the same per-read outputs."""
import ctypes as C
import numpy as np
import pytest
import torch
from oracle import orc
import nvbio_b200 as nb
from nvbio_b200 import aln
from nvbio_b200.bam import ContigTable, numbered_names
from nvbio_b200.pipeline import MapqParams, ReseedParams
from nvbio_b200.strings import pack_symbols
from tests import read_layouts as rl
from tests.gpu_util import require_gpu
from tests.pipeline_oracle import seed_extend_oracle
from tests.test_gpu_all import repeat_genome, make_reads
from tests.test_gpu_finish import se_world  # noqa: F401  (the single-end world fixture)
from tests.test_gpu_paired_traceback import world, PAIR_KEYS, MAPQ_KEYS  # noqa: F401  (the paired world fixture)

pytestmark = pytest.mark.gpu
WIDTHS = ((2, True), (2, False), (4, True), (4, False))
LOCAL = dict(seed_len=20, seed_interval=10, band_len=31, type=aln.LOCAL, both_strands=True, max_seed_hits=50)


def se_params(sname, lay):
    """LOCAL seed + extend under the constant scheme ("const") or the quality-table one with the layout's qualities ("qual")"""
    if sname == "qual":
        return nb.SeedExtendParams(**LOCAL, scheme=aln.QualityGotohScheme(2, 2, 6, 5, 3, 5, 3), read_quals=lay.quals)
    return nb.SeedExtendParams(**LOCAL, scheme=aln.SimpleGotohScheme(2, -2, -5, -3))


N_EVERY = 5


def with_n(reads, seed):
    """the 4-bit batch: the same reads with two N's in every N_EVERY-th one (reads 0, N_EVERY, ...)"""
    rng = np.random.default_rng(seed)
    out = [r.copy() for r in reads]
    for r in out[::N_EVERY]:
        r[rng.integers(0, len(r), 2)] = 4
    return out


def u(t):
    torch.cuda.synchronize()
    t = t.detach().cpu()
    return t.numpy().view(np.uint32) if t.dtype == torch.int32 else t.numpy()


def masked(rows, n):
    """rows[i, :n[i]] with the rest zeroed (capacity-bound outputs hold nothing past their count)"""
    rows, n = u(rows).copy(), u(n).astype(np.int64)
    keep = np.arange(rows.shape[-1]) < np.minimum(n, rows.shape[-1]).reshape(n.shape + (1,))
    rows[~keep] = 0
    return rows


def diff(want, got, what):
    """None, or the first field (in order) where got differs from want, and the first row there.  Fields whose last axis is sized from
    the set's `length` (ops, CIGAR, MD) are compared over the narrower width, the rest of the wider one being zero"""
    for k, a in want.items():
        b = got[k]
        if isinstance(a, bytes):
            if a != b:
                i = next((j for j in range(min(len(a), len(b))) if a[j] != b[j]), min(len(a), len(b)))
                return "%s: %s differs (%d vs %d bytes), first at byte %d" % (what, k, len(a), len(b), i)
            continue
        if a.ndim >= 2 and a.shape[:-1] == b.shape[:-1] and a.shape[-1] != b.shape[-1]:
            w = min(a.shape[-1], b.shape[-1])
            if a[..., w:].any() or b[..., w:].any():
                return "%s: %s has entries past width %d" % (what, k, w)
            a, b = a[..., :w], b[..., :w]
        if a.shape != b.shape:
            return "%s: %s has shape %s, not %s" % (what, k, b.shape, a.shape)
        if not np.array_equal(a, b):
            at = tuple(int(v) for v in np.argwhere(a != b)[0])
            return "%s: %s differs, first at read / row %s: %s vs %s" % (what, k, at, a[at[:1]].reshape(-1)[:12].tolist(),
                                                                           b[at[:1]].reshape(-1)[:12].tolist())
    return None


def check_same(want, got, what):
    msg = diff(want, got, what)
    assert msg is None, msg


def for_each_layout(reads, quals, run, entry, paired=False, widths=WIDTHS, layouts=None, alias_keys=()):
    """run(layout) -> outputs for the reads in every layout x width, against the concat big-endian run of the same reads at that width;
    the 2-bit and 4-bit concat runs of the N-free reads against each other; per-read alias_keys equal for reads sharing a string.
    Equal-length layouts get the reads cut to the shortest one."""
    lmin = min(len(r) for r in reads)
    groups = (("ragged", reads, quals), ("fixed", [r[:lmin] for r in reads], [q[:lmin] for q in quals]))
    ran = set()
    for group, rr, qq in groups:
        names = [l for l in rl.layouts_for(paired, group == "fixed") if (l in rl.FIXED_ONLY) == (group == "fixed") or l == "concat"]
        if layouts is not None:
            names = [l for l in names if l in layouts or l == "concat"]
        if names == ["concat"]:
            continue
        sym = {2: rr, 4: with_n(rr, 11)}
        ref = {b: run(rl.build(sym[b], qq, b, True, "concat")) for b in (2, 4)}
        check_same(ref[2], run(rl.build(rr, qq, 4, True, "concat")), "%s, cross-width (%s reads)" % (entry, group))
        for name in names:
            for bits, be in widths:
                if name == "concat" and be:
                    continue
                lay = rl.build(sym[bits], qq, bits, be, name, seed=bits + 2 * be)
                got = run(lay)
                what = "%s, layout %s, %d-bit %s" % (entry, name, bits, "big-endian" if be else "little-endian")
                check_same(ref[bits], got, what)
                if name == "aliased" and alias_keys:
                    check_aliases(lay, sym[bits], got, alias_keys, what)
                ran.add(name)
                del lay, got
        torch.cuda.empty_cache()
    return ran


def check_aliases(lay, reads, got, keys, what):
    spans = {}
    for i, (o, r) in enumerate(zip(lay.off.tolist(), reads)):
        spans.setdefault((o, len(r)), []).append(i)
    groups = [g for g in spans.values() if len(g) > 1]
    assert groups, what
    for k in keys:
        for g in groups:
            assert all(np.array_equal(got[k][g[0]], got[k][i]) for i in g[1:]), "%s: %s differs between reads %s sharing a string" % (what, k, g)


# ---- single end ---------------------------------------------------------------------------------------------------------------------

def se_reads(w):
    return rl.with_aliases(w["reads"][:240], w["quals"][:240], np.random.default_rng(21))


def set_path(p):
    nb.lib().nvb_debug_pipeline_path(C.c_int(p))


SE_KEYS = ("best_score", "best_pos", "n_hits")
HIT_KEYS = ("hit_read", "hit_window", "hit_score", "hit_sink")
SE_TB_KEYS = ("best_ops", "best_n_ops", "best_begin", "best_strand")
SE_MAPQ_KEYS = ("second_score", "second_pos", "second_strand", "mapq")


def se_outputs(ws, tag, out, hits=False):
    for k in SE_KEYS:
        out[tag + k] = u(getattr(ws, k))
    kept = int(ws.n_hits[0])
    if hits:
        for k in HIT_KEYS:
            out[tag + k] = u(getattr(ws, k))[:kept]
    if ws.best_ops is not None:
        out[tag + "best_ops"] = masked(ws.best_ops, ws.best_n_ops)
        for k in SE_TB_KEYS[1:]:
            out[tag + k] = u(getattr(ws, k))
    if ws.mapq is not None:
        for k in SE_MAPQ_KEYS:
            out[tag + k] = u(getattr(ws, k))
    return out


def finish_outputs(f, tag, out):
    out[tag + "cigar"] = masked(f.cigar, f.n_cigar)
    out[tag + "md"] = masked(f.md, f.md_len)
    for k in ("n_cigar", "md_len", "edits"):
        out[tag + k] = u(getattr(f, k))
    return out


@pytest.mark.parametrize("path", [0, 1])
def test_seed_extend_every_layout(se_world, path):
    """seed_extend plain, keep_hits, traceback and mapq (constant and quality schemes), then finish and BAM records with layout-indexed
    qualities; path 1 = the per-hit extension path"""
    w = se_world
    reads, quals = se_reads(w)
    n, lmax = len(reads), max(len(r) for r in reads)
    mq = MapqParams.local(lmax + 16)
    contigs = ContigTable(["c0", "c1"], [w["G"] // 2, w["G"] - w["G"] // 2])
    names = numbered_names(n)

    def run(lay):
        out = {}
        set_path(path)
        try:
            for sname in ("const", "qual"):
                params = se_params(sname, lay)
                hc = 64 * n
                se_outputs(nb.seed_extend(w["fmi"], w["gw"], lay.reads, params, hit_capacity=hc), sname + "/plain:", out)
                se_outputs(nb.seed_extend(w["fmi"], w["gw"], lay.reads, params, hit_capacity=hc, keep_hits=True), sname + "/hits:", out, True)
                se_outputs(nb.seed_extend(w["fmi"], w["gw"], lay.reads, params, hit_capacity=hc, traceback=True), sname + "/tb:", out)
                ws = nb.seed_extend(w["fmi"], w["gw"], lay.reads, params, hit_capacity=hc, traceback=True, mapq=mq, keep_hits=True)
                se_outputs(ws, sname + "/mapq:", out, True)
                f = nb.finish_alignments(w["gw"], lay.reads, ws.best_ops, ws.best_n_ops, ws.best_begin, ws.best_strand, genome_len=w["G"])
                finish_outputs(f, sname + "/finish:", out)
                out[sname + "/bam"] = nb.bam_records(ws, f, lay.reads, contigs, names, quals=lay.quals).to_bytes()
        finally:
            set_path(0)
        return out

    ran = for_each_layout(reads, quals, run, "seed_extend (path %d)" % path,
                          alias_keys=["%s/mapq:%s" % (s, k) for s in ("const", "qual") for k in SE_KEYS[:2] + SE_TB_KEYS + SE_MAPQ_KEYS])
    assert ran == set(rl.layouts_for(False, True))


def test_concat_anchor_against_oracle(se_world):
    """the reference of every layout comparison: the concat big-endian run against the oracle composition, per hit and per read"""
    w = se_world
    reads, quals = se_reads(w)
    O = orc.Oracle()
    idx = O.build_index(w["g"])
    for sname in ("const", "qual"):
        lay = rl.build(reads, quals, 2, True, "concat")
        params = se_params(sname, lay)
        ws = nb.seed_extend(w["fmi"], w["gw"], lay.reads, params, hit_capacity=64 * len(reads), keep_hits=True)
        want = seed_extend_oracle(O, idx, w["g"], reads, params, quals=quals if sname == "qual" else None)
        kept, total, _ = [int(v) for v in ws.n_hits.cpu()]
        assert kept == total == want["n_hits"], sname
        assert np.array_equal(u(ws.hit_read)[:kept].astype(np.int64), want["hit_string"]), sname
        assert np.array_equal(u(ws.hit_window)[:kept].astype(np.int64), want["hit_window"]), sname
        assert np.array_equal(ws.hit_score.cpu().numpy()[:kept].astype(np.int64), want["hit_score"]), sname
        assert np.array_equal(u(ws.hit_sink)[:kept].astype(np.int64), want["hit_sink"]), sname
        assert np.array_equal(ws.best_score.cpu().numpy().astype(np.int64), want["best_score"]), sname
        assert np.array_equal(u(ws.best_pos).astype(np.int64), want["best_pos"]), sname


def test_seed_extend_reseed_every_layout(se_world):
    w = se_world
    reads, quals = se_reads(w)
    n, lmax = len(reads), max(len(r) for r in reads)
    mq, rp = MapqParams.local(lmax + 16), ReseedParams.local(lmax + 16, max_reseed=2)

    def run(lay):
        out = {}
        for sname in ("const", "qual"):
            params = se_params(sname, lay)
            ws = nb.seed_extend_reseed(w["fmi"], w["gw"], lay.reads, params, rp, traceback=True, mapq=mq, keep_hits=True, hit_capacity=64 * n)
            se_outputs(ws, sname + ":", out, True)
            out[sname + ":rounds"], out[sname + ":active"] = u(ws.rounds), u(ws.active)
        return out

    for_each_layout(reads, quals, run, "seed_extend_reseed", alias_keys=["const:best_score", "const:mapq", "qual:rounds"])


def test_map_seeds_big_endian_layouts(se_world):
    """map_seeds reads big-endian sets only (little-endian ones are refused, tests/test_read_layouts.py).  nvBowtie seeds against the
    index of the reversed genome.  The reads are exact copies of either genome strand, so that every exact seed search finds ranges: each
    read without an N must find some, the one stored last (ending on symbol 2^32 - 1 under high) included"""
    w = se_world
    rng = np.random.default_rng(23)
    reads = []
    for _ in range(240):
        L = int(rng.integers(60, 151)); x = int(rng.integers(0, w["G"] - L))
        r = w["g"][x:x + L].copy()
        reads.append(np.where(r < 4, 3 - r, r)[::-1].copy() if rng.random() < 0.5 else r)
    quals = [rng.integers(2, 41, len(r)).astype(np.uint8) for r in reads]
    reads, quals = rl.with_aliases(reads, quals, rng)
    ridx = orc.Oracle().build_index(np.ascontiguousarray(w["g"][::-1]))
    fmi_rev = nb.FMIndexDevice.from_host(ridx.bwt_occ, ridx.ssa, ridx.L2, ridx.n, ridx.primary)

    def run(lay):
        out = {}
        rs = lay.reads
        ln = u(rs.lengths).astype(np.int64) if rs.lengths is not None else np.full(rs.count, rs.length, np.int64)
        top = int(np.argmax(lay.off + ln))
        for alg in (nb.MAP_EXACT, nb.MAP_APPROX):
            hits, counts, reseed, stats = nb.map_seeds(fmi_rev, lay.reads, algorithm=alg, seed_len=20 if alg == nb.MAP_EXACT else 16,
                                                      seed_freq=10, max_hits=40, subseed_len=8)
            for k, v in (("hits", hits), ("counts", counts), ("reseed", reseed), ("stats", stats)):
                out["%d:%s" % (alg, k)] = u(v)
        c = out["%d:counts" % nb.MAP_EXACT]
        has_n = (np.arange(rs.count) % N_EVERY == 0) if rs.bits == 4 else np.zeros(rs.count, bool)
        assert (c[~has_n] > 0).all(), (lay.name, rs.bits, np.nonzero((c == 0) & ~has_n)[0][:8])
        assert has_n[top] or c[top] > 0, (lay.name, rs.bits, top)
        return out

    for_each_layout(reads, quals, run, "map_seeds", widths=((2, True), (4, True)), alias_keys=["0:counts", "1:stats"])


def test_fm_queries_every_layout(se_world):
    """match, match_approx and FMIndexFilterDevice.rank / locate on poisoned query sets: seeds of the genome (every other one mutated),
    10-22 symbols"""
    w = se_world
    rng = np.random.default_rng(8)
    q = []
    for i in range(600):
        L = int(rng.integers(10, 23)); st = int(rng.integers(0, w["G"] - L))
        s = w["g"][st:st + L].copy()
        if i % 2:
            s[int(rng.integers(L // 2, L))] ^= 1
        q.append(s)
    qq = [np.zeros(len(s), np.uint8) for s in q]

    def run(lay):
        out = {"match": u(nb.match(w["fmi"], lay.reads)),
               "match_fc": u(nb.match(w["fmi"], lay.reads, flags=nb.MATCH_FORWARD_ORDER | nb.MATCH_COMPLEMENT))}
        # the queries are forward genome text: the default (reversed) consumption order finds them; FORWARD_ORDER reads them the other way
        for exact_len, fe, flags in ((10, True, 0), (0, False, nb.MATCH_FORWARD_ORDER)):
            r, c, s = nb.match_approx(w["fmi"], lay.reads, exact_len, fe, max_out=80, flags=flags)
            out["approx%d:ranges" % exact_len], out["approx%d:counts" % exact_len], out["approx%d:sums" % exact_len] = u(r), u(c), u(s)
        flt = nb.FMIndexFilterDevice()
        h = flt.rank(w["fmi"], lay.reads)
        out["filter:n_hits"] = np.array([h])
        out["filter:ranges"], out["filter:slots"] = u(flt.ranges()), u(flt.slots())
        out["filter:hits"] = u(flt.locate(0, min(h, 20000)))
        m = out["match"]
        assert (m[:, 0] <= m[:, 1]).mean() > 0.3 and h > 0 and (out["approx10:counts"] > 0).mean() > 0.3, lay.name
        return out

    for_each_layout(q, qq, run, "FM-index queries", layouts=("concat", "sparse", "aliased", "stride_odd", "high", "slack"))


# ---- seed_extend_all on the repeat genome -------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def repeat_world():
    require_gpu()
    O = orc.Oracle()
    g = repeat_genome()
    gw = torch.from_numpy(pack_symbols(g, 2, True).view(np.int32)).cuda()
    idx = O.build_index(g)
    fmi = nb.FMIndexDevice.from_host(idx.bwt_occ, idx.ssa, idx.L2, idx.n, idx.primary)
    rng = np.random.default_rng(31)
    reads = make_reads(g, n_reads=200, L=100, ragged=True, seed=29)
    quals = [rng.integers(2, 41, len(r)).astype(np.uint8) for r in reads]
    reads, quals = rl.with_aliases(reads, quals, rng)
    return dict(g=g, gw=gw, fmi=fmi, G=len(g), reads=reads, quals=quals)


@pytest.mark.parametrize("k", [0, 3])
def test_seed_extend_all_every_layout(repeat_world, k):
    w = repeat_world
    reads, quals, n = w["reads"], w["quals"], len(w["reads"])
    mq = MapqParams.local(max(len(r) for r in reads) + 16)
    contigs = ContigTable(["r0", "r1"], [w["G"] // 3, w["G"] - w["G"] // 3])
    names = numbered_names(n)

    def run(lay):
        out = {}
        for sname in ("const", "qual"):
            params = se_params(sname, lay)
            al = nb.seed_extend_all(w["fmi"], w["gw"], lay.reads, params, mq, k, capacity=16 * n + 1024, hit_capacity=1000 * n)
            t = sname + ":"
            for f in ("best_score", "best_pos", "second_score", "second_pos", "second_strand", "mapq", "n_hits", "first", "count"):
                out[t + f] = u(getattr(al, f))
            c = int(al.count[0])
            for f in ("read", "score", "pos", "n_ops", "begin", "strand"):
                out[t + f] = u(getattr(al, f))[:c]
            out[t + "ops"] = masked(al.ops, al.n_ops)[:c]
            f = nb.finish_alignments(w["gw"], al.strings(lay.reads), al.ops, al.n_ops, al.begin, al.strand, genome_len=w["G"])
            fo = finish_outputs(f, "", {})
            for key, v in fo.items():
                out[t + "finish:" + key] = v[:c]
            out[t + "bam"] = nb.bam_records_all(al, f, lay.reads, contigs, names, quals=lay.quals).to_bytes()
        return out

    for_each_layout(reads, quals, run, "seed_extend_all (k = %d)" % k, alias_keys=["const:best_score", "qual:mapq", "qual:second_score"])


# ---- paired end ---------------------------------------------------------------------------------------------------------------------

def paired_reads(w):
    """the paired world's mates (mate 1 of every pair, then mate 2), with some mate 2s replaced by copies or infixes of earlier reads"""
    n = w["n_pairs"]
    r, q = rl.with_aliases(w["reads"], w["quals"], np.random.default_rng(41), every=23)
    return r, q, n


@pytest.mark.parametrize("reseed", [False, True])
def test_seed_extend_paired_every_layout(world, reseed):
    """seed_extend_paired with MAPQ and traceback (constant and quality schemes), then finish and paired BAM records; with reseed,
    seed_extend_paired_reseed at max_reseed 2"""
    w = world
    reads, quals, n_pairs = paired_reads(w)
    lmax = max(len(r) for r in reads)
    mq = MapqParams.local(lmax + 16)
    pair = nb.PairParams(min_frag=0, max_frag=420, min_mate_score=50)
    G = int(w["idx"].n)
    contigs = ContigTable(["p0"], [G])
    names = numbered_names(n_pairs)

    def run(lay):
        out = {}
        for sname in ("const", "qual"):
            params = se_params(sname, lay)
            if reseed:
                ws = nb.seed_extend_paired_reseed(w["fmi"], w["gw"], lay.reads, params, pair, ReseedParams.local(lmax + 16, max_reseed=2),
                                                  mapq=mq, traceback=True, hit_capacity=128 * n_pairs)
            else:
                ws = nb.seed_extend_paired(w["fmi"], w["gw"], lay.reads, params, pair, hit_capacity=128 * n_pairs, mapq=mq, traceback=True)
            t = sname + ":"
            for k in PAIR_KEYS + MAPQ_KEYS + ("mate_n_ops", "mate_begin", "n_hits"):
                out[t + k] = u(getattr(ws, k))
            out[t + "mate_ops"] = masked(ws.mate_ops, ws.mate_n_ops)
            if reseed:
                out[t + "rounds"], out[t + "active"] = u(ws.rounds), u(ws.active)
            f = nb.finish_alignments(w["gw"], lay.reads, ws.mate_ops, ws.mate_n_ops, ws.mate_begin, ws.mate_strand, genome_len=G)
            finish_outputs(f, t + "finish:", out)
            out[t + "bam"] = nb.bam_records(ws, f, lay.reads, contigs, names, quals=lay.quals).to_bytes()
        return out

    ran = for_each_layout(reads, quals, run, "seed_extend_paired%s" % ("_reseed" if reseed else ""), paired=True)
    assert "mates_interleaved" in ran and "high" in ran
