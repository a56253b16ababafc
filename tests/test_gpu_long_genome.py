"""The FM-index, seed + extend and the occ build on genomes longer than 2^31 bases: rows, SA values, text positions and k-mer table
entries above 2^31, SA ranges above 2^31 and FMIndexFilter slot totals above 2^32.

The genomes are T = A^F . R (tests/long_genome.py), whose suffix array is known in closed form, so the device makes their index without a
suffix sort.  Two configurations, built one at a time:
    A: F = 2^31 - 2^21, R straddles 2^31; n ~ 2.15e9 < 0xC0000000, so two-row context table entries carry the marker
    B: F = 0xC0000000 - 2^21, R straddles 0xC0000000; n ~ 3.22e9, so they do not, and real range ends at or above 0xC0000000 exist
Each is checked in three index forms: SA every 16 rows without a table, a 16-byte context table (k = 8) with the per-row array, and a
wide table (k = 12, larger than L2) with the per-row array.  Everything that involves R is compared with the few-Mbp partner
T' = A^F' . R, which the device suffix-sorts itself: rows >= 1 and positions move by F - F'.  Queries of A's alone are compared with
their closed-form range sizes, and the seed range sums of reads that hold them -- which wrap a uint32 on T -- with nvBowtie's reseed
rule evaluated on those sizes.  The output chain (finish, BAM, SAM, sort and BAI) runs with contigs that begin past 2^31.  Last, a
synthetic BWT of n = 2^32 - 2 and 2^32 - 64 symbols pins the occ build at the top of the range."""
import numpy as np
import pytest
import torch

import nvbio_b200 as nb
from nvbio_b200.fmindex import FMIndexDevice, FMIndexFilterDevice, MATCH_COMPLEMENT, MATCH_FORWARD_ORDER
from nvbio_b200.strings import PackedStringSet, pack_symbols
from nvbio_b200.synth import gather_symbols
from tests import bai_oracle
from tests.gpu_util import require_gpu
from tests.long_genome import LongGenome, a_runs, device_bwt, device_genome, device_index, device_sa

pytestmark = pytest.mark.gpu

R_LEN = 1 << 22
F_PARTNER = 1 << 20
CONFIGS = {"A": (1 << 31) - (1 << 21), "B": 0xC0000000 - (1 << 21)}
FORMS = ("plain", "ctx8", "wide12")
FLAGS = (0, MATCH_COMPLEMENT, MATCH_FORWARD_ORDER, MATCH_FORWARD_ORDER | MATCH_COMPLEMENT)


def _u32(t: torch.Tensor) -> np.ndarray:
    return t.detach().cpu().numpy().view(np.uint32).astype(np.int64)


def _i32(a) -> torch.Tensor:
    return torch.from_numpy(np.asarray(a, np.int64).astype(np.uint32).view(np.int32)).cuda()


def _make_R():
    rng = np.random.default_rng(2024)
    R = rng.integers(0, 4, R_LEN).astype(np.uint8)
    R[1000:1020] = 0                          # a 20-long A-run (the longest), so that A^s queries up to 20 also hit R
    R[1020] = 2
    R[0], R[-1] = 1, 3
    return R


def _form(base: FMIndexDevice, sa: torch.Tensor, gw: torch.Tensor, form: str) -> FMIndexDevice:
    """one index form over base's occ table and the full suffix array sa"""
    if form == "plain":
        return FMIndexDevice(base.bwt_occ, sa[::16].clone(), base.L2, base.length, base.primary, sa_interval=16)
    idx = FMIndexDevice(base.bwt_occ, sa, base.L2, base.length, base.primary, sa_interval=1)
    idx.build_ktab(8 if form == "ctx8" else 12, located=True, text=gw)
    assert idx.struct().ktab_located == (3 if form == "ctx8" else 5), form
    return idx


class Genome:
    def __init__(self, lg: LongGenome, sa: torch.Tensor):
        self.lg, self.sa = lg, sa
        self.gw = device_genome(lg)
        self.idx = device_index(lg, sa, 1)
        self.n = lg.n

    def form(self, name):
        torch.cuda.empty_cache()                           # build_ktab sizes its arrays by the device's free memory
        return _form(self.idx, self.sa, self.gw, name)


@pytest.fixture(scope="module")
def partner():
    require_gpu()
    R = _make_R()
    rw = torch.from_numpy(pack_symbols(R).view(np.int32)).cuda()
    _, sa_R = FMIndexDevice.from_text(rw, R_LEN, want_sa=True, sa_interval=1)
    sa_R = _u32(sa_R)
    lg = LongGenome(R, F_PARTNER, sa_R)
    gw = device_genome(lg)
    # the partner is suffix-sorted by the device; the closed form must give the same suffix array
    fmi, sa = FMIndexDevice.from_text(gw, lg.n, want_sa=True, sa_interval=1)
    assert fmi.primary == lg.primary
    assert np.array_equal(_u32(sa)[1:], np.concatenate([np.arange(lg.h), lg.tail]))
    sa[0] = -1                                             # the `$` row as the index keeps it
    g = Genome(lg, sa)
    assert np.array_equal(_u32(g.idx.bwt_occ), _u32(fmi.bwt_occ)) and g.idx.L2 == fmi.L2
    return g, sa_R


@pytest.fixture(scope="module", params=sorted(CONFIGS))
def cfg(request, partner):
    p, sa_R = partner
    torch.cuda.reset_peak_memory_stats()
    lg = LongGenome(p.lg.R, CONFIGS[request.param], sa_R)
    g = Genome(lg, device_sa(lg))
    g.name, g.p, g.d = request.param, p, lg.shift(p.lg)
    g.mark = CONFIGS[request.param] + (1 << 21)            # 2^31 or 0xC0000000: the R offset 2^21 sits there
    yield g
    print("\nlong genome %s: n = %d, peak device memory %.1f GB" % (g.name, g.n, torch.cuda.max_memory_allocated() / 1e9))
    del g
    torch.cuda.empty_cache()


# -- occ table and rank --------------------------------------------------------------------------------------------------
_LUT = None


def _byte_counts():
    """[4, 256]: occurrences of each symbol among the 4 symbols of a byte"""
    global _LUT
    if _LUT is None:
        b = torch.arange(256)
        _LUT = torch.stack([sum((((b >> (2 * i)) & 3) == c).to(torch.int64) for i in range(4)) for c in range(4)]).cuda()
    return _LUT


def _block_counts(words: torch.Tensor) -> torch.Tensor:
    """int64 [n_blocks, 4]: symbols of each 64-symbol block of 2-bit words (4 words per block), in chunks"""
    out = []
    lut = _byte_counts()
    for lo in range(0, words.numel(), 1 << 26):
        by = words[lo:lo + (1 << 26)].view(torch.uint8).to(torch.int64).view(-1, 16)
        out.append(torch.stack([lut[c][by].sum(1) for c in range(4)], 1))
    return torch.cat(out)


def test_occ_table_and_rank(cfg):
    """from_bwt's interleaved BWT words and counters and its L2 against popcounts of the BWT words on the device; rank and rank4 at
    2^31 +- 1, the primary row, 0xC0000000 +- 1, n - 1 and n against the same counts"""
    lg, idx, n = cfg.lg, cfg.idx, cfg.n
    blocks = idx.bwt_occ.view(-1, 8)
    bwt = blocks[:, :4].reshape(-1).contiguous()
    assert torch.equal(bwt, device_bwt(lg))              # (the builder's padding symbols are zero)
    cnt = _block_counts(bwt)
    excl = torch.cumsum(cnt, 0) - cnt
    assert torch.equal(blocks[:, 4:].to(torch.int64) & 0xFFFFFFFF, excl)
    tot = cnt.sum(0).cpu().numpy()
    tot[0] -= len(cnt) * 64 - n                          # padding symbols are A's
    assert idx.L2 == [0] + np.cumsum(tot).tolist()

    def rank_ref(k):
        if k == n:
            return tot
        s = k - 1 if k >= lg.primary else k              # stored-BWT symbol of row k; rows [0, k] = stored [0, s]
        b = s // 64
        base = excl[b].cpu().numpy()
        w = bwt[4 * b:4 * b + 4].cpu().numpy().view(np.uint32)
        sym = np.array([(int(w[i // 16]) >> (30 - 2 * (i % 16))) & 3 for i in range(s % 64 + 1)])
        return base + np.bincount(sym, minlength=4)

    ks = sorted({(1 << 31) - 1, 1 << 31, (1 << 31) + 1, lg.primary, 0xC0000000 - 1, 0xC0000000, 0xC0000000 + 1, n - 1, n})
    ks = [k for k in ks if k <= n]
    want = np.stack([rank_ref(k) for k in ks])
    got4 = _u32(nb.rank4(idx, _i32(ks)))
    assert np.array_equal(got4, want)
    for c in range(4):
        got = _u32(nb.rank(idx, _i32(ks), torch.full((len(ks),), c, dtype=torch.uint8, device="cuda")))
        assert np.array_equal(got, want[:, c])


# -- match -----------------------------------------------------------------------------------------------------------------
def _seeds(R, count, ln, seed):
    rng = np.random.default_rng(seed)
    pos = rng.integers(0, len(R) - ln, count)
    pos[:64] = (1 << 21) - np.arange(64) * 7          # across the configuration's mark
    pos[64:72] = len(R) - ln                          # ending at n
    sym = R[pos[:, None] + np.arange(ln)]
    return PackedStringSet.fixed(torch.from_numpy(pack_symbols(sym.reshape(-1)).view(np.int32)).cuda(), count, ln)


def _same_ranges(got: np.ndarray, want: np.ndarray, d: int):
    """T's ranges = T''s moved by d (non-empty ones); empty on both or on neither"""
    ne = want[:, 0] <= want[:, 1]
    assert np.array_equal(ne, got[:, 0] <= got[:, 1])
    assert np.array_equal(got[ne], want[ne] + d)
    return int(ne.sum())


def test_match_seeds(cfg):
    """100K 22-mers of R, both orientations and strands, in every index form: the partner's ranges through the row map"""
    q = _seeds(cfg.lg.R, 100_000, 22, 1)
    for form in FORMS:
        idx, pidx = cfg.form(form), cfg.p.form(form)
        for fl in FLAGS:
            hits = _same_ranges(_u32(nb.match(idx, q, fl)), _u32(nb.match(pidx, q, fl)), cfg.d)
            assert fl or hits == 100_000, (form, fl)
        del idx, pidx


def _query_set(qs):
    lens = np.array([len(x) for x in qs])
    return PackedStringSet.from_symbols(np.concatenate(qs), np.concatenate([[0], np.cumsum(lens)[:-1]]), lens)


def _a_queries(R):
    """A^s, and A^s . R[:q] across the run's end"""
    a = [np.zeros(s, np.uint8) for s in (1, 12, 20, 21, 32)]
    b = [np.concatenate([np.zeros(s, np.uint8), R[:q]]) for s in (1, 12, 20, 21, 32) for q in (1, 3, 8, 30)]
    return a, b


def test_a_run_ranges(cfg):
    """ranges of A^s are rows 1 .. a_run_range_size(s) (above 2^31 rows here), those of A^s . R[:q] the partner's moved by d with
    boundary_range_size(s, q) rows -- in every form"""
    lg = cfg.lg
    a, b = _a_queries(lg.R)
    qa, qb = _query_set(a), _query_set(b)
    for form in FORMS:
        idx, pidx = cfg.form(form), cfg.p.form(form)
        got = _u32(nb.match(idx, qa))
        want = np.array([[1, lg.a_run_range_size(len(x))] for x in a])
        assert np.array_equal(got, want), form
        if cfg.n > 0xC0000000:
            assert (want[:, 1] > 1 << 31).all()
        got, pw = _u32(nb.match(idx, qb)), _u32(nb.match(pidx, qb))
        _same_ranges(got, pw, cfg.d)
        sizes = np.maximum(got[:, 1] - got[:, 0] + 1, 0)
        s_q = [(s, q) for s in (1, 12, 20, 21, 32) for q in (1, 3, 8, 30)]
        assert sizes.tolist() == [lg.boundary_range_size(s, q) for s, q in s_q], form
        del idx, pidx


# -- locate --------------------------------------------------------------------------------------------------------------
def test_locate(cfg):
    """locate, locate_init + locate_lookup and locate_sorted over the sampled SA (and locate over the full one) at rows 0, the primary,
    2^31 +- 1, 0xC0000000 +- 1, n and random rows, against the suffix array; locate also on the full SA with each table and per-row array"""
    n, lg = cfg.n, cfg.lg
    rng = np.random.default_rng(3)
    rows = [0, lg.primary, (1 << 31) - 1, 1 << 31, (1 << 31) + 1, 0xC0000000 - 1, 0xC0000000, 0xC0000000 + 1, n - 1, n]
    rows = [r for r in rows if r <= n] + rng.integers(0, n + 1, 20_000).tolist() + (n - rng.integers(0, lg.r + lg.m, 20_000)).tolist()
    r = _i32(rows)
    want_pos = _u32(cfg.sa[r.long() & 0xFFFFFFFF])         # row 0: 0xFFFFFFFF
    plain = cfg.form("plain")
    assert np.array_equal(_u32(nb.locate(plain, r)), want_pos)
    assert np.array_equal(_u32(nb.locate(cfg.idx, r)), want_pos)
    for form in ("ctx8", "wide12"):
        idx = cfg.form(form)
        assert np.array_equal(_u32(nb.locate(idx, r)), want_pos), form
        del idx
    sr, st = nb.locate_init(plain, r)
    assert np.array_equal(_u32(nb.locate_lookup(plain, sr, st)), want_pos)
    assert np.array_equal(_u32(nb.locate_sorted(plain, r)), want_pos)


# -- FMIndexFilter -------------------------------------------------------------------------------------------------------
def test_filter_slots_above_2_32(cfg):
    """a batch of A-rich queries whose hits exceed 2^32: slots = the closed-form cumulative range sizes; locate(b, e) on windows at 0,
    around 2^32 and at the end = (SA of the slot's row, query id)"""
    lg = cfg.lg
    qs = [np.zeros(s, np.uint8) for s in (1, 2, 3, 12)] + [R_q for R_q in (lg.R[:22], lg.R[5000:5022])]
    want_sizes = [lg.a_run_range_size(s) for s in (1, 2, 3, 12)] + [1, 1]
    f = FMIndexFilterDevice()
    plain = cfg.form("plain")
    total = f.rank(plain, _query_set(qs))
    slots = np.cumsum(want_sizes)
    assert total == slots[-1] > 1 << 32
    assert np.array_equal(f.slots().cpu().numpy(), slots)
    ranges = _u32(f.ranges())
    for b in (0, (1 << 32) - 3000, total - 3000):
        h = _u32(f.locate(b, b + 3000))
        hit = np.arange(b, b + 3000)
        qid = np.searchsorted(slots, hit, side="right")
        row = ranges[qid, 0] + hit - np.concatenate([[0], slots])[qid]
        assert np.array_equal(h[:, 1], qid)
        assert np.array_equal(h[:, 0], _u32(cfg.sa[torch.from_numpy(row).cuda()]))


# -- context tables ------------------------------------------------------------------------------------------------------
def _text_before(gw: torch.Tensor, pos: torch.Tensor, want: int) -> torch.Tensor:
    """the (up to) `want` symbols before each text position, symbol pos - 1 lowest (none for 0xFFFFFFFF)"""
    out = torch.zeros_like(pos)
    for t in range(1, want + 1):
        ok = (pos >= t) & (pos != 0xFFFFFFFF)
        out |= torch.where(ok, gather_symbols(gw, torch.where(ok, pos - t, 0)), 0) << (2 * (t - 1))
    return out


def test_context_table_entries(cfg):
    """two-row entries of the 16-byte context table: marked (n < 0xC0000000) or plain {x, x + 1, SA[x], SA[x + 1]} (n above it), as
    their builder intends; and match() with each table = match() without"""
    q = _seeds(cfg.lg.R, 100_000, 22, 2)
    a, b = _a_queries(cfg.lg.R)
    qa = _query_set(a + b)
    base = {fl: _u32(nb.match(cfg.idx, q, fl)) for fl in FLAGS}
    base_a = _u32(nb.match(cfg.idx, qa))
    for form in ("ctx8", "wide12"):
        idx = cfg.form(form)
        t = idx.ktab.view(-1, 8 if form == "wide12" else 4)[:, :4].to(torch.int64) & 0xFFFFFFFF
        x, y = t[:, 0], t[:, 1]
        if cfg.n < 0xC0000000:
            two = y >= 0xC0000000                          # every range end is a row below 0xC0000000: these are markers
            assert int((y == x + 1).sum()) == 0
        else:
            two = y == x + 1
            assert int(((x <= y) & (y >= 0xC0000000)).sum()) > 0     # real ranges ending at rows the marker would claim
        if form == "wide12":
            assert int(two.sum()) > 1000
        xs = x[two]
        sa0, sa1 = cfg.sa[xs].to(torch.int64) & 0xFFFFFFFF, cfg.sa[xs + 1].to(torch.int64) & 0xFFFFFFFF
        assert torch.equal(t[two, 2], sa0) and torch.equal(t[two, 3], sa1)
        if cfg.n < 0xC0000000:
            # the marker's 7 + 7 context symbols: the text before SA[x] and SA[x + 1], read at positions above 2^31
            yv = y[two]
            assert torch.equal(yv & 0x3FFF, _text_before(cfg.gw, sa0, 7)) and torch.equal((yv >> 14) & 0x3FFF, _text_before(cfg.gw, sa1, 7))
            if form == "wide12":
                assert int((sa0 > 1 << 31).sum()) > 1000
        del t, x, y, two, xs, sa0, sa1
        for fl in FLAGS:
            assert np.array_equal(_u32(nb.match(idx, q, fl)), base[fl]), (form, fl)
        assert np.array_equal(_u32(nb.match(idx, qa)), base_a), form
        del idx


# -- map_seeds and seed + extend -----------------------------------------------------------------------------------------
def _reads(R, count, ln, seed, mark_off, boundary=(1, 5, 12, 20, 40, 75, 149)):
    """reads of R (T coordinates = F + offset) with 1 % substitutions, half reverse-complemented; some end exactly at R's end, some
    cover the configuration's mark, and the last ones are A^s . R[:ln - s] boundary reads for s in `boundary`"""
    rng = np.random.default_rng(seed)
    off = rng.integers(0, len(R) - ln + 1, count)
    off[:200] = mark_off - rng.integers(0, ln, 200)
    off[200:220] = len(R) - ln
    sym = R[off[:, None] + np.arange(ln)].copy()
    sub = rng.random(sym.shape) < 0.01
    sym[sub] = (sym[sub] + rng.integers(1, 4, int(sub.sum()))) % 4
    for i, s in enumerate(boundary):
        sym[-1 - i] = np.concatenate([np.zeros(s, np.uint8), R[:ln - s]])
    rc = np.arange(count) % 2 == 1
    sym[rc] = (3 - sym[rc])[:, ::-1]
    return sym


def _read_set(sym, bits):
    c, ln = sym.shape
    return PackedStringSet.from_symbols(sym.reshape(-1), np.arange(c) * ln, np.full(c, ln), bits=bits)


def _moved(a: np.ndarray, d: int) -> np.ndarray:
    """the partner's text positions on T: moved by d, but for none (0xFFFFFFFF) and those deep in the A-run, which A^s seeds reach
    through their first rows (SA = 0, 1, 2, ... on both)"""
    return np.where((a == 0xFFFFFFFF) | (a < F_PARTNER // 2), a, a + d)


def test_map_seeds(cfg):
    """nvBowtie's seed mapping (EXACT and APPROX) of reads from R: the partner's hits through the row map, counts, reseed flags
    and range statistics equal (boundary reads whose A's hold a whole seed have other range sizes on T and are left out)"""
    sym = _reads(cfg.lg.R, 20_000, 100, 4, 1 << 21, boundary=(1, 5, 12, 20))
    rs = _read_set(sym, 2)
    for form in FORMS:
        idx, pidx = cfg.form(form), cfg.p.form(form)
        for alg in (nb.MAP_EXACT, nb.MAP_APPROX):
            h, c, rsd, st = nb.map_seeds(idx, rs, algorithm=alg)
            ph, pc, prsd, pst = nb.map_seeds(pidx, rs, algorithm=alg)
            assert torch.equal(c, pc) and torch.equal(rsd, prsd) and torch.equal(st, pst), (form, alg)
            k = torch.arange(h.shape[1], device="cuda")[None, :] < c[:, None]
            assert torch.equal(h[..., 1][k], ph[..., 1][k])
            assert np.array_equal(_u32(h[..., 0][k]), _u32(ph[..., 0][k]) + cfg.d), (form, alg)
        del idx, pidx


def test_seed_extend(cfg):
    """seed + extend of 20K reads from R (2- and 4-bit) and of boundary reads: best score, position, second best and MAPQ, and the
    traced alignment equal the partner's after the position rule"""
    sym = _reads(cfg.lg.R, 20_000, 150, 5, 1 << 21)
    mq = nb.MapqParams.local(150)
    params = nb.SeedExtendParams()
    for form in ("plain", "wide12"):
        idx, pidx = cfg.form(form), cfg.p.form(form)
        for bits in (2, 4):
            rs = _read_set(sym, bits)
            w = nb.seed_extend(idx, cfg.gw, rs, params, mapq=mq)
            pw = nb.seed_extend(pidx, cfg.p.gw, rs, params, mapq=mq)
            assert torch.equal(w.best_score, pw.best_score) and torch.equal(w.mapq, pw.mapq), (form, bits)
            assert torch.equal(w.second_score, pw.second_score) and torch.equal(w.second_strand, pw.second_strand)
            assert np.array_equal(_u32(w.best_pos), _moved(_u32(pw.best_pos), cfg.d))
            assert np.array_equal(_u32(w.second_pos), _moved(_u32(pw.second_pos), cfg.d))
            assert float((w.best_score > 150).float().mean()) > 0.95
            pos = _u32(w.best_pos)
            assert ((pos >= cfg.mark - 150) & (pos < cfg.mark + 150)).sum() > 50 and (pos >= cfg.n - 2).any()
        rs = _read_set(sym, 2)
        w = nb.seed_extend(idx, cfg.gw, rs, params, traceback=True)
        pw = nb.seed_extend(pidx, cfg.p.gw, rs, params, traceback=True)
        assert torch.equal(w.best_n_ops, pw.best_n_ops) and torch.equal(w.best_ops, pw.best_ops) and torch.equal(w.best_strand, pw.best_strand)
        b, pb = _u32(w.best_begin), _u32(pw.best_begin)
        assert np.array_equal(b[:, 1], pb[:, 1]) and np.array_equal(b[:, 0], _moved(pb[:, 0], cfg.d))
        del idx, pidx


def _same(ws, pws, keys, pos_keys, d, what):
    """outputs equal, positions (pos_keys; the genome column of (n, 2) begins) through the position rule"""
    for k in keys:
        assert torch.equal(getattr(ws, k), getattr(pws, k)), (what, k)
    for k in pos_keys:
        a, b = _u32(getattr(ws, k)), _u32(getattr(pws, k))
        if k.endswith("begin"):
            assert np.array_equal(a[..., 1], b[..., 1]), (what, k)
            a, b = a[..., 0], b[..., 0]
        assert np.array_equal(a, _moved(b, d)), (what, k)


def test_seed_extend_reseed_all_and_streaming(cfg):
    """seed_extend_reseed (max_reseed 2, MAPQ, traceback), seed_extend_all (k = 3) and one StreamingSeedExtend batch on reads from R:
    the partner's outputs after the position rule, rounds and per-round read counts equal (100 random reads, whose seeds find nothing,
    go on to the later rounds)"""
    sym = _reads(cfg.lg.R, 20_000, 150, 6, 1 << 21)
    sym[300:400] = np.random.default_rng(9).integers(0, 4, (100, 150))
    rs = _read_set(sym, 2)
    params = nb.SeedExtendParams()
    mq = nb.MapqParams.local(150)
    rp = nb.ReseedParams.local(150, max_reseed=2)
    for form in ("plain", "wide12"):
        idx, pidx = cfg.form(form), cfg.p.form(form)
        w = nb.seed_extend_reseed(idx, cfg.gw, rs, params, rp, traceback=True, mapq=mq)
        pw = nb.seed_extend_reseed(pidx, cfg.p.gw, rs, params, rp, traceback=True, mapq=mq)
        _same(w, pw, ("best_score", "second_score", "second_strand", "mapq", "rounds", "active", "best_n_ops", "best_ops", "best_strand"),
              ("best_pos", "second_pos", "best_begin"), cfg.d, (form, "reseed"))
        assert int(w.active[1]) >= 100
        del w, pw
        a = nb.seed_extend_all(idx, cfg.gw, rs, params, mq, 3)
        pa = nb.seed_extend_all(pidx, cfg.p.gw, rs, params, mq, 3)
        assert torch.equal(a.count, pa.count) and int(a.count[0]) == int(a.count[1]) > rs.count // 2
        c = int(a.count[0])
        for k in ("first", "best_score", "second_score", "mapq"):
            assert torch.equal(getattr(a, k), getattr(pa, k)), (form, "all", k)
        for k in ("read", "score", "n_ops", "ops", "strand"):
            assert torch.equal(getattr(a, k)[:c], getattr(pa, k)[:c]), (form, "all", k)
        assert np.array_equal(_u32(a.pos[:c]), _moved(_u32(pa.pos[:c]), cfg.d))
        b, pb = _u32(a.begin[:c]), _u32(pa.begin[:c])
        assert np.array_equal(b[:, 1], pb[:, 1]) and np.array_equal(b[:, 0], _moved(pb[:, 0], cfg.d))
        del a, pa, idx, pidx
    # the streaming entry point on T: the direct call's results
    pad = np.zeros((len(sym), 160), np.uint8)
    pad[:, :150] = sym
    host = torch.from_numpy(pack_symbols(pad.reshape(-1), pad_words=0).view(np.int32).reshape(len(sym), 10).copy()).pin_memory()
    w = nb.seed_extend(cfg.idx, cfg.gw, rs, params)
    st = nb.StreamingSeedExtend(cfg.idx, cfg.gw, params, len(sym), 150, 10, depth=2)
    try:
        sc, ps, _ = st.result(st.submit(host))
        assert torch.equal(sc, w.best_score.cpu()) and torch.equal(ps, w.best_pos.cpu())
    finally:
        st.close()


def _pairs(R, count, ln, seed, mark_off):
    """pairs inside R (FR, fragments of 200-400 bases), some across the configuration's mark and some ending at R's end: mate 1 of every
    pair, then mate 2"""
    rng = np.random.default_rng(seed)
    frag = rng.integers(200, 401, count)
    off = rng.integers(0, len(R) - 400, count)
    off[:100] = mark_off - rng.integers(0, 400, 100)
    off[100:110] = len(R) - frag[100:110]
    m1 = R[off[:, None] + np.arange(ln)]
    m2 = R[(off + frag - ln)[:, None] + np.arange(ln)]
    m2 = (3 - m2)[:, ::-1]
    sym = np.concatenate([m1, m2])
    sub = rng.random(sym.shape) < 0.01
    sym[sub] = (sym[sub] + rng.integers(1, 4, int(sub.sum()))) % 4
    return sym


def test_seed_extend_paired(cfg):
    """paired-end seed + extend with MAPQ and traceback on 5K pairs inside R: pair scores and flags, mates' scores, strands, MAPQ,
    traces and rescue counts equal the partner's, mate positions and begins through the position rule"""
    rs = _read_set(_pairs(cfg.lg.R, 5000, 150, 7, 1 << 21), 2)
    params = nb.SeedExtendParams()
    mq = nb.MapqParams.local(150)
    pair = nb.PairParams(min_frag=0, max_frag=500, min_mate_score=80)
    for form in ("plain", "wide12"):
        idx, pidx = cfg.form(form), cfg.p.form(form)
        w = nb.seed_extend_paired(idx, cfg.gw, rs, params, pair, mapq=mq, traceback=True)
        pw = nb.seed_extend_paired(pidx, cfg.p.gw, rs, params, pair, mapq=mq, traceback=True)
        _same(w, pw, ("pair_score", "pair_flags", "mate_score", "mate_strand", "n_rescue", "second_pair_score", "second_mate_strand",
                      "mate_second_score", "mate_mapq", "mate_ops", "mate_n_ops"), ("mate_pos", "second_mate_pos", "mate_begin"), cfg.d,
              (form, "paired"))
        pos = _u32(w.mate_pos)
        assert (pos != 0xFFFFFFFF).mean() > 0.95 and ((pos >= cfg.mark - 400) & (pos < cfg.mark + 400)).sum() > 50
        del w, pw, idx, pidx


def test_all_a_reads_reseed_rule(cfg):
    """reads of A's alone: their seeds' ranges are rows 1 .. a_run_range_size(L), which the seed range sums add in wrapping uint32
    arithmetic (nvBowtie's rule, pipeline_core.cuh reseed_read).  On T these sums wrap.  map_seeds' range statistics and reseed flags,
    and seed_extend_reseed's rounds of boundary reads A^s . R[:150 - s] (whose A's hold whole seeds), equal that rule on the closed-form
    sizes; rep_seeds 2^28 makes the wrap decide some flags"""
    lg = cfg.lg
    assert a_runs(3 - lg.R).max() < 20                      # no T-run of a seed's length: the reverse-complement seeds find nothing
    lens = np.arange(22, 151, 2)
    rs = PackedStringSet.from_symbols(np.zeros(int(lens.sum()), np.uint8), np.concatenate([[0], np.cumsum(lens)[:-1]]), lens)
    REP, M32 = 1 << 28, 1 << 32

    def flagged(cnt, size):
        return (cnt == 0) | ((cnt * size) % M32 >= (REP * cnt) % M32)

    cnt = (lens - 22) // 10 + 1
    _, _, rsd, st = nb.map_seeds(cfg.idx, rs, rep_seeds=REP)
    st = _u32(st)
    assert np.array_equal(st[:, 1], cnt) and np.array_equal(st[:, 0], (cnt * lg.a_run_range_size(22)) % M32)
    want = flagged(cnt, lg.a_run_range_size(22))
    assert np.array_equal(rsd.cpu().numpy().astype(bool), want) and (~want).any()

    # seed_extend_reseed: a read of A's alone finds no alignment on either genome (its seeds' ranges are far wider than max_seed_hits),
    # which flags it whatever its sums; boundary reads A^s . R[:150 - s] align at F - s, so their flags are the sums' alone
    params = nb.SeedExtendParams()
    rp = nb.ReseedParams.local(150, max_reseed=2, rep_seeds=REP)
    w = nb.seed_extend_reseed(cfg.idx, cfg.gw, rs, params, rp)
    pw = nb.seed_extend_reseed(cfg.p.idx, cfg.p.gw, rs, params, rp)
    assert torch.equal(w.best_score, pw.best_score) and torch.equal(w.best_pos, pw.best_pos) and (w.rounds == 3).all()
    ss = np.arange(20, 131, 2)
    sym = np.stack([np.concatenate([np.zeros(k, np.uint8), lg.R[:150 - k]]) for k in ss])
    size = _seed_sizes(lg, params.seed_len)
    rounds = np.ones(len(ss), np.int64)
    for r in range(rp.max_reseed):
        o = r * (params.seed_interval // (rp.max_reseed + 1))
        for i, row in enumerate(sym):
            sz = [size(st[p:p + params.seed_len]) for st in (row, (3 - row)[::-1]) for p in range(o, 150 - params.seed_len + 1, params.seed_interval)]
            c = sum(1 for z in sz if z)
            rounds[i] += int(rounds[i] == r + 1 and (c == 0 or sum(sz) % M32 >= (REP * c) % M32))
    rs = _read_set(sym, 2)
    w = nb.seed_extend_reseed(cfg.idx, cfg.gw, rs, params, rp)
    got, pos, score = w.rounds.cpu().numpy().astype(np.int64), _u32(w.best_pos), w.best_score.cpu().numpy()
    true = (pos == lg.F - ss + 150) & (score == 300)        # aligned at F - s (best_pos = the end, exclusive): flags are the sums' alone
    assert true[ss <= 44].all()
    assert np.array_equal(got[true], rounds[true]) and (rounds[true] == 1).any()
    # longer A-prefixes: the run's hits fill the read's max_seed_hits and it finds no alignment (as on the partner): flagged every round
    none = score == np.iinfo(np.int32).min
    assert none[ss >= 48].all() and (got[none] == rp.max_reseed + 1).all()

def _seed_sizes(lg, ln):
    """the range size on T of any ln-symbol seed: A's alone from the closed form; otherwise its occurrences inside R plus the one
    at the run's end when it is A^j . R[:ln - j]"""
    key = np.zeros(lg.r - ln + 1, np.int64)
    for i in range(ln):
        key = key * 4 + lg.R[i:lg.r - ln + 1 + i]
    uniq, cnt = np.unique(key, return_counts=True)

    def size(seed):
        if not seed.any():
            return lg.a_run_range_size(ln)
        k = 0
        for v in seed:
            k = k * 4 + int(v)
        j = np.searchsorted(uniq, k)
        inside = int(cnt[j]) if j < len(uniq) and uniq[j] == k else 0
        lead = int(np.argmax(seed != 0))
        return inside + int(lead >= 1 and np.array_equal(seed[lead:], lg.R[:ln - lead]))
    return size


def _contigs(F, r, pieces, piece):
    """the run tiled into `pieces` contigs (the last of them 2^18 long, right before R) plus one contig for R"""
    head = F - (1 << 18)
    lens = [piece] * (pieces - 1) + [head - piece * (pieces - 1)] if piece else [head // pieces] * (pieces - 1) + [head - head // pieces * (pieces - 1)]
    return nb.ContigTable(["run%d" % i for i in range(pieces)] + ["runZ", "R"], lens + [1 << 18, r])


def test_output_chain(cfg):
    """finish_alignments -> bam_records -> sam_text on T, with the run tiled into 500 Mbp contigs (so that contigs begin past 2^31) and
    one contig for R: byte-identical to the partner's SAM text under contigs of the same names; sort_bam_records + bam_index on T's
    records equal tests/bai_oracle.py"""
    sym = _reads(cfg.lg.R, 20_000, 150, 8, 1 << 21)
    rs = _read_set(sym, 2)
    params = nb.SeedExtendParams()
    mq = nb.MapqParams.local(150)
    pieces = -(-(cfg.lg.F - (1 << 18)) // 500_000_000)
    sams = []
    for g, contigs in ((cfg, _contigs(cfg.lg.F, cfg.lg.r, pieces, 500_000_000)), (cfg.p, _contigs(cfg.p.lg.F, cfg.p.lg.r, pieces, 0))):
        assert contigs.genome_len == g.n and contigs.begin[-2] == g.lg.F
        w = nb.seed_extend(g.idx, g.gw, rs, params, traceback=True, mapq=mq)
        f = nb.finish_alignments(g.gw, rs, w.best_ops, w.best_n_ops, w.best_begin, w.best_strand, genome_len=g.n)
        recs = nb.bam_records(w, f, rs, contigs, nb.numbered_names(rs.count, "r"))
        sams.append(nb.sam_text(recs, contigs).to_bytes())
        if g is cfg:
            t_recs, t_contigs = recs, contigs
    assert sams[0] == sams[1] and sams[0].count(b"\tR\t") > 19_000
    off = t_recs.offsets.cpu().numpy()
    s = nb.sort_bam_records(t_recs)
    srt = s.to_bytes()
    soff = s.offsets.cpu().numpy()
    blocks = nb.bgzf_compress(s.data[:int(soff[-1])])
    boff = blocks.offsets.cpu().numpy()
    bai = nb.bam_index(s, blocks, 1000, t_contigs)
    assert bai == bai_oracle.bai_bytes([srt[soff[i]:soff[i + 1]] for i in range(len(off) - 1)], boff, 1000, len(t_contigs.names))


# -- the top of the range --------------------------------------------------------------------------------------------------
WORD = 0x1B1B1B1B                                   # A C G T A C G T ...: four of each symbol


@pytest.mark.parametrize("n", [(1 << 32) - 2, (1 << 32) - 64])
def test_occ_build_at_the_top_of_the_range(n):
    """from_bwt on a synthetic BWT of n symbols (one repeated word, a few hundred random words at the start, around 2^31 and at the end):
    L2, the block counters around the planted words and the last block's, and rank / rank4 at n - 1 and n against the closed form.
    (n + 63) / 64 in uint32 arithmetic gives 0 blocks at n = 2^32 - 2."""
    require_gpu()
    n_words = ((n + 63) // 64) * 4
    rng = np.random.default_rng(n & 0xFFFF)
    planted = np.concatenate([np.arange(0, 256), np.arange((1 << 27) - 128, (1 << 27) + 128), np.arange(n_words - 256, n_words)])
    vals = rng.integers(0, 1 << 32, len(planted), dtype=np.uint64).astype(np.uint32)
    words = torch.full((n_words,), WORD - (1 << 32) if WORD >= 1 << 31 else WORD, dtype=torch.int32, device="cuda")
    words[torch.from_numpy(planted).cuda()] = torch.from_numpy(vals.view(np.int32)).cuda()
    idx = FMIndexDevice.from_bwt(words, n, 1, None)

    def sym_counts(w, keep=16):
        return np.array([sum(((int(w) >> (30 - 2 * i)) & 3) == c for i in range(keep)) for c in range(4)], np.int64)

    pc = np.stack([sym_counts(v) for v in vals]) - 4        # planted words' excess over the repeated word
    padding = n_words * 16 - n                              # the last word's unused symbols

    def prefix(s):
        """counts of stored symbols [0, s) (s a multiple of 16)"""
        wcount = s // 16
        return 4 * wcount + pc[planted < wcount].sum(0)

    last = vals[-1]
    tot = prefix(n_words * 16) - sym_counts(last) + sym_counts(last, 16 - padding)
    assert idx.L2 == [0] + np.cumsum(tot).tolist()
    blocks = idx.bwt_occ.view(-1, 8)
    assert blocks.shape[0] == n_words // 4
    check = np.unique(np.concatenate([planted // 4, planted // 4 + 1, rng.integers(0, n_words // 4, 1000)]))
    check = check[check < n_words // 4]
    got = _u32(blocks[torch.from_numpy(check).cuda(), 4:])
    want = np.stack([prefix(64 * k) for k in check])
    assert np.array_equal(got, want)
    # rank at n - 1 (stored symbol n - 2 with the primary at 1) and n
    ks = [n - 1, n]
    at = 16 - padding - 1                                   # stored symbol n - 1 in the last word
    want = np.stack([tot - np.eye(4, dtype=np.int64)[(int(last) >> (30 - 2 * at)) & 3], tot])
    got4 = _u32(nb.rank4(idx, _i32(ks)))
    assert np.array_equal(got4, want)
    for c in range(4):
        assert np.array_equal(_u32(nb.rank(idx, _i32(ks), torch.full((2,), c, dtype=torch.uint8, device="cuda"))), want[:, c])

