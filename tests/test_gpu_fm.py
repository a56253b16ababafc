"""-m gpu: FM-index parity through the C ABI (nvbio_b200 python mirror -> libnvbio_b200.so) against
the golden fixtures produced by the reference and against the oracle on fresh seeded inputs."""
import os
import numpy as np
import pytest
import torch
from oracle import orc
import nvbio_b200 as nb
from nvbio_b200.strings import pack_symbols, PackedStringSet
from tests.gpu_util import require_gpu, dev_u32, host_u32, mask_pad

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module")
def O():
    require_gpu()
    return orc.Oracle()


def upload(idx):
    return nb.FMIndexDevice.from_host(idx["bwt_occ"] if isinstance(idx, dict) else idx.bwt_occ,
                                      idx["ssa"] if isinstance(idx, dict) else idx.ssa,
                                      idx["L2"] if isinstance(idx, dict) else idx.L2,
                                      idx["n"] if isinstance(idx, dict) else idx.n,
                                      idx["primary"] if isinstance(idx, dict) else idx.primary)


def test_golden_fixtures(O):
    g = np.load(os.path.join(GOLD, "fmindex.npz"))
    for name in ("rand", "rep", "allA", "tiny"):
        text = g[f"{name}_text"]
        n = len(text)
        fmi = nb.FMIndexDevice.from_host(g[f"{name}_bwt_occ"], g[f"{name}_ssa"], g[f"{name}_L2"], n, int(g[f"{name}_primary"][0]))
        q = PackedStringSet.from_symbols(g[f"{name}_q"], g[f"{name}_q_off"], g[f"{name}_q_len"], bits=2)
        assert np.array_equal(host_u32(nb.match(fmi, q)), g[f"{name}_ranges"]), name
        assert np.array_equal(host_u32(nb.locate(fmi, dev_u32(g[f"{name}_rows"]))), g[f"{name}_pos"]), name
        k, c = dev_u32(g[f"{name}_rank_k"]), torch.from_numpy(g[f"{name}_rank_c"]).cuda()
        assert np.array_equal(host_u32(nb.rank(fmi, k, c)), g[f"{name}_rank_out"]), name
        # rank4 == the four single-symbol ranks (rank_test.cu:55-86 checks rank_all against running counts)
        r4 = host_u32(nb.rank4(fmi, k))
        for cc in range(4):
            want4 = host_u32(nb.rank(fmi, k, torch.full_like(c, cc)))
            assert np.array_equal(r4[:, cc], want4), (name, cc)


@pytest.mark.parametrize("n", [1, 2, 63, 64, 65, 1000, 50021, 300000])
def test_device_index_build_matches_oracle(O, n):
    rng = np.random.default_rng(n)
    text = rng.integers(0, 4, n).astype(np.uint8)
    ref = O.build_index(text)
    words = dev_u32(pack_symbols(text, 2, True))
    fmi, sa = nb.FMIndexDevice.from_text(words, n, want_sa=True)
    assert np.array_equal(host_u32(sa).astype(np.int64), ref.sa.astype(np.int64))
    assert fmi.primary == ref.primary
    assert np.array_equal(np.array(fmi.L2, np.uint32), ref.L2)
    assert np.array_equal(mask_pad(host_u32(fmi.bwt_occ), n), mask_pad(ref.bwt_occ, n))
    assert np.array_equal(host_u32(fmi.ssa), ref.ssa)


@pytest.mark.parametrize("kind", ["allA", "period2", "period7", "blocks", "long_repeat"])
def test_device_suffix_sort_repetitive(O, kind):
    """ties far beyond the 32-symbol radix key: exercises the prefix-doubling rounds"""
    rng = np.random.default_rng(5)
    if kind == "allA":
        text = np.zeros(5000, np.uint8)
    elif kind == "period2":
        text = np.tile(np.array([1, 2], np.uint8), 3000)[:5999]
    elif kind == "period7":
        text = np.tile(rng.integers(0, 4, 7).astype(np.uint8), 1200)
    elif kind == "blocks":
        blk = rng.integers(0, 4, 300).astype(np.uint8)
        text = np.concatenate([blk, blk, rng.integers(0, 4, 50).astype(np.uint8), blk, blk[:200]])
    else:
        a = rng.integers(0, 4, 20000).astype(np.uint8)
        text = np.concatenate([a, rng.integers(0, 4, 13).astype(np.uint8), a[:15000]])
    n = len(text)
    ref = O.build_index(text)
    fmi, sa = nb.FMIndexDevice.from_text(dev_u32(pack_symbols(text, 2, True)), n, want_sa=True)
    assert np.array_equal(host_u32(sa).astype(np.int64), ref.sa.astype(np.int64)), kind
    assert fmi.primary == ref.primary
    assert np.array_equal(mask_pad(host_u32(fmi.bwt_occ), n), mask_pad(ref.bwt_occ, n))


def _queries(rng, text, nq, lo=1, hi=30, n_frac=0.0):
    n = len(text)
    lens = rng.integers(lo, hi + 1, nq).astype(np.uint32)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint32)
    q = rng.integers(0, 4, int(lens.sum())).astype(np.uint8)
    for i in range(0, nq, 2):
        L = int(lens[i])
        if n > L:
            st = int(rng.integers(0, n - L + 1)); q[offs[i]:offs[i] + L] = text[st:st + L]
    if n_frac:
        for i in rng.integers(0, nq, int(nq * n_frac)):
            q[offs[i] + rng.integers(0, lens[i])] = 4
    return q, offs, lens


@pytest.mark.parametrize("bits,be,layout", [pytest.param(b, e, "concat", id="%d-%s" % (b, e)) for b, e in
                                             ((2, True), (2, False), (4, True), (4, False), (8, False))] +
                                            [pytest.param(b, e, "sparse", id="%d-%s-sparse" % (b, e)) for b, e in
                                             ((2, True), (2, False), (4, True), (4, False))])
def test_match_all_stream_formats(O, bits, be, layout):
    """every stream format, concatenated and as a sparse set (permuted storage order, gaps of random symbols, tests/read_layouts.py)"""
    from tests import read_layouts as rl
    rng = np.random.default_rng(bits * 2 + be)
    text = rng.integers(0, 4, 70001).astype(np.uint8)
    idx = O.build_index(text)
    fmi = upload(idx)
    q, offs, lens = _queries(rng, text, 20000, n_frac=0.02 if bits > 2 else 0.0)
    want, _ = O.match(idx, q, offs, lens)
    if layout == "sparse":
        reads = [q[o:o + l] for o, l in zip(offs, lens)]
        qs = rl.build(reads, None, bits, be, "sparse", seed=bits).reads
    else:
        qs = PackedStringSet.from_symbols(q, offs, lens, bits=bits, big_endian=be)
    got = host_u32(nb.match(fmi, qs))
    assert np.array_equal(got, want)
    # nvBowtie's reverse-complement seed search: forward order + complement on the forward index
    if bits == 2 and layout == "concat":
        rc = np.concatenate([(3 - q[o:o + l])[::-1] for o, l in zip(offs, lens)]).astype(np.uint8)
        want_rc, _ = O.match(idx, rc, offs, lens)
        got_rc = host_u32(nb.match(fmi, PackedStringSet.from_symbols(q, offs, lens, bits=2, big_endian=be),
                                   flags=nb.MATCH_FORWARD_ORDER | nb.MATCH_COMPLEMENT))
        assert np.array_equal(got_rc, want_rc)


def test_empty_and_degenerate(O):
    text = np.random.default_rng(2).integers(0, 4, 1000).astype(np.uint8)
    idx = O.build_index(text)
    fmi = upload(idx)
    # zero queries
    q = PackedStringSet.from_symbols(np.zeros(4, np.uint8), np.zeros(0, np.uint32), np.zeros(0, np.uint32))
    assert nb.match(fmi, q).shape[0] == 0
    # zero-length query -> the whole range (0, n) as in the reference
    q = PackedStringSet.from_symbols(np.zeros(4, np.uint8), [0, 1], [0, 1])
    r = host_u32(nb.match(fmi, q))
    assert tuple(r[0]) == (0, 1000)
    # fixed-stride set == offsets set
    sym = np.random.default_rng(3).integers(0, 4, 22 * 64).astype(np.uint8)
    a = PackedStringSet.from_symbols(sym, np.arange(64) * 22, np.full(64, 22))
    b = PackedStringSet.fixed(a.words, 64, 22)
    assert torch.equal(nb.match(fmi, a), nb.match(fmi, b))


def test_filter_rank_locate(O):
    """FMIndexFilter semantics (filter_inl.h:268-402): ranges, uint64 slots, hits = (text pos, query id)"""
    rng = np.random.default_rng(17)
    text = np.tile(rng.integers(0, 4, 4000).astype(np.uint8), 3)     # every seed occurs >= 3 times
    idx = O.build_index(text)
    fmi = upload(idx)
    q, offs, lens = _queries(rng, text, 3000, lo=6, hi=14)
    want, _ = O.match(idx, q, offs, lens)
    flt = nb.FMIndexFilterDevice()
    n_hits = flt.rank(fmi, PackedStringSet.from_symbols(q, offs, lens))
    assert np.array_equal(host_u32(flt.ranges()), want)
    sizes = np.where(want[:, 0] <= want[:, 1], want[:, 1].astype(np.int64) - want[:, 0] + 1, 0)
    slots = np.cumsum(sizes)
    assert n_hits == int(slots[-1])
    assert np.array_equal(flt.slots().cpu().numpy(), slots)
    # expected hits in slot order
    rows = np.concatenate([np.arange(x, x + s, dtype=np.uint32) for (x, _), s in zip(want, sizes)])
    qid = np.repeat(np.arange(len(sizes), dtype=np.uint32), sizes)
    pos = O.locate(idx, rows)
    for b, e in ((0, n_hits), (17, min(n_hits, 5000)), (n_hits - 1, n_hits)):
        hits = host_u32(flt.locate(b, e))
        assert np.array_equal(hits[:, 0], pos[b:e]) and np.array_equal(hits[:, 1], qid[b:e])
    # located text really carries the query (fmindex_test.cu:611-664)
    hits = host_u32(flt.locate(0, min(n_hits, 2000)))
    for p, i in hits[::97]:
        L = int(lens[i]); assert np.array_equal(text[p:p + L], q[offs[i]:offs[i] + L])


def test_large_index_properties():
    """size-independent properties on a 20 Mbp device-built index: every sampled seed hits its own
    position; ranges are stable under query permutation; forward+complement == reverse complement."""
    require_gpu()
    from nvbio_b200 import synth
    n = 20_000_000
    words = synth.random_genome_words(n)
    fmi, _ = nb.FMIndexDevice.from_text(words, n)
    assert sum(fmi.L2[i + 1] - fmi.L2[i] for i in range(4)) == n
    sw, pos = synth.sample_seeds(words, n, 200_000, 22)
    q = PackedStringSet.fixed(sw.reshape(-1), 200_000, 22, stride=32)
    r = nb.match(fmi, q)
    x = r[:, 0].to(torch.int64) & 0xFFFFFFFF
    y = r[:, 1].to(torch.int64) & 0xFFFFFFFF
    assert bool((x <= y).all())
    one = (x == y)
    assert one.float().mean() > 0.99
    located = nb.locate(fmi, r[:, 0][one].contiguous()).to(torch.int64) & 0xFFFFFFFF
    assert torch.equal(located, pos[one])
    perm = torch.randperm(200_000, device="cuda")
    q2 = PackedStringSet.fixed(sw[perm].contiguous().reshape(-1), 200_000, 22, stride=32)
    assert torch.equal(nb.match(fmi, q2), r[perm])


@pytest.mark.parametrize("k", [1, 5, 9])
def test_ktab_gives_identical_ranges(O, k):
    """the k-mer range table (an extension) only replaces the first k LF steps: ranges stay bit-identical,
    including empty ranges (the reference's early exit), N's and queries shorter than k"""
    rng = np.random.default_rng(k)
    text = rng.integers(0, 4, 90001).astype(np.uint8)
    idx = O.build_index(text)
    plain = upload(idx)
    tab = upload(idx).build_ktab(k)
    assert tab.ktab.shape[0] == 4 ** k
    # table entries themselves == match() of every k-mer
    kmers = np.array([[(u >> (2 * (k - 1 - j))) & 3 for j in range(k)] for u in range(min(4 ** k, 4096))], np.uint8)
    want_tab, _ = O.match(idx, kmers.reshape(-1), np.arange(len(kmers)) * k, np.full(len(kmers), k))
    assert np.array_equal(host_u32(tab.ktab)[:len(kmers)], want_tab)
    q, offs, lens = _queries(rng, text, 30000, lo=1, hi=28, n_frac=0.03)
    want, _ = O.match(idx, q, offs, lens)
    for bits, be in ((4, True), (8, False)):
        qs = PackedStringSet.from_symbols(q, offs, lens, bits=bits, big_endian=be)
        assert np.array_equal(host_u32(nb.match(tab, qs)), want)
    q2 = np.where(q > 3, 0, q).astype(np.uint8)
    qs = PackedStringSet.from_symbols(q2, offs, lens, bits=2)
    for flags in (0, nb.MATCH_FORWARD_ORDER | nb.MATCH_COMPLEMENT, nb.MATCH_FORWARD_ORDER, nb.MATCH_COMPLEMENT):
        assert torch.equal(nb.match(tab, qs, flags=flags), nb.match(plain, qs, flags=flags)), flags
    # 16-byte "located" entries {x, y, SA[x], SA[y]} (nvb_fm_build_ktab_located; needs the full suffix array): same ranges from every entry
    # point, and SA[x] stored for exactly the single-row k-mers
    full, _ = nb.FMIndexDevice.from_text(dev_u32(pack_symbols(text, 2, True)), len(text), sa_interval=1)
    loc = full.build_ktab(k, located=True)
    t16 = host_u32(loc.ktab)
    assert t16.shape == (4 ** k, 4) and np.array_equal(t16[:len(kmers), :2], want_tab)
    single = t16[:, 0] == t16[:, 1]
    assert np.array_equal(t16[single, 2], host_u32(full.ssa)[t16[single, 0]]) and (single.any() or k < 9)
    two = t16[:, 1] == t16[:, 0] + 1                        # two-row ranges carry both SA values
    assert np.array_equal(t16[two, 2], host_u32(full.ssa)[t16[two, 0]]) and np.array_equal(t16[two, 3], host_u32(full.ssa)[t16[two, 1]])
    for flags in (0, nb.MATCH_FORWARD_ORDER | nb.MATCH_COMPLEMENT):
        assert torch.equal(nb.match(loc, qs, flags=flags), nb.match(plain, qs, flags=flags)), flags
    # ... + text context (nvb_fm_build_ktab_context): the last word of a one-row entry = the up to 16 symbols before SA[x]
    tw = dev_u32(np.concatenate([pack_symbols(text, 2, True), np.zeros(2, np.uint32)]))
    ctx = full.build_ktab(k, located=True, text=tw)
    assert ctx.ktab_located == 2
    c16 = host_u32(ctx.ktab)
    assert np.array_equal(c16[:, 0], t16[:, 0]) and np.array_equal(c16[:, 2], t16[:, 2]) and np.array_equal(c16[~single, 3], t16[~single, 3])
    # two-row entries: y = x + 1 is implied by a marker; the freed bits hold the 7 symbols before SA[x] and before SA[x + 1]
    assert np.array_equal(c16[~two, 1], t16[~two, 1]) and (c16[two, 1] >> 30 == 3).all()
    def before(pos, want):
        cnt = 0 if pos == 0xFFFFFFFF else min(pos, want)
        v = 0
        for sym in text[pos - cnt:pos] if cnt else []:
            v = (v << 2) | int(sym)
        return v
    for v in np.flatnonzero(two)[:: max(1, int(two.sum()) // 300)]:
        assert int(c16[v, 1]) == (0xC0000000 | before(int(c16[v, 2]), 7) | (before(int(c16[v, 3]), 7) << 14)), v
    for v in np.flatnonzero(single)[:: max(1, int(single.sum()) // 500)]:
        pos = int(c16[v, 2])
        cnt = 0 if pos == 0xFFFFFFFF else min(pos, 16)
        want_ctx = 0
        for sym in text[pos - cnt:pos] if cnt else []:
            want_ctx = (want_ctx << 2) | int(sym)
        assert int(c16[v, 3]) == want_ctx, (v, pos)
    for flags in (0, nb.MATCH_FORWARD_ORDER | nb.MATCH_COMPLEMENT):
        assert torch.equal(nb.match(ctx, qs, flags=flags), nb.match(plain, qs, flags=flags)), flags
    with pytest.raises(nb.NvbError):
        upload(idx).build_ktab(k, located=True)                 # sampled SA: unsupported


@pytest.mark.parametrize("interval", [1, 2, 4, 16, 32])
def test_sampled_sa_interval(O, interval):
    """denser (or sparser) SA sampling than the reference's SA_INT=16 locates the same positions"""
    rng = np.random.default_rng(interval)
    n = 40007
    text = rng.integers(0, 4, n).astype(np.uint8)
    ref = O.build_index(text)
    fmi, _ = nb.FMIndexDevice.from_text(dev_u32(pack_symbols(text, 2, True)), n, sa_interval=interval)
    assert fmi.ssa.numel() == (n + interval) // interval
    want_ssa = ref.sa[::interval].astype(np.uint32).copy(); want_ssa[0] = 0xFFFFFFFF
    assert np.array_equal(host_u32(fmi.ssa), want_ssa)
    rows = rng.integers(0, n + 1, 5000).astype(np.uint32); rows[:3] = (0, ref.primary, n)
    assert np.array_equal(host_u32(nb.locate(fmi, dev_u32(rows))), O.locate(ref, rows))


def test_match_approx_one_mismatch(O):
    """nvBowtie's map<find_exact> core (rank4-based one-substitution search) against its characterisation through the pinned
    exact match(): every single-substitution variant in push order, then the exact match"""
    from tests.test_host_core import approx_expected
    rng = np.random.default_rng(31)
    n = 60000
    text = rng.integers(0, 4, n).astype(np.uint8)
    idx = O.build_index(text)
    fmi = upload(idx)
    nq = 1500
    lens = rng.integers(10, 23, nq).astype(np.uint32)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint32)
    q = rng.integers(0, 4, int(lens.sum())).astype(np.uint8)
    for i in range(nq):
        L = int(lens[i]); st = int(rng.integers(0, n - L))
        cons = text[st:st + L][::-1].copy()             # consumed order = reversed text order
        if i % 3:
            cons[int(rng.integers(L // 2, L))] ^= 2
        if i % 23 == 0:
            cons[int(rng.integers(0, L))] = 4
        q[offs[i]:offs[i] + L] = cons
    qs = PackedStringSet.from_symbols(q, offs, lens, bits=4, big_endian=True)
    for exact_len, find_exact in ((10, True), (0, False)):
        want = approx_expected(O, idx, q, offs, lens, exact_len, find_exact, True, False)
        ranges, counts, sums = nb.match_approx(fmi, qs, exact_len, find_exact, max_out=80, flags=nb.MATCH_FORWARD_ORDER)
        r, c, s = host_u32(ranges), host_u32(counts), host_u32(sums)
        for i in range(nq):
            got = [tuple(x) for x in r[i, :c[i]]]
            assert got == want[i], (i, exact_len)
            assert s[i] == sum(y - x + 1 for x, y in want[i])


@pytest.mark.parametrize("interval", [16, 4, 1])
def test_two_phase_and_sorted_locate(O, interval):
    """nvBowtie's two-pass locate (locate_init -> locate_lookup, locate_inl.h:122-210) through a sorting permutation, and the
    radix-sorted one-pass variant (aligner_best_approx.h:737-756): positions == nvbio::locate for every row, in input order"""
    require_gpu()
    rng = np.random.default_rng(interval)
    n = 50_000
    text = np.concatenate([rng.integers(0, 4, n // 2), np.tile(rng.integers(0, 4, 97), n)[: n - n // 2]]).astype(np.uint8)
    idx = O.build_index(text)
    ssa = idx.sa[::interval].astype(np.uint32).copy(); ssa[0] = 0xFFFFFFFF
    fmi = nb.FMIndexDevice.from_host(idx.bwt_occ, ssa, idx.L2, idx.n, idx.primary, sa_interval=interval)
    rows = rng.integers(0, n + 1, 20000).astype(np.uint32); rows[:3] = (0, idx.primary, n)
    want = O.locate(idx, rows)
    d_rows = dev_u32(rows)
    perm = dev_u32(rng.permutation(len(rows)).astype(np.uint32))
    for p in (None, perm):
        r, t = nb.locate_init(fmi, d_rows, p)
        assert (host_u32(r) % interval == 0).all()             # a sampled row; the number of LF steps is geometric, not bounded by the interval
        assert np.array_equal(host_u32(nb.locate_lookup(fmi, r, t, p)), want)
    assert np.array_equal(host_u32(nb.locate_sorted(fmi, d_rows)), want)
    assert np.array_equal(host_u32(nb.locate(fmi, d_rows)), want)


def test_generic_rank_dictionary_gpu():
    """nvb_dict_rank / nvb_dict_rank4 / nvb_dict_build_occ (SURVEY 8a row a6) == the reference's rank_dictionary over plain 32- / 64-bit
    word streams and build_occurrence_table<2,K> (committed fixture generated by running the reference)"""
    require_gpu()
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "generic_rank.npz"))
    for i, (wb, K, n) in enumerate(g["cfgs"]):
        wb, K, n = int(wb), int(K), int(n)
        sdt, tdt = (np.int32, torch.int32) if wb == 32 else (np.int64, torch.int64)
        words = torch.from_numpy(np.concatenate([g[f"words{i}"], np.zeros(4, g[f"words{i}"].dtype)]).view(sdt)).cuda()
        occ = torch.from_numpy(g[f"occ{i}"].view(sdt).copy()).cuda()
        qi = g[f"qi{i}"]
        qi_dev = torch.from_numpy((qi & (0xFFFFFFFF if wb == 32 else 0xFFFFFFFFFFFFFFFF)).astype(np.uint32 if wb == 32 else np.uint64).view(sdt)).cuda()
        qc = torch.from_numpy(g[f"qc{i}"].copy()).cuda()
        mask = np.uint64(0xFFFFFFFF if wb == 32 else 0xFFFFFFFFFFFFFFFF)
        got = nb.dict_rank(words, occ, K, qi_dev, qc).cpu().numpy().view(np.uint32 if wb == 32 else np.uint64).astype(np.uint64)
        assert np.array_equal(got, g[f"ranks{i}"]), (wb, K, n)
        all4 = nb.dict_rank(words, occ, K, qi_dev).cpu().numpy().view(np.uint32 if wb == 32 else np.uint64).astype(np.uint64)
        assert np.array_equal(all4[np.arange(len(qi)), g[f"qc{i}"]], g[f"ranks{i}"])
        built, counts = nb.dict_build_occ(words, n, K, index_bits=wb)
        assert np.array_equal(built.cpu().numpy().view(np.uint32 if wb == 32 else np.uint64), g[f"occ{i}"]), (wb, K, n)
        assert counts == [int((g[f"text{i}"] == c).sum()) for c in range(4)]
