"""-m gpu: up to k distinct alignments per read (nvb_seed_extend_all) against the oracle composition (tests/pipeline_oracle.py's per-hit
outputs + the selection rule, tests/all_oracle.py) on a genome with planted repeat families; rank 0 / rank 1 against the best-alignment
and MAPQ calls, every alignment's trace against the banded traceback of its job alone, capacity cuts, paths and read lengths."""
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
from tests.all_oracle import all_oracle, all_records
from tests.mapq_oracle import INT_MIN

pytestmark = pytest.mark.gpu

N_GENOME = 200_000


def rc(s):
    return np.where(s < 4, 3 - s, s)[::-1].astype(np.uint8)


def repeat_genome(seed=5):
    """repeat families for reads up to 512 bp: a 12-copy family (exact copies, copies with 1-3 substitutions per 100 bp, a copy with a 1 bp
    deletion and one with a 1 bp insertion, two reverse-complemented copies, two copies 40 bp apart) and a copy running into the genome's end"""
    rng = np.random.default_rng(seed)
    g = rng.integers(0, 4, N_GENOME).astype(np.uint8)
    a = g[10_000:10_600].copy()
    for st in (20_000, 30_000, 40_000):
        g[st:st + 600] = a
    for st, step in ((50_000, 100), (60_000, 50), (70_000, 33)):
        c = a.copy(); c[step // 2::step] = (c[step // 2::step] + 1) % 4
        g[st:st + 600] = c
    g[80_000:80_599] = np.delete(a, 300)                                           # 1 bp deletion
    g[90_000:90_601] = np.insert(a, 300, (a[300] + 1) % 4)                          # 1 bp insertion
    g[100_000:100_600] = rc(a); g[110_000:110_600] = rc(a)                         # reverse complement
    g[120_000:120_600] = a; g[120_040:120_640] = a                                 # two copies 40 bp apart (closer than len/2)
    g[N_GENOME - 300:] = a[:300]                                                   # a copy at the genome's end
    return g


def make_reads(g, n_reads=500, L=100, ragged=False, seed=7):
    rng = np.random.default_rng(seed)
    reads = []
    for i in range(n_reads):
        ln = int(rng.integers(L - 40, L + 1)) if ragged else L
        kind = i % 8
        if kind < 5:                                                               # from the repeat family
            p = 10_000 + int(rng.integers(0, 600 - ln + 1))
        elif kind == 5:                                                            # the genome's end
            p = N_GENOME - ln - int(rng.integers(0, 60))
        else:
            p = int(rng.integers(0, N_GENOME - ln))
        r = g[p:p + ln].copy()
        if kind == 6:
            m = rng.random(ln) < 0.1
            r[m] = (r[m] + 1) % 4
        if rng.random() < 0.5:
            r = rc(r)
        reads.append(r)
    return reads


def packed(reads, bits=2, L=None):
    lens = np.array([len(r) for r in reads], np.uint32)
    offs = (np.cumsum(lens) - lens).astype(np.uint32)
    rs = PackedStringSet.from_symbols(np.concatenate(reads), offs, lens, bits=bits, big_endian=True)
    if L is not None:
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


def lists(al):
    """per read: [(score, pos, strand)] of its stored alignments in rank order"""
    torch.cuda.synchronize()
    first = host_u32(al.first).astype(np.int64)
    stored = int(al.count[0])
    sc, pos, st = al.score.cpu().numpy()[:stored], host_u32(al.pos)[:stored], al.strand.cpu().numpy()[:stored]
    out = []
    for r in range(al.n_reads):
        b, e = first[r], first[r + 1]
        out.append([(int(sc[i]), int(pos[i]), int(st[i])) for i in range(b, e)] if e <= stored else None)
    return out


def run(fmi, gw, rs, params, mq, k, capacity=None, hit_capacity=None):
    """seed_extend_all with room for every hit and, for k = 0, 16 alignments per read on average"""
    if capacity is None and k == 0:
        capacity = 16 * rs.count + 1024
    return nb.seed_extend_all(fmi, gw, rs, params, mq, k, capacity=capacity, hit_capacity=hit_capacity or 1000 * rs.count)


def check(O, g, gw, idx, fmi, reads, rs, params, mq, k, quals=None):
    hc = 1000 * rs.count
    al = run(fmi, gw, rs, params, mq, k)
    ref = nb.seed_extend(fmi, gw, rs, params, hit_capacity=hc, traceback=True, mapq=mq)
    torch.cuda.synchronize()
    assert int(al.n_hits[0]) == int(al.n_hits[1])
    for f in ("best_score", "best_pos", "second_score", "second_pos", "second_strand", "mapq", "n_hits"):
        assert torch.equal(getattr(al, f), getattr(ref, f)), f
    strands = 2 if params.both_strands else 1
    lens = np.array([len(r) for r in reads])
    se = seed_extend_oracle(O, idx, g, reads, params, quals=quals)
    min_score = mq.min_score.cpu().numpy()
    want = all_oracle(se, lens, strands, min_score, k)
    got = lists(al)
    end = se["hit_window"][:, 0] + se["hit_sink"][:, 0]
    n_al = 0
    for r in range(len(reads)):
        w = [(int(se["hit_score"][h]), int(end[h]), int(se["hit_string"][h]) % strands) for h in want[r]]
        assert got[r] == w, (r, got[r], w)
        n_al += len(w)
    assert int(al.count[0]) == int(al.count[1]) == n_al
    # rank 0 = the best alignment and its traceback, rank 1 = the second best
    first = host_u32(al.first).astype(np.int64)
    best_score, best_pos, bst = ref.best_score.cpu().numpy(), host_u32(ref.best_pos), ref.best_strand.cpu().numpy()
    has_best = np.array([len(x) > 0 for x in got])
    above = (best_score != INT_MIN) & (best_score >= min_score[lens])
    assert np.array_equal(has_best, above)
    rows = np.nonzero(has_best)[0]
    f0 = first[rows]
    assert np.array_equal(al.score.cpu().numpy()[f0], best_score[rows]) and np.array_equal(host_u32(al.pos)[f0], best_pos[rows])
    assert np.array_equal(al.strand.cpu().numpy()[f0], bst[rows])
    assert torch.equal(al.n_ops[f0], ref.best_n_ops[rows]) and torch.equal(al.begin[f0], ref.best_begin[rows])
    assert torch.equal(al.ops[f0], ref.best_ops[rows])
    sec, spos, sst = ref.second_score.cpu().numpy(), host_u32(ref.second_pos), ref.second_strand.cpu().numpy()
    for r in rows:
        if k != 1:
            if len(got[r]) > 1:
                assert got[r][1] == (int(sec[r]), int(spos[r]), int(sst[r])), r
            else:
                assert sec[r] == INT_MIN, r
    # every alignment's trace = the banded traceback of its (strand, window) job alone
    hits = [h for r in range(len(reads)) for h in want[r]]
    if hits:
        strs = [reads[int(se["hit_string"][h]) // strands] if int(se["hit_string"][h]) % strands == 0 else rc(reads[int(se["hit_string"][h]) // strands])
                for h in hits]
        pats = packed(strs, bits=rs.bits)
        win = se["hit_window"][hits]
        txt = PackedStringSet(words=gw, bits=2, big_endian=True, offsets=torch.from_numpy(win[:, 0].astype(np.uint32).view(np.int32)).cuda(),
                              lengths=torch.from_numpy((win[:, 1] - win[:, 0]).astype(np.uint32).view(np.int32)).cuda(),
                              stride=0, length=int((win[:, 1] - win[:, 0]).max()), count=len(hits))
        q = None
        if quals is not None:
            q = torch.from_numpy(np.concatenate([quals[int(se["hit_string"][h]) // strands] if int(se["hit_string"][h]) % strands == 0
                                                 else quals[int(se["hit_string"][h]) // strands][::-1] for h in hits])).cuda()
        tb = aln.batch_banded_alignment_traceback(params.band_len, aln.make_gotoh_aligner(params.type, params.scheme), pats, txt, quals=q,
                                                  max_ops=al.max_ops)
        torch.cuda.synchronize()
        n = len(hits)
        assert torch.equal(al.n_ops[:n], tb["n_ops"])
        begin = tb["source"].clone()
        begin[:, 0] += torch.from_numpy(win[:, 0].astype(np.int64)).cuda().to(torch.int32)
        assert torch.equal(al.begin[:n], begin)
        for i in range(n):
            m = int(tb["n_ops"][i])
            assert torch.equal(al.ops[i, :m], tb["ops"][i, :m]), i
    return al, got


LOCAL = dict(seed_len=20, seed_interval=10, band_len=31, type=aln.LOCAL, both_strands=True, max_seed_hits=50)


@pytest.mark.parametrize("k", [1, 2, 5, 0])
def test_all_local_vs_oracle(setup, k):
    O, g, gw, idx, fmi = setup
    reads = make_reads(g, seed=7 + k)
    rs = packed(reads, L=100)
    params = nb.SeedExtendParams(**LOCAL, scheme=aln.SimpleGotohScheme(2, -2, -5, -3))
    al, got = check(O, g, gw, idx, fmi, reads, rs, params, MapqParams.local(100), k)
    counts = np.array([len(x) for x in got])
    if k != 1:
        assert (counts > 1).sum() > 0.3 * len(reads)                     # the repeat family
        assert counts.max() == (k or counts.max())
    if k == 0:
        assert counts.max() >= 8


@pytest.mark.parametrize("k", [2, 0])
def test_all_4bit_ragged_and_paths(setup, k):
    """4-bit reads with N, ragged lengths; the per-hit path and job de-duplication off give the same stored alignments"""
    O, g, gw, idx, fmi = setup
    reads = make_reads(g, ragged=True, seed=17 + k)
    rng = np.random.default_rng(3)
    for r in reads[::7]:
        r[rng.integers(0, len(r), 2)] = 4
    rs = packed(reads, bits=4, L=100)
    params = nb.SeedExtendParams(**LOCAL, scheme=aln.SimpleGotohScheme(2, -2, -5, -3))
    mq = MapqParams.local(100)
    al, got = check(O, g, gw, idx, fmi, reads, rs, params, mq, k)
    L_ = nb.lib()
    L_.nvb_debug_pipeline_path(C.c_int(1))
    try:
        assert lists(run(fmi, gw, rs, params, mq, k)) == got
    finally:
        L_.nvb_debug_pipeline_path(C.c_int(0))
    params.dedup_jobs = False
    assert lists(run(fmi, gw, rs, params, mq, k)) == got


@pytest.mark.parametrize("k", [1, 5])
def test_all_end_to_end(setup, k):
    O, g, gw, idx, fmi = setup
    reads = make_reads(g, seed=21 + k)
    rs = packed(reads, L=100)
    params = nb.SeedExtendParams(seed_len=22, seed_interval=10, band_len=31, type=aln.SEMI_GLOBAL, both_strands=True, max_seed_hits=50,
                                 scheme=aln.SimpleGotohScheme(0, -6, -5, -3))
    check(O, g, gw, idx, fmi, reads, rs, params, MapqParams.end_to_end(100), k)


def test_all_quality_scheme(setup):
    O, g, gw, idx, fmi = setup
    reads = make_reads(g, seed=33)
    rng = np.random.default_rng(9)
    quals = [rng.integers(0, 50, len(r)).astype(np.uint8) for r in reads]
    rs = packed(reads, L=100)
    sch = aln.QualityGotohScheme(match_bonus=2, mm_min=2, mm_max=6, read_gap_const=5, read_gap_coeff=3, ref_gap_const=5, ref_gap_coeff=3)
    params = nb.SeedExtendParams(**LOCAL, scheme=sch, read_quals=torch.from_numpy(np.concatenate(quals)).cuda())
    check(O, g, gw, idx, fmi, reads, rs, params, MapqParams.local(100), 2, quals=quals)


@pytest.mark.parametrize("L", [300, 512])
def test_all_long_reads(setup, L):
    O, g, gw, idx, fmi = setup
    reads = make_reads(g, n_reads=120, L=L, ragged=True, seed=L)
    rs = packed(reads, L=L)
    params = nb.SeedExtendParams(**LOCAL, scheme=aln.SimpleGotohScheme(2, -2, -5, -3))
    al, got = check(O, g, gw, idx, fmi, reads, rs, params, MapqParams.local(L), 0)
    assert sum(len(x) > 1 for x in got) > 10


def test_all_capacity_cut_and_empty(setup):
    """a capacity that cuts mid-batch stores exactly the whole reads that fit; traceback slices past the stored ones are no-ops;
    no reads: d_first = [0], count = (0, 0)"""
    O, g, gw, idx, fmi = setup
    reads = make_reads(g, seed=5)
    rs = packed(reads, L=100)
    params = nb.SeedExtendParams(**LOCAL, scheme=aln.SimpleGotohScheme(2, -2, -5, -3))
    mq = MapqParams.local(100)
    full = run(fmi, gw, rs, params, mq, 0)
    want = lists(full)
    first = host_u32(full.first).astype(np.int64)
    total = int(first[-1])
    assert int(full.count[0]) == int(full.count[1]) == total
    cap = int(first[len(reads) // 2]) + 1                                # one slot into the next read's range
    cut = run(fmi, gw, rs, params, mq, 0, capacity=cap)
    got = lists(cut)
    assert torch.equal(cut.first, full.first)
    last = max(r for r in range(len(reads)) if first[r + 1] <= cap)
    assert int(cut.count[0]) == int(first[last + 1]) and int(cut.count[1]) == total
    for r in range(len(reads)):
        assert got[r] == (want[r] if first[r + 1] <= cap else None), r
    s = int(cut.count[0])
    for f in ("read", "score", "pos", "n_ops", "begin", "strand"):
        assert torch.equal(getattr(cut, f)[:s], getattr(full, f)[:s]), f
    # a capacity of several slices of n_reads each, most of them past the stored alignments
    many = run(fmi, gw, rs, params, mq, 1, capacity=5 * len(reads) + 7)
    one = run(fmi, gw, rs, params, mq, 1)
    assert lists(many) == lists(one)
    # n_reads = 0
    e = PackedStringSet.fixed(rs.words, 0, 100, stride=112)
    z = nb.seed_extend_all(fmi, gw, e, params, mq, 2, capacity=4, hit_capacity=16)
    torch.cuda.synchronize()
    assert int(z.first[0]) == 0 and z.count.tolist() == [0, 0]


def test_all_strings_view(setup):
    """strings(reads): slot i is read read[i] over the reads' own words"""
    O, g, gw, idx, fmi = setup
    reads = make_reads(g, n_reads=64, seed=9)
    rs = packed(reads, L=100)
    params = nb.SeedExtendParams(**LOCAL, scheme=aln.SimpleGotohScheme(2, -2, -5, -3))
    al = run(fmi, gw, rs, params, MapqParams.local(100), 0)
    v = al.strings(rs)
    torch.cuda.synchronize()
    s = int(al.count[0])
    rd = al.read[:s].long()
    assert v.words is rs.words and v.count == al.capacity
    assert torch.equal(v.offsets[:s], rs.offsets[rd]) and torch.equal(v.lengths[:s], rs.lengths[rd])


@pytest.mark.parametrize("k,bits", [(3, 2), (0, 4)])
def test_all_bam_records(setup, k, bits, tmp_path):
    """BAM records of the stored alignments equal the restatement (tests/all_oracle.py on tests/bam_oracle.py) byte for byte, on contigs
    cut under some copies of the family; the coordinate-sorted file reads back through htslib (where built) with one non-secondary record
    per read and NH equal to the read's mapped records, and its BAI is built (status 0)"""
    from oracle.ref_bam import RefBam
    O, g, gw, idx, fmi = setup
    reads = make_reads(g, n_reads=300, seed=60 + k)
    rng = np.random.default_rng(k)
    quals = [rng.integers(0, 42, len(r)).astype(np.uint8) for r in reads]
    rs = packed(reads, bits=bits, L=100)
    params = nb.SeedExtendParams(**LOCAL, scheme=aln.SimpleGotohScheme(2, -2, -5, -3))
    al = run(fmi, gw, rs, params, MapqParams.local(100), k, capacity=None if k else 8 * rs.count)
    cuts = [20_300, 40_000, 60_590, 100_010, 150_000]                       # inside, at and near copies of the family
    cb = [0] + cuts + [N_GENOME]
    contigs = nb.ContigTable(["c%d" % i for i in range(len(cb) - 1)], list(np.diff(cb)))
    names = ["r%d" % i for i in range(len(reads))]
    q = torch.from_numpy(np.concatenate(quals)).cuda()
    f = nb.finish_alignments(gw, al.strings(rs), al.ops, al.n_ops, al.begin, al.strand, genome_len=N_GENOME)
    recs = nb.bam_records_all(al, f, rs, contigs, names, quals=q)
    torch.cuda.synchronize()
    A = al.capacity
    inp = dict(reads=reads, quals=quals, n_ops=al.n_ops.cpu().numpy(), begin=host_u32(al.begin).reshape(-1, 2), strand=al.strand.cpu().numpy(),
               cigar=host_u32(f.cigar).reshape(A, -1), n_cigar=host_u32(f.n_cigar), md=f.md.cpu().numpy().reshape(A, -1),
               md_len=host_u32(f.md_len), edits=host_u32(f.edits).reshape(A, 4), score=al.score.cpu().numpy(), mapq=al.mapq.cpu().numpy(),
               second=al.second_score.cpu().numpy(), pair_flags=None, contig_begin=np.array(cb, np.int64), contig_names=contigs.names,
               contig_lengths=list(np.diff(cb)), names=names)
    first = host_u32(al.first)
    want, cnt = all_records(inp, first, al.capacity)
    assert recs.counts.cpu().tolist() == cnt
    assert recs.offsets.numel() == len(want) + 1
    assert recs.to_bytes() == b"".join(w for w, _ in want)
    flags = np.array([int.from_bytes(w[18:20], "little") for w, _ in want])
    assert (flags & 0x100).sum() > 50 and cnt[2] > 0                       # secondary records, and alignments cut by a contig end
    path = str(tmp_path / "all.bam")
    nb.write_sorted_bam(path, contigs, recs)
    if RefBam.available():
        lines = RefBam().format(path).splitlines()
        assert len(lines) == len(want)
        primary, nh, mapped = {}, {}, {}
        for ln in lines:
            fl = ln.split("\t")
            flag = int(fl[1])
            if not flag & 0x100:
                primary[fl[0]] = primary.get(fl[0], 0) + 1
            if not flag & 0x4:
                mapped[fl[0]] = mapped.get(fl[0], 0) + 1
                nh[fl[0]] = [int(t[5:]) for t in fl[11:] if t.startswith("NH:i:")][0]
        assert all(primary.get(nm) == 1 for nm in names)
        assert all(nh[nm] == mapped[nm] for nm in mapped)
