"""-m gpu: nvb_finish_alignments on the device.  On the outputs of nvb_seed_extend_traceback (planted-repeat genome, 1 % substitutions and
1-3 bp indels, reads at and past both genome ends, 2- and 4-bit reads with N, both strands, LOCAL / SEMI_GLOBAL / GLOBAL, bands 15 / 31,
constant and quality schemes) and of nvb_seed_extend_paired_traceback (rescued mates included) every field equals tests/finish_oracle.py on
the same device outputs, MD + CIGAR rebuild the reference span and NM = XM + I + D; crafted batches through the entry point cover the
hand-built op streams, capacity truncation and n = 0."""
import numpy as np
import pytest
import torch
from oracle import orc
import nvbio_b200 as nb
from nvbio_b200 import aln
from nvbio_b200.strings import PackedStringSet, pack_symbols
from tests import finish_oracle as fo
from tests.gpu_util import require_gpu
from tests.test_finish_host import Batch, build_case, HAND
from tests.test_gpu_paired_traceback import world, run as run_paired  # noqa: F401  (the paired world fixture)

NONE = 0xFFFFFFFF


def check_device(f, reads, strand, ops, n_ops, begin, gsym, glen):
    """every alignment of a FinishedAlignments against the restatement; returns (finished, with indels, with clips, with columns past the end)"""
    torch.cuda.synchronize()
    cig, ncig = f.cigar.cpu().numpy().view(np.uint32), f.n_cigar.cpu().numpy().view(np.uint32)
    md, mdl, ed = f.md.cpu().numpy(), f.md_len.cpu().numpy().view(np.uint32), f.edits.cpu().numpy().view(np.uint32)
    max_ops = ops.shape[1]
    stats = np.zeros(4, np.int64)
    for a in range(len(reads)):
        cigar, m, e = fo.finish(ops[a], n_ops[a], max_ops, begin[a], strand[a], reads[a], gsym, glen)
        got = ([(int(v) >> 4, int(v) & 15) for v in cig[a, :ncig[a]]], bytes(md[a, :mdl[a]]).decode(), tuple(int(v) for v in ed[a]))
        assert got == (cigar, m, e), (a, int(strand[a]), begin[a].tolist(), fo.cigar_text(cigar), m)
        if n_ops[a] == 0 or e[0] == NONE:
            continue
        x = int(begin[a][0]); M = sum(k for k, op in cigar if op == 0); D = sum(k for k, op in cigar if op == 2)
        assert fo.rebuild_reference(cigar, m, reads[a], strand[a]) == "".join(fo.ref_char(gsym, glen, x + c) for c in range(M + D))
        assert e[0] == e[1] + sum(k for k, op in cigar if op in (1, 2))
        stats += (1, any(op in (1, 2) for _, op in cigar), any(op == 4 for _, op in cigar), x + M + D > glen)
    return stats


@pytest.fixture(scope="module")
def se_world():
    """200 kbp genome with a planted repeat family and a tandem repeat; 400 reads of 90-150 bp (1 % substitutions, a 1-3 bp indel in a
    third of them, half reverse-complemented), 40 of them at position 0..5 or running up to 12 bp past the genome's end"""
    require_gpu()
    O = orc.Oracle()
    rng = np.random.default_rng(404)
    G = 200_000
    g = rng.integers(0, 4, G).astype(np.uint8)
    unit = g[1000:1800].copy()
    for p in (20_000, 70_000, 130_000, 170_000):
        u = unit.copy(); m = rng.random(len(u)) < 0.01; u[m] = rng.integers(0, 4, int(m.sum())); g[p:p + len(u)] = u
    g[50_000:51_000] = np.tile(g[50_000:50_040], 25)
    idx = O.build_index(g)
    fmi = nb.FMIndexDevice.from_host(idx.bwt_occ, idx.ssa, idx.L2, idx.n, idx.primary)
    gw = torch.from_numpy(pack_symbols(g, 2, True).view(np.int32)).cuda()
    reads = []
    for i in range(400):
        L = int(rng.integers(90, 151))
        x = int(rng.integers(0, 6)) if i < 20 else (G - L + int(rng.integers(-4, 13)) if i < 40 else
                                                      int(rng.choice([20_000, 70_000, 1000])) + int(rng.integers(0, 500)) if i < 80 else int(rng.integers(0, G - L)))
        r = np.concatenate([g[x:x + L], rng.integers(0, 4, max(0, x + L - G)).astype(np.uint8)])[:L]
        m = rng.random(L) < 0.01; r[m] = rng.integers(0, 4, int(m.sum()))
        if rng.random() < 0.33:
            k, d = int(rng.integers(20, L - 20)), int(rng.integers(1, 4))
            r = np.concatenate([r[:k], r[k + d:]]) if rng.random() < 0.5 else np.concatenate([r[:k], rng.integers(0, 4, d).astype(np.uint8), r[k:]])
        if rng.random() < 0.5:
            r = fo.strand_read(r, 1)
        reads.append(r.astype(np.uint8))
    quals = [rng.integers(2, 41, len(r)).astype(np.uint8) for r in reads]
    return dict(g=g, G=G, fmi=fmi, gw=gw, reads=reads, quals=quals, rng=rng)


def read_set(reads, bits):
    lens = np.array([len(r) for r in reads], np.uint32)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint32)
    return PackedStringSet.from_symbols(np.concatenate(reads), offs, lens, bits=bits, big_endian=True)


@pytest.mark.gpu
@pytest.mark.parametrize("bits", [2, 4])
def test_single_end_traceback_outputs(se_world, bits):
    w = se_world
    rng = np.random.default_rng(9 + bits)
    reads = [r.copy() for r in w["reads"]]
    if bits == 4:
        for r in reads:
            r[rng.random(len(r)) < 0.005] = 4
    rs = read_set(reads, bits)
    q = torch.from_numpy(np.concatenate(w["quals"])).cuda()
    total = np.zeros(4, np.int64)
    for typ in (aln.LOCAL, aln.SEMI_GLOBAL, aln.GLOBAL):
        for band in (15, 31):
            for qual in (False, True):
                scheme = aln.QualityGotohScheme(2 if typ == aln.LOCAL else 0, 2, 6, 5, 3, 5, 3) if qual else \
                    aln.SimpleGotohScheme(2, -2, -5, -3) if typ == aln.LOCAL else aln.SimpleGotohScheme(0, -6, -5, -3)
                params = nb.SeedExtendParams(seed_len=20, seed_interval=10, band_len=band, type=typ, both_strands=True, max_seed_hits=50,
                                             scheme=scheme, read_quals=q if qual else None)
                ws = nb.seed_extend(w["fmi"], w["gw"], rs, params, traceback=True, hit_capacity=64 * len(reads))
                f = nb.finish_alignments(w["gw"], rs, ws.best_ops, ws.best_n_ops, ws.best_begin, ws.best_strand, genome_len=w["G"])
                torch.cuda.synchronize()
                ops, n_ops = ws.best_ops.cpu().numpy(), ws.best_n_ops.cpu().numpy()
                begin, strand = ws.best_begin.cpu().numpy().view(np.uint32), ws.best_strand.cpu().numpy()
                assert f.cigar.shape[1] == ws.max_ops + 2 and f.md.shape[1] == 3 * ws.max_ops + 1
                st = check_device(f, reads, strand, ops, n_ops, begin, w["g"], w["G"])
                assert st[0] > 0.8 * len(reads), (typ, band, qual, st)
                total += st
    assert total[1] > 100 and total[2] > 50 and (strand == 1).any() and (strand == 0).any()


@pytest.mark.gpu
@pytest.mark.parametrize("qual", [False, True])
def test_paired_traceback_outputs(world, qual):
    w = world
    pair = nb.PairParams(min_frag=0, max_frag=420, min_mate_score=50)
    got, ws = run_paired(w, pair, qual=qual)
    rescued = ((got["pair_flags"] == 2) | (got["pair_flags"] == 4)).sum()
    assert rescued > 0
    lens = np.array([len(r) for r in w["reads"]], np.uint32)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint32)
    rs = PackedStringSet.from_symbols(np.concatenate(w["reads"]), offs, lens, bits=2, big_endian=True)
    f = nb.finish_alignments(w["gw"], rs, ws.mate_ops, ws.mate_n_ops, ws.mate_begin, ws.mate_strand, genome_len=int(w["idx"].n))
    n = 2 * w["n_pairs"]
    ops, n_ops = got["mate_ops"].reshape(n, -1), got["mate_n_ops"].reshape(n)
    begin, strand = got["mate_begin"].reshape(n, 2).view(np.uint32), got["mate_strand"].reshape(n)
    st = check_device(f, w["reads"], strand, ops, n_ops, begin, w["gsym"], int(w["idx"].n))
    assert st[0] > 0.8 * n and st[1] > 20


def crafted(rng, genome, bits):
    G = len(genome)
    b = Batch(genome)
    for script in HAND + ([[("N", 1)], [("M", 3), ("N", 2), ("X", 1), ("N", 1), ("M", 2)]] if bits == 4 else []):
        for strand in (0, 1):
            for x in (0, 777, G - 1300):
                r, ops, beg = build_case(rng, genome, G, x, script, strand, bits)
                b.add(r, strand, ops, beg)
    for strand in (0, 1):
        for script, x in (([("M", 40)], G - 10), ([("M", 5), ("D", 3), ("M", 5)], G - 6), ([("S", 3), ("M", 33), ("S", 2)], G - 17)):
            r, ops, beg = build_case(rng, genome, G, x, script, strand, bits)
            b.add(r, strand, ops, beg)
    r, ops, beg = build_case(rng, genome, G, 500, [("M", 30), ("I", 2), ("M", 10)], 0, bits)
    b.add(r, 0, ops, beg, n_ops=b.max_ops + 1)
    b.add(r, 0, ops, (NONE, 0))
    b.add(r, 0, ops, (500, 1))
    b.add(r, 0, ops[:0], (NONE, NONE))
    return b


def device_batch(b, bits):
    rs = read_set(b.reads, bits)
    gw = torch.from_numpy(pack_symbols(b.genome[:b.genome_len], 2, True).view(np.int32)).cuda()
    ops = torch.from_numpy(np.stack(b.ops)).cuda()
    n_ops = torch.from_numpy(np.array(b.n_ops, np.uint32).view(np.int32)).cuda()
    begin = torch.from_numpy(np.array(b.begin, np.uint32).reshape(-1, 2).view(np.int32)).cuda()
    strand = torch.from_numpy(np.array(b.strand, np.uint8)).cuda()
    return rs, gw, ops, n_ops, begin, strand


@pytest.mark.gpu
@pytest.mark.parametrize("bits", [2, 4])
def test_crafted_batches(bits):
    require_gpu()
    rng = np.random.default_rng(55 + bits)
    genome = rng.integers(0, 4, 20_000).astype(np.uint8)
    b = crafted(rng, genome, bits)
    rs, gw, ops, n_ops, begin, strand = device_batch(b, bits)
    f = nb.finish_alignments(gw, rs, ops, n_ops, begin, strand, genome_len=b.genome_len)
    st = check_device(f, b.reads, np.array(b.strand), np.stack(b.ops), np.array(b.n_ops), np.array(b.begin, np.uint32).reshape(-1, 2), genome, b.genome_len)
    assert st[3] > 0
    ed = f.edits.cpu().numpy().view(np.uint32)
    assert (ed[-4:-1, 0] == NONE).all() and not ed[-1].any()
    i = [a for a in range(len(b)) if b.n_ops[a] == 1000 and b.strand[a] == 0][0]
    assert f.md_string(i) == "1000" and f.cigar_string(i) == "1000M"
    # capacity truncation: runs / bytes beyond max_cigar / max_md are counted and not stored; a sentinel after the last slot stays
    for mc, mm in ((1, 1), (2, 7)):
        g = nb.finish_alignments(gw, rs, ops, n_ops, begin, strand, max_cigar=mc, max_md=mm, genome_len=b.genome_len)
        torch.cuda.synchronize()
        assert torch.equal(g.n_cigar, f.n_cigar) and torch.equal(g.md_len, f.md_len) and torch.equal(g.edits, f.edits)
        for a in range(len(b)):
            kc, km = min(mc, int(f.n_cigar[a])), min(mm, int(f.md_len[a]))
            assert torch.equal(g.cigar[a, :kc], f.cigar[a, :kc]) and torch.equal(g.md[a, :km], f.md[a, :km])
        # the same call into buffers one slot larger than the arrays it is told about
        from nvbio_b200._lib import lib, BestAlignmentOutStruct, FinishOutStruct
        import ctypes as C
        n = len(b)
        cig = torch.full((n * mc + 1,), 0x5A5A5A5A, dtype=torch.int32, device="cuda"); md = torch.full((n * mm + 1,), 0x5A, dtype=torch.uint8, device="cuda")
        aux = torch.zeros((3, n), dtype=torch.int32, device="cuda"); edits = torch.zeros((n, 4), dtype=torch.int32, device="cuda")
        A = BestAlignmentOutStruct(); A.d_ops, A.max_ops, A.d_n_ops, A.d_begin, A.d_strand = ops.data_ptr(), ops.shape[1], n_ops.data_ptr(), begin.data_ptr(), strand.data_ptr()
        O = FinishOutStruct(); O.d_cigar, O.max_cigar, O.d_n_cigar, O.d_md, O.max_md, O.d_md_len, O.d_edits = \
            cig.data_ptr(), mc, aux[0].data_ptr(), md.data_ptr(), mm, aux[1].data_ptr(), edits.data_ptr()
        rd = rs.struct()
        assert lib().nvb_finish_alignments(C.c_void_p(gw.data_ptr()), C.c_uint32(b.genome_len), C.byref(rd), C.c_uint32(n), C.byref(A), C.byref(O),
                                           C.c_void_p(torch.cuda.current_stream().cuda_stream)) == 0
        torch.cuda.synchronize()
        assert int(cig[-1]) == 0x5A5A5A5A and int(md[-1]) == 0x5A
        for a in range(n):                                   # the stored slots; the others keep the fill
            kc, km = min(mc, int(g.n_cigar[a])), min(mm, int(g.md_len[a]))
            assert torch.equal(cig[a * mc:a * mc + kc], g.cigar[a, :kc]) and torch.equal(md[a * mm:a * mm + km], g.md[a, :km])
            assert (cig[a * mc + kc:(a + 1) * mc] == 0x5A5A5A5A).all() and (md[a * mm + km:(a + 1) * mm] == 0x5A).all()
        # n = 0: nothing is touched
        assert lib().nvb_finish_alignments(C.c_void_p(gw.data_ptr()), C.c_uint32(b.genome_len), C.byref(rd), C.c_uint32(0), C.byref(A), C.byref(O),
                                           C.c_void_p(torch.cuda.current_stream().cuda_stream)) == 0
        torch.cuda.synchronize()
        assert int(cig[-1]) == 0x5A5A5A5A and int(md[-1]) == 0x5A
    z = nb.finish_alignments(gw, PackedStringSet(words=rs.words, bits=bits, big_endian=True, offsets=rs.offsets[:0], lengths=rs.lengths[:0],
                                                 stride=0, length=rs.length, count=0), ops[:0], n_ops[:0], begin[:0], strand[:0], genome_len=b.genome_len)
    torch.cuda.synchronize()
    assert z.cigar.shape[0] == 0 and z.edits.shape == (0, 4)
