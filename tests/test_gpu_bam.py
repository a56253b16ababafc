"""-m gpu: nvb_bam_records on the device.  Single end: seed_extend(traceback=True, mapq=...) -> finish_alignments -> bam_records on a genome
cut into contigs with boundaries planted under read positions, some contigs shorter than a read, and reads past the genome's end (LOCAL and
SEMI_GLOBAL, constant and quality schemes, 2- and 4-bit reads).  Paired: the paired traceback flow with rescued mates.  Every record equals
tests/bam_oracle.py on the same device outputs and d_counts its tallies; write_bam's file reads back through htslib (where oracle/_ref is
built); a capacity that cuts mid-batch stores exactly the records that fit, offsets complete; n = 0 works."""
import ctypes as C
import numpy as np
import pytest
import torch
import nvbio_b200 as nb
from nvbio_b200 import aln
from nvbio_b200.pipeline import MapqParams
from oracle.ref_bam import RefBam
from tests import bam_oracle as bo
from tests.gpu_util import require_gpu
from tests.test_gpu_finish import se_world, read_set  # noqa: F401  (the single-end world fixture)
from tests.test_gpu_paired_traceback import world, run as run_paired  # noqa: F401  (the paired world fixture)


def planted_contigs(begin, n_ops, G, rng, short=True):
    """cuts 30 bases into every 6th aligned read (so its span crosses a contig boundary), random cuts and, with `short`, contigs of 40 / 60 bp"""
    cuts = set(int(x) for x in rng.integers(1, G, 10))
    al = np.nonzero(n_ops > 0)[0]
    for a in al[::6]:
        x = int(begin[a][0]) + 30
        if 0 < x < G:
            cuts.add(x)
    if short:
        cuts |= {1000, 1040, 1100}
    cb = [0] + sorted(cuts) + [G]
    lens = np.diff(cb)
    return nb.ContigTable(["ctg%d" % i for i in range(len(lens))], lens)


def host_inputs(reads, quals, n_ops, begin, strand, f, score, mapq, second, pair_flags, contigs, names):
    torch.cuda.synchronize()
    return dict(reads=reads, quals=quals, n_ops=n_ops.reshape(-1).cpu().numpy().view(np.uint32),
                begin=begin.reshape(-1, 2).cpu().numpy().view(np.uint32), strand=strand.reshape(-1).cpu().numpy(),
                cigar=f.cigar.cpu().numpy().view(np.uint32), n_cigar=f.n_cigar.cpu().numpy().view(np.uint32), md=f.md.cpu().numpy(),
                md_len=f.md_len.cpu().numpy().view(np.uint32), edits=f.edits.cpu().numpy().view(np.uint32),
                score=score.reshape(-1).cpu().numpy(), mapq=None if mapq is None else mapq.reshape(-1).cpu().numpy(),
                second=None if second is None else second.reshape(-1).cpu().numpy(),
                pair_flags=None if pair_flags is None else pair_flags.cpu().numpy().view(np.uint32),
                contig_begin=contigs.begin, contig_names=contigs.names, contig_lengths=list(contigs.lengths), names=names)


def check_records(recs, inp):
    """every record and the tallies equal the restatement; returns the counts"""
    torch.cuda.synchronize()
    want, cnt = bo.records(inp)
    off = recs.offsets.cpu().numpy()
    data = recs.data.cpu().numpy().tobytes()
    assert recs.stored() == len(want)
    for k, (w, sam) in enumerate(want):
        assert data[off[k]:off[k + 1]] == w, (k, sam)
    assert recs.counts.cpu().numpy().tolist() == cnt
    return cnt


@pytest.mark.gpu
@pytest.mark.parametrize("bits", [2, 4])
def test_single_end(se_world, bits, tmp_path):
    w = se_world
    rng = np.random.default_rng(21 + bits)
    reads = [r.copy() for r in w["reads"]]
    if bits == 4:
        for r in reads:
            r[rng.random(len(r)) < 0.005] = 4
    rs = read_set(reads, bits)
    q = torch.from_numpy(np.concatenate(w["quals"])).cuda()
    names = nb.numbered_names(len(reads), "se%d_" % bits)
    total = np.zeros(4, np.int64)
    for typ in (aln.LOCAL, aln.SEMI_GLOBAL):
        for qual in (False, True):
            scheme = aln.QualityGotohScheme(2 if typ == aln.LOCAL else 0, 2, 6, 5, 3, 5, 3) if qual else \
                aln.SimpleGotohScheme(2, -2, -5, -3) if typ == aln.LOCAL else aln.SimpleGotohScheme(0, -6, -5, -3)
            params = nb.SeedExtendParams(seed_len=20, seed_interval=10, band_len=31, type=typ, both_strands=True, max_seed_hits=50,
                                         scheme=scheme, read_quals=q if qual else None)
            mq = MapqParams.local(160) if typ == aln.LOCAL else MapqParams.end_to_end(160)
            ws = nb.seed_extend(w["fmi"], w["gw"], rs, params, traceback=True, mapq=mq, hit_capacity=64 * len(reads))
            f = nb.finish_alignments(w["gw"], rs, ws.best_ops, ws.best_n_ops, ws.best_begin, ws.best_strand, genome_len=w["G"])
            torch.cuda.synchronize()
            contigs = planted_contigs(ws.best_begin.cpu().numpy().view(np.uint32), ws.best_n_ops.cpu().numpy(), w["G"], rng)
            recs = nb.bam_records(ws, f, rs, contigs, names, quals=q if qual else None)
            inp = host_inputs(reads, w["quals"] if qual else None, ws.best_n_ops, ws.best_begin, ws.best_strand, f, ws.best_score,
                              ws.mapq, ws.second_score, None, contigs, names)
            cnt = check_records(recs, inp)
            total += cnt
            if typ == aln.LOCAL and qual and RefBam.available():
                p = str(tmp_path / ("se%d.bam" % bits))
                nb.write_bam(p, nb.bam_header(contigs), [recs])
                want, _ = bo.records(inp)
                assert RefBam().format(p) == "".join(s + "\n" for _, s in want)
    assert total[1] > 0.6 * total[0] and total[2] > 20, total


@pytest.mark.gpu
@pytest.mark.parametrize("qual", [False, True])
def test_paired(world, qual):
    w = world
    rng = np.random.default_rng(31 + qual)
    pair = nb.PairParams(min_frag=0, max_frag=420, min_mate_score=50)
    got, ws = run_paired(w, pair, qual=qual, mapq=MapqParams.local(120))
    assert ((got["pair_flags"] == 2) | (got["pair_flags"] == 4)).sum() > 0
    lens = np.array([len(r) for r in w["reads"]], np.uint32)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint32)
    rs = nb.PackedStringSet.from_symbols(np.concatenate(w["reads"]), offs, lens, bits=2, big_endian=True)
    G = int(w["idx"].n)
    f = nb.finish_alignments(w["gw"], rs, ws.mate_ops, ws.mate_n_ops, ws.mate_begin, ws.mate_strand, genome_len=G)
    torch.cuda.synchronize()
    contigs = planted_contigs(ws.mate_begin.reshape(-1, 2).cpu().numpy().view(np.uint32), ws.mate_n_ops.reshape(-1).cpu().numpy(), G, rng)
    names = nb.numbered_names(w["n_pairs"], "pair")
    q = torch.from_numpy(np.concatenate(w["quals"])).cuda() if qual else None
    recs = nb.bam_records(ws, f, rs, contigs, names, quals=q)
    inp = host_inputs(w["reads"], w["quals"] if qual else None, ws.mate_n_ops, ws.mate_begin, ws.mate_strand, f, ws.mate_score,
                      ws.mate_mapq, ws.mate_second_score, ws.pair_flags, contigs, names)
    cnt = check_records(recs, inp)
    assert cnt[2] > 10 and cnt[1] > 0.6 * cnt[0], cnt
    # a capacity that cuts mid-batch: exactly the records that fit are stored, offsets and counts complete
    off = recs.offsets.cpu().numpy()
    cap = int(off[len(off) // 2] + 7)
    cut = nb.bam_records(ws, f, rs, contigs, names, quals=q, capacity=cap)
    torch.cuda.synchronize()
    k = int(np.searchsorted(off[1:], cap, side="right"))
    assert torch.equal(cut.offsets, recs.offsets) and torch.equal(cut.counts, recs.counts) and cut.stored() == k
    assert cut.data[:int(off[k])].cpu().numpy().tobytes() == recs.data[:int(off[k])].cpu().numpy().tobytes()


@pytest.mark.gpu
def test_records_larger_than_the_staging_span_and_n_zero():
    """records longer than the write kernel's 32 KiB staging span are composed in place; n = 0 writes offsets[0] = 0 and zero counts"""
    require_gpu()
    from nvbio_b200._lib import lib, BamInStruct, BamOutStruct
    from tests.golden.make_bam_golden import fixture_inputs
    inp = fixture_inputs(False, 5, n=40)
    for a in (3, 4, 20):                                     # 25,000-symbol unaligned reads: 37.5 KB records
        inp["n_ops"][a] = 0; inp["reads"][a] = np.random.default_rng(a).integers(0, 5, 25_000).astype(np.uint8)
    inp["quals"] = [np.full(len(r), 30, np.uint8) for r in inp["reads"]]
    want, cnt = bo.records(inp)
    n = len(want)
    lens = np.array([len(r) for r in inp["reads"]], np.uint32)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint32)
    rs = nb.PackedStringSet.from_symbols(np.concatenate(inp["reads"]), offs, lens, bits=4, big_endian=True)
    t = lambda x, dt: torch.from_numpy(np.ascontiguousarray(np.asarray(x).astype(dt))).cuda()  # noqa: E731
    dq = t(np.concatenate(inp["quals"]), np.uint8)
    nbytes = [nm.encode() for nm in inp["names"]]
    dn = t(np.frombuffer(b"".join(nbytes), np.uint8), np.uint8)
    dno = t(np.concatenate([[0], np.cumsum([len(x) for x in nbytes])]).astype(np.int64), np.int32)
    keep = dict(n_ops=t(inp["n_ops"], np.int32), begin=t(inp["begin"].astype(np.int64), np.int32), strand=t(inp["strand"], np.uint8),
                cigar=t(inp["cigar"].astype(np.int64), np.int32), n_cigar=t(inp["n_cigar"], np.int32), md=t(inp["md"], np.uint8),
                md_len=t(inp["md_len"], np.int32), edits=t(inp["edits"].astype(np.int64), np.int32), score=t(inp["score"], np.int32),
                cb=t(inp["contig_begin"].astype(np.int64), np.int32))
    a = BamInStruct()
    a.reads = rs.struct(); a.d_read_quals = dq.data_ptr()
    a.d_n_ops, a.d_begin, a.d_strand = keep["n_ops"].data_ptr(), keep["begin"].data_ptr(), keep["strand"].data_ptr()
    a.finish.d_cigar, a.finish.max_cigar, a.finish.d_n_cigar = keep["cigar"].data_ptr(), inp["cigar"].shape[1], keep["n_cigar"].data_ptr()
    a.finish.d_md, a.finish.max_md, a.finish.d_md_len = keep["md"].data_ptr(), inp["md"].shape[1], keep["md_len"].data_ptr()
    a.finish.d_edits, a.d_score = keep["edits"].data_ptr(), keep["score"].data_ptr()
    a.d_contig_begin, a.n_contigs = keep["cb"].data_ptr(), len(inp["contig_begin"]) - 1
    a.d_names, a.d_name_offsets = dn.data_ptr(), dno.data_ptr()
    total = sum(len(x) for x, _ in want)
    data = torch.full((total + 64,), 0x5A, dtype=torch.uint8, device="cuda")
    offsets = torch.empty(n + 1, dtype=torch.int64, device="cuda"); counts = torch.empty(4, dtype=torch.int32, device="cuda")
    o = BamOutStruct(); o.d_records, o.capacity, o.d_offsets, o.d_counts = data.data_ptr(), total, offsets.data_ptr(), counts.data_ptr()
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    tb = C.c_size_t(0)
    assert lib().nvb_bam_records(C.byref(a), C.c_uint32(n), C.byref(o), None, C.byref(tb), s) == -2 and tb.value > 0
    temp = torch.empty(tb.value, dtype=torch.uint8, device="cuda")
    assert lib().nvb_bam_records(C.byref(a), C.c_uint32(n), C.byref(o), C.c_void_p(temp.data_ptr()), C.byref(tb), s) == 0
    torch.cuda.synchronize()
    assert data[:total].cpu().numpy().tobytes() == b"".join(x for x, _ in want)
    assert (data[total:] == 0x5A).all() and counts.cpu().tolist() == cnt
    assert max(len(x) for x, _ in want) > 32768
    # n = 0
    offsets.fill_(7); counts.fill_(7)
    assert lib().nvb_bam_records(C.byref(a), C.c_uint32(0), C.byref(o), None, C.byref(tb), s) == 0
    torch.cuda.synchronize()
    assert int(offsets[0]) == 0 and counts.cpu().tolist() == [0, 0, 0, 0]
