"""-m gpu: the chain after seed + extend at the genome and batch size bench.py times.  The rest of the suite runs the traceback, MAPQ,
pairing and rescue, finish, BAM records, sort, BGZF and BAI on genomes of a few hundred kbp and batches of a few thousand reads; here they
run on bench.py's 1.9 Gbp index (full suffix array, 15-mer located table with text context, built exactly as bench.build_index builds it)
and on bench's own batches, which differ from the small worlds in what matters:

  * coordinates up to 1.9e9: windows and rescue windows clipped at the genome's end, finish reading the genome for MD, contig look-up of
    a global position, BAI bins and linear-index windows on contigs 2^29 long (the longest the BAI allows);
  * more scored alignments than the resident grid (16 CTAs of 256 threads per SM): the kernels that stride over a device-side count
    (the per-read winner, second-best reduce, candidate scatter, DP scatter and finalize) loop more than once;
  * the index layout build_ktab picks from the free device memory (32-byte table entries, the per-row array), and the same call without
    the per-row array;
  * a BAM stream of about a million records, compressed into thousands of BGZF members, sorted and indexed whole.

  1. single end: bench.make_reads' 1M x 150 bp batch plus ~1,300 planted reads (the genome's end, 2^29 and 2^30, contig boundaries,
     indels, 15 % substitutions, reads found nowhere) and a 4-bit batch with N.  Sampled reads (every 64th, every planted one and up to
     4,000 from each rare group) against the oracle composition run on those reads alone: best, second and MAPQ (mapq_oracle), the
     traceback (the banded traceback of the read's best job alone), finish (finish_oracle) and BAM records (bam_oracle).  The whole
     stream: sort against a stable numpy argsort, BGZF members against zlib and at a second grid size, BAI against bai_oracle.  The same
     call without the per-row array gives identical outputs.
  2. paired end: bench's 500K-pair batch plus planted pairs (rescue windows clipped at both genome ends, fragments across 2^29, fragments
     longer than max_frag, swapped second mates).  Sampled pairs against pair_mapq_oracle; mate traces against the banded traceback of the
     mate's own best job or the full-matrix traceback of its rescue job, replayed to their score and end; finish and paired BAM records;
     sort, BGZF and BAI of the whole stream; the streaming API (nvb_pipeline, paired) returns the direct call's outputs.

Each per-read (per-pair) output depends on that read (pair) alone once no hit is dropped and every rescue job runs, so the oracle runs
on the sample only.  The fixture needs an 80 GB part."""
import ctypes as C
import gc
import time
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import bench
import nvbio_b200 as nb
from nvbio_b200 import aln, synth
from nvbio_b200.pipeline import MapqParams
from nvbio_b200.strings import PackedStringSet, pack_symbols
from oracle import orc
from tests import bai_oracle, bam_oracle
from tests.gpu_util import require_gpu, host_u32
from tests.mapq_oracle import mapq_oracle
from tests.pair_mapq_oracle import pair_mapq_oracle
from tests.pipeline_oracle import seed_extend_oracle, best_hits
from tests.test_bgzf_host import BLOCK, MAX_MEMBER, check_member
from tests.test_gpu_finish import check_device
from tests.test_gpu_paired_traceback import strand_string, replay, PAIR_KEYS, TB_KEYS, MAPQ_KEYS

pytestmark = pytest.mark.gpu

N = 1_900_000_000                                     # bench.py --genome-mbp 1900
L = bench.READ_LEN
B29, B30 = 1 << 29, 1 << 30
FIXED_CUTS = (B29, B30, 3 * B29, 1_800_000_000)       # contigs of exactly 2^29 up to 3 * 2^29, then two shorter ones
INT_MIN = -2**31
NONE = 0xFFFFFFFF
GROUP = 4000                                          # reads (pairs) sampled from each rare group
HEADER_BYTES = 4321                                   # the BAM header's compressed size: it shifts every virtual offset alike


def params():
    """bench.py's SeedExtendParams"""
    return nb.SeedExtendParams(seed_len=bench.SEED_LEN, seed_interval=bench.SEED_INTERVAL, band_len=bench.BAND, type=aln.LOCAL,
                               both_strands=True, max_seed_hits=100, dedup_jobs=True, scheme=aln.SimpleGotohScheme(*bench.SCHEME))


def resident_grid_threads():
    """the largest grid of the kernels that stride over a device-side count (pipeline.cu resident_grid), in threads"""
    return torch.cuda.get_device_properties(0).multi_processor_count * 16 * 256


def rc(r):
    return np.where(r < 4, 3 - r, r)[::-1].astype(np.uint8)


def mutate(r, rate, rng):
    r = r.copy()
    m = rng.random(len(r)) < rate
    r[m] = (r[m] + 1 + rng.integers(0, 3, int(m.sum()))) % 4
    return r


def pack_rows(reads, wpr):
    """150 bp symbol arrays -> int32 words [n, wpr], the layout of bench's batches (2-bit big endian, wpr words per read)"""
    flat = np.zeros((len(reads), wpr * 16), np.uint8)
    for a, r in enumerate(reads):
        flat[a, :len(r)] = r
    return torch.from_numpy(pack_symbols(flat.reshape(-1), 2, True).view(np.int32)[:len(reads) * wpr].copy()).reshape(len(reads), wpr)


def unpack_rows(words, n_sym=L):
    return bench._unpack_rows(np.ascontiguousarray(words).view(np.uint32), n_sym)


def spread(idx, k):
    """up to k entries of idx, evenly spaced (deterministic)"""
    if len(idx) <= k:
        return idx
    return idx[np.linspace(0, len(idx) - 1, k).astype(np.int64)]


def dev_u32(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint32).view(np.int32)).cuda()


def contig_table(cut_at):
    """FIXED_CUTS plus a cut at every position of cut_at past 2^29 (the first contig stays 2^29 long); the last contig ends at the
    genome's end"""
    cuts = sorted(set(FIXED_CUTS) | set(int(x) for x in cut_at if B29 < int(x) < N))
    lens = np.diff([0] + cuts + [N])
    assert lens.max() <= B29 and lens[0] == B29
    return nb.ContigTable(["chr%d" % i for i in range(len(lens))], lens)


# ---------------------------------------------------------------------------------------------------------------------------------------
# the index, as bench.build_index builds it with its defaults
# ---------------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def H():
    require_gpu()
    _, total = torch.cuda.mem_get_info()
    if total < 75e9:
        pytest.skip("needs an 80 GB part")
    gc.collect()
    torch.cuda.empty_cache()                             # the suffix sort needs all but a few GB of the part
    t0 = time.perf_counter()
    genome = synth.random_genome_words(N)
    fmi, _ = nb.FMIndexDevice.from_text(genome, N, sa_interval=1)
    torch.cuda.empty_cache()
    fmi.build_ktab(15, located=True, text=genome)
    torch.cuda.synchronize()
    print("\nindex: %.0f s; ktab_k %d, ktab_located %d, ktab_wide %s, rows %s; %.1f GB of %.1f GB free" %
          (time.perf_counter() - t0, fmi.ktab_k, fmi.ktab_located, fmi.ktab_wide, fmi.rows is not None,
           torch.cuda.mem_get_info()[0] / 1e9, total / 1e9), flush=True)
    # host side for the oracle: the index in the reference's format and the genome as 1-byte symbols, unpacked in chunks
    idx = orc._Index(n=N, primary=fmi.primary, bwt_occ=host_u32(fmi.bwt_occ), ssa=host_u32(fmi.ssa[::16].contiguous()),
                     L2=np.array(fmi.L2, np.uint32))
    gw = host_u32(genome)
    g = np.empty(N, np.uint8)
    sh = (30 - 2 * np.arange(16)).astype(np.uint32)
    step = 1 << 22
    for w in range(0, N // 16, step):
        c = min(step, N // 16 - w)
        g[16 * w:16 * (w + c)] = ((gw[w:w + c, None] >> sh) & 3).astype(np.uint8).reshape(-1)
    assert N % 16 == 0
    print("host copies: %.0f s" % (time.perf_counter() - t0), flush=True)
    return SimpleNamespace(genome=genome, fmi=fmi, idx=idx, g=g, O=orc.Oracle(), grid=resident_grid_threads())


# ---------------------------------------------------------------------------------------------------------------------------------------
# checks shared by both tests
# ---------------------------------------------------------------------------------------------------------------------------------------
def assert_same(got, want, sel, what):
    for k in got:
        bad = np.flatnonzero(got[k] != want[k])
        assert len(bad) == 0, (what, k, len(bad), [(int(sel[i % len(sel)]), got[k].reshape(-1)[i].item(), want[k].reshape(-1)[i].item())
                                                    for i in bad[:5]])


def banded_traceback_of_jobs(H, pats, win, bits, max_ops):
    """aln.batch_banded_alignment_traceback of (pattern, genome window) jobs: (n_ops, ops, begin = (genome start, read start))"""
    p = params()
    lens = np.array([len(x) for x in pats], np.uint32)
    P = PackedStringSet.from_symbols(np.concatenate(pats), np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint32), lens, bits=bits)
    tl = (win[:, 1] - win[:, 0]).astype(np.uint32)
    T = PackedStringSet(words=H.genome, bits=2, big_endian=True, offsets=dev_u32(win[:, 0]), lengths=dev_u32(tl), stride=0,
                        length=int(tl.max()), count=len(pats))
    tb = aln.batch_banded_alignment_traceback(p.band_len, aln.make_gotoh_aligner(p.type, p.scheme), P, T, max_ops=max_ops)
    torch.cuda.synchronize()
    src = host_u32(tb["source"]).astype(np.int64)
    begin = np.stack([win[:, 0] + src[:, 0], src[:, 1]], axis=1)
    return host_u32(tb["n_ops"]).astype(np.int64), tb["ops"].cpu().numpy(), begin


def check_traces(n_ops, ops, begin, want_n, want_ops, want_begin, sel, what):
    assert np.array_equal(n_ops, want_n), (what, [int(sel[i]) for i in np.flatnonzero(n_ops != want_n)[:5]])
    assert np.array_equal(begin, want_begin), (what, [int(sel[i]) for i in np.flatnonzero((begin != want_begin).any(1))[:5]])
    for i in range(len(n_ops)):
        assert np.array_equal(ops[i, :n_ops[i]], want_ops[i, :n_ops[i]]), (what, int(sel[i]))


def sliced_finish(f, t):
    return SimpleNamespace(cigar=f.cigar[t], n_cigar=f.n_cigar[t], md=f.md[t], md_len=f.md_len[t], edits=f.edits[t])


def check_records(raw, off, rec_index, inp, what):
    """bam_oracle.records(inp) == the device records rec_index (host bytes raw, offsets off)"""
    want, cnt = bam_oracle.records(inp)
    assert len(want) == len(rec_index)
    for (wb, sam), k in zip(want, rec_index):
        assert raw[off[k]:off[k + 1]] == wb, (what, int(k), sam)
    return cnt


def record_keys(data, off):
    """(refID, pos) of every record as uint32, read from the record headers"""
    h = data[off[:-1, None] + np.arange(4, 12)[None, :]]
    v = np.ascontiguousarray(h).view("<u4")
    return v[:, 0], v[:, 1]


def check_stream(recs, contigs, what):
    """sort, BGZF and BAI of a whole record stream; returns (records, BGZF members)"""
    t0 = time.perf_counter()
    off = recs.offsets.cpu().numpy()
    n = len(off) - 1
    assert recs.stored() == n
    raw = recs.data[:int(off[-1])].cpu().numpy()
    s = nb.sort_bam_records(recs)
    torch.cuda.synchronize()
    ref, pos = record_keys(raw, off)
    order = np.argsort((ref.astype(np.uint64) << np.uint64(32)) | pos.astype(np.uint64), kind="stable")
    assert np.array_equal(s.order.cpu().numpy(), order), what
    lens = np.diff(off)
    soff = np.concatenate([[0], np.cumsum(lens[order])]).astype(np.int64)
    assert np.array_equal(s.offsets.cpu().numpy(), soff), what
    rb = raw.tobytes()
    srt = s.to_bytes()
    assert srt == b"".join(rb[off[i]:off[i + 1]] for i in order), what
    # BGZF: every member bounded, with a valid header, CRC-32 and ISIZE, inflating to its 0xFF00 input bytes
    blocks = nb.bgzf_compress(s.data[:int(soff[-1])])
    z = blocks.to_bytes()
    boff = blocks.offsets.cpu().numpy()
    nbk = -(-len(srt) // BLOCK)
    assert blocks.n_blocks == nbk and blocks.stored() == nbk and len(z) == boff[-1], what
    for i in range(nbk):
        m = z[boff[i]:boff[i + 1]]
        assert len(m) <= MAX_MEMBER
        check_member(m, srt[i * BLOCK:(i + 1) * BLOCK])
    try:
        nb.lib().nvb_debug_bgzf_grid(C.c_uint32(37))
        z2 = nb.bgzf_compress(s.data[:int(soff[-1])]).to_bytes()
    finally:
        nb.lib().nvb_debug_bgzf_grid(C.c_uint32(0))
    assert z2 == z, what
    # BAI of the whole sorted stream
    bai = nb.bam_index(s, blocks, HEADER_BYTES, contigs)
    want = bai_oracle.bai_bytes([srt[soff[i]:soff[i + 1]] for i in range(n)], boff, HEADER_BYTES, len(contigs.names))
    assert bai == want, what
    top = int(pos[ref != NONE].max()) if (ref != NONE).any() else -1
    print("%s: %d records, %.0f MB, %d BGZF members (%.0f MB), BAI %d bytes, largest pos %d; %.0f s" %
          (what, n, len(srt) / 1e6, nbk, len(z) / 1e6, len(bai), top, time.perf_counter() - t0), flush=True)
    assert top > 1 << 28, what                          # BAI windows past 2^14 on a contig
    return n, nbk


# ---------------------------------------------------------------------------------------------------------------------------------------
# 1. single end
# ---------------------------------------------------------------------------------------------------------------------------------------
def planted_reads(g, rng):
    """150 bp reads at the places the small worlds do not reach; (reads, kind of each)"""
    out, kind = [], []

    def add(r, k):
        out.append((rc(r) if rng.random() < 0.5 else r).astype(np.uint8)); kind.append(k)
    for k in range(0, 200, 2):                                      # ending at and within 200 bp of the genome's end
        add(g[N - L - k:N - k].copy(), "end")
    for k in (1, 3, 9, 15, 16, 40):                                 # running past it
        add(np.concatenate([g[N - L + k:], rng.integers(0, 4, k).astype(np.uint8)]), "past")
    for b in FIXED_CUTS:                                            # across 2^29, 2^30 and every fixed contig boundary
        for k in range(1, L, 3):
            add(mutate(g[b - k:b - k + L], 0.01, rng), "boundary")
    for _ in range(200):                                            # a 1-3 bp deletion or insertion
        p, q, d = int(rng.integers(0, N - 2 * L)), int(rng.integers(20, L - 20)), int(rng.integers(1, 4))
        r = g[p:p + L + 8].copy()
        r = np.concatenate([r[:q], r[q + d:]]) if rng.random() < 0.5 else np.concatenate([r[:q], rng.integers(0, 4, d).astype(np.uint8), r[q:]])
        add(r[:L], "indel")
    for _ in range(600):                                            # ~15 % substitutions: second bests and MAPQ below the maximum
        p = int(rng.integers(0, N - L))
        add(mutate(g[p:p + L], 0.15, rng), "sub15")
    for _ in range(200):                                            # found nowhere
        add(rng.integers(0, 4, L).astype(np.uint8), "none")
    return out, kind


def run_single(H, rs, n):
    mq = MapqParams.local(L)
    ws = nb.seed_extend(H.fmi, H.genome, rs, params(), traceback=True, mapq=mq, hit_capacity=24 * n)
    torch.cuda.synchronize()
    return ws, mq


SE_OUT = ("best_score", "best_pos", "n_hits", "best_ops", "best_n_ops", "best_begin", "best_strand", "second_score", "second_pos",
          "second_strand", "mapq")


def check_single(H, ws, mq, f, raw, off, contigs, names, reads, sel, bits, what):
    """the sampled reads sel (symbols `reads`) of one seed_extend(traceback=True, mapq=...) call against the oracle composition"""
    t0 = time.perf_counter()
    p = params()
    se = seed_extend_oracle(H.O, H.idx, H.g, reads, p)
    lens = np.array([len(r) for r in reads])
    want = mapq_oracle(se, lens, 2, mq.min_score.cpu().numpy(), mq.match_bonus)
    t = torch.from_numpy(sel).cuda()
    got = dict(best_score=ws.best_score[t].cpu().numpy().astype(np.int64), best_pos=host_u32(ws.best_pos[t]).astype(np.int64),
               best_strand=ws.best_strand[t].cpu().numpy().astype(np.int64), second_score=ws.second_score[t].cpu().numpy().astype(np.int64),
               second_pos=host_u32(ws.second_pos[t]).astype(np.int64), second_strand=ws.second_strand[t].cpu().numpy().astype(np.int64),
               mapq=ws.mapq[t].cpu().numpy().astype(np.int64))
    assert_same(got, want, sel, what)
    # traceback: the banded traceback of the read's best job alone
    n_ops, ops, begin = ws.best_n_ops[t].cpu().numpy().astype(np.int64), ws.best_ops[t].cpu().numpy(), host_u32(ws.best_begin[t])
    strand = ws.best_strand[t].cpu().numpy()
    bh = best_hits(se, len(reads))
    none = np.flatnonzero(bh < 0)
    assert (n_ops[none] == 0).all() and (begin[none] == NONE).all(), what
    rows = np.flatnonzero(bh >= 0)
    h = bh[rows]
    st = se["hit_string"][h] % 2
    pats = [reads[r] if s == 0 else rc(reads[r]) for r, s in zip(rows, st)]
    wn, wo, wb = banded_traceback_of_jobs(H, pats, se["hit_window"][h], bits, ws.max_ops)
    check_traces(n_ops[rows], ops[rows], begin[rows].astype(np.int64), wn, wo, wb, sel[rows], what + ("traceback",))
    gapped = int(sum(np.isin(ops[r, :n_ops[r]], (1, 2)).any() for r in rows))
    # finish: CIGAR, MD and NM / XM / XO / XG
    stats = check_device(sliced_finish(f, t), reads, strand, ops, n_ops, begin, H.g, N)
    # BAM records of the sample, from the inputs sliced to it
    inp = dict(reads=reads, quals=None, n_ops=n_ops.astype(np.uint32), begin=begin, strand=strand, cigar=host_u32(f.cigar[t]),
               n_cigar=host_u32(f.n_cigar[t]), md=f.md[t].cpu().numpy(), md_len=host_u32(f.md_len[t]), edits=host_u32(f.edits[t]),
               score=ws.best_score[t].cpu().numpy(), mapq=ws.mapq[t].cpu().numpy(), second=ws.second_score[t].cpu().numpy(), pair_flags=None,
               contig_begin=contigs.begin, contig_names=contigs.names, contig_lengths=list(contigs.lengths), names=[names[i] for i in sel])
    cnt = check_records(raw, off, sel, inp, what + ("bam",))
    print("%s: %d reads sampled, %d aligned (%d gapped), %d with a second, %d with MAPQ < 44; finish %s; records %s; %.0f s" %
          (what, len(sel), len(rows), gapped, int((want["second_score"] != INT_MIN).sum()), int((want["mapq"] < 44).sum()),
           stats.tolist(), cnt, time.perf_counter() - t0), flush=True)
    return want, gapped, stats


def test_single_end_chain(H):
    rng = np.random.default_rng(1900)
    dev = H.genome.device
    n_bench = 1_000_000
    bw = bench.make_reads(H.genome, N, n_bench, 0, dev)                   # rank 0's first timed batch
    wpr = bw.shape[1]
    planted, kinds = planted_reads(H.g, rng)
    words = torch.cat([bw, pack_rows(planted, wpr).to(dev)]).contiguous()
    n = words.shape[0]
    rs = PackedStringSet.fixed(words.reshape(-1), n, L, stride=wpr * 16)
    ws, mq = run_single(H, rs, n)
    kept, total, jobs = [int(v) for v in ws.n_hits.cpu()]
    print("single end: %d reads, %d hits kept of %d, %d scored alignments, resident grid %d threads" % (n, kept, total, jobs, H.grid),
          flush=True)
    assert kept == total
    assert jobs > H.grid                                    # the grid-stride loops run more than once

    # the sample: every 64th read, every planted read, up to GROUP reads of each rare group
    best = ws.best_score.cpu().numpy()
    end = host_u32(ws.best_pos).astype(np.int64)
    col = torch.arange(ws.max_ops, device=dev)
    gapped = (((ws.best_ops == 1) | (ws.best_ops == 2)) & (col[None, :] < ws.best_n_ops[:, None])).any(1).cpu().numpy()
    second = ws.second_score.cpu().numpy() != INT_MIN
    low = ws.mapq.cpu().numpy() < 44
    cuts = np.array(FIXED_CUTS + (N,), np.int64)
    near = (best != INT_MIN) & (np.abs(end[:, None] - cuts[None, :]) <= 1000).any(1)
    groups = dict(none=best == INT_MIN, gapped=gapped, second=second, low_mapq=low & (best != INT_MIN), near_boundary=near)
    sel = [np.arange(0, n, 64), np.arange(n_bench, n)] + [spread(np.flatnonzero(m), GROUP) for m in groups.values()]
    sel = np.unique(np.concatenate(sel))
    print("groups in the batch: %s; sampled %d reads" % ({k: int(v.sum()) for k, v in groups.items()}, len(sel)), flush=True)
    for k, v in groups.items():
        assert v[sel].sum() > 0, k
    host_words = words.cpu().numpy()
    reads = [planted[i - n_bench] if i >= n_bench else unpack_rows(host_words[i:i + 1])[0] for i in sel]

    # contigs: FIXED_CUTS, cuts 30 bp into every 40th sampled aligned read, the last ending at the genome's end
    begin = host_u32(ws.best_begin)
    al = sel[ws.best_n_ops.cpu().numpy()[sel] > 0]
    contigs = contig_table(begin[al[::40], 0].astype(np.int64) + 30)
    names = nb.numbered_names(n, "r")
    f = nb.finish_alignments(H.genome, rs, ws.best_ops, ws.best_n_ops, ws.best_begin, ws.best_strand, genome_len=N)
    recs = nb.bam_records(ws, f, rs, contigs, names)
    torch.cuda.synchronize()
    off = recs.offsets.cpu().numpy()
    raw = recs.data[:int(off[-1])].cpu().numpy().tobytes()
    want, n_gapped, stats = check_single(H, ws, mq, f, raw, off, contigs, names, reads, sel, 2, ("single end",))
    assert n_gapped > 0 and stats[1] > 0 and stats[2] > 0   # gapped traces, CIGARs with indels and soft clips were checked
    assert (want["best_pos"] > B30).sum() > 1000
    check_stream(recs, contigs, "single-end stream")
    del recs, f, raw

    # the same call without the per-row array: every output identical
    first = {k: getattr(ws, k).clone() for k in SE_OUT}
    del ws
    gc.collect(); torch.cuda.empty_cache()
    rows = H.fmi.rows
    if rows is None:
        print("layout: the index has no per-row array here; the call without it is the call above", flush=True)
    else:
        H.fmi.rows = None
        try:
            ws2, _ = run_single(H, rs, n)
        finally:
            H.fmi.rows = rows
        for k in SE_OUT:
            assert torch.equal(getattr(ws2, k), first[k]), ("without rows", k)
        del ws2
    del first

    # 4-bit reads with N: sampled and planted reads, ~0.5 % of their symbols N
    four = []
    for r in reads[::16] + [planted[i] for i in range(0, len(planted), 4)]:
        r = r.copy(); r[rng.random(L) < 0.005] = 4; four.append(r)
    lens = np.full(len(four), L, np.uint32)
    rs4 = PackedStringSet.from_symbols(np.concatenate(four), (np.arange(len(four)) * L).astype(np.uint32), lens, bits=4)
    ws4, mq4 = run_single(H, rs4, len(four))
    assert int(ws4.n_hits[0]) == int(ws4.n_hits[1])
    f4 = nb.finish_alignments(H.genome, rs4, ws4.best_ops, ws4.best_n_ops, ws4.best_begin, ws4.best_strand, genome_len=N)
    names4 = nb.numbered_names(len(four), "n")
    recs4 = nb.bam_records(ws4, f4, rs4, contigs, names4)
    torch.cuda.synchronize()
    off4 = recs4.offsets.cpu().numpy()
    raw4 = recs4.data[:int(off4[-1])].cpu().numpy().tobytes()
    check_single(H, ws4, mq4, f4, raw4, off4, contigs, names4, four, np.arange(len(four)), 4, ("4-bit",))


# ---------------------------------------------------------------------------------------------------------------------------------------
# 2. paired end
# ---------------------------------------------------------------------------------------------------------------------------------------
def planted_pairs(g, rng, donors):
    """(mate 1 list, mate 2 list): FR pairs whose rescue windows are clipped at both genome ends, fragments across 2^29, fragments longer
    than max_frag, chimeric pairs that pair at two loci (the random genome has hardly any second-best pair otherwise), and second mates
    taken from other pairs (donors: mate symbols of far-away pairs)"""
    m1, m2 = [], []

    def pair(left, frag, hard, swap):
        fw, rv = g[left:left + L].copy(), rc(g[left + frag - L:left + frag])
        if hard == 1:
            fw = mutate(fw, 0.15, rng)
        elif hard == 2:
            rv = mutate(rv, 0.15, rng)
        a, b = (rv, fw) if swap else (fw, rv)
        m1.append(mutate(a, 0.005, rng)); m2.append(b)
    for k in range(40):
        frag = int(rng.integers(L + 10, 420))
        pair(int(rng.integers(0, 40)), frag, 1, k & 1)               # reverse anchor near 0: its window [end - 500, end) starts below 0
        pair(N - frag - int(rng.integers(0, 40)), frag, 2, k & 1)    # forward anchor near the end: its window runs past the end
        pair(N - frag - int(rng.integers(0, 40)), frag, 0, k & 1)
        pair(B29 - int(rng.integers(20, frag - 20)), frag, k % 3, k & 1)   # across the 2^29 contig boundary
        pair(int(rng.integers(0, N - 2000)), int(rng.integers(520, 1500)), 0, k & 1)   # longer than max_frag
    for _ in range(100):                  # chimeric pairs: each mate is half locus A, half locus B, so both loci pair (a second pair)
        a, b, frag = int(rng.integers(0, N - 1000)), int(rng.integers(0, N - 1000)), int(rng.integers(280, 320))
        m1.append(np.concatenate([g[a:a + L // 2], g[b + L // 2:b + L]]))
        m2.append(rc(np.concatenate([g[a + frag - L:a + frag - L // 2], g[b + frag - L // 2:b + frag]])))
    for d in donors:                                                 # a second mate from another pair
        p, frag = int(rng.integers(0, N - 1000)), int(rng.integers(250, 450))
        m1.append(mutate(g[p:p + L], 0.005, rng)); m2.append(d)
    return m1, m2


def pair_outputs(ws, keys):
    torch.cuda.synchronize()
    return {k: getattr(ws, k).clone() for k in keys}


def test_paired_chain(H):
    rng = np.random.default_rng(500)
    dev = H.genome.device
    nbp = 500_000
    bw, _, _ = synth.sample_pairs(H.genome, N, nbp, L, frag_mean=350.0, frag_sd=30.0, sub_rate=0.01, hard_frac=0.05, hard_sub_rate=0.2,
                                  device=dev, seed=0x51ED, mut_seed=0xC0FFEE)        # bench.paired_end_config's batch, rank 0
    wpr = bw.shape[1]
    hw = bw.cpu().numpy()
    donors = [unpack_rows(hw[nbp + i:nbp + i + 1])[0] for i in range(1000, 1060)]
    p1, p2 = planted_pairs(H.g, rng, donors)
    n_pl = len(p1)
    words = torch.cat([bw[:nbp], pack_rows(p1, wpr).to(dev), bw[nbp:], pack_rows(p2, wpr).to(dev)]).contiguous()
    NP = nbp + n_pl
    rs = PackedStringSet.fixed(words.reshape(-1), 2 * NP, L, stride=wpr * 16)
    p = params()
    pair = nb.PairParams(min_frag=0, max_frag=500, min_mate_score=80)
    mq = MapqParams.local(L)
    ws = nb.seed_extend_paired(H.fmi, H.genome, rs, p, pair, hit_capacity=24 * 2 * NP, mapq=mq, traceback=True)
    torch.cuda.synchronize()
    kept, total, jobs = [int(v) for v in ws.n_hits.cpu()]
    run, wanted = [int(v) for v in ws.n_rescue.cpu()]
    flags = ws.pair_flags.cpu().numpy()
    print("paired: %d pairs, %d hits kept of %d, %d scored alignments, resident grid %d threads; rescue jobs run %d of %d wanted; "
          "flags %s" % (NP, kept, total, jobs, H.grid, run, wanted, np.bincount(flags, minlength=5).tolist()), flush=True)
    assert kept == total and run == wanted
    assert jobs > H.grid

    # the sample: every 64th pair, every planted pair, up to GROUP rescued and GROUP unpaired pairs
    resc = np.flatnonzero((flags == 2) | (flags == 4))
    unp = np.flatnonzero(flags == 0)
    sel = np.unique(np.concatenate([np.arange(0, NP, 64), np.arange(nbp, NP), spread(resc, GROUP), spread(unp, GROUP)]))
    ns = len(sel)
    hwords = words.cpu().numpy()
    reads = [unpack_rows(hwords[m * NP + q:m * NP + q + 1])[0] for m in range(2) for q in sel]
    t = torch.from_numpy(sel).cuda()
    rows = np.concatenate([sel, NP + sel])
    tr = torch.from_numpy(rows).cuda()
    t0 = time.perf_counter()
    ms = mq.min_score.cpu().numpy()
    want = pair_mapq_oracle(H.O, H.idx, H.g, reads, p, pair, ns, ms, mq.match_bonus)
    u32 = ("mate_pos", "second_mate_pos")
    got = {}
    for k in ("pair_score", "pair_flags", "second_pair_score"):
        got[k] = getattr(ws, k)[t].cpu().numpy().astype(np.int64)
    for k in ("mate_score", "mate_pos", "mate_strand", "second_mate_pos", "second_mate_strand", "mate_second_score", "mate_mapq"):
        v = getattr(ws, k)[:, t].cpu().numpy()
        got[k] = (v.view(np.uint32) if k in u32 else v).astype(np.int64)
    assert_same(got, {k: want[k] for k in got}, sel, ("paired",))
    fl = want["pair_flags"]
    n_second = int((want["second_pair_score"] != INT_MIN).sum())
    print("paired sample: %d pairs, flags %s, %d with a second pair; oracle %.0f s" % (ns, np.bincount(fl, minlength=5).tolist(), n_second,
                                                                                       time.perf_counter() - t0), flush=True)
    assert (fl == 1).sum() > 0 and ((fl == 2) | (fl == 4)).sum() > 100 and (fl == 0).sum() > 0 and n_second >= 50

    # mate traces: a mate keeping its own best = the banded traceback of its best job; a rescued mate = the full-matrix traceback of its
    # rescue job; every aligned mate's ops replay to its score and end
    se = seed_extend_oracle(H.O, H.idx, H.g, reads, p)
    bh = best_hits(se, 2 * ns)
    mn = ws.mate_n_ops.reshape(-1)[tr].cpu().numpy().astype(np.int64)
    mops = ws.mate_ops.reshape(2 * NP, -1)[tr].cpu().numpy()
    mbeg = host_u32(ws.mate_begin.reshape(2 * NP, 2)[tr]).astype(np.int64)
    mstrand = got["mate_strand"].reshape(-1)
    mscore, mpos = got["mate_score"].reshape(-1), got["mate_pos"].reshape(-1)
    rescued = np.zeros(2 * ns, bool)
    rescued[np.flatnonzero(fl == 2)] = True
    rescued[ns + np.flatnonzero(fl == 4)] = True
    own = np.flatnonzero(~rescued & (bh >= 0))
    lost = np.flatnonzero(~rescued & (bh < 0))
    assert (mn[lost] == 0).all() and (mbeg[lost] == NONE).all()
    h = bh[own]
    st = se["hit_string"][h] % 2
    wn, wo, wb = banded_traceback_of_jobs(H, [reads[r] if s == 0 else rc(reads[r]) for r, s in zip(own, st)], se["hit_window"][h], 2,
                                          ws.max_ops)
    check_traces(mn[own], mops[own], mbeg[own], wn, wo, wb, rows[own], ("paired", "own best"))
    rr = np.flatnonzero(rescued)
    pats, t_off, t_len = [], [], []
    for r in rr:
        a = r + ns if r < ns else r - ns                             # the anchor: the other mate of the pair
        hb = bh[a]
        ae = int(se["hit_window"][hb][0] + se["hit_sink"][hb][0])
        ast = int(se["hit_string"][hb] % 2)
        if ast == 0:
            to = max(ae - len(reads[a]), 0); te = min(to + pair.max_frag, N)
        else:
            to, te = max(ae - pair.max_frag, 0), ae
        pats.append(strand_string(reads[r], np.zeros(L, np.uint8), 1 - ast)[0])
        t_off.append(to); t_len.append(te - to)
    lens = np.full(len(pats), L, np.uint32)
    P = PackedStringSet.from_symbols(np.concatenate(pats), (np.arange(len(pats)) * L).astype(np.uint32), lens, bits=2)
    T = PackedStringSet(words=H.genome, bits=2, big_endian=True, offsets=dev_u32(t_off), lengths=dev_u32(t_len), stride=0,
                        length=int(max(t_len)), count=len(pats))
    fm = aln.batch_alignment_traceback(aln.make_gotoh_aligner(aln.LOCAL, p.scheme), P, T, max_ops=ws.max_ops)
    torch.cuda.synchronize()
    src, snk = host_u32(fm["source"]).astype(np.int64), host_u32(fm["sink"]).astype(np.int64)
    t_off = np.array(t_off, np.int64)
    assert np.array_equal(fm["score"].cpu().numpy().astype(np.int64), mscore[rr])
    assert np.array_equal(t_off + snk[:, 0], mpos[rr])
    check_traces(mn[rr], mops[rr], mbeg[rr], host_u32(fm["n_ops"]).astype(np.int64), fm["ops"].cpu().numpy(),
                 np.stack([t_off + src[:, 0], src[:, 1]], axis=1), rows[rr], ("paired", "rescued"))
    clipped = int(sum((t_off[i] == 0) or (t_off[i] + t_len[i] == N) for i in range(len(rr))))
    for r in np.flatnonzero(mpos != NONE):
        pat, _ = strand_string(reads[r], np.zeros(L, np.uint8), int(mstrand[r]))
        assert replay(mops[r], mn[r], mbeg[r], pat, None, H.g, p.scheme) == (int(mscore[r]), int(mpos[r])), int(rows[r])
    print("paired traces: %d own best, %d rescued (%d windows clipped at a genome end), %d without an alignment" %
          (len(own), len(rr), clipped, len(lost)), flush=True)
    assert clipped > 0

    # finish and paired BAM records (records 2q and 2q + 1 of pair q)
    f = nb.finish_alignments(H.genome, rs, ws.mate_ops, ws.mate_n_ops, ws.mate_begin, ws.mate_strand, genome_len=N)
    torch.cuda.synchronize()
    stats = check_device(sliced_finish(f, tr), reads, mstrand, mops, mn, mbeg, H.g, N)
    al = rows[mn > 0]
    contigs = contig_table(mbeg[mn > 0][::40, 0] + 30)
    names = nb.numbered_names(NP, "p")
    recs = nb.bam_records(ws, f, rs, contigs, names)
    torch.cuda.synchronize()
    off = recs.offsets.cpu().numpy()
    raw = recs.data[:int(off[-1])].cpu().numpy().tobytes()
    inp = dict(reads=reads, quals=None, n_ops=mn.astype(np.uint32), begin=mbeg.astype(np.uint32), strand=mstrand.astype(np.uint8),
               cigar=host_u32(f.cigar[tr]), n_cigar=host_u32(f.n_cigar[tr]), md=f.md[tr].cpu().numpy(), md_len=host_u32(f.md_len[tr]),
               edits=host_u32(f.edits[tr]), score=mscore.astype(np.int32), mapq=got["mate_mapq"].reshape(-1).astype(np.uint8),
               second=got["mate_second_score"].reshape(-1).astype(np.int32), pair_flags=fl.astype(np.uint32),
               contig_begin=contigs.begin, contig_names=contigs.names, contig_lengths=list(contigs.lengths), names=[names[q] for q in sel])
    rec_index = np.stack([2 * sel, 2 * sel + 1], axis=1).reshape(-1)
    cnt = check_records(raw, off, rec_index, inp, ("paired", "bam"))
    print("paired finish %s, records %s, %d aligned mates sampled" % (stats.tolist(), cnt, len(al)), flush=True)
    check_stream(recs, contigs, "paired stream")
    del recs, f, raw

    # bench's own rescue capacity: identical outputs when every wanted job fits, otherwise reported
    first = pair_outputs(ws, PAIR_KEYS + MAPQ_KEYS + TB_KEYS)
    del ws
    gc.collect(); torch.cuda.empty_cache()
    cap = max(NP // 4, 1024)
    if wanted <= cap:
        capped = nb.PairParams(min_frag=0, max_frag=500, min_mate_score=80, rescue_capacity=cap)
        ws2 = nb.seed_extend_paired(H.fmi, H.genome, rs, p, capped, hit_capacity=24 * 2 * NP, mapq=mq, traceback=True)
        for k in first:
            assert torch.equal(getattr(ws2, k), first[k]), ("rescue capacity", k)
        del ws2
        print("rescue capacity %d (bench's): %d wanted fit, outputs identical" % (cap, wanted), flush=True)
    else:
        print("rescue capacity %d (bench's) is below the %d jobs wanted: bench's timed configuration drops rescues" % (cap, wanted),
              flush=True)
    gc.collect(); torch.cuda.empty_cache()

    # the streaming API (nvb_pipeline, paired, bench's shape at depth 2) returns the direct call's pair outputs
    st = nb.StreamingSeedExtend(H.fmi, H.genome, p, 2 * NP, L, wpr, hit_capacity=24 * 2 * NP, depth=2, pair=pair)
    try:
        res = {k: v.clone() for k, v in st.result(st.submit(words.cpu().pin_memory())).items()}
    finally:
        st.close()
    for k in PAIR_KEYS:
        assert torch.equal(res[k].reshape(first[k].shape), first[k].cpu()), ("streaming", k)
