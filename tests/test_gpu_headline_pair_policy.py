"""-m gpu: the paired chain at the genome and batch size bench.py times, under a pairing policy other than FR.  test_gpu_headline_chain.py's
paired test runs FR with min_frag 0; here bench's paired batch is generated in RF (synth.sample_pairs(..., orientation="rf")) and mapped
under RF with min_frag 200, --no-overlap, discordant pairs and --no-mixed, plus planted RF pairs whose rescue windows are clipped at 0 and
at the genome's end (1.9e9).  Sampled pairs against pair_policy_oracle.pair_mapq_oracle; mate traces against the banded traceback of
the mate's own best job or the full-matrix traceback of its RF rescue window, replayed to their score and end; paired BAM records,
discordant pairs included, against bam_oracle; sort, BGZF and BAI of the whole stream.  nvb_pipeline refuses discordant pairs, so the
streaming API runs without them and returns the direct call's outputs.  The fixture (the 1.9 Gbp index) needs an 80 GB part."""
import gc
import time

import numpy as np
import pytest
import torch

import nvbio_b200 as nb
from nvbio_b200 import aln, synth
from nvbio_b200.pipeline import MapqParams
from nvbio_b200.strings import PackedStringSet
from tests import pair_policy_oracle as ppo
from tests.gpu_util import host_u32
from tests.pipeline_oracle import seed_extend_oracle, best_hits
from tests.test_gpu_finish import check_device
from tests.test_gpu_paired_traceback import strand_string, replay, PAIR_KEYS
from tests.test_gpu_pair_policy_edges import mates
from tests.test_gpu_headline_chain import (H, N, L, GROUP, INT_MIN, NONE, params, rc, mutate, pack_rows, unpack_rows, spread, dev_u32,  # noqa: F401
                                           contig_table, assert_same, banded_traceback_of_jobs, check_traces, sliced_finish, check_records,
                                           check_stream)

pytestmark = pytest.mark.gpu

POLICY = "rf"


def planted_pairs(g, rng):
    """RF pairs at both genome ends, either mate first: the mate nearest the end 15 % substituted, so that the other anchors a window
    clipped at 0 (a left window) or at N (a right one); exact pairs on fragments of 300 (the shortest --no-overlap allows for 150 bp
    mates) and of max_frag; mates of two far-apart loci (discordant: bench's batch has no unpaired pair) and mates whose other mate is
    found nowhere (unpaired, reported unaligned under --no-mixed)"""
    m1, m2 = [], []
    for k in range(80):
        odd = k & 1
        frag = int(rng.integers(320, 480))
        for left, hard in ((int(rng.integers(0, 40)), "left"), (N - frag - int(rng.integers(0, 40)), "right")):
            (a, b), lm = mates(g, POLICY, odd, left, frag, (L, L))
            pair = [mutate(a, 0.005, rng), mutate(b, 0.005, rng)]
            h = lm if hard == "left" else 1 - lm
            pair[h] = mutate(pair[h], 0.15, rng)
            m1.append(pair[0]); m2.append(pair[1])
    for frag in (300, 500) * 10:
        (a, b), _ = mates(g, POLICY, len(m1) & 1, int(rng.integers(0, N - 1000)), frag, (L, L))
        m1.append(a); m2.append(b)
    for k in range(150):
        (a, b), _ = mates(g, POLICY, k & 1, int(rng.integers(0, N - 1000)), 350, (L, L))
        q = int(rng.integers(0, N - 1000))
        far = g[q:q + L] if k & 2 else rc(g[q:q + L])
        m1.append(mutate(a, 0.005, rng)); m2.append(mutate(far, 0.005, rng) if k < 100 else rng.integers(0, 4, L).astype(np.uint8))
    return m1, m2


def test_rf_paired_chain(H):
    rng = np.random.default_rng(501)
    dev = H.genome.device
    nbp = 500_000
    bw, _, _ = synth.sample_pairs(H.genome, N, nbp, L, frag_mean=350.0, frag_sd=30.0, sub_rate=0.01, hard_frac=0.05, hard_sub_rate=0.2,
                                  device=dev, seed=0x51ED, mut_seed=0xC0FFEE, orientation=POLICY)   # bench's paired batch, read in RF
    wpr = bw.shape[1]
    p1, p2 = planted_pairs(H.g, rng)
    n_pl = len(p1)
    words = torch.cat([bw[:nbp], pack_rows(p1, wpr).to(dev), bw[nbp:], pack_rows(p2, wpr).to(dev)]).contiguous()
    del bw
    NP = nbp + n_pl
    rs = PackedStringSet.fixed(words.reshape(-1), 2 * NP, L, stride=wpr * 16)
    p = params()
    pair = nb.PairParams(min_frag=200, max_frag=500, min_mate_score=80, policy=POLICY, overlap=False, discordant=True, mixed=False)
    mq = MapqParams.local(L)
    t0 = time.perf_counter()
    ws = nb.seed_extend_paired(H.fmi, H.genome, rs, p, pair, hit_capacity=24 * 2 * NP, mapq=mq, traceback=True)
    torch.cuda.synchronize()
    kept, total, _ = [int(v) for v in ws.n_hits.cpu()]
    run, wanted = [int(v) for v in ws.n_rescue.cpu()]
    flags = ws.pair_flags.cpu().numpy()
    print("\nrf paired: %d pairs, %d hits kept of %d; rescue jobs %d of %d; flags %s; %.1f s" %
          (NP, kept, total, run, wanted, np.bincount(flags, minlength=9).tolist(), time.perf_counter() - t0), flush=True)
    assert kept == total and run == wanted
    assert (flags == nb.PAIR_CONCORDANT).mean() > 0.8

    # the sample: every 128th pair, every planted pair, up to GROUP rescued, discordant and unpaired pairs
    groups = dict(rescued=np.flatnonzero((flags == 2) | (flags == 4)), discordant=np.flatnonzero(flags == nb.PAIR_DISCORDANT),
                  unpaired=np.flatnonzero(flags == 0))
    sel = np.unique(np.concatenate([np.arange(0, NP, 128), np.arange(nbp, NP)] + [spread(v, GROUP) for v in groups.values()]))
    ns = len(sel)
    hwords = words.cpu().numpy()
    reads = [unpack_rows(hwords[m * NP + q:m * NP + q + 1])[0] for m in range(2) for q in sel]
    t = torch.from_numpy(sel).cuda()
    rows = np.concatenate([sel, NP + sel])
    tr = torch.from_numpy(rows).cuda()
    t0 = time.perf_counter()
    want = ppo.pair_mapq_oracle(H.O, H.idx, H.g, reads, p, pair, ns, mq.min_score.cpu().numpy(), mq.match_bonus)
    got = {k: getattr(ws, k)[t].cpu().numpy().astype(np.int64) for k in ("pair_score", "pair_flags", "second_pair_score")}
    for k in ("mate_score", "mate_pos", "mate_strand", "second_mate_pos", "second_mate_strand", "mate_second_score", "mate_mapq"):
        v = getattr(ws, k)[:, t].cpu().numpy()
        got[k] = (v.view(np.uint32) if k in ("mate_pos", "second_mate_pos") else v).astype(np.int64)
    assert_same(got, {k: np.asarray(want[k], np.int64) for k in got}, sel, ("rf paired",))
    fl = got["pair_flags"]
    n_second = int((got["second_pair_score"] != INT_MIN).sum())
    print("rf sample: %d pairs, flags %s, %d with a second pair; oracle %.0f s" % (ns, np.bincount(fl, minlength=9).tolist(), n_second,
                                                                                   time.perf_counter() - t0), flush=True)
    assert (fl == 1).sum() > 0 and ((fl == 2) | (fl == 4)).sum() > 100 and (fl == 0).sum() > 0 and (fl == 8).sum() > 0

    # mate traces: a mate keeping its own best = the banded traceback of its best job; a rescued mate = the full-matrix traceback of its
    # RF rescue window (strand of the policy); --no-mixed mates: none; every aligned mate's ops replay to its score and end
    se = seed_extend_oracle(H.O, H.idx, H.g, reads, p)
    bh = best_hits(se, 2 * ns)
    mn = ws.mate_n_ops.reshape(-1)[tr].cpu().numpy().astype(np.int64)
    mops = ws.mate_ops.reshape(2 * NP, -1)[tr].cpu().numpy()
    mbeg = host_u32(ws.mate_begin.reshape(2 * NP, 2)[tr]).astype(np.int64)
    mstrand, mscore, mpos = got["mate_strand"].reshape(-1), got["mate_score"].reshape(-1), got["mate_pos"].reshape(-1)
    rescued = np.zeros(2 * ns, bool)
    rescued[np.flatnonzero(fl == 2)] = True
    rescued[ns + np.flatnonzero(fl == 4)] = True
    placed = mpos != NONE
    own = np.flatnonzero(~rescued & placed)
    assert (mn[~placed] == 0).all() and (mbeg[~placed] == NONE).all()
    assert (bh[own] >= 0).all()
    h = bh[own]
    st = se["hit_string"][h] % 2
    wn, wo, wb = banded_traceback_of_jobs(H, [reads[r] if s == 0 else strand_string(reads[r], np.zeros(L, np.uint8), 1)[0]
                                              for r, s in zip(own, st)], se["hit_window"][h], 2, ws.max_ops)
    check_traces(mn[own], mops[own], mbeg[own], wn, wo, wb, rows[own], ("rf paired", "own best"))
    rr = np.flatnonzero(rescued)
    pats, t_off, t_len = [], [], []
    for r in rr:
        a = r + ns if r < ns else r - ns                             # the anchor: the other mate of the pair
        hb = bh[a]
        ae = int(se["hit_window"][hb][0] + se["hit_sink"][hb][0])
        to, te, ot = ppo.rescue_window(POLICY, False, 0 if a < ns else 1, int(se["hit_string"][hb] % 2), max(ae - L, 0), ae, pair.max_frag, N)
        assert mstrand[r] == ot
        pats.append(strand_string(reads[r], np.zeros(L, np.uint8), ot)[0])
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
                 np.stack([t_off + src[:, 0], src[:, 1]], axis=1), rows[rr], ("rf paired", "rescued"))
    clip0 = int((t_off == 0).sum())
    clipN = int((t_off + np.array(t_len) == N).sum())
    for r in np.flatnonzero(placed):
        pat, _ = strand_string(reads[r], np.zeros(L, np.uint8), int(mstrand[r]))
        assert replay(mops[r], mn[r], mbeg[r], pat, None, H.g, p.scheme) == (int(mscore[r]), int(mpos[r])), int(rows[r])
    print("rf traces: %d own best, %d rescued (windows clipped: %d at 0, %d at the end)" % (len(own), len(rr), clip0, clipN), flush=True)
    assert clip0 > 0 and clipN > 0

    # finish and paired BAM records, discordant pairs included, against the oracle
    f = nb.finish_alignments(H.genome, rs, ws.mate_ops, ws.mate_n_ops, ws.mate_begin, ws.mate_strand, genome_len=N)
    torch.cuda.synchronize()
    check_device(sliced_finish(f, tr), reads, mstrand, mops, mn, mbeg, H.g, N)
    contigs = contig_table(mbeg[mn > 0][::40, 0] + 30)
    names = nb.numbered_names(NP, "q")
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
    cnt = check_records(raw, off, rec_index, inp, ("rf paired", "bam"))
    disc_recs = 0
    for i, k in enumerate(rec_index):
        flag = int.from_bytes(raw[off[k] + 18:off[k] + 20], "little")
        if fl[i // 2] == nb.PAIR_DISCORDANT and not flag & 0xC:
            assert flag & 0x1 and not flag & 0x2
            disc_recs += 1
    print("rf records %s, %d discordant records with both mates placed" % (cnt, disc_recs), flush=True)
    assert disc_recs > 0
    check_stream(recs, contigs, "rf paired stream")
    del recs, f, raw, ws
    gc.collect(); torch.cuda.empty_cache()

    # the streaming API (nvb_pipeline, paired, depth 2) without discordant pairs returns the direct call's outputs
    plain = nb.PairParams(min_frag=200, max_frag=500, min_mate_score=80, policy=POLICY, overlap=False, mixed=False)
    direct = nb.seed_extend_paired(H.fmi, H.genome, rs, p, plain, hit_capacity=24 * 2 * NP)
    torch.cuda.synchronize()
    first = {k: getattr(direct, k).cpu() for k in PAIR_KEYS}
    del direct
    gc.collect(); torch.cuda.empty_cache()
    st = nb.StreamingSeedExtend(H.fmi, H.genome, p, 2 * NP, L, wpr, hit_capacity=24 * 2 * NP, depth=2, pair=plain)
    try:
        res = {k: v.clone() for k, v in st.result(st.submit(words.cpu().pin_memory())).items()}
    finally:
        st.close()
    for k in PAIR_KEYS:
        assert torch.equal(res[k].reshape(first[k].shape), first[k]), ("streaming", k)
    f2 = first["pair_flags"].numpy()
    assert (f2 == 0).sum() > 0 and not (f2 == nb.PAIR_DISCORDANT).any()
