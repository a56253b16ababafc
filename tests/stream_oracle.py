"""TEST INFRASTRUCTURE: the BAM records of a batch of host reads computed by the oracles alone, with no device output in between -- what
the BAM mode of nvb_pipeline (StreamingBam) must return for the batch.  The stage oracles are composed as the device chain composes its
stages:

  - single end: pipeline_oracle.seed_extend_oracle, then mapq_oracle (second best and BowtieMapq2);
  - paired: pair_policy_oracle.pair_mapq_oracle under the pair's policy and options;
  - the winning alignment's ops: the oracle's banded traceback of the read's best job, or for a rescued mate the full-matrix traceback of
    its rescue window (pair_policy_oracle.rescue_window around the anchor's best, the rule tests/test_gpu_paired_traceback.py uses);
  - finish_oracle.finish, then the CIGAR and MD stored up to max_cigar / max_md with their full counts, as nvb_finish_alignments stores
    them, so that bam_oracle marks a truncated record unfinished exactly as the header states;
  - bam_oracle.records.

Each stage oracle reads only what the previous oracle produced, so a hand-off convention the device stages share (op order, begin,
strand, mate order, per-read length, the quality rows) is checked against the header's statement of it, not against itself."""
import numpy as np
from tests import bam_oracle, finish_oracle, pair_policy_oracle, pipeline_oracle
from tests.mapq_oracle import mapq_oracle
from tests.pipeline_oracle import best_hits, _scheme_args

NONE = 0xFFFFFFFF


def _rc(r):
    return np.where(r < 4, 3 - r, r)[::-1].astype(np.uint8)


def _oriented(read, qual, strand):
    """(symbols, qualities) of the strand an alignment is of"""
    if strand == 0:
        return read, qual
    return _rc(read), (qual[::-1] if qual is not None else None)


def _traceback(O, genome_sym, jobs, params, max_ops, full):
    """jobs: (pattern, qualities or None, window begin, window end).  The oracle's banded (or full-matrix) traceback of every job:
    (n_ops, ops END -> START, begin = (genome, pattern) coordinates of the first aligned column, score, genome end)"""
    scheme6, qtab = _scheme_args(params.scheme)
    lens = np.array([len(j[0]) for j in jobs], np.uint32)
    t_off = np.array([j[2] for j in jobs], np.uint32)
    t_len = np.array([j[3] - j[2] for j in jobs], np.uint32)
    args = (np.concatenate([j[0] for j in jobs]), (np.cumsum(lens) - lens).astype(np.uint32), lens, genome_sym, t_off, t_len)
    qual = np.concatenate([j[1] for j in jobs]) if qtab is not None else None
    if full:
        o = O.gotoh_full_traceback(params.type, scheme6, *args, max_ops=max_ops, qual=qual, qtab=qtab)
    else:
        o = O.banded_traceback(params.band_len, params.type, scheme6, *args, max_ops=max_ops, qual=qual, qtab=qtab)
    t = t_off.astype(np.int64)
    begin = np.stack([t + o["source"][:, 0], o["source"][:, 1].astype(np.int64)], axis=1)
    return o["n_ops"].astype(np.int64), o["ops"], begin, o["score"].astype(np.int64), t + o["sink"][:, 0]


def chain(O, idx, genome_sym, reads, lengths, quals, names, params, mapq, pair, contigs, max_ops, max_cigar, max_md):
    """reads: symbols [n, >= length] (paired: mate 1 of every pair, then mate 2); lengths: per-read lengths or None (every row whole);
    quals: base qualities [n, >= length] or None; names: one per read (per pair); params: the SeedExtendParams of the stream (qualities
    score only under a quality table); mapq: its MapqParams; pair: PairParams or None; contigs: a ContigTable; max_ops / max_cigar /
    max_md: the stream's maxima, resolved (no 0).  Returns dict(records = [record bytes], counts = [records, mapped, off-contig,
    unfinished], pair_flags (or None), rescued = the rescued mates' read indices)."""
    n = len(reads)
    lens = np.array([len(r) for r in reads] if lengths is None else lengths, np.int64)
    rd = [np.asarray(reads[i][:lens[i]], np.uint8) for i in range(n)]
    qs = None if quals is None else [np.asarray(quals[i][:lens[i]], np.uint8) for i in range(n)]
    oq = qs if _scheme_args(params.scheme)[1] is not None else None
    ms = mapq.min_score.cpu().numpy().astype(np.int64)
    se = pipeline_oracle.seed_extend_oracle(O, idx, genome_sym, rd, params, quals=oq)
    bh = best_hits(se, n)
    strand = np.zeros(n, np.int64)
    rescued = np.zeros(n, bool)
    if pair is None:
        m = mapq_oracle(se, lens, 2, ms, mapq.match_bonus)
        score, mq, second, flags = m["best_score"], m["mapq"], m["second_score"], None
        own = bh >= 0
    else:
        h = n // 2
        pm = pair_policy_oracle.pair_mapq_oracle(O, idx, genome_sym, rd, params, pair, h, ms, mapq.match_bonus, quals=oq)
        score, mq, second = pm["mate_score"].reshape(-1), pm["mate_mapq"].reshape(-1), pm["mate_second_score"].reshape(-1)
        pos, mstrand, flags = pm["mate_pos"].reshape(-1), pm["mate_strand"].reshape(-1), pm["pair_flags"]
        rescued[np.flatnonzero(flags == 2)] = True
        rescued[h + np.flatnonzero(flags == 4)] = True
        own = (bh >= 0) & ~rescued & (pos != NONE)                  # (--no-mixed reports both mates of an unpaired pair unaligned)
    n_ops = np.zeros(n, np.int64)
    ops = np.zeros((n, max_ops), np.uint8)
    begin = np.full((n, 2), NONE, np.int64)
    rows = np.flatnonzero(own)
    if len(rows):
        hh = bh[rows]
        st = se["hit_string"][hh] % 2
        jobs = [_oriented(rd[r], None if qs is None else qs[r], s) + tuple(se["hit_window"][b]) for r, s, b in zip(rows, st, hh)]
        n_ops[rows], ops[rows], begin[rows], _, _ = _traceback(O, genome_sym, jobs, params, max_ops, False)
        strand[rows] = st
    rr = np.flatnonzero(rescued)
    if len(rr):
        policy, overlap, _, _ = pair_policy_oracle.pair_options(pair)
        jobs, ost = [], []
        for r in rr:
            o, q = divmod(int(r), h)
            a = (1 - o) * h + q                                      # the anchor: the other mate, at its own best
            wb, we, ot = pair_policy_oracle.rescue_window(policy, overlap, 1 - o, int(mstrand[a]), max(int(pos[a]) - int(lens[a]), 0),
                                                          int(pos[a]), pair.max_frag, idx.n)
            jobs.append(_oriented(rd[r], None if qs is None else qs[r], ot) + (wb, we))
            ost.append(ot)
        tn, to, tb, tsc, tend = _traceback(O, genome_sym, jobs, params, max_ops, True)
        assert np.array_equal(tsc, score[rr]) and np.array_equal(tend, pos[rr]), "the rescue traceback is not the pairing's alignment"
        n_ops[rr], ops[rr], begin[rr], strand[rr] = tn, to, tb, ost
    cigar = np.zeros((n, max_cigar), np.uint32)
    n_cigar = np.zeros(n, np.uint32)
    md = np.zeros((n, max_md), np.uint8)
    md_len = np.zeros(n, np.uint32)
    edits = np.zeros((n, 4), np.uint32)
    for r in range(n):
        c, m_, e = finish_oracle.finish(ops[r], n_ops[r], max_ops, begin[r], strand[r], rd[r], genome_sym, idx.n)
        enc = [k << 4 | op for k, op in c][:max_cigar]
        mdb = np.frombuffer(m_.encode(), np.uint8)[:max_md]
        cigar[r, :len(enc)], n_cigar[r] = enc, len(c)
        md[r, :len(mdb)], md_len[r] = mdb, len(m_)
        edits[r] = e
    inp = dict(reads=rd, quals=qs, n_ops=n_ops, begin=begin, strand=strand, cigar=cigar, n_cigar=n_cigar, md=md, md_len=md_len,
               edits=edits, score=score, mapq=mq, second=second, pair_flags=flags, contig_begin=contigs.begin,
               contig_names=contigs.names, names=[nm.decode() if isinstance(nm, bytes) else nm for nm in names])
    out, counts = bam_oracle.records(inp)
    return dict(records=[b for b, _ in out], counts=counts, pair_flags=flags, rescued=rr)


def records(O, idx, genome_sym, reads, lengths, quals, names, params, mapq, pair, contigs, max_ops, max_cigar, max_md):
    """the concatenated BAM record bytes of chain(...)"""
    return b"".join(chain(O, idx, genome_sym, reads, lengths, quals, names, params, mapq, pair, contigs, max_ops, max_cigar,
                          max_md)["records"])
