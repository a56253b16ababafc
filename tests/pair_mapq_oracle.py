"""Restatement of the second-best pair and paired MAPQ of nvb_seed_extend_paired_mapq (test infrastructure): the rule of
include/nvbio_b200.h by brute force over every combination of the mates' candidates (no merging, no search), applied to the oracle
composition of the paired stage (tests/pipeline_oracle.py) and nvBowtie's BowtieMapq2 restated in tests/mapq_oracle.py."""
import numpy as np
from tests.mapq_oracle import bowtie_mapq2, mapq_oracle, INT_MIN
from tests.pipeline_oracle import seed_extend_oracle, seed_extend_paired_oracle, _scheme_args, best_hits, EMPTY_SINK

NONE_TIE = 0xFFFFFFFF


def _distinct(p, t, bp, bt, length):
    """io::distinct_alignments (mapq_oracle.distinct) over arrays"""
    d = length // 2
    return (t != bt) | (p < bp - min(bp, d)) | (p > ((bp + d) & 0xFFFFFFFF))


def second_pair(c1, c2, len1, len2, star, min_frag, max_frag, rescues=()):
    """c1 / c2: mate 1's / mate 2's candidates (score, strand, end, tie), already at or above the min score; star = ((end, strand) of P*'s
    mate 1, of its mate 2); rescues: (anchor mate, pair score, anchor end, anchor strand, anchor tie, rescued end).  Every combination of
    one candidate of each mate is tested (no merging, no search).  Returns (score, ((end1, strand1), (end2, strand2))) of the second-best
    pair, or None."""
    A = np.array(c1, np.int64).reshape(-1, 4)[:, None, :]
    B = np.array(c2, np.int64).reshape(-1, 4)[None, :, :]
    e1, t1, e2, t2 = A[..., 2], A[..., 1], B[..., 2], B[..., 1]
    b1, b2 = np.where(e1 > len1, e1 - len1, 0), np.where(e2 > len2, e2 - len2, 0)
    fw1 = t1 == 0
    fb, fe, rb, re_ = np.where(fw1, b1, b2), np.where(fw1, e1, e2), np.where(fw1, b2, b1), np.where(fw1, e2, e1)
    ok = (t1 != t2) & (fb <= rb) & (fe <= re_) & (re_ > fb) & (re_ - fb >= min_frag) & (re_ - fb <= max_frag)
    ok = np.broadcast_to(ok, (A.shape[0], B.shape[1]))
    i, j = np.nonzero(ok)
    S = (A[i, 0, 0] + B[0, j, 0]).tolist()
    cols = [S, A[i, 0, 3].tolist(), B[0, j, 3].tolist(), A[i, 0, 2].tolist(), A[i, 0, 1].tolist(), B[0, j, 2].tolist(), B[0, j, 1].tolist()]
    for a, sc, ae, at, ai, oe in rescues:
        m1, m2 = ((ae, at, ai), (oe, 1 - at, NONE_TIE)) if a == 0 else ((oe, 1 - at, NONE_TIE), (ae, at, ai))
        for c, v in zip(cols, (sc, m1[2], m2[2], m1[0], m1[1], m2[0], m2[1])):
            c.append(v)
    S, I1, I2, E1, T1, E2, T2 = (np.array(c, np.int64) for c in cols)
    keep = _distinct(E1, T1, star[0][0], star[0][1], len1) | _distinct(E2, T2, star[1][0], star[1][1], len2)
    if not keep.any():
        return None
    k = np.flatnonzero(keep)[np.lexsort((I2[keep], I1[keep], -S[keep]))[0]]
    return int(S[k]), ((int(E1[k]), int(T1[k])), (int(E2[k]), int(T2[k])))


def rescue_jobs(O, idx, genome_sym, reads, params, pair, n_pairs, single, redo, quals=None):
    """every opposite-mate job of the paired stage as the header states it, scored by the oracle's full-matrix Gotoh: (pair, anchor,
    window begin, score, sink.x) of the first rescue_capacity jobs, and the number wanted.  single: the mates' single-end bests
    (mapq_oracle); redo[p]: the pair was not concordant as it stood"""
    jobs = []
    for p in np.flatnonzero(redo):
        for a in range(2):
            ra = a * n_pairs + p
            if single["best_score"][ra] == INT_MIN or single["best_score"][ra] < pair.min_mate_score:
                continue
            end, ln = int(single["best_pos"][ra]), len(reads[ra])
            o = reads[(1 - a) * n_pairs + p]
            oq = quals[(1 - a) * n_pairs + p] if quals is not None else None
            if single["best_strand"][ra] == 0:
                to = max(end - ln, 0); te = min(to + pair.max_frag, idx.n)
                pat, pq = np.where(o < 4, 3 - o, o)[::-1].astype(np.uint8), (oq[::-1] if oq is not None else None)
            else:
                to, te = max(end - pair.max_frag, 0), end
                pat, pq = o, oq
            if te - to >= 1 and len(pat) >= 1:
                jobs.append((int(p), a, pat, to, te - to, pq))
    cap = 2 * n_pairs if pair.rescue_capacity is None else pair.rescue_capacity
    run = jobs[:cap]
    if not run:
        return [], len(jobs)
    p_len = np.array([len(j[2]) for j in run], np.uint32)
    scheme, qtab = _scheme_args(params.scheme)
    rs, rx, _ = O.gotoh_full(params.type, scheme, np.concatenate([j[2] for j in run]), (np.cumsum(p_len) - p_len).astype(np.uint32), p_len,
                             genome_sym, np.array([j[3] for j in run], np.uint32), np.array([j[4] for j in run], np.uint32),
                             qual=np.concatenate([j[5] for j in run]) if quals is not None else None, qtab=qtab)
    return [(p, a, to, int(s), int(x)) for (p, a, _, to, _, _), s, x in zip(run, rs, rx)], len(jobs)


def pair_mapq_oracle(O, idx, genome_sym, reads, params, pair, n_pairs, min_score, match_bonus, quals=None):
    """the oracle composition of every nvb_seed_extend_paired_mapq output (int64 arrays; mates as [2, n_pairs])"""
    pe = seed_extend_paired_oracle(O, idx, genome_sym, reads, params, pair, n_pairs, quals=quals)
    se = seed_extend_oracle(O, idx, genome_sym, reads, params, quals=quals)
    lens = np.array([len(r) for r in reads], np.int64)
    ms = np.asarray(min_score, np.int64)
    single = mapq_oracle(se, lens, 2, ms, match_bonus)
    best_h = best_hits(se, len(reads))                             # every read's best hit (its tie index): max score, then smallest hit
    rescues, wanted = rescue_jobs(O, idx, genome_sym, reads, params, pair, n_pairs, single, pe["pair_flags"] != 1, quals=quals)
    assert (len(rescues), wanted) == tuple(pe["n_rescue"])         # the same jobs as the paired composition ran
    end = se["hit_window"][:, 0] + se["hit_sink"][:, 0] if len(se["hit_string"]) else np.zeros(0, np.int64)
    cands = [[] for _ in reads]
    for h, s in enumerate(se["hit_string"]):
        r = int(s) // 2
        if se["hit_sink"][h][0] != EMPTY_SINK and se["hit_score"][h] >= ms[lens[r]]:
            cands[r].append((int(se["hit_score"][h]), int(s) % 2, int(end[h]), h))
    resc = {}
    for p, a, to, rs, x in rescues:
        if rs >= pair.min_mate_score and rs >= ms[lens[(1 - a) * n_pairs + p]]:
            ra = a * n_pairs + p
            resc.setdefault(p, []).append((a, int(se["hit_score"][best_h[ra]]) + rs, int(single["best_pos"][ra]), int(single["best_strand"][ra]),
                                           int(best_h[ra]), to + x))
    out = dict(pair_score=pe["pair_score"], pair_flags=pe["pair_flags"], mate_score=pe["mate_score"], mate_pos=pe["mate_pos"],
               mate_strand=pe["mate_strand"], n_rescue=pe["n_rescue"],
               second_pair_score=np.full(n_pairs, INT_MIN, np.int64), second_mate_pos=np.full((2, n_pairs), 0xFFFFFFFF, np.int64),
               second_mate_strand=np.zeros((2, n_pairs), np.int64), mate_second_score=single["second_score"].reshape(2, n_pairs),
               mate_mapq=single["mapq"].reshape(2, n_pairs).copy())
    for p in range(n_pairs):
        if pe["pair_flags"][p] == 0:
            continue
        l1, l2 = int(lens[p]), int(lens[n_pairs + p])
        star = ((int(pe["mate_pos"][0, p]), int(pe["mate_strand"][0, p])), (int(pe["mate_pos"][1, p]), int(pe["mate_strand"][1, p])))
        sp = second_pair(cands[p], cands[n_pairs + p], l1, l2, star, pair.min_frag, pair.max_frag, resc.get(p, ()))
        if sp is not None:
            out["second_pair_score"][p] = sp[0]
            for k in range(2):
                out["second_mate_pos"][k, p], out["second_mate_strand"][k, p] = sp[1][k]
        q = bowtie_mapq2(pe["pair_score"][p], sp is not None, sp[0] if sp is not None else 0, l1 + l2, match_bonus, ms[l1] + ms[l2])
        out["mate_mapq"][:, p] = int(q)
    return out
