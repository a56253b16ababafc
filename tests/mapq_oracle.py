"""Restatement of the second-best / MAPQ outputs of nvb_seed_extend_mapq (test infrastructure): nvBowtie's BowtieMapq2
(nvBowtie/bowtie2/cuda/mapq.h:142-331) in numpy float32, and the second-best rule of include/nvbio_b200.h applied to the per-hit
outputs of the oracle composition (tests/pipeline_oracle.py)."""
import numpy as np
from tests.pipeline_oracle import best_hits, EMPTY_SINK

INT_MIN = -2**31


def bowtie_mapq2(best, has_second, second, length, match_bonus, min_score):
    """BowtieMapq2 of unpaired reads, vectorised: the reference's float32 operations in the same order (arrays broadcast)"""
    best, has, second, length, bonus, ms = np.broadcast_arrays(np.asarray(best, np.int64), np.asarray(has_second) != 0,
                                                               np.asarray(second, np.int64), np.asarray(length, np.int64),
                                                               np.asarray(match_bonus, np.int64), np.asarray(min_score, np.int64))
    f32 = np.float32
    max_s = (length * bonus).astype(np.int32).astype(f32)
    min_s = ms.astype(np.int32).astype(f32)
    diff = max_s - min_s
    b = best.astype(np.int32).astype(f32)
    bo = b - min_s
    top = bo == diff
    bd = np.abs(np.abs(b) - np.abs(second.astype(np.int32).astype(f32)))

    def over(c):
        return bo >= diff * f32(c)

    def dif(c):
        return bd >= diff * f32(c)

    def w(c, x, y):
        return np.where(c, x, y)

    e2e_one = np.select([over(0.8), over(0.7), over(0.6), over(0.5), over(0.4), over(0.3)], [42, 40, 24, 23, 8, 3], 0)
    e2e_two = np.select(
        [dif(0.9), dif(0.8), dif(0.7), dif(0.6), dif(0.5), dif(0.4), dif(0.3), dif(0.2), dif(0.1), bd > 0],
        [w(top, 39, 33), w(top, 38, 27), w(top, 37, 26), w(top, 36, 22),
         w(top, 35, w(over(0.84), 25, w(over(0.68), 16, 5))),
         w(top, 34, w(over(0.84), 21, w(over(0.68), 14, 4))),
         w(top, 32, w(over(0.88), 18, w(over(0.67), 15, 3))),
         w(top, 31, w(over(0.88), 17, w(over(0.67), 11, 0))),
         w(top, 30, w(over(0.88), 12, w(over(0.67), 7, 0))),
         w(over(0.67), 6, 2)],
        w(over(0.67), 1, 0))
    loc_one = np.select([over(0.8), over(0.7), over(0.6), over(0.5), over(0.4), over(0.3)], [44, 42, 41, 36, 28, 24], 22)
    loc_two = np.select(
        [dif(0.9), dif(0.8), dif(0.7), dif(0.6), dif(0.5), dif(0.4), dif(0.3), dif(0.2), dif(0.1), bd > 0],
        [40, 39, 38, 37,
         w(top, 35, w(over(0.5), 25, 20)), w(top, 34, w(over(0.5), 21, 19)), w(top, 33, w(over(0.5), 18, 16)),
         w(top, 32, w(over(0.5), 17, 12)), w(top, 31, w(over(0.5), 14, 9)), w(over(0.5), 11, 2)],
        w(over(0.5), 1, 0))
    q = np.where(bonus == 0, np.where(has, e2e_two, e2e_one), np.where(has, loc_two, loc_one))
    return np.where(b < min_s, 0, q).astype(np.uint8)


def distinct(p, t, bp, bt, length):
    """io::distinct_alignments(p, t, bp, bt, len/2) in uint32 arithmetic"""
    d = length // 2
    return t != bt or p < bp - min(bp, d) or p > ((bp + d) & 0xFFFFFFFF)


def mapq_oracle(se, lengths, strands, min_score, match_bonus):
    """se: seed_extend_oracle's result; lengths: read lengths; min_score: the table (index = read length).  Returns dict of
    best_score, best_pos, best_strand, second_score, second_pos, second_strand, mapq (int64 arrays, one entry per read)."""
    n = len(lengths)
    hs, score = se["hit_string"], se["hit_score"]
    end = se["hit_window"][:, 0] + se["hit_sink"][:, 0] if len(hs) else np.zeros(0, np.int64)
    best_h = best_hits(se, n, strands)
    out = {k: np.zeros(n, np.int64) for k in ("best_score", "best_pos", "best_strand", "second_score", "second_pos", "second_strand")}
    out["best_score"][:] = INT_MIN; out["best_pos"][:] = 0xFFFFFFFF
    out["second_score"][:] = INT_MIN; out["second_pos"][:] = 0xFFFFFFFF
    for r in range(n):
        if best_h[r] >= 0:
            b = best_h[r]
            out["best_score"][r], out["best_pos"][r], out["best_strand"][r] = score[b], end[b], int(hs[b]) % strands
    second_h = np.full(n, -1, np.int64)
    for h, s in enumerate(hs):
        r = int(s) // strands
        ln = int(lengths[r])
        if se["hit_sink"][h][0] == EMPTY_SINK or score[h] < min_score[ln] or not distinct(int(end[h]), int(s) % strands, int(out["best_pos"][r]), int(out["best_strand"][r]), ln):
            continue
        if second_h[r] < 0 or score[h] > score[second_h[r]]:
            second_h[r] = h
    for r in range(n):
        if second_h[r] >= 0:
            h = second_h[r]
            out["second_score"][r], out["second_pos"][r], out["second_strand"][r] = score[h], end[h], int(hs[h]) % strands
    lengths = np.asarray(lengths, np.int64)
    has = second_h >= 0
    out["mapq"] = bowtie_mapq2(out["best_score"], has, np.where(has, out["second_score"], 0), lengths, match_bonus,
                               np.asarray(min_score, np.int64)[lengths]).astype(np.int64)
    return out
