"""Oracle composition of nvb_seed_extend_reseed (test infrastructure): seed_extend_oracle's primitives (the oracle's FM-index match and
locate, its banded Gotoh) driven round by round with the seed offset, the active set and the flag rule of include/nvbio_b200.h, and
mapq_oracle over the union of the rounds' hits."""
import numpy as np
from tests.pipeline_oracle import EMPTY_SINK, best_hits, _scheme_args
from tests.mapq_oracle import mapq_oracle

INT_MIN = -2**31
U32 = 0xFFFFFFFF


def reseed_offset(r, interval, max_reseed):
    """read offset of round r's first seed: r * floor(I / (max_reseed + 1))"""
    return r * (interval // (max_reseed + 1))


def reseed_flag(range_sum, range_count, rep_seeds, aligned):
    """the flag rule in wrapping uint32 arithmetic: no range, mean range size >= rep_seeds, or no alignment reaching the min score"""
    return range_count == 0 or (range_sum & U32) >= ((rep_seeds * range_count) & U32) or not aligned


def range_stats(ranges, valid):
    """(range_sum, range_count) of one read's seeds: the non-empty SA ranges of its valid seeds, full sizes, uint32 sum"""
    s = c = 0
    for (x, y), v in zip(ranges, valid):
        if v and int(x) <= int(y):
            s = (s + int(y) - int(x) + 1) & U32
            c += 1
    return s, c


def seed_positions(length, K, L, I, o):
    """the seed slots k = 0 .. K-1 of a string of this length in a round with offset o: (start, valid)"""
    return [(o + k * I, o + k * I + L <= length) for k in range(K)]


def _strings(read, q, strands):
    out = [(read, q)]
    if strands == 2:
        out.append((np.where(read < 4, 3 - read, read)[::-1].astype(np.uint8), None if q is None else q[::-1]))
    return out


def seed_extend_reseed_oracle(O, idx, genome_sym, reads, params, max_reseed, rep_seeds, min_score, hit_capacity, match_bonus=None,
                              quals=None):
    """reads: list of uint8 arrays (symbol 4 = N); min_score: the table indexed by read length.  Returns dict of
    rounds (per read), active (per round), stats (per round: dict read -> (range_sum, range_count)), flags (per round: dict read -> bool,
    rounds 0 .. max_reseed - 1), hit_string / hit_window / hit_score / hit_sink / hit_round (the kept hits of all rounds, round-major,
    original string ids), n_hits = (kept, found) and, with match_bonus, mapq_oracle's best / second / MAPQ over the union (else the best)."""
    L, I, B = params.seed_len, params.seed_interval, params.band_len
    strands = 2 if params.both_strands else 1
    n_reads = len(reads)
    max_len = max(len(r) for r in reads)
    K = (max_len - L) // I + 1
    scheme, qtab = _scheme_args(params.scheme)
    lengths = np.array([len(r) for r in reads], np.int64)
    rounds = np.zeros(n_reads, np.int64)
    active_counts, stats_all, flags_all = [], [], []
    hs, hw, hsc, hsk, hround = [], [], [], [], []
    kept_total = found_total = 0
    active = list(range(n_reads))
    for r in range(max_reseed + 1):
        if not active:
            active_counts.append(0); stats_all.append({})
            continue
        active_counts.append(len(active))
        o = reseed_offset(r, I, max_reseed)
        for rd in active:
            rounds[rd] = r + 1
        # seeds of the round's strings in (read, strand, k) order; a seed with an N has an empty range
        q, off, ln, valid, owner = [], [], [], [], []
        pos = 0
        strs = []
        for rd in active:
            for t, (s, sq) in enumerate(_strings(reads[rd], quals[rd] if quals is not None else None, strands)):
                strs.append((rd, t, s, sq))
                for p, v in seed_positions(len(s), K, L, I, o):
                    v = v and bool(np.all(s[p:p + L] < 4))
                    if v:
                        q.append(s[p:p + L]); off.append(pos); ln.append(L); pos += L
                    else:
                        off.append(pos); ln.append(0)
                    valid.append(v); owner.append(len(strs) - 1)
        qcat = np.concatenate(q) if q else np.zeros(1, np.uint8)
        ranges, _ = O.match(idx, qcat, np.array(off, np.uint32), np.array(ln, np.uint32))
        # hits in slot order, the round's capacity what the earlier rounds left
        stats = {rd: [0, 0] for rd in active}
        hits = []                      # (string index into strs, seed start, SA row)
        for qi, ((x, y), v) in enumerate(zip(ranges, valid)):
            si = owner[qi]
            if not v or int(x) > int(y):
                continue
            st = stats[strs[si][0]]
            st[0] = (st[0] + int(y) - int(x) + 1) & U32; st[1] += 1
            k = qi % K
            for j in range(min(int(y) - int(x) + 1, params.max_seed_hits)):
                hits.append((si, o + k * I, int(x) + j))
        found_total += len(hits)
        hits = hits[:max(hit_capacity - kept_total, 0)]
        kept_total += len(hits)
        stats_all.append({rd: tuple(v) for rd, v in stats.items()})
        if hits:
            tpos = O.locate(idx, np.array([h[2] for h in hits], np.uint32))
            p_sym, p_q, p_off, p_len, t_off, t_len = [], [], [], [], [], []
            po = 0
            for (si, sb, _), tp in zip(hits, tpos):
                rd, t, s, sq = strs[si]
                diag = int(tp) - sb if int(tp) > sb else 0
                gb = diag - B // 2 if diag > B // 2 else 0
                ge = min(gb + len(s) + B, idx.n)
                p_sym.append(s); p_off.append(po); p_len.append(len(s)); po += len(s)
                if quals is not None:
                    p_q.append(sq)
                t_off.append(gb); t_len.append(ge - gb)
                hs.append(rd * strands + t); hw.append((gb, ge)); hround.append(r)
            score, sx, sy, _ = O.banded_gotoh(B, params.type, scheme, np.concatenate(p_sym), np.array(p_off, np.uint32),
                                              np.array(p_len, np.uint32), genome_sym, np.array(t_off, np.uint32), np.array(t_len, np.uint32),
                                              qual=np.concatenate(p_q) if quals is not None else None, qtab=qtab)
            hsc.extend(int(v) for v in score); hsk.extend((int(a), int(b)) for a, b in zip(sx, sy))
        if r == max_reseed:
            break
        se = _se(hs, hw, hsc, hsk)
        best_h = best_hits(se, n_reads, strands)
        flags = {}
        for rd in active:
            b = best_h[rd]
            aligned = b >= 0 and se["hit_score"][b] >= min_score[len(reads[rd])]
            flags[rd] = reseed_flag(stats[rd][0], stats[rd][1], rep_seeds, aligned)
        flags_all.append(flags)
        active = [rd for rd in active if flags[rd]]
    se = _se(hs, hw, hsc, hsk)
    out = dict(rounds=rounds, active=np.array(active_counts, np.int64), stats=stats_all, flags=flags_all, hit_string=se["hit_string"],
               hit_window=se["hit_window"], hit_score=se["hit_score"], hit_sink=se["hit_sink"], hit_round=np.array(hround, np.int64),
               n_hits=(kept_total, found_total & U32), best_h=best_hits(se, n_reads, strands))
    if match_bonus is not None:
        out.update(mapq_oracle(se, lengths, strands, np.asarray(min_score, np.int64), match_bonus))
    return out


def _se(hs, hw, hsc, hsk):
    return dict(hit_string=np.array(hs, np.int64), hit_window=np.array(hw, np.int64).reshape(-1, 2), hit_score=np.array(hsc, np.int64),
                hit_sink=np.array(hsk, np.int64).reshape(-1, 2))
