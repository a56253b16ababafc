"""Oracle composition of the seed+extend pipeline (test infrastructure): the same stages as
nvbio_b200/csrc/pipeline.cu, each stage computed by the CPU oracle / reference library."""
import numpy as np

EMPTY_SINK = 0xFFFFFFFF      # sink.x of a job the banded DP reports empty (window shorter than the read)


def best_hits(se, n_reads, strands=2):
    """every read's best hit (index into se's hits, -1 = none): max score, ties -> smallest hit index; empty jobs are skipped"""
    best_h = np.full(n_reads, -1, np.int64)
    for h, s in enumerate(se["hit_string"]):
        r = int(s) // strands
        if se["hit_sink"][h][0] == EMPTY_SINK:
            continue
        if best_h[r] < 0 or se["hit_score"][h] > se["hit_score"][best_h[r]]:
            best_h[r] = h
    return best_h


def _scheme_args(sch):
    """(scheme tuple, qtab or None) of a SimpleGotohScheme / QualityGotohScheme / a scheme object with separate pattern and text gap
    costs (match, mismatch, pgo, pge, tgo, tge)"""
    if hasattr(sch, "table_host"):
        return (sch.match_bonus, int(sch.table_host[0, 1]), sch.pgo, sch.pge, sch.tgo, sch.tge), sch.table_host
    if hasattr(sch, "tgo"):
        return (sch.match, sch.mismatch, sch.pgo, sch.pge, sch.tgo, sch.tge), None
    return (sch.match, sch.mismatch, sch.gap_open, sch.gap_ext), None


def seed_extend_oracle(O, idx, genome_sym, reads, params, quals=None):
    """reads: list of uint8 arrays; quals: optional list of uint8 arrays (base qualities, with a QualityGotohScheme).
    Returns dict(best_score, best_pos, hit_string, hit_window, hit_score, hit_sink, n_hits)."""
    L, I, B = params.seed_len, params.seed_interval, params.band_len
    n = idx.n
    strands = 2 if params.both_strands else 1
    strings, squals = [], []
    for i, r in enumerate(reads):
        strings.append(r)
        if quals is not None:
            squals.append(quals[i])
        if strands == 2:
            rc = np.where(r < 4, 3 - r, r)[::-1].astype(np.uint8)
            strings.append(rc)
            if quals is not None:
                squals.append(quals[i][::-1])
    max_len = max(len(r) for r in reads)
    K = (max_len - L) // I + 1
    # seeds
    q, off, ln, valid = [], [], [], []
    o = 0
    for s in strings:
        for k in range(K):
            p = k * I
            if p + L <= len(s):
                q.append(s[p:p + L]); off.append(o); ln.append(L); o += L; valid.append(True)
            else:
                off.append(o); ln.append(0); valid.append(False)
    qcat = np.concatenate(q) if q else np.zeros(1, np.uint8)
    ranges, _ = O.match(idx, qcat, np.array(off, np.uint32), np.array(ln, np.uint32))
    hit_string, rows, seed_k = [], [], []
    for qi, ((x, y), v) in enumerate(zip(ranges, valid)):
        if not v or x > y:
            continue
        sz = min(int(y) - int(x) + 1, params.max_seed_hits)
        for j in range(sz):
            hit_string.append(qi // K); seed_k.append(qi % K); rows.append(int(x) + j)
    rows = np.array(rows, np.uint32)
    pos = O.locate(idx, rows) if len(rows) else np.zeros(0, np.uint32)
    p_sym, p_q, p_off, p_len, t_off, t_len, wins = [], [], [], [], [], [], []
    po = 0
    for s, k, p in zip(hit_string, seed_k, pos):
        ln_s = len(strings[s])
        sb = k * I
        diag = int(p) - sb if int(p) > sb else 0
        gb = diag - B // 2 if diag > B // 2 else 0
        ge = min(gb + ln_s + B, n)
        p_sym.append(strings[s]); p_off.append(po); p_len.append(ln_s); po += ln_s
        if quals is not None:
            p_q.append(squals[s])
        t_off.append(gb); t_len.append(ge - gb); wins.append((gb, ge))
    scheme, qtab = _scheme_args(params.scheme)
    if hit_string:
        score, sx, sy, _ = O.banded_gotoh(B, params.type, scheme, np.concatenate(p_sym), np.array(p_off, np.uint32), np.array(p_len, np.uint32),
                                          genome_sym, np.array(t_off, np.uint32), np.array(t_len, np.uint32),
                                          qual=np.concatenate(p_q) if quals is not None else None, qtab=qtab)
    else:
        score = np.zeros(0, np.int32); sx = sy = np.zeros(0, np.uint32)
    best_score = np.full(len(reads), -2**31, np.int64)
    best_pos = np.full(len(reads), 0xFFFFFFFF, np.int64)
    for h, s in enumerate(hit_string):
        r = s // strands
        if int(sx[h]) == EMPTY_SINK:                 # a window shorter than the read: the DP's empty result is not an alignment
            continue
        if int(score[h]) > best_score[r]:
            best_score[r] = int(score[h]); best_pos[r] = t_off[h] + int(sx[h])
    return dict(best_score=best_score, best_pos=best_pos, hit_string=np.array(hit_string, np.int64),
                hit_window=np.array(wins, np.int64).reshape(-1, 2), hit_score=score.astype(np.int64),
                hit_sink=np.stack([sx.astype(np.int64), sy.astype(np.int64)], axis=1) if len(sx) else np.zeros((0, 2), np.int64),
                n_hits=len(hit_string))


def seed_extend_paired_oracle(O, idx, genome_sym, reads, params, pair, n_pairs, quals=None):
    """Oracle composition of nvb_seed_extend_paired: the single-end composition above for the 2*n_pairs mates, the pairing rules of
    include/nvbio_b200.h restated in Python, and the opposite-mate rescue scored by the oracle's full-matrix Gotoh.
    reads: mate 1 of every pair, then mate 2.  Returns dict(pair_score, pair_flags, mate_score[2,n], mate_pos[2,n], mate_strand[2,n],
    n_rescue)."""
    se = seed_extend_oracle(O, idx, genome_sym, reads, params, quals=quals)
    glen = idx.n
    strands = 2
    best_h = best_hits(se, len(reads), strands)
    INT_MIN = -2**31

    def mate(r):
        h = best_h[r]
        if h < 0:
            return dict(has=False, score=INT_MIN, strand=0, beg=0xFFFFFFFF, end=0xFFFFFFFF, len=0)
        s = int(se["hit_string"][h])
        ln = len(reads[r])
        end = int(se["hit_window"][h][0] + se["hit_sink"][h][0])
        return dict(has=True, score=int(se["hit_score"][h]), strand=s % strands, beg=max(end - ln, 0), end=end, len=ln)

    cap = 2 * n_pairs if pair.rescue_capacity is None else pair.rescue_capacity
    pair_score = np.full(n_pairs, INT_MIN, np.int64); pair_flags = np.zeros(n_pairs, np.int64)
    mate_score = np.full((2, n_pairs), INT_MIN, np.int64); mate_pos = np.full((2, n_pairs), 0xFFFFFFFF, np.int64)
    mate_strand = np.zeros((2, n_pairs), np.int64)
    jobs = []          # (pair, anchor, pattern symbols, window begin, window length)
    for p in range(n_pairs):
        m = [mate(p), mate(n_pairs + p)]
        for k in range(2):
            mate_score[k, p], mate_pos[k, p], mate_strand[k, p] = m[k]["score"], m[k]["end"], m[k]["strand"]
        conc = m[0]["has"] and m[1]["has"] and m[0]["strand"] != m[1]["strand"]
        if conc:
            f, r = (m[0], m[1]) if m[0]["strand"] == 0 else (m[1], m[0])
            frag = r["end"] - f["beg"]
            conc = f["beg"] <= r["beg"] and f["end"] <= r["end"] and r["end"] > f["beg"] and pair.min_frag <= frag <= pair.max_frag
        if conc:
            pair_score[p] = m[0]["score"] + m[1]["score"]; pair_flags[p] = 1
            continue
        for a in range(2):
            if not (m[a]["has"] and m[a]["score"] >= pair.min_mate_score):
                continue
            o = reads[(1 - a) * n_pairs + p]
            oq = quals[(1 - a) * n_pairs + p] if quals is not None else None
            if m[a]["strand"] == 0:
                to = m[a]["beg"]; te = min(to + pair.max_frag, glen)
                pat = np.where(o < 4, 3 - o, o)[::-1].astype(np.uint8)
                pq = oq[::-1] if oq is not None else None
            else:
                to = max(m[a]["end"] - pair.max_frag, 0); te = m[a]["end"]
                pat = o
                pq = oq
            if te - to >= 1 and len(pat) >= 1:
                jobs.append((p, a, pat, to, te - to, pq))
    wanted = len(jobs)
    run = jobs[:cap]
    if run:
        pats = np.concatenate([j[2] for j in run])
        p_len = np.array([len(j[2]) for j in run], np.uint32)
        p_off = (np.cumsum(p_len) - p_len).astype(np.uint32)
        t_off = np.array([j[3] for j in run], np.uint32); t_len = np.array([j[4] for j in run], np.uint32)
        scheme, qtab = _scheme_args(params.scheme)
        rs, rx, _ = O.gotoh_full(params.type, scheme, pats, p_off, p_len, genome_sym, t_off, t_len,
                                 qual=np.concatenate([j[5] for j in run]) if quals is not None else None, qtab=qtab)
        cand = {}
        for (p, a, _, to, _, _), s, x in zip(run, rs, rx):
            if int(s) < pair.min_mate_score:
                continue
            tot = int(mate_score[a, p]) + int(s)
            if p not in cand or tot > cand[p][0]:
                cand[p] = (tot, a, int(s), to + int(x))
        for p, (tot, a, s, pos) in cand.items():
            o = 1 - a
            pair_score[p] = tot; pair_flags[p] = 2 if o == 0 else 4
            mate_score[o, p] = s; mate_pos[o, p] = pos; mate_strand[o, p] = 1 - mate_strand[a, p]
    return dict(pair_score=pair_score, pair_flags=pair_flags, mate_score=mate_score, mate_pos=mate_pos, mate_strand=mate_strand,
                n_rescue=(len(run), wanted))
