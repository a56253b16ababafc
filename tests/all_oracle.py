"""Restatement of the selection rule of nvb_seed_extend_all (test infrastructure): include/nvbio_b200.h's rule in plain Python, applied
to candidate lists and to the per-hit outputs of the oracle composition (tests/pipeline_oracle.py)."""
import numpy as np
from tests.pipeline_oracle import EMPTY_SINK
from tests.mapq_oracle import distinct


def select(score, tie, end, strand, sink_x, length, min_score, k):
    """indices of the admitted candidates in rank order: the aligned ones reaching min_score, by (score desc, tie asc), each admitted
    when distinct from every one admitted before it; at most k (0 = no limit)"""
    cand = [i for i in range(len(score)) if int(sink_x[i]) != EMPTY_SINK and int(score[i]) >= int(min_score)]
    cand.sort(key=lambda i: (-int(score[i]), int(tie[i])))
    adm = []
    for i in cand:
        if k and len(adm) >= k:
            break
        if all(distinct(int(end[i]), int(strand[i]), int(end[a]), int(strand[a]), int(length)) for a in adm):
            adm.append(i)
    return adm


def all_oracle(se, lengths, strands, min_score, k):
    """se: seed_extend_oracle's result; lengths: read lengths; min_score: the table (index = read length).  Returns, per read, the
    admitted hit indices in rank order (a hit is its own tie index)"""
    n = len(lengths)
    hs = se["hit_string"]
    end = se["hit_window"][:, 0] + se["hit_sink"][:, 0] if len(hs) else np.zeros(0, np.int64)
    by_read = [[] for _ in range(n)]
    for h, s in enumerate(hs):
        by_read[int(s) // strands].append(h)
    out = []
    for r in range(n):
        h = np.array(by_read[r], np.int64)
        if not len(h):
            out.append([])
            continue
        adm = select(se["hit_score"][h], h, end[h], hs[h] % strands, se["hit_sink"][h, 0], lengths[r], min_score[int(lengths[r])], k)
        out.append([int(h[i]) for i in adm])
    return out


def all_records(inp, first, capacity):
    """nvb_bam_records_all restated on tests/bam_oracle.py: (list of (bam bytes, sam line), counts [records, mapped, off-contig,
    unfinished or beyond capacity]).  inp: as bam_oracle.records takes it, but n_ops / begin / strand / cigar / n_cigar / md / md_len /
    edits / score indexed by ALIGNMENT and reads / quals / names / mapq / second by READ; pair_flags None"""
    from tests import bam_oracle as bo
    per_aln = ("n_ops", "begin", "strand", "cigar", "n_cigar", "md", "md_len", "edits", "score")
    n_reads = len(inp["reads"])
    out, cnt = [], [0, 0, 0, 0]

    def one(r, a, primary, nh):
        t = dict(inp)
        for f in per_aln:
            t[f] = inp[f][a:a + 1] if a is not None else (np.zeros(1, np.int64) if f == "n_ops" else inp[f][:1])
        t["reads"], t["names"] = [inp["reads"][r]], [inp["names"][r]]
        t["quals"] = None if inp["quals"] is None else [inp["quals"][r]]
        mapq = None if inp["mapq"] is None else [int(inp["mapq"][r])]
        second = None if inp["second"] is None else [int(inp["second"][r])]
        t["mapq"] = mapq if primary else [255]
        t["second"] = second if primary else None
        me = bo.place(t, 0)
        bam, sam = bo.record(t, 0, me, None, 0)
        if a is None or me[0] != 1:
            return bam, sam
        body = bytearray(bam[4:])
        if not primary:
            flag = int.from_bytes(body[14:16], "little") | 0x100
            body[14:16] = flag.to_bytes(2, "little")
            f = sam.split("\t"); f[1] = str(flag); sam = "\t".join(f)
        body += bo.int_tag("NH", nh)
        return len(body).to_bytes(4, "little") + bytes(body), sam + "\tNH:i:%d" % nh

    for r in range(n_reads):
        b, e = int(first[r]), int(first[r + 1])
        mapped = []
        if e <= capacity:
            for a in range(b, e):
                st = bo.place(inp, a)[0]
                if st == 1:
                    mapped.append(a)
                elif st:
                    cnt[st] += 1
        else:
            cnt[3] += 1
        cnt[1] += len(mapped)
        if not mapped:
            out.append(one(r, None, True, 0))
        for i, a in enumerate(mapped):
            out.append(one(r, a, i == 0, len(mapped)))
    cnt[0] = len(out)
    return out, cnt
