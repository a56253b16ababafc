"""Writes tests/golden/bam.npz: htslib's BAM bytes (sam_parse1 + bam_write1, oracle/_ref/libnvbio_ref_bam.so) of the SAM lines that
tests/bam_oracle.py gives for fixture_inputs(), hts_reg2bin at the bin-level edges, and the .ann files nvbio's save_bns writes for
ann_fixtures().  Run where oracle/_ref is built:  python -m tests.golden.make_bam_golden"""
import os
import tempfile
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "bam.npz")
TAG_EDGES = [-32769, -32768, -129, -128, -1, 0, 127, 128, 255, 256, 65535, 65536]
QNAME = [c for c in range(33, 127) if c != ord("@")]


def reg2bin_points():
    pts = []
    for sh in (14, 17, 20, 23, 26):
        for m in (1, 2, 3):
            v = m << sh
            for d in (-1, 0, 1):
                pts.append(v + d)
    return sorted(set(pts))


def name(rng, L):
    return "".join(chr(int(c)) for c in rng.choice(QNAME, L))


def fixture_inputs(paired, seed=5, n=240):
    """hand-built inputs of n alignments (CIGARs consistent with the read lengths; MD and edits arbitrary, the record stage copies them)
    on a genome of 5 contigs, covering every tag-type edge, names of 1 and 254 bytes, both strands, N, with and without qualities"""
    rng = np.random.default_rng(seed + (100 if paired else 0))
    contig_names = ["chr1", "chrM", "c3", "tiny", "last_one"]
    contig_lengths = [40_000, 60, 300_000, 90, 20_000_000]
    cb = np.concatenate([[0], np.cumsum(contig_lengths)]).astype(np.int64)
    G = int(cb[-1])
    max_cigar, max_md = 8, 40
    reads, n_ops, begin, strand = [], np.zeros(n, np.uint32), np.zeros((n, 2), np.uint32), np.zeros(n, np.uint8)
    cigar, n_cigar = np.zeros((n, max_cigar), np.uint32), np.zeros(n, np.uint32)
    md, md_len = np.zeros((n, max_md), np.uint8), np.zeros(n, np.uint32)
    edits = np.zeros((n, 4), np.uint32)
    for a in range(n):
        L = int(rng.integers(1, 160))
        r = rng.integers(0, 4, L).astype(np.uint8)
        r[rng.random(L) < 0.03] = 4
        reads.append(r)
        kind = rng.random()
        if kind < 0.08:
            continue                                              # unaligned
        s0 = int(rng.integers(0, min(L, 4)))
        s1 = int(rng.integers(0, min(L - s0, 4)))
        core = L - s0 - s1
        ins = int(rng.integers(0, min(core, 3))) if core > 2 else 0
        m1 = (core - ins) // 2
        m2 = core - ins - m1
        d = int(rng.integers(0, 3))
        runs = [(s0, 4), (m1, 0), (ins, 1), (d, 2), (m2, 0), (s1, 4)]
        runs = [(k, op) for k, op in runs if k]
        merged = []
        for k, op in runs:
            if merged and merged[-1][1] == op:
                merged[-1] = (merged[-1][0] + k, op)
            else:
                merged.append((k, op))
        rlen = sum(k for k, op in merged if op in (0, 2))
        where = rng.random()
        if where < 0.2:                                           # near a contig end: inside, exactly at it, one past, off the genome
            c = int(rng.integers(1, len(cb)))
            x = int(cb[c]) - rlen + int(rng.integers(-2, 3))
        else:
            x = int(rng.integers(0, G - 200))
        x = max(0, x)
        n_ops[a] = max(1, core + d)
        begin[a] = (x, s0)
        strand[a] = int(rng.integers(0, 2))
        if kind < 0.12:
            edits[a] = (0xFFFFFFFF, 0, 0, 0)                      # not finished
            continue
        n_cigar[a] = len(merged) if kind > 0.15 else max_cigar + 1  # a few truncated CIGARs
        for i, (k, op) in enumerate(merged[:max_cigar]):
            cigar[a, i] = k << 4 | op
        m = "%d" % int(rng.integers(0, 200)) if rng.random() < 0.9 else ""
        if rng.random() < 0.5:
            m += "A0^CG3T"
        md_len[a] = len(m) if kind < 0.9 else max_md + 3          # and a few truncated MDs
        md[a, :min(len(m), max_md)] = np.frombuffer(m.encode(), np.uint8)[:max_md]
        edits[a] = [TAG_EDGES[(a + j) % len(TAG_EDGES)] & 0xFFFFFFFF if TAG_EDGES[(a + j) % len(TAG_EDGES)] >= 0 else int(rng.integers(0, 9))
                    for j in range(4)]
    score = np.array([TAG_EDGES[a % len(TAG_EDGES)] for a in range(n)], np.int32)
    second = np.array([TAG_EDGES[(a * 7) % len(TAG_EDGES)] if a % 5 else -(1 << 31) for a in range(n)], np.int32)
    n_names = n // 2 if paired else n
    names = [name(rng, 1 if i == 0 else (254 if i == 1 else int(rng.integers(1, 30)))) for i in range(n_names)]
    if paired:
        h = n // 2
        for p in range(0, h, 9):                                  # equal begins
            begin[h + p] = begin[p]; n_ops[h + p] = n_ops[p]; n_cigar[h + p] = n_cigar[p]; cigar[h + p] = cigar[p]
            edits[h + p] = edits[p]; md_len[h + p] = md_len[p]; md[h + p] = md[p]; reads[h + p] = reads[p].copy()
        for p in range(3, h, 11):                                 # both mates unaligned
            n_ops[p] = n_ops[h + p] = 0
    quals = [rng.integers(0, 42, len(r)).astype(np.uint8) for r in reads]
    pair_flags = rng.choice([0, 1, 2, 4], n // 2).astype(np.uint32) if paired else None
    return dict(reads=reads, quals=quals if seed % 2 else None, n_ops=n_ops, begin=begin, strand=strand, cigar=cigar, n_cigar=n_cigar,
                md=md, md_len=md_len, edits=edits, score=score, mapq=rng.integers(0, 61, n).astype(np.uint8) if paired else None,
                second=second if paired else None, pair_flags=pair_flags, contig_begin=cb, contig_names=contig_names,
                contig_lengths=contig_lengths, names=names)


def ann_fixtures():
    """(names, annotations, lengths) of the .ann files: a name with a comment, one without, 1 and 40 contigs"""
    return [(["chr1", "chr2_random", "chrM"], ["Homo sapiens chromosome 1", "", "mitochondrion  two  spaces"], [1000, 77, 16569]),
            (["only"], [""], [5]),
            (["c%d" % i for i in range(40)], ["comment %d" % i if i % 3 else "" for i in range(40)], [100 + 7 * i for i in range(40)])]


def main():
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    from oracle.ref_bam import RefBam, save_bns
    from tests import bam_oracle as bo
    R = RefBam()
    lines, recs, lens, hdrs = [], [], [], []
    for paired in (False, True):
        for seed in (5, 6):
            inp = fixture_inputs(paired, seed)
            out, _ = bo.records(inp)
            hdr = bo.header_text(inp["contig_names"], inp["contig_lengths"])
            got = R.encode(hdr, [s for _, s in out])
            lines += [s for _, s in out]; recs += got; lens.append(len(out)); hdrs.append(hdr)
    pts = reg2bin_points()
    bins = [[R.reg2bin(b, e) for e in (b + 1, b + 2, b + 16384, b + 131072)] for b in pts]
    anns = []
    with tempfile.TemporaryDirectory() as d:
        for i, (names, annos, lengths) in enumerate(ann_fixtures()):
            offs = np.concatenate([[0], np.cumsum(lengths)[:-1]])
            save_bns(os.path.join(d, "g%d" % i), names, annos, offs, lengths, np.arange(len(names)), int(np.sum(lengths)))
            anns.append(open(os.path.join(d, "g%d.ann" % i)).read())
    np.savez_compressed(OUT, lines=np.array("\n".join(lines)), headers=np.array("\x00".join(hdrs)), batch_sizes=np.array(lens),
                        records=np.frombuffer(b"".join(recs), np.uint8), record_sizes=np.array([len(r) for r in recs]),
                        reg2bin_points=np.array(pts, np.int64), reg2bin=np.array(bins, np.int64), ann=np.array("\x00".join(anns)))
    print("wrote", OUT, len(recs), "records")


if __name__ == "__main__":
    main()
