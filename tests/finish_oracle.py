"""TEST INFRASTRUCTURE: a plain restatement of nvb_finish_alignments (include/nvbio_b200.h) from (ops, n_ops, begin, strand, read,
genome), written from the header's semantics and not from the kernel, plus nvBowtie's MDS token vector restated from
finish_alignment_kernel (nvBowtie/bowtie2/cuda/traceback_inl.h:584-674) and helpers that decode MD + CIGAR back into the reference."""
import numpy as np

NONE = 0xFFFFFFFF
BAD = (NONE, 0, 0, 0)
MDS_MATCH, MDS_MISMATCH, MDS_INSERTION, MDS_DELETION = 0, 1, 2, 3


def strand_read(read, strand):
    """the symbols the alignment is of: the read, or its reverse complement (c < 4 ? 3 - c : c)"""
    read = np.asarray(read, dtype=np.uint8)
    return read if strand == 0 else np.where(read < 4, 3 - read, read)[::-1].astype(np.uint8)


def ref_char(genome, genome_len, x):
    return "ACGT"[int(genome[x])] if x < genome_len else "N"


def op_runs(ops, n_ops):
    """[(op, length)] START -> END from ops END -> START"""
    runs = []
    for op in np.asarray(ops[:n_ops], dtype=np.int64)[::-1]:
        if runs and runs[-1][0] == op:
            runs[-1][1] += 1
        else:
            runs.append([int(op), 1])
    return [(o, k) for o, k in runs]


def finish(ops, n_ops, max_ops, begin, strand, read, genome, genome_len):
    """(cigar [(length, op)] with op 0 M / 1 I / 2 D / 4 S, md str, (NM, XM, XO, XG)) of one alignment; read = the caller's symbols"""
    n_ops, bx, by = int(n_ops), int(begin[0]), int(begin[1])
    L = len(read)
    if n_ops == 0:
        return [], "", (0, 0, 0, 0)
    if n_ops > max_ops or bx == NONE:
        return [], "", BAD
    ops = np.asarray(ops[:n_ops])
    if (ops > 2).any():
        return [], "", BAD
    M, I = int((ops == 0).sum()), int((ops == 1).sum())
    if by > L or M + I > L - by:
        return [], "", BAD
    r = strand_read(read, strand)
    cigar = [(by, 4)] if by else []
    md, run = "", 0
    nm = xm = xo = xg = 0
    x, y = bx, by
    for op, k in op_runs(ops, n_ops):
        cigar.append((k, op))
        if op == 0:
            for _ in range(k):
                g = int(genome[x]) if x < genome_len else 4
                if g < 4 and r[y] < 4 and r[y] == g:
                    run += 1
                else:
                    md += "%d%s" % (run, ref_char(genome, genome_len, x)); run = 0; xm += 1
                x += 1; y += 1
        elif op == 1:
            y += k; nm += k; xo += 1; xg += k - 1
        else:
            md += "%d^%s" % (run, "".join(ref_char(genome, genome_len, x + c) for c in range(k))); run = 0
            x += k; nm += k; xo += 1; xg += k - 1
    md += "%d" % run
    if L - y:
        cigar.append((L - y, 4))
    return cigar, md, (nm + xm, xm, xo, xg)


def cigar_text(cigar):
    return "".join("%d%s" % (k, "MIDNSHP=X"[op]) for k, op in cigar)


def rebuild_reference(cigar, md, read, strand):
    """the genome span [begin.x, begin.x + M + D) rebuilt from MD + CIGAR + the read alone (what a SAM consumer does)"""
    r = strand_read(read, strand)
    cols, i = [], 0                                      # one entry per M / D column: '=' a match, a base a mismatch, lower case deleted
    while i < len(md):
        if md[i].isdigit():
            j = i
            while j < len(md) and md[j].isdigit():
                j += 1
            cols += ["="] * int(md[i:j]); i = j
        elif md[i] == "^":
            j = i + 1
            while j < len(md) and md[j].isalpha():
                j += 1
            cols += list(md[i + 1:j].lower()); i = j
        else:
            cols.append(md[i]); i += 1
    out, y, c = [], 0, 0
    for k, op in cigar:
        if op in (1, 4):
            y += k; continue
        for _ in range(k):
            e = cols[c]; c += 1
            if op == 2:
                assert e.islower(), (md, cigar)
                out.append(e.upper())
            else:
                assert not e.islower(), (md, cigar)
                out.append("ACGTN"[int(r[y])] if e == "=" else e); y += 1
    assert c == len(cols), (md, cigar)
    return "".join(out)


def mds_vector(ops, n_ops, begin, strand, read, genome, genome_len):
    """nvBowtie's MDS byte vector (traceback_inl.h:584-674: two length bytes, then MATCH n (n <= 255, merged), MISMATCH read base,
    INSERTION l + read bases, DELETION l + reference bases) of the aligned part of an alignment -- soft clips left out, see DESIGN.md.
    Bases are 2-bit codes, a read N and a column past the genome's end 4."""
    r = strand_read(read, strand)
    v = [0, 0]
    mds_op = 4
    x, y = int(begin[0]), int(begin[1])
    for op, k in op_runs(ops, int(n_ops)):
        if op != 0:
            mds_op = MDS_DELETION if op == 2 else MDS_INSERTION
            v += [mds_op, k]
        for _ in range(k):
            if op == 0:
                g = int(genome[x]) if x < genome_len else 4
                if int(r[y]) == g and g < 4:
                    if mds_op == MDS_MATCH and v[-1] < 255:
                        v[-1] += 1
                    else:
                        v += [MDS_MATCH, 1]; mds_op = MDS_MATCH
                else:
                    v += [MDS_MISMATCH, int(r[y])]; mds_op = MDS_MISMATCH
                x += 1; y += 1
            elif op == 1:
                v.append(int(r[y])); y += 1
            else:
                v.append(int(genome[x]) if x < genome_len else 4); x += 1
    v[0], v[1] = len(v) & 0xFF, len(v) >> 8
    return np.array(v, dtype=np.uint8)
