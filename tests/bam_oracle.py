"""TEST INFRASTRUCTURE: a plain restatement of nvb_bam_records (include/nvbio_b200.h) written from the header's rules and not from the
kernels.  For every record it gives both the BAM bytes and the SAM line, so that htslib's encoding of the line can be compared with the
bytes.  Inputs are host arrays laid out like the C inputs (a dict, see `records`)."""
import struct
import numpy as np

NONE = 0xFFFFFFFF
INT_MIN = -(1 << 31)
NT16 = {0: 1, 1: 2, 2: 4, 3: 8}
CIGAR_OPS = "MIDNSHP=X"


def reg2bin(beg, end):
    """the specification's reg2bin (SAMv1 section 5.3)"""
    end -= 1
    if beg >> 14 == end >> 14:
        return ((1 << 15) - 1) // 7 + (beg >> 14)
    if beg >> 17 == end >> 17:
        return ((1 << 12) - 1) // 7 + (beg >> 17)
    if beg >> 20 == end >> 20:
        return ((1 << 9) - 1) // 7 + (beg >> 20)
    if beg >> 23 == end >> 23:
        return ((1 << 6) - 1) // 7 + (beg >> 23)
    if beg >> 26 == end >> 26:
        return ((1 << 3) - 1) // 7 + (beg >> 26)
    return 0


def int_tag(name, v):
    """an integer tag as htslib's SAM parser types it"""
    if v < 0:
        t, f = ("c", "<b") if v >= -128 else (("s", "<h") if v >= -32768 else ("i", "<i"))
    else:
        t, f = ("C", "<B") if v <= 255 else (("S", "<H") if v <= 65535 else ("I", "<I"))
    return name.encode() + t.encode() + struct.pack(f, v)


def strand_symbols(read, strand):
    read = np.asarray(read, np.uint8)
    return read if strand == 0 else np.where(read < 4, 3 - read, read)[::-1]


def place(inp, a):
    """(state, ref, pos, rlen, strand): state 0 unaligned, 1 mapped, 2 off its contig, 3 not finished whole"""
    if int(inp["n_ops"][a]) == 0:
        return (0, -1, -1, 0, 0)
    nc, ml = int(inp["n_cigar"][a]), int(inp["md_len"][a])
    if int(inp["edits"][a][0]) == NONE or nc > inp["cigar"].shape[1] or nc > 65535 or ml > inp["md"].shape[1]:
        return (3, -1, -1, 0, 0)
    rlen = sum(int(c) >> 4 for c in inp["cigar"][a][:nc] if int(c) & 15 in (0, 2))
    bx = int(inp["begin"][a][0])
    cb = inp["contig_begin"]
    r = int(np.searchsorted(cb, bx, side="right")) - 1
    r = min(r, len(cb) - 2)
    if bx >= cb[r + 1] or bx + rlen > cb[r + 1]:
        return (2, -1, -1, 0, 0)
    return (1, r, bx - int(cb[r]), rlen, 1 if int(inp["strand"][a]) else 0)


def record(inp, k, me, mate, pflag):
    """(bam bytes, sam line) of record k"""
    paired = mate is not None
    n = len(inp["n_ops"])
    a = (k & 1) * (n // 2) + (k >> 1) if paired else k
    name = inp["names"][k >> 1 if paired else k][:254]
    mapped = me[0] == 1
    flag = (0x10 if me[4] else 0) if mapped else 0x4
    ref = pos = nref = npos = -1
    tlen, bin_ = 0, 4680
    if paired:
        mm = mate[0] == 1
        flag |= 0x1 | (0x80 if k & 1 else 0x40)
        if pflag in (1, 2, 4) and mapped and mm:                 # concordant or rescued; a discordant pair (8) is not proper
            flag |= 0x2
        if not mm:
            flag |= 0x8
        elif mate[4]:
            flag |= 0x20
        if mapped:
            ref, pos = me[1], me[2]
            if mm:
                nref, npos = mate[1], mate[2]
                if mate[1] == me[1]:
                    t = max(me[2] + me[3], mate[2] + mate[3]) - min(me[2], mate[2])
                    tlen = t if (me[2] < mate[2] or (me[2] == mate[2] and not k & 1)) else -t
            else:
                nref, npos = me[1], me[2]
        elif mm:
            ref = nref = mate[1]; pos = npos = mate[2]
            bin_ = reg2bin(pos, pos + 1)
    elif mapped:
        ref, pos = me[1], me[2]
    read = inp["reads"][a]
    L = len(read)
    strand = me[4] if mapped else 0
    sym = strand_symbols(read, strand)
    q = None if inp["quals"] is None else np.asarray(inp["quals"][a], np.uint8)
    if q is not None and strand:
        q = q[::-1]
    cigar = [int(c) for c in inp["cigar"][a][:int(inp["n_cigar"][a])]] if mapped else []
    if mapped:
        bin_ = reg2bin(pos, pos + me[3])
    mapq = (int(inp["mapq"][a]) if inp["mapq"] is not None else 255) if mapped else 0
    tags, sam_tags = b"", []
    if mapped:
        e = [int(v) for v in inp["edits"][a]]
        vals = [("NM", e[0]), ("AS", int(inp["score"][a]))]
        if inp["second"] is not None and int(inp["second"][a]) != INT_MIN:
            vals.append(("XS", int(inp["second"][a])))
        vals += [("XM", e[1]), ("XO", e[2]), ("XG", e[3])]
        for nm, v in vals:
            tags += int_tag(nm, v); sam_tags.append("%s:i:%d" % (nm, v))
        ml = int(inp["md_len"][a])
        if ml:
            md = bytes(inp["md"][a][:ml])
            tags += b"MDZ" + md + b"\0"; sam_tags.append("MD:Z:" + md.decode())
    seq = bytearray((L + 1) // 2)
    for i, c in enumerate(sym):
        seq[i >> 1] |= (15 if c > 3 else NT16[int(c)]) << (4 if i % 2 == 0 else 0)
    qual = bytes([0xFF] * L) if q is None else bytes(q)
    nameb = name.encode() + b"\0"
    core = struct.pack("<iiIIiiii", ref, pos, bin_ << 16 | mapq << 8 | len(nameb), flag << 16 | len(cigar), L, nref, npos, tlen)
    body = core + nameb + b"".join(struct.pack("<I", c) for c in cigar) + bytes(seq) + qual + tags
    bam = struct.pack("<i", len(body)) + body
    cnames = inp["contig_names"]
    rname = cnames[ref] if ref >= 0 else "*"
    rnext = "*" if nref < 0 else ("=" if nref == ref else cnames[nref])
    sam = "\t".join([name, str(flag), rname, str(pos + 1), str(mapq), "".join("%d%s" % (c >> 4, CIGAR_OPS[c & 15]) for c in cigar) or "*",
                     rnext, str(npos + 1), str(tlen), "".join("ACGTN"[min(int(c), 4)] for c in sym) or "*",
                     "*" if q is None else "".join(chr(int(v) + 33) for v in q)] + sam_tags)
    return bam, sam


def records(inp):
    """(list of (bam bytes, sam line) per record, counts [records, mapped, off-contig, unfinished]).  inp: reads (caller symbols per
    alignment), quals (per alignment or None), n_ops, begin [n, 2], strand, cigar [n, max_cigar], n_cigar, md [n, max_md], md_len,
    edits [n, 4], score, mapq / second (or None), pair_flags (or None), contig_begin, contig_names, names"""
    n = len(inp["n_ops"])
    out, cnt = [], [n, 0, 0, 0]
    pl = [place(inp, a) for a in range(n)]
    for p in pl:
        if p[0]:
            cnt[p[0]] += 1
    if inp["pair_flags"] is None:
        for k in range(n):
            out.append(record(inp, k, pl[k], None, 0))
    else:
        h = n // 2
        for p in range(h):
            pf = int(inp["pair_flags"][p])
            out.append(record(inp, 2 * p, pl[p], pl[h + p], pf))
            out.append(record(inp, 2 * p + 1, pl[h + p], pl[p], pf))
    return out, cnt


def header_text(contig_names, contig_lengths):
    return "@HD\tVN:1.0\tSO:unsorted\n" + "".join("@SQ\tSN:%s\tLN:%d\n" % (nm, ln) for nm, ln in zip(contig_names, contig_lengths))
