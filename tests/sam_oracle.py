"""TEST INFRASTRUCTURE: a plain restatement of nvb_sam_format's line rule (include/nvbio_b200.h), written from the header and htslib's
sam_format1 and not from the kernels: BAM record bytes (block_size included) -> the SAM line ('\\n' included), or None when the record is
rejected."""
import struct

CIGAR_OPS = "MIDNSHP=X"
SEQ = "=ACMGRSVTWYHKDBN"
INT_TAGS = {"c": "<b", "C": "<B", "s": "<h", "S": "<H", "i": "<i", "I": "<I"}


def _i32(v):
    return (v + (1 << 31)) % (1 << 32) - (1 << 31)


def line(rec: bytes, ref_names) -> bytes:
    n = len(rec)
    if n < 36 or struct.unpack_from("<I", rec)[0] + 4 != n:
        return None
    ref, pos, bmn, fnc, l_seq, nref, npos, tlen = struct.unpack_from("<iiIIIiii", rec, 4)
    l_name, mapq, flag, nc = bmn & 0xFF, (bmn >> 8) & 0xFF, fnc >> 16, fnc & 0xFFFF
    if not (-1 <= ref < len(ref_names) and -1 <= nref < len(ref_names)):
        return None
    cg = 36 + l_name
    sq = cg + 4 * nc
    ql = sq + (l_seq + 1) // 2
    aux = ql + l_seq
    if l_name < 2 or aux > n or rec[cg - 1] != 0:
        return None
    ops = struct.unpack_from("<%dI" % nc, rec, cg)
    if any(op & 15 > 8 for op in ops):
        return None
    f = [rec[36:cg - 1], str(flag).encode(), b"*" if ref < 0 else ref_names[ref], str(_i32(pos + 1)).encode(), str(mapq).encode(),
         b"".join(b"%d%s" % (op >> 4, CIGAR_OPS[op & 15].encode()) for op in ops) or b"*",
         b"*" if nref < 0 else (b"=" if nref == ref else ref_names[nref]), str(_i32(npos + 1)).encode(), str(tlen).encode()]
    if l_seq:
        f.append("".join(SEQ[rec[sq + (i >> 1)] >> (0 if i & 1 else 4) & 15] for i in range(l_seq)).encode())
        f.append(b"*" if rec[ql] == 0xFF else bytes(q + 33 for q in rec[ql:aux]))
    else:
        f += [b"*", b"*"]
    p = aux
    while n - p >= 4:
        key, t = rec[p:p + 2], chr(rec[p + 2])
        p += 3
        if t == "Z":
            z = rec.find(b"\0", p)
            if z < 0:
                return None
            f.append(key + b":Z:" + rec[p:z])
            p = z + 1
        elif t in INT_TAGS:
            k = struct.calcsize(INT_TAGS[t])
            if p + k > n:
                return None
            f.append(key + b":i:%d" % struct.unpack_from(INT_TAGS[t], rec, p)[0])
            p += k
        else:
            return None
    if p != n:
        return None
    return b"\t".join(f) + b"\n"


def text(data: bytes, offsets, ref_names):
    """(the text of every record of a stream, [rejected, first rejected index or 0xFFFFFFFF]); ref_names as str or bytes"""
    names = [nm.encode() if isinstance(nm, str) else bytes(nm) for nm in ref_names]
    out, bad, first = [], 0, 0xFFFFFFFF
    for i in range(len(offsets) - 1):
        ln = line(data[int(offsets[i]):int(offsets[i + 1])], names)
        if ln is None:
            bad += 1
            first = min(first, i)
            ln = b""
        out.append(ln)
    return out, [bad, first]
