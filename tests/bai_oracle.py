"""Serial restatement of the coordinate order of nvb_bam_sort and of the BAI rules of nvb_bam_index (include/nvbio_b200.h): records in,
index bytes out; plus a parser of BAI bytes into {refID: (bins, linear index)} for comparisons with htslib's index."""
import struct
import numpy as np

BLOCK = 0xFF00
META_BIN = 37450
EOF_LEN = 28


def sort_key(rec: bytes):
    ref, pos = struct.unpack_from("<II", rec, 4)
    return (ref, pos)


def sort_records(recs):
    """(order, sorted records): Python's stable sort on (refID as uint32, pos as uint32)"""
    order = sorted(range(len(recs)), key=lambda i: sort_key(recs[i]))
    return order, [recs[i] for i in order]


def split_records(raw: bytes):
    out, o = [], 0
    while o < len(raw):
        k = struct.unpack_from("<I", raw, o)[0] + 4
        out.append(raw[o:o + k]); o += k
    return out


def reg2bin(beg, end):
    end -= 1
    for s, t in ((14, 4681), (17, 585), (20, 73), (23, 9), (26, 1)):
        if beg >> s == end >> s:
            return t + (beg >> s)
    return 0


def rec_fields(rec: bytes):
    """refID, pos, end (pos + rlen), bin, mapped"""
    ref, pos = struct.unpack_from("<ii", rec, 4)
    l_name = rec[12]
    n_cigar, flag = struct.unpack_from("<HH", rec, 16)
    rlen = 0
    for k in range(n_cigar):
        c = struct.unpack_from("<I", rec, 36 + l_name + 4 * k)[0]
        if c & 15 in (0, 2, 3, 7, 8):
            rlen += c >> 4
    rlen = rlen or 1
    if ref < 0:
        return ref, pos, pos + rlen, 4680, not flag & 4
    return ref, pos, pos + rlen, reg2bin(pos, pos + rlen), not flag & 4


def voffsets(recs, block_offsets, header_bytes):
    """virtual offset of every record's start, and F (the file size << 16)"""
    bo = np.asarray(block_offsets, np.int64)
    starts, u = [], 0
    for r in recs:
        starts.append(((header_bytes + int(bo[u // BLOCK])) << 16) | (u % BLOCK))
        u += len(r)
    return starts, (header_bytes + int(bo[-1]) + EOF_LEN) << 16


def build_index(recs, block_offsets, header_bytes, n_refs):
    """{refID: (bins {bin: [(beg, end)]}, linear [..]), n_no_coor} by the rules, the records in nvb_bam_sort order"""
    starts, F = voffsets(recs, block_offsets, header_bytes)
    fields = [rec_fields(r) for r in recs]
    nxt = starts[1:] + [F]
    refs = {}
    n_no_coor = 0
    for i, (ref, pos, end, b, mapped) in enumerate(fields):
        if ref < 0:
            n_no_coor += 1
            continue
        assert ref < n_refs
        R = refs.setdefault(ref, {"chunks": [], "first": starts[i], "mapped": 0, "unmapped": 0, "lin": {}})
        if R["chunks"] and R["chunks"][-1][0] == b and R["chunks"][-1][2] == starts[i]:
            R["chunks"][-1][2] = nxt[i]
        else:
            R["chunks"].append([b, starts[i], nxt[i]])
        R["mapped" if mapped else "unmapped"] += 1
        if mapped:
            for w in range(pos >> 14, ((end - 1) >> 14) + 1):
                R["lin"].setdefault(w, starts[i])
    out = {}
    for ref, R in refs.items():
        bins = {}
        for b, s, e in R["chunks"]:
            bins.setdefault(b, []).append((s, e))
        for lvl in range(5, 0, -1):
            first, nxt_first = ((1 << 3 * lvl) - 1) // 7, ((1 << 3 * lvl + 3) - 1) // 7
            for b in sorted(k for k in bins if first <= k < nxt_first):
                ch = sorted(bins[b])
                bins[b] = ch
                if (ch[-1][1] >> 16) - (ch[0][0] >> 16) < 65536 and (b - 1) >> 3 in bins:
                    bins[(b - 1) >> 3] += ch
                    del bins[b]
        for b in bins:
            ch = sorted(bins[b])
            m = [list(ch[0])]
            for s, e in ch[1:]:
                if m[-1][1] >> 16 >= s >> 16:
                    m[-1][1] = max(m[-1][1], e)
                else:
                    m.append([s, e])
            bins[b] = [tuple(c) for c in m]
        bins[META_BIN] = [(R["first"], R["chunks"][-1][2]), (R["mapped"], R["unmapped"])]
        n_intv = max(R["lin"]) + 1 if R["lin"] else 0
        lin, prev = [], None
        for w in range(n_intv):
            v = R["lin"].get(w)
            if v is None:
                v = R["first"] if prev is None else prev
            lin.append(v)
            if w in R["lin"]:
                prev = v
        out[ref] = (bins, lin)
    return out, n_no_coor


def serialise(index, n_no_coor, n_refs) -> bytes:
    """BAI bytes, bins in ascending order"""
    out = [b"BAI\1", struct.pack("<i", n_refs)]
    for r in range(n_refs):
        bins, lin = index.get(r, ({}, []))
        out.append(struct.pack("<i", len(bins)))
        for b in sorted(bins):
            out.append(struct.pack("<Ii", b, len(bins[b])))
            out += [struct.pack("<QQ", s, e) for s, e in bins[b]]
        out.append(struct.pack("<i", len(lin)))
        out += [struct.pack("<Q", v) for v in lin]
    out.append(struct.pack("<Q", n_no_coor))
    return b"".join(out)


def bai_bytes(recs, block_offsets, header_bytes, n_refs) -> bytes:
    index, n_no_coor = build_index(recs, block_offsets, header_bytes, n_refs)
    return serialise(index, n_no_coor, n_refs)


def parse_bai(data: bytes):
    """({refID: (bins {bin: [(beg, end)]}, linear [..])} with the refIDs that have bins or entries, n_no_coor, n_ref)"""
    assert data[:4] == b"BAI\1"
    (n_ref,) = struct.unpack_from("<i", data, 4)
    o, out = 8, {}
    for r in range(n_ref):
        (nb,) = struct.unpack_from("<i", data, o); o += 4
        bins = {}
        for _ in range(nb):
            b, nc = struct.unpack_from("<Ii", data, o); o += 8
            bins[b] = [struct.unpack_from("<QQ", data, o + 16 * k) for k in range(nc)]
            o += 16 * nc
        (ni,) = struct.unpack_from("<i", data, o); o += 4
        lin = list(struct.unpack_from("<%dQ" % ni, data, o)); o += 8 * ni
        if bins or lin:
            out[r] = (bins, lin)
    n_no_coor = struct.unpack_from("<Q", data, o)[0] if o + 8 <= len(data) else None
    return out, n_no_coor, n_ref
