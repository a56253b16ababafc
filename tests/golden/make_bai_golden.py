"""Writes tests/golden/bai.npz: for each synthetic case of cases(), the unsorted records, the framing of the sorted records by write_bam's
host path (header members' size, member offsets of the records) and htslib's index of that file (bam_index_build,
oracle/_ref/libnvbio_ref_bai.so).  Run where oracle/_ref is built:  python -m tests.golden.make_bai_golden"""
import os
import struct
import tempfile
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "bai.npz")
BLOCK = 0xFF00


def reg2bin(beg, end):
    end -= 1
    for s, t in ((14, 4681), (17, 585), (20, 73), (23, 9), (26, 1)):
        if beg >> s == end >> s:
            return t + (beg >> s)
    return 0


def record(name, ref, pos, flag=0, cigar=((0, 100),), l_seq=None, qual=None, mapq=60):
    """one BAM record (block_size first); cigar: (op, length) pairs, op in BAM's MIDNSHP=X numbering; qual: bytes of l_seq or None"""
    if l_seq is None:
        l_seq = sum(ln for op, ln in cigar if op in (0, 1, 4, 7, 8))
    qn = name.encode() + b"\0"
    cig = b"".join(struct.pack("<I", ln << 4 | op) for op, ln in cigar)
    rlen = sum(ln for op, ln in cigar if op in (0, 2, 3, 7, 8)) or 1
    b = reg2bin(pos, pos + rlen) if ref >= 0 else 4680
    seq = bytes([0x12]) * ((l_seq + 1) // 2)
    q = qual if qual is not None else b"\xff" * l_seq
    core = struct.pack("<iiBBHHHiiii", ref, pos, len(qn), mapq if not flag & 4 else 0, b, len(cigar), flag, l_seq, -1, -1, 0)
    body = core + qn + cig + seq + q
    return struct.pack("<i", len(body)) + body


def unmapped(name, ref=-1, pos=-1, l_seq=100):
    return record(name, ref, pos, flag=4, cigar=(), l_seq=l_seq)


def cases():
    """name -> (contig lengths, records in an unsorted order)"""
    rng = np.random.default_rng(2024)
    out = {}

    def reads(ref, n, lo, hi, tag, read_len=100, p_unmapped=0.0):
        recs = []
        for k, p in enumerate(rng.integers(lo, hi - read_len, n)):
            if rng.random() < p_unmapped:
                recs.append(unmapped("%s_%d" % (tag, k), ref, int(p)))
            else:
                recs.append(record("%s_%d" % (tag, k), ref, int(p), flag=16 * int(rng.integers(0, 2)), cigar=((0, read_len),)))
        return recs

    # one contig, with and without unplaced records
    base = reads(0, 3000, 0, 1_000_000, "a", p_unmapped=0.05)
    out["one_contig"] = ([1_000_000], base)
    out["one_contig_unplaced"] = ([1_000_000], base + [unmapped("u%d" % k) for k in range(40)])
    out["only_unplaced"] = ([5000, 7000], [unmapped("u%d" % k) for k in range(300)])
    # 3,000 contigs, most of them empty, one with only unmapped-placed records
    lens = [int(x) for x in rng.integers(2_000, 60_000, 3000)]
    recs = []
    for r in sorted(rng.choice(3000, 60, replace=False)):
        recs += reads(int(r), int(rng.integers(1, 40)), 0, lens[r], "m%d" % r)
    recs += [unmapped("pu%d" % k, 5, int(p)) for k, p in enumerate(rng.integers(0, lens[5], 30))]
    recs += [unmapped("u%d" % k) for k in range(7)]
    out["many_contigs"] = (lens, [recs[i] for i in rng.permutation(len(recs))])
    # records whose end falls exactly on a 0xFF00 boundary of the uncompressed stream: equal-size records, in sorted order already
    r0 = record("x" * 200, 0, 0)
    k = BLOCK // len(r0) + 1
    pad = k * len(r0) - BLOCK                              # shorten the first record's name by `pad` bytes
    assert pad < 200
    out["block_boundary"] = ([200_000], [record("x" * (200 - pad), 0, 0)] + [record("x" * 200, 0, 50 * i) for i in range(1, 3 * k)])
    # a 100 kbp deletion among short reads, and bins at every level (long N skips)
    recs = reads(0, 400, 0, 600_000, "d")
    recs.append(record("del", 0, 123_456, cigar=((0, 50), (2, 100_000), (0, 50))))
    spans = [100, 30_000, 200_000, 2_000_000, 20_000_000, 70_000_000]
    for i, sp in enumerate(spans):
        for j in range(3):
            p = int(rng.integers(0, 150_000_000 - sp))
            recs.append(record("lv%d_%d" % (i, j), 0, p, cigar=((0, 50), (3, sp), (0, 50))))
    recs.append(record("lv_edge", 0, (1 << 26) - 60, cigar=((0, 120),)))   # across the 2^26 boundary: bin 0
    out["deletion_levels"] = ([150_000_000], [recs[i] for i in rng.permutation(len(recs))])
    # dense small bins that merge upward, and sparse incompressible records whose chunks stay apart
    recs = reads(0, 4000, 0, 300_000, "dn", read_len=60)
    for i in range(40):
        q = bytes(rng.integers(0, 94, 6000, dtype=np.uint8) + 33)
        recs.append(record("sp%d" % i, 0, 400_000 + 20_000 * i, cigar=((0, 6000),), qual=q))
        recs.append(record("sq%d" % i, 0, 400_000 + 20_000 * i + 3000, cigar=((0, 6000),), qual=q[::-1]))
    out["dense_sparse"] = ([2_000_000], [recs[i] for i in rng.permutation(len(recs))])
    return out


def header(lens):
    from nvbio_b200.bam import ContigTable, bam_header
    return bam_header(ContigTable(["c%d" % i for i in range(len(lens))], lens), sort_order="coordinate")


def frame(hdr: bytes, recs):
    """write_bam's host framing of header + records: (file bytes, header_bytes, member offsets of the records)"""
    from nvbio_b200.bam import _bgzf_block, _BGZF_EOF
    hz = b"".join(_bgzf_block(hdr[i:i + BLOCK]) for i in range(0, len(hdr), BLOCK))
    raw = b"".join(recs)
    blocks = [_bgzf_block(raw[i:i + BLOCK]) for i in range(0, len(raw), BLOCK)]
    offs = np.concatenate([[0], np.cumsum([len(b) for b in blocks])]).astype(np.int64)
    return hz + b"".join(blocks) + _BGZF_EOF, len(hz), offs


def htslib_index(data: bytes) -> bytes:
    from oracle.ref_bai import RefBai
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "f.bam")
        with open(p, "wb") as f:
            f.write(data)
        return RefBai().index(p)


def main():
    from tests.bai_oracle import sort_records
    arrays = {}
    for name, (lens, recs) in cases().items():
        _, srt = sort_records(recs)
        data, hb, offs = frame(header(lens), srt)
        arrays[name + "/lens"] = np.asarray(lens, np.int64)
        arrays[name + "/records"] = np.frombuffer(b"".join(recs), np.uint8)
        arrays[name + "/header_bytes"] = np.int64(hb)
        arrays[name + "/block_offsets"] = offs
        arrays[name + "/htslib_bai"] = np.frombuffer(htslib_index(data), np.uint8)
    np.savez_compressed(OUT, **arrays)
    print("wrote", OUT, sorted({k.split("/")[0] for k in arrays}))


if __name__ == "__main__":
    main()
