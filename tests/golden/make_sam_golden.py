"""Writes tests/golden/sam.npz: the text htslib's sam_format1 (oracle/_ref/libnvbio_ref_bam.so, ref_bam_format) gives for hand-built BAM
records that none of the record writers produce but nvb_sam_format's rule covers: l_seq 0, QUAL 0xFF, RNEXT naming another contig, POS
-1, every CIGAR op 0-8, I values above 2^31, TLEN = INT_MIN, every integer tag type at its edges, every SEQ code, 1- and 254-byte names.
Run where oracle/_ref is built:  python -m tests.golden.make_sam_golden"""
import os
import struct
import tempfile
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "sam.npz")
REF_NAMES = ["chr1", "chrM", "contig_three", "x"]
REF_LENGTHS = [1000, 16569, 300000, 7]
INT_MIN, INT_MAX = -(1 << 31), (1 << 31) - 1


def int_tag(key, t, v):
    return key.encode() + t.encode() + struct.pack({"c": "<b", "C": "<B", "s": "<h", "S": "<H", "i": "<i", "I": "<I"}[t], v)


def z_tag(key, s):
    return key.encode() + b"Z" + s + b"\0"


def record(name=b"r", flag=0, ref=-1, pos=-1, mapq=0, cigar=(), nref=-1, npos=-1, tlen=0, seq=(), qual=None, tags=b"", bin_=4680):
    """BAM bytes (block_size included); seq: 4-bit codes; qual: bytes, or None for 0xFF * l_seq"""
    nm = name + b"\0"
    s = bytearray((len(seq) + 1) // 2)
    for i, c in enumerate(seq):
        s[i >> 1] |= c << (4 if i % 2 == 0 else 0)
    q = bytes([0xFF] * len(seq)) if qual is None else bytes(qual)
    core = struct.pack("<iiIIiiii", ref, pos, bin_ << 16 | mapq << 8 | len(nm), flag << 16 | len(cigar), len(seq), nref, npos, tlen)
    body = core + nm + b"".join(struct.pack("<I", c) for c in cigar) + bytes(s) + q + tags
    return struct.pack("<i", len(body)) + body


def edge_records():
    rng = np.random.default_rng(17)
    seq = lambda n: [int(x) for x in rng.integers(0, 16, n)]             # noqa: E731
    qual = lambda n: bytes(int(x) for x in rng.integers(0, 94, n))        # noqa: E731
    ints = b"".join(int_tag(k, t, v) for k, t, v in [("Xa", "c", -128), ("Xb", "c", 127), ("Xc", "C", 0), ("Xd", "C", 255), ("Xe", "s", -32768),
                                                     ("Xf", "s", 32767), ("Xg", "S", 65535), ("Xh", "i", INT_MIN), ("Xi", "i", INT_MAX),
                                                     ("Xj", "I", 0), ("Xk", "I", (1 << 31) + 1), ("Xl", "I", (1 << 32) - 1)])
    recs = [
        record(b"no_seq"),                                                                     # l_seq 0, unplaced, POS -1
        record(b"no_seq_placed", flag=0x10, ref=0, pos=5, mapq=60, cigar=(5 << 4 | 4,), tags=z_tag("MD", b"")),
        record(b"qual_ff", flag=0x4, seq=seq(9)),                                              # QUAL 0xFF: '*'
        record(b"all_codes", ref=1, pos=0, mapq=255, cigar=(16 << 4,), seq=list(range(16)) + [15, 0, 1], qual=qual(19)),
        record(b"other_contig", flag=0x1 | 0x40, ref=0, pos=999, mapq=3, cigar=(2 << 4,), nref=2, npos=299999, tlen=0, seq=seq(2), qual=qual(2)),
        record(b"same_contig", flag=0x1 | 0x80, ref=3, pos=0, mapq=0, cigar=(7 << 4,), nref=3, npos=0, tlen=-7, seq=seq(7), qual=qual(7)),
        record(b"mate_unplaced_ref", flag=0x4, ref=-1, pos=-1, nref=2, npos=-1, seq=seq(3), qual=qual(3)),
        record(b"every_op", ref=2, pos=100, mapq=17, cigar=tuple((i + 1) << 4 | i for i in range(9)) + ((1 << 28) - 1 << 4 | 0,),
               seq=seq(11), qual=qual(11)),
        record(b"tlen_min", flag=0x1, ref=0, pos=INT_MAX - 1, nref=0, npos=INT_MAX - 1, tlen=INT_MIN, seq=seq(1), qual=qual(1)),
        record(b"tlen_max", flag=0x1, ref=0, pos=0, nref=1, npos=0, tlen=INT_MAX, seq=seq(4), qual=qual(4)),
        record(b"int_tags", ref=0, pos=1, cigar=(3 << 4,), seq=seq(3), qual=qual(3), tags=ints),
        record(b"z_tags", ref=0, pos=1, seq=seq(2), qual=qual(2), tags=z_tag("ZA", b"") + z_tag("ZB", b"hello world 1^2") + int_tag("NM", "C", 3)),
        record(b"q" * 254, flag=0xFFFF, ref=1, pos=123, mapq=42, cigar=(1 << 4 | 1, 4 << 4), nref=1, npos=122, tlen=-5, seq=seq(5), qual=qual(5)),
        record(b"A", seq=seq(150), qual=qual(150), tags=int_tag("AS", "s", -300) + int_tag("XS", "I", 3000000000)),
    ]
    return recs


def main():
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    from oracle.ref_bam import RefBam
    from nvbio_b200.bam import ContigTable, bam_header, write_bam
    recs = edge_records()
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "edges.bam")
        write_bam(p, bam_header(ContigTable(REF_NAMES, REF_LENGTHS)), [b"".join(recs)])
        text = RefBam().format(p)
    np.savez_compressed(OUT, records=np.frombuffer(b"".join(recs), np.uint8), record_sizes=np.array([len(r) for r in recs]),
                        text=np.array(text))
    print("wrote", OUT, len(recs), "records")


if __name__ == "__main__":
    main()
