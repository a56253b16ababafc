"""CPU: nvb_sam_format's per-record routines (sam_core.cuh), compiled for the host by tests/host/sam_harness.cu, against the restatement in
tests/sam_oracle.py, against tests/bam_oracle.py's SAM lines (which tests/golden/bam.npz pins to htslib) and against htslib's sam_format1
(live where oracle/_ref is built, else tests/golden/sam.npz): records of traced and finished alignments, single end and paired, sorted, and
-k streams with secondary records and NH; hand-built edge records; every rejection condition; a capacity cut; n = 0; the header text;
write_sam read back by htslib; the entry point's argument checks."""
import ctypes as C
import os
import struct
import subprocess
import numpy as np
import pytest
from oracle.ref_bam import RefBam
from nvbio_b200 import bam as nbam
from nvbio_b200 import sam as nsam
from tests import bam_oracle as bo
from tests import sam_oracle as so
from tests.golden.make_bam_golden import fixture_inputs
from tests.golden.make_sam_golden import edge_records, REF_NAMES, REF_LENGTHS, record, int_tag, z_tag
from tests.test_bam_host import traced_inputs, HF, genome, LIVE  # noqa: F401  (HF, genome: fixtures)

HERE = os.path.dirname(os.path.abspath(__file__))


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


@pytest.fixture(scope="module")
def H(tmp_path_factory):
    so_path = str(tmp_path_factory.mktemp("sam_harness") / "libsam_harness.so")
    from nvbio_b200.build import NVCC
    subprocess.check_call([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "-Wno-deprecated-declarations",
                           "-Xcompiler", "-fPIC", "-shared", "-o", so_path, os.path.join(HERE, "host", "sam_harness.cu")])
    return C.CDLL(so_path)


def run_host(H, recs, ref_names, capacity=None, base=0):
    """the harness on a list of record bytes (laid out from byte `base` of the buffer): (text buffer, offsets, rejected)"""
    data = np.frombuffer(b"\0" * base + b"".join(recs) + b"\0", np.uint8).copy()
    off = np.concatenate([[0], np.cumsum([len(r) for r in recs])]).astype(np.uint64) + base
    names = [nm.encode() for nm in ref_names]
    nb = np.frombuffer(b"".join(names) + b"\0", np.uint8).copy()
    no = np.concatenate([[0], np.cumsum([len(x) for x in names])]).astype(np.uint32)
    n = len(recs)
    cap = (5 * len(data)) // 2 + n * 200 if capacity is None else capacity
    text = np.full(cap + 16, 0xA5, np.uint8)
    o = np.zeros(n + 1, np.uint64); rej = np.zeros(2, np.uint32)
    H.hh_sam(_p(data), _p(off), C.c_uint32(n), _p(nb), _p(no), C.c_uint32(len(names)), _p(text), C.c_uint64(cap), _p(o), _p(rej))
    return text, o, rej


def lines_of(text, o):
    return [text[int(o[i]):int(o[i + 1])].tobytes() for i in range(len(o) - 1)]


def check(H, recs, ref_names, want_lines=None):
    """harness == restatement (== want_lines when given), nothing rejected; returns the text"""
    text, o, rej = run_host(H, recs, ref_names)
    got = lines_of(text, o)
    want, bad = so.text(b"".join(recs), np.concatenate([[0], np.cumsum([len(r) for r in recs])]), ref_names)
    assert bad == [0, 0xFFFFFFFF] and rej.tolist() == bad
    assert got == want
    if want_lines is not None:
        assert got == [(s + "\n").encode() for s in want_lines]
    return b"".join(got)


def bam_file(path, ref_names, ref_lengths, recs):
    nbam.write_bam(path, nbam.bam_header(nbam.ContigTable(ref_names, ref_lengths)), [b"".join(recs)])
    return path


# ---- records of the writers' rules -------------------------------------------------------------------------------------------------

def test_golden_bam_records(H):
    """the records of tests/golden/bam.npz (htslib's bytes of bam_oracle's lines: every integer tag edge, 1- and 254-byte names,
    cross-contig mates, both-unmapped pairs, equal begins) format to exactly those lines"""
    g = np.load(os.path.join(HERE, "golden", "bam.npz"))
    lines = str(g["lines"]).split("\n")
    sizes = g["record_sizes"]; raw = g["records"].tobytes()
    recs = [raw[o - s:o] for o, s in zip(np.cumsum(sizes), sizes)]
    names = fixture_inputs(False, 5)["contig_names"]
    check(H, recs, names, lines)


@pytest.mark.parametrize("bits", [2, 4])
@pytest.mark.parametrize("paired", [False, True])
def test_traced_records(H, HF, genome, bits, paired, tmp_path):
    """records of alignments traced by the oracle and finished by the host build of finish (test_bam_host's batches): the line of every
    record is bam_oracle's; htslib's sam_format1 of the .bam agrees where it is built; their coordinate order formats the same lines"""
    rng = np.random.default_rng(70 + 10 * bits + paired)
    for i, (typ, band) in enumerate([(1, 31), (2, 15), (0, 63)]):
        inp = traced_inputs(HF, rng, genome, bits, paired, band=band, typ=typ, quals=i % 2 == 0, mapq=i != 2)
        want, _ = bo.records(inp)
        recs = [w for w, _ in want]
        text = check(H, recs, inp["contig_names"], [s for _, s in want])
        if LIVE:
            p = bam_file(str(tmp_path / "t.bam"), inp["contig_names"], inp["contig_lengths"], recs)
            assert RefBam().format(p).encode() == text
        # coordinate order (refID, pos as unsigned, stable), as nvb_bam_sort gives it
        key = [(struct.unpack_from("<I", r, 4)[0], struct.unpack_from("<I", r, 8)[0]) for r in recs]
        order = sorted(range(len(recs)), key=lambda k: key[k])
        check(H, [recs[k] for k in order], inp["contig_names"], [want[k][1] for k in order])


def test_all_records_with_secondary_and_nh(H, HF, genome):
    """-k streams (nvb_bam_records_all's rule, tests/all_oracle.py): primary and secondary records with NH"""
    from tests.test_all_host import all_inputs
    from tests.all_oracle import all_records
    rng = np.random.default_rng(55)
    secondary = nh = 0
    for bits in (2, 4):
        inp, first = all_inputs(HF, rng, genome, bits, quals=bits == 2, mapq=True)
        want, _ = all_records(inp, first, int(first[-1]))
        check(H, [w for w, _ in want], inp["contig_names"], [s for _, s in want])
        secondary += sum(int.from_bytes(w[18:20], "little") & 0x100 != 0 for w, _ in want)
        nh += sum("\tNH:i:" in s for _, s in want)
    assert secondary > 0 and nh > 0


# ---- hand-built records -----------------------------------------------------------------------------------------------------------

def test_edge_records_match_htslib(H, tmp_path):
    """l_seq 0, QUAL 0xFF, RNEXT naming another contig, POS -1, every CIGAR op, I above 2^31, TLEN = INT_MIN, every integer tag edge:
    the harness equals htslib's text (live where oracle/_ref is built, else tests/golden/sam.npz) and the restatement"""
    recs = edge_records()
    g = np.load(os.path.join(HERE, "golden", "sam.npz"))
    assert g["records"].tobytes() == b"".join(recs)
    want = str(g["text"])
    if LIVE:
        assert RefBam().format(bam_file(str(tmp_path / "e.bam"), REF_NAMES, REF_LENGTHS, recs)) == want
    text = check(H, recs, REF_NAMES, want.split("\n")[:-1])
    for s in (b"\t*\t0\t0\t*\t*\t0\t0\t*\t*\n", b"\t*\t0\t0\t*\tcontig_three\t0\t0\t", b"\t-2147483648\t", b"XS:i:3000000000",
              b"Xl:i:4294967295", b"1M2I3D4N5S6H7P8=9X268435455M"):
        assert s in text, s


def rejected_cases():
    """(what, record bytes) of records nvb_sam_format rejects"""
    good = record(b"bad", ref=0, pos=3, cigar=(4 << 4,), seq=[1, 2, 4, 8], qual=b"\x01\x02\x03\x04", tags=int_tag("NM", "C", 1) + z_tag("MD", b"4"))
    core_end = 36 + 4
    cases = [("extent != block_size + 4", good + b"\0"),
             ("block_size too small", struct.pack("<i", len(good) - 5) + good[4:]),
             ("shorter than the fixed fields", good[:30]),
             ("name runs past the end", good[:12] + struct.pack("<I", (struct.unpack_from("<I", good, 12)[0] & ~0xFF) | 250) + good[16:]),
             ("empty name", record(b"", ref=0, pos=3, seq=[1], qual=b"\x01")),
             ("name not NUL-terminated", good[:core_end - 1] + b"x" + good[core_end:]),
             ("refID below -1", good[:4] + struct.pack("<i", -2) + good[8:]),
             ("refID = n_refs", good[:4] + struct.pack("<i", len(REF_NAMES)) + good[8:]),
             ("next_refID = n_refs", good[:24] + struct.pack("<i", len(REF_NAMES)) + good[28:]),
             ("CIGAR op 9", good[:core_end] + struct.pack("<I", 4 << 4 | 9) + good[core_end + 4:]),
             ("CIGAR runs past the end", good[:16] + struct.pack("<I", 200) + good[20:]),
             ("SEQ / QUAL run past the end", good[:20] + struct.pack("<I", 60) + good[24:]),
             ("tag type A", record(b"bad", seq=[1], qual=b"\x01", tags=b"XAA" + b"x")),
             ("tag type f", record(b"bad", seq=[1], qual=b"\x01", tags=b"XFf" + struct.pack("<f", 1.5))),
             ("tag type B", record(b"bad", seq=[1], qual=b"\x01", tags=b"XBBC" + struct.pack("<I", 1) + b"\x01")),
             ("Z without NUL", record(b"bad", seq=[1], qual=b"\x01", tags=b"MDZ" + b"10A5")),
             ("i runs past the end", record(b"bad", seq=[1], qual=b"\x01", tags=b"NMi" + b"\x01\x02")),
             ("S runs past the end", record(b"bad", seq=[1], qual=b"\x01", tags=int_tag("NM", "C", 1) + b"XSS\x01")),
             ("1 byte after the last tag", record(b"bad", seq=[1], qual=b"\x01", tags=int_tag("NM", "C", 1) + b"X")),
             ("3 bytes after the last tag", record(b"bad", seq=[1], qual=b"\x01", tags=int_tag("NM", "C", 1) + b"XYC"))]
    return good, cases


def test_rejected_records(H):
    """every rejection condition: the record gets a line of 0 bytes, is counted, and its valid neighbours' lines are unchanged"""
    good, cases = rejected_cases()
    neigh = edge_records()
    assert so.line(good, [n.encode() for n in REF_NAMES]) is not None
    want, _ = so.text(b"".join(neigh), np.concatenate([[0], np.cumsum([len(r) for r in neigh])]), REF_NAMES)
    for what, bad in cases:
        assert so.line(bad, [n.encode() for n in REF_NAMES]) is None, what
        for at in (0, 5, len(neigh)):
            recs = neigh[:at] + [bad, bad] + neigh[at:]
            text, o, rej = run_host(H, recs, REF_NAMES, base=3)
            got = lines_of(text, o)
            assert rej.tolist() == [2, at], what
            assert got[at] == got[at + 1] == b"", what
            assert got[:at] + got[at + 2:] == want, what


def test_capacity_stores_exactly_the_prefix(H):
    inp = fixture_inputs(True, 5)
    recs = [w for w, _ in bo.records(inp)[0]]
    full, o, _ = run_host(H, recs, inp["contig_names"])
    cap = int(o[37]) + 5                                     # cuts line 37
    cut, o2, _ = run_host(H, recs, inp["contig_names"], capacity=cap)
    assert np.array_equal(o, o2)
    assert cut[:int(o[37])].tobytes() == full[:int(o[37])].tobytes() and (cut[int(o[37]):] == 0xA5).all()


def test_n_zero(H):
    text, o, rej = run_host(H, [], REF_NAMES)
    assert o.tolist() == [0] and rej.tolist() == [0, 0xFFFFFFFF]


def test_header_is_the_bam_header_text():
    t = nbam.ContigTable(REF_NAMES, REF_LENGTHS)
    for so_ in ("unsorted", "coordinate"):
        h = nsam.sam_header(t, program="prog", sort_order=so_)
        assert nbam.sam_header_text(nbam.bam_header(t, program="prog", sort_order=so_)) == h
        assert h.startswith("@HD\tVN:1.0\tSO:%s\n@SQ\tSN:chr1\tLN:1000\n" % so_) and h.endswith("@PG\tID:prog\tPN:prog\n")
    with pytest.raises(ValueError):
        nsam.sam_header(t, sort_order="random")


def test_write_sam_round_trip(H, tmp_path):
    """write_sam's file is the header then the lines; htslib (where built) reads it back as SAM and formats the same lines"""
    inp = fixture_inputs(True, 5)
    want, _ = bo.records(inp)
    recs = [w for w, _ in want]
    text, o, _ = run_host(H, recs, inp["contig_names"])
    body = text[:int(o[-1])].tobytes()
    t = nbam.ContigTable(inp["contig_names"], inp["contig_lengths"])
    hdr = nsam.sam_header(t, program="test")
    p = str(tmp_path / "out.sam")
    k = int(o[100])
    assert nsam.write_sam(p, hdr, [body[:k], body[k:]]) == len(hdr) + len(body)
    assert open(p, "rb").read() == hdr.encode() + body
    assert body.decode() == "".join(s + "\n" for _, s in want)
    if LIVE:
        assert RefBam().format(p) == body.decode()


def test_argument_validation_without_gpu():
    """nvb_sam_format rejects NULL out / temp_bytes / d_offsets / d_rejected, a NULL d_text with capacity > 0, NULL records with n > 0,
    NULL names with n_refs > 0 and n >= 2^31 - 1 with NVB_E_INVALID (-1) before any CUDA call"""
    from nvbio_b200 import _lib
    from nvbio_b200._lib import SamOutStruct
    L = _lib.lib()

    def good():
        o = SamOutStruct(); o.d_text, o.capacity, o.d_offsets, o.d_rejected = 16, 1 << 20, 16, 16
        return o

    def call(o, n=8, recs=16, offs=16, names=16, name_off=16, n_refs=3, tb=True):
        t = C.c_size_t(0)
        return L.nvb_sam_format(C.c_void_p(recs) if recs else None, C.c_void_p(offs) if offs else None, C.c_uint32(n),
                                C.c_void_p(names) if names else None, C.c_void_p(name_off) if name_off else None, C.c_uint32(n_refs),
                                C.byref(o) if o is not None else None, None, C.byref(t) if tb else None, None)
    assert call(None) == -1 and call(good(), tb=False) == -1
    for f in ("d_offsets", "d_rejected", "d_text"):
        o = good(); setattr(o, f, None); assert call(o) == -1, f
    assert call(good(), recs=0) == -1 and call(good(), offs=0) == -1
    assert call(good(), names=0) == -1 and call(good(), name_off=0) == -1
    assert call(good(), n=0x7FFFFFFF) == -1
