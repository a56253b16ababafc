"""-m gpu: nvb_sam_format on the device.  The text of every chain equals tests/sam_oracle.py on the same record bytes and, where
oracle/_ref is built, htslib's sam_format1 of the .bam written from them: single end (LOCAL and SEMI_GLOBAL, constant and quality
schemes, 2- and 4-bit reads with N), paired with rescued mates, bam_records_all at k = 8 on a planted repeat family, sort_bam_records of
several batches.  Also: records larger than the write kernel's spans at unaligned offsets, a mid-batch capacity cut, n = 0, a record
corrupted in device memory, and write_sam of the chain read back through htslib."""
import ctypes as C
import numpy as np
import pytest
import torch
import nvbio_b200 as nb
from nvbio_b200 import aln
from nvbio_b200.pipeline import MapqParams
from nvbio_b200._lib import lib, SamOutStruct
from oracle.ref_bam import RefBam
from tests import sam_oracle as so
from tests.gpu_util import require_gpu
from tests.golden.make_sam_golden import record, int_tag, z_tag, edge_records, REF_NAMES, REF_LENGTHS
from tests.test_gpu_bam import planted_contigs
from tests.test_gpu_finish import se_world, read_set  # noqa: F401  (the single-end world fixture)
from tests.test_gpu_paired_traceback import world, run as run_paired  # noqa: F401  (the paired world fixture)
from tests.test_gpu_bam_sort import chain_records
from tests.test_gpu_all import setup  # noqa: F401  (the repeat-family fixture)


def check_text(t: nb.SamText, data: bytes, offsets, contigs, tmp_path=None):
    """the device lines equal the restatement's (and htslib's, where built); returns the text"""
    torch.cuda.synchronize()
    want, bad = so.text(data, offsets, contigs.names)
    off = t.offsets.cpu().numpy()
    text = t.data[:int(off[-1])].cpu().numpy().tobytes()
    assert t.rejected.cpu().numpy().view(np.uint32).tolist() == bad == [0, 0xFFFFFFFF]
    assert t.stored() == len(want)
    assert [text[off[i]:off[i + 1]] for i in range(len(want))] == want
    if tmp_path is not None and RefBam.available():
        p = str(tmp_path / "r.bam")
        nb.write_bam(p, nb.bam_header(contigs), [data])
        assert RefBam().format(p).encode() == text
    return text


def host(recs):
    torch.cuda.synchronize()
    return recs.to_bytes(), recs.offsets.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("bits", [2, 4])
def test_single_end(se_world, bits, tmp_path):
    w = se_world
    rng = np.random.default_rng(121 + bits)
    reads = [r.copy() for r in w["reads"]]
    if bits == 4:
        for r in reads:
            r[rng.random(len(r)) < 0.005] = 4
    rs = read_set(reads, bits)
    q = torch.from_numpy(np.concatenate(w["quals"])).cuda()
    names = nb.numbered_names(len(reads), "se%d_" % bits)
    for typ in (aln.LOCAL, aln.SEMI_GLOBAL):
        for qual in (False, True):
            scheme = aln.QualityGotohScheme(2 if typ == aln.LOCAL else 0, 2, 6, 5, 3, 5, 3) if qual else \
                aln.SimpleGotohScheme(2, -2, -5, -3) if typ == aln.LOCAL else aln.SimpleGotohScheme(0, -6, -5, -3)
            params = nb.SeedExtendParams(seed_len=20, seed_interval=10, band_len=31, type=typ, both_strands=True, max_seed_hits=50,
                                         scheme=scheme, read_quals=q if qual else None)
            mq = MapqParams.local(160) if typ == aln.LOCAL else MapqParams.end_to_end(160)
            ws = nb.seed_extend(w["fmi"], w["gw"], rs, params, traceback=True, mapq=mq, hit_capacity=64 * len(reads))
            f = nb.finish_alignments(w["gw"], rs, ws.best_ops, ws.best_n_ops, ws.best_begin, ws.best_strand, genome_len=w["G"])
            torch.cuda.synchronize()
            contigs = planted_contigs(ws.best_begin.cpu().numpy().view(np.uint32), ws.best_n_ops.cpu().numpy(), w["G"], rng)
            recs = nb.bam_records(ws, f, rs, contigs, names, quals=q if qual else None)
            t = nb.sam_text(recs, contigs)
            data, off = host(recs)
            text = check_text(t, data, off, contigs, tmp_path if qual else None)
            if typ == aln.LOCAL and qual:
                # write_sam of the chain reads back through htslib (sam_open reads SAM text) as the same lines
                p = str(tmp_path / "se.sam")
                hdr = nb.sam_header(contigs)
                assert nb.write_sam(p, hdr, [t]) == len(hdr) + len(text)
                if RefBam.available():
                    assert RefBam().format(p).encode() == text


@pytest.mark.gpu
def test_paired_and_capacity_cut(world, tmp_path):
    w = world
    pair = nb.PairParams(min_frag=0, max_frag=420, min_mate_score=50)
    got, ws = run_paired(w, pair, qual=True, mapq=MapqParams.local(120))
    assert ((got["pair_flags"] == 2) | (got["pair_flags"] == 4)).sum() > 0
    lens = np.array([len(r) for r in w["reads"]], np.uint32)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint32)
    rs = nb.PackedStringSet.from_symbols(np.concatenate(w["reads"]), offs, lens, bits=2, big_endian=True)
    G = int(w["idx"].n)
    f = nb.finish_alignments(w["gw"], rs, ws.mate_ops, ws.mate_n_ops, ws.mate_begin, ws.mate_strand, genome_len=G)
    torch.cuda.synchronize()
    contigs = planted_contigs(ws.mate_begin.reshape(-1, 2).cpu().numpy().view(np.uint32), ws.mate_n_ops.reshape(-1).cpu().numpy(), G,
                              np.random.default_rng(3))
    q = torch.from_numpy(np.concatenate(w["quals"])).cuda()
    recs = nb.bam_records(ws, f, rs, contigs, nb.numbered_names(w["n_pairs"], "pair"), quals=q)
    data, roff = host(recs)
    t = nb.sam_text(recs, contigs)
    text = check_text(t, data, roff, contigs, tmp_path)
    # a capacity that cuts mid-batch stores exactly the lines that fit, equal to the uncut prefix; offsets complete
    off = t.offsets.cpu().numpy()
    cap = int(off[len(off) // 2] + 7)
    cut = nb.sam_text(recs, contigs, capacity=cap)
    torch.cuda.synchronize()
    k = int(np.searchsorted(off[1:], cap, side="right"))
    assert torch.equal(cut.offsets, t.offsets) and cut.stored() == k
    assert cut.to_bytes() == text[:int(off[k])]
    with pytest.raises(ValueError):
        nb.write_sam(str(tmp_path / "cut.sam"), nb.sam_header(contigs), [cut])


@pytest.mark.gpu
def test_all_k8(setup, tmp_path):
    """bam_records_all at k = 8 on the planted repeat family: primary and secondary records with NH"""
    from tests.test_gpu_all import make_reads, packed, run, LOCAL, N_GENOME
    O, g, gw, idx, fmi = setup
    reads = make_reads(g, n_reads=300, seed=68)
    rs = packed(reads, bits=2, L=100)
    params = nb.SeedExtendParams(**LOCAL, scheme=aln.SimpleGotohScheme(2, -2, -5, -3))
    al = run(fmi, gw, rs, params, MapqParams.local(100), 8)
    cb = [0, 20_300, 40_000, 60_590, 100_010, 150_000, N_GENOME]
    contigs = nb.ContigTable(["c%d" % i for i in range(len(cb) - 1)], list(np.diff(cb)))
    f = nb.finish_alignments(gw, al.strings(rs), al.ops, al.n_ops, al.begin, al.strand, genome_len=N_GENOME)
    recs = nb.bam_records_all(al, f, rs, contigs, ["r%d" % i for i in range(len(reads))])
    data, off = host(recs)
    text = check_text(nb.sam_text(recs, contigs), data, off, contigs, tmp_path)
    lines = text.split(b"\n")[:-1]
    assert sum(int(ln.split(b"\t")[1]) & 0x100 != 0 for ln in lines) > 50 and all(b"\tNH:i:" in ln for ln in lines if not int(ln.split(b"\t")[1]) & 4)


@pytest.mark.gpu
def test_sorted_batches(se_world, tmp_path):
    """sort_bam_records of several batches, then sam_text with the coordinate-sorted header"""
    b2, contigs = chain_records("se", se_world, 2, False)
    b4, _ = chain_records("se", se_world, 4, True)
    s = nb.sort_bam_records([b2, b4, b2])
    torch.cuda.synchronize()
    text = check_text(nb.sam_text(s, contigs), s.to_bytes(), s.offsets.cpu().numpy(), contigs, tmp_path)
    assert nb.sam_header(contigs, sort_order="coordinate").startswith("@HD\tVN:1.0\tSO:coordinate\n")
    pos = [(int(ln.split(b"\t")[2][1:]) if ln.split(b"\t")[2] != b"*" else 1 << 40, int(ln.split(b"\t")[3])) for ln in text.split(b"\n")[:-1]]
    assert pos == sorted(pos)


def _format(data: torch.Tensor, offsets: torch.Tensor, names, n, capacity, text):
    """one raw nvb_sam_format call: (offsets, rejected) tensors"""
    raw = [nm.encode() for nm in names]
    dn = torch.frombuffer(bytearray(b"".join(raw)), dtype=torch.uint8).cuda()
    dno = torch.from_numpy(np.concatenate([[0], np.cumsum([len(x) for x in raw])]).astype(np.int32)).cuda()
    out_off = torch.full((n + 1,), -1, dtype=torch.int64, device="cuda")
    rej = torch.full((2,), 7, dtype=torch.int32, device="cuda")
    o = SamOutStruct()
    o.d_text, o.capacity, o.d_offsets, o.d_rejected = text.data_ptr() if text is not None else None, capacity, out_off.data_ptr(), rej.data_ptr()
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    args = (C.c_void_p(data.data_ptr()), C.c_void_p(offsets.data_ptr()), C.c_uint32(n), C.c_void_p(dn.data_ptr()), C.c_void_p(dno.data_ptr()),
            C.c_uint32(len(names)), C.byref(o))
    tb = C.c_size_t(0)
    err = lib().nvb_sam_format(*args, None, C.byref(tb), s)
    assert err == (0 if n == 0 else -2)
    temp = torch.empty(max(tb.value, 1), dtype=torch.uint8, device="cuda")
    assert lib().nvb_sam_format(*args, C.c_void_p(temp.data_ptr()), C.byref(tb), s) == 0
    torch.cuda.synchronize()
    return out_off.cpu().numpy(), rej.cpu().numpy().view(np.uint32).tolist()


@pytest.mark.gpu
def test_large_records_corruption_and_n_zero():
    """25 kbp unaligned reads (records and lines larger than the write kernel's spans) among the edge records, at an odd byte offset and
    written to an odd text address; a record whose tag type byte is corrupted in device memory is rejected without disturbing the other
    lines; n = 0 writes offsets[0] = 0 and rejected = (0, 0xFFFFFFFF)"""
    require_gpu()
    rng = np.random.default_rng(9)
    big = [record(b"long%d" % i, flag=4, seq=[int(x) for x in rng.integers(0, 16, 25_000 + i)],
                  qual=bytes(int(x) for x in rng.integers(0, 60, 25_000 + i)), tags=int_tag("NM", "C", i) + z_tag("MD", b"25000"))
           for i in range(3)]
    edges = edge_records()
    recs = edges[:4] + [big[0]] + edges[4:9] + big[1:] + edges[9:] * 20
    base = 3
    raw = b"\0" * base + b"".join(recs)
    data = torch.frombuffer(bytearray(raw), dtype=torch.uint8).cuda()
    off_h = (np.concatenate([[0], np.cumsum([len(r) for r in recs])]) + base).astype(np.int64)
    offsets = torch.from_numpy(off_h).cuda()
    want, bad = so.text(raw, off_h, REF_NAMES)
    total = sum(len(x) for x in want)
    assert max(len(x) for x in want) > 50_000 and max(len(r) for r in recs) > 37_000
    text = torch.full((total + 64,), 0x5A, dtype=torch.uint8, device="cuda")
    n = len(recs)
    o, rej = _format(data, offsets, REF_NAMES, n, total, text[5:])
    got = text[5:5 + total].cpu().numpy().tobytes()
    assert rej == bad == [0, 0xFFFFFFFF] and got == b"".join(want) and (text[5 + total:] == 0x5A).all() and (text[:5] == 0x5A).all()
    # corrupt the type byte of the first tag of record 10 (the int_tags record) in device memory
    k = 10
    aux = so_aux(recs[k])
    data[int(off_h[k]) + aux + 2] = ord("q")
    o2, rej2 = _format(data, offsets, REF_NAMES, n, total, text)
    got2 = [text[int(o2[i]):int(o2[i + 1])].cpu().numpy().tobytes() for i in range(n)]
    assert rej2 == [1, k] and got2[k] == b"" and got2[:k] + got2[k + 1:] == want[:k] + want[k + 1:]
    # n = 0
    o3, rej3 = _format(data, offsets, REF_NAMES, 0, 0, None)
    assert o3[0] == 0 and rej3 == [0, 0xFFFFFFFF]


def so_aux(rec: bytes) -> int:
    """byte offset of a record's first tag"""
    import struct
    l_name = rec[12]
    nc = struct.unpack_from("<H", rec, 16)[0]
    l_seq = struct.unpack_from("<I", rec, 20)[0]
    return 36 + l_name + 4 * nc + (l_seq + 1) // 2 + l_seq
