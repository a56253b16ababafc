"""-m gpu: nvb_bam_sort and nvb_bam_index on the device.  Sort: bytes, offsets and order equal Python's stable sort of the host bytes on the
single-end and paired seed + extend -> finish -> BAM records chains (2- and 4-bit reads, with and without qualities) and on synthetic
streams (the BAI cases of tests/golden/make_bai_golden.py, ties in the thousands, pos 0 and contig ends, records larger than the staging
span, n = 0 and 1, all unplaced, a list of three batches, a capacity that cuts mid-stream); repeated calls and a side stream give the same
bytes.  Index: byte-equal to tests/bai_oracle.py on every case through the real bgzf_compress; a shuffled input gives status 1.  End to
end, where oracle/_ref is built: write_sorted_bam reads back through htslib as the unsorted file's SAM lines reordered, htslib indexes it
like we do up to the two deviations, and htslib's region queries through our .bai return the brute-force overlap sets."""
import gzip
import shutil
import numpy as np
import pytest
import torch
import ctypes as C
import nvbio_b200 as nb
from nvbio_b200 import aln
from nvbio_b200.pipeline import MapqParams
from nvbio_b200._lib import lib, check, BamSortOutStruct
from oracle.ref_bam import RefBam
from oracle.ref_bai import RefBai
from tests import bai_oracle as bo
from tests.gpu_util import require_gpu
from tests.golden.make_bai_golden import cases, record, unmapped
from tests.test_gpu_finish import se_world, read_set  # noqa: F401  (the single-end world fixture)
from tests.test_gpu_paired_traceback import world, run as run_paired  # noqa: F401  (the paired world fixture)

CASES = cases()


def as_batch(recs) -> nb.BamRecords:
    raw = b"".join(recs)
    off = np.concatenate([[0], np.cumsum([len(r) for r in recs])]).astype(np.int64)
    data = torch.frombuffer(bytearray(raw), dtype=torch.uint8).cuda() if raw else torch.empty(0, dtype=torch.uint8, device="cuda")
    return nb.BamRecords(data=data, offsets=torch.from_numpy(off).cuda(), counts=torch.zeros(4, dtype=torch.int32, device="cuda"))


def check_sort(recs, s=None):
    if s is None:
        s = nb.sort_bam_records(as_batch(recs))
    torch.cuda.synchronize()
    order, srt = bo.sort_records(recs)
    assert s.order.cpu().tolist() == order
    assert s.offsets.cpu().tolist() == np.concatenate([[0], np.cumsum([len(r) for r in srt])]).astype(np.int64).tolist()
    assert s.to_bytes() == b"".join(srt)
    return srt


def contig_table(lens):
    return nb.ContigTable(["c%d" % i for i in range(len(lens))], lens)


def check_index(recs, lens, header_bytes=1234):
    s = nb.sort_bam_records(as_batch(recs))
    blocks = nb.bgzf_compress(s.data[:int(s.offsets[-1])])
    got = nb.bam_index(s, blocks, header_bytes, contig_table(lens))
    _, srt = bo.sort_records(recs)
    want = bo.bai_bytes(srt, blocks.offsets.cpu().numpy(), header_bytes, len(lens))
    assert got == want
    return got


def chain_records(kind, w, bits=2, qual=False):
    if kind == "se":
        rng = np.random.default_rng(41 + bits)
        reads = [r.copy() for r in w["reads"]]
        if bits == 4:
            for r in reads:
                r[rng.random(len(r)) < 0.005] = 4
        rs = read_set(reads, bits)
        q = torch.from_numpy(np.concatenate(w["quals"])).cuda() if qual else None
        params = nb.SeedExtendParams(seed_len=20, seed_interval=10, band_len=31, type=aln.LOCAL, both_strands=True, max_seed_hits=50,
                                     scheme=aln.SimpleGotohScheme(2, -2, -5, -3))
        ws = nb.seed_extend(w["fmi"], w["gw"], rs, params, traceback=True, mapq=MapqParams.local(160), hit_capacity=64 * len(reads))
        f = nb.finish_alignments(w["gw"], rs, ws.best_ops, ws.best_n_ops, ws.best_begin, ws.best_strand, genome_len=w["G"])
        contigs = nb.ContigTable(["c0", "c1", "c2"], [w["G"] // 3, w["G"] // 3, w["G"] - 2 * (w["G"] // 3)])
        return nb.bam_records(ws, f, rs, contigs, nb.numbered_names(len(reads), "se"), quals=q), contigs
    pair = nb.PairParams(min_frag=0, max_frag=420, min_mate_score=50)
    _, ws = run_paired(w, pair, qual=qual, mapq=MapqParams.local(120))
    lens = np.array([len(r) for r in w["reads"]], np.uint32)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint32)
    rs = nb.PackedStringSet.from_symbols(np.concatenate(w["reads"]), offs, lens, bits=bits, big_endian=True)
    G = int(w["idx"].n)
    f = nb.finish_alignments(w["gw"], rs, ws.mate_ops, ws.mate_n_ops, ws.mate_begin, ws.mate_strand, genome_len=G)
    contigs = nb.ContigTable(["c0", "c1"], [G // 2, G - G // 2])
    q = torch.from_numpy(np.concatenate(w["quals"])).cuda() if qual else None
    return nb.bam_records(ws, f, rs, contigs, nb.numbered_names(w["n_pairs"], "pair"), quals=q), contigs


@pytest.mark.gpu
@pytest.mark.parametrize("bits", [2, 4])
@pytest.mark.parametrize("qual", [False, True])
def test_sort_and_index_single_end(se_world, bits, qual):
    require_gpu()
    recs, contigs = chain_records("se", se_world, bits, qual)
    raw = bo.split_records(recs.to_bytes())
    check_sort(raw, nb.sort_bam_records(recs))
    check_index(raw, contigs.lengths.tolist())


@pytest.mark.gpu
@pytest.mark.parametrize("qual", [False, True])
def test_sort_and_index_paired(world, qual):
    require_gpu()
    recs, contigs = chain_records("pe", world, 2, qual)
    raw = bo.split_records(recs.to_bytes())
    check_sort(raw, nb.sort_bam_records(recs))
    check_index(raw, contigs.lengths.tolist())


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(CASES))
def test_cases(case):
    require_gpu()
    lens, recs = CASES[case]
    check_sort(recs)
    check_index(recs, lens)


def synthetic():
    rng = np.random.default_rng(7)
    out = {}
    out["ties"] = [record("t%d" % k, int(k % 2), 777, flag=16 * (k % 3 == 0)) for k in range(5000)]
    out["edges"] = [record("e%d" % k, k % 3, p, cigar=((0, 40),)) for k, p in enumerate([0, 9960, 0, 4960, 0, 19960] * 5)]
    big = bytes(rng.integers(33, 120, 40_000, dtype=np.uint8))
    out["large"] = [record("L%d" % k, 0, int(p), cigar=((0, 40_000),), qual=big) for k, p in enumerate(rng.integers(0, 1_000_000, 9))] + \
        [record("s%d" % k, 0, int(p)) for k, p in enumerate(rng.integers(0, 1_000_000, 500))]
    out["one"] = [record("one", 1, 5)]
    out["unplaced"] = [unmapped("u%d" % k, l_seq=int(k % 150) + 1) for k in range(2000)]
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["ties", "edges", "large", "one", "unplaced"])
def test_synthetic(case):
    require_gpu()
    recs = synthetic()[case]
    lens = [1_000_000, 10_000, 20_000]
    srt = check_sort(recs)
    check_index(recs, lens)
    if case == "ties":
        assert [bo.sort_key(r) for r in srt] == sorted(bo.sort_key(r) for r in recs)


@pytest.mark.gpu
def test_empty_list_capacity_determinism():
    require_gpu()
    e = nb.sort_bam_records(as_batch([]))
    torch.cuda.synchronize()
    assert e.n == 0 and e.offsets.cpu().tolist() == [0] and e.to_bytes() == b""
    assert check_index([], [100, 200]) == bo.bai_bytes([], [0], 1234, 2)
    lens, recs = CASES["one_contig_unplaced"]
    thirds = [recs[:1000], recs[1000:1001], recs[1001:]]
    s = nb.sort_bam_records([as_batch(t) for t in thirds])
    check_sort(recs, s)
    # a capacity that cuts mid-stream: offsets whole, a prefix of the records stored
    b = as_batch(recs)
    n, cap = len(recs), int(s.offsets[len(recs) // 2]) + 7
    out = torch.full((cap + 64,), 0xAB, dtype=torch.uint8, device="cuda")
    off = torch.empty(n + 1, dtype=torch.int64, device="cuda")
    o = BamSortOutStruct()
    o.d_records, o.capacity, o.d_offsets = out.data_ptr(), cap, off.data_ptr()
    tb = C.c_size_t(0)
    args = (C.c_void_p(b.data.data_ptr()), C.c_void_p(b.offsets.data_ptr()), C.c_uint32(n), C.byref(o))
    assert lib().nvb_bam_sort(*args, None, C.byref(tb), None) == -2
    temp = torch.empty(tb.value, dtype=torch.uint8, device="cuda")
    check(lib().nvb_bam_sort(*args, C.c_void_p(temp.data_ptr()), C.byref(tb), None), "nvb_bam_sort")
    torch.cuda.synchronize()
    assert torch.equal(off, s.offsets)
    k = int(np.searchsorted(off.cpu().numpy()[1:], cap, side="right"))
    stored = int(off[k])
    got = out.cpu().numpy().tobytes()
    assert got[:stored] == s.to_bytes()[:stored] and set(got[stored:]) == {0xAB}
    # repeated calls and a side stream
    a = nb.sort_bam_records(b).to_bytes()
    assert nb.sort_bam_records(b).to_bytes() == a
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        c = nb.sort_bam_records(b, stream=side)
    side.synchronize()
    assert c.to_bytes() == a


@pytest.mark.gpu
def test_unsorted_and_unknown_refs_are_refused():
    require_gpu()
    lens, recs = CASES["one_contig"]
    b = as_batch(recs)                                     # not sorted
    srt = nb.SortedBamRecords(data=b.data, offsets=b.offsets, order=torch.arange(len(recs), dtype=torch.int32, device="cuda"))
    blocks = nb.bgzf_compress(b.data)
    with pytest.raises(ValueError, match="status 1"):
        nb.bam_index(srt, blocks, 100, contig_table(lens))
    s = nb.sort_bam_records(as_batch(synthetic()["edges"]))      # refIDs 0-2
    blocks = nb.bgzf_compress(s.data[:int(s.offsets[-1])])
    with pytest.raises(ValueError, match="status 2"):
        nb.bam_index(s, blocks, 100, contig_table([10_000_000]))
    assert len(nb.bam_index(s, blocks, 100, contig_table([10_000_000] * 3))) > 8


@pytest.mark.gpu
@pytest.mark.skipif(not (RefBam.available() and RefBai.available()), reason="oracle/_ref is not built here")
def test_write_sorted_bam_end_to_end(world, tmp_path):
    require_gpu()
    recs, contigs = chain_records("pe", world, 2, True)
    unsorted_path, path = str(tmp_path / "u.bam"), str(tmp_path / "s.bam")
    nb.write_bam(unsorted_path, nb.bam_header(contigs), [recs])
    nb.write_sorted_bam(path, contigs, recs)
    lines_u, lines_s = RefBam().format(unsorted_path).splitlines(), RefBam().format(path).splitlines()
    assert sorted(lines_u) == sorted(lines_s) and lines_u != lines_s
    assert "\tSO:coordinate\n" in nb.bam.sam_header_text(gzip.decompress(open(path, "rb").read()))
    ours = open(path + ".bai", "rb").read()
    copy = str(tmp_path / "h.bam")
    shutil.copy(path, copy)
    hts = RefBai().index(copy)                             # htslib accepts the order
    a, a_nc, _ = bo.parse_bai(ours)
    b, b_nc, _ = bo.parse_bai(hts)
    assert a == {r: ({k: [tuple(c) for c in v] for k, v in b[r][0].items()}, b[r][1]) for r in b}
    assert b_nc == min(a_nc, 1)
    # region queries through our index against the brute-force overlap sets
    raw = bo.split_records(nb.sort_bam_records(recs).to_bytes())
    fields = [bo.rec_fields(r) for r in raw]
    rng = np.random.default_rng(3)
    qs = []
    for _ in range(1000):
        t = int(rng.integers(0, len(contigs.names)))
        beg = int(rng.integers(0, int(contigs.lengths[t])))
        qs.append((t, beg, beg + int(rng.integers(1, 5000))))
    for t, ln in enumerate(contigs.lengths.tolist()):
        qs += [(t, 0, 1), (t, ln - 1, ln), (t, 0, ln), (t, ln - 200, ln + 1000)]
    for t, beg, end in qs:
        want = sorted(lines_s[i] for i, (ref, pos, e, _, _) in enumerate(fields) if ref == t and pos < end and e > beg)
        assert sorted(RefBai().query(path, t, beg, end)) == want, (t, beg, end)
