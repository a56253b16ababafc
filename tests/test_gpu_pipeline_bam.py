"""-m gpu: the BAM mode of nvb_pipeline (StreamingBam) against the direct chain on the same batch and device: seed_extend(traceback=True,
mapq=...) / seed_extend_paired(traceback=True, mapq=...) -> finish_alignments -> bam_records [-> bgzf_compress].  Without compression the
payload is byte-identical to the records; with it, to bgzf_compress of them, and it inflates to them.  Single end and paired (FR; RF with
--no-overlap, --no-mixed and discordant pairs, rescued mates present), LOCAL and SEMI_GLOBAL, the constant and the quality-table scheme,
2- and 4-bit reads with N, mixed lengths, names of 1, 254 and more bytes, contigs cut under alignments, short last batches and a batch
where nothing aligns; depth 1-3, waits out of order, a slot reused without a wait, two compute streams; write_bam of the batches read
back through gzip and htslib (where oracle/_ref is built).  Also the device-count BGZF hook against nvb_bgzf_compress."""
import ctypes as C
import gzip
import zlib
import numpy as np
import pytest
import torch
import nvbio_b200 as nb
from nvbio_b200 import aln, synth
from nvbio_b200._lib import lib, check, BgzfOutStruct
from nvbio_b200.pipeline import MapqParams
from nvbio_b200.strings import PackedStringSet
from oracle.ref_bam import RefBam
from tests.gpu_util import require_gpu, host_u32

pytestmark = pytest.mark.gpu

G = 400_000
L = 150


@pytest.fixture(scope="module")
def world():
    require_gpu()
    gw = synth.random_genome_words(G, seed=4711)
    fmi, _ = nb.FMIndexDevice.from_text(gw, G)
    w = host_u32(gw)
    gsym = ((w[:, None] >> (30 - 2 * np.arange(16, dtype=np.uint32))) & 3).reshape(-1)[:G].astype(np.uint8)
    # contigs every ~1 kbp: about one 150 bp alignment in seven crosses a boundary
    cuts = np.unique(np.concatenate([np.arange(997, G, 997), np.random.default_rng(5).integers(1, G, 50)]))
    cb = np.concatenate([[0], cuts, [G]])
    contigs = nb.ContigTable(["chr%d" % i for i in range(len(cb) - 1)], np.diff(cb))
    return dict(gw=gw, fmi=fmi, gsym=gsym, contigs=contigs)


def revcomp(s):
    return np.where(s < 4, 3 - s, s)[::-1]


def pack_rows(sym, bits):
    """[n, L] symbols -> [n, wpr] big-endian words (int32 bit patterns), padded with zero symbols"""
    spw = 32 // bits
    n, ln = sym.shape
    wpr = -(-ln // spw)
    s = np.zeros((n, wpr * spw), np.uint32)
    s[:, :ln] = sym
    sh = (32 - bits - bits * np.arange(spw, dtype=np.uint32)).astype(np.uint32)
    return (s.reshape(n, wpr, spw) << sh).sum(axis=2, dtype=np.uint64).astype(np.uint32).view(np.int32)


def se_reads(gsym, n, rng, n_frac=0.0):
    pos = rng.integers(0, G - L, n)
    r = np.stack([gsym[p:p + L] for p in pos])
    sub = rng.random(r.shape) < 0.02
    r = np.where(sub, (r + rng.integers(1, 4, r.shape)) & 3, r).astype(np.uint8)
    r = np.stack([revcomp(x) if i % 2 else x for i, x in enumerate(r)])
    if n_frac:
        r[rng.random(r.shape) < n_frac] = 4
    return r


def pe_reads(gsym, n_pairs, rng, orientation, n_frac=0.0):
    """mate 1 of every pair, then mate 2; fragments 250-420 bp (a max_frag of 330 leaves some pairs apart), every 11th pair's mates
    20-70 kbp apart"""
    m1, m2 = [], []
    for i in range(n_pairs):
        frag = int(rng.integers(250, 420))
        p = int(rng.integers(0, G - frag))
        a, b = gsym[p:p + L].copy(), gsym[p + frag - L:p + frag].copy()
        if i % 7 == 3:                                               # a mate with many substitutions: rescue material
            b = np.where(rng.random(L) < 0.15, (b + 1) & 3, b).astype(np.uint8)
        elif i % 11 == 5:                                            # mates far apart: no rescue reaches them, so a discordant pair
            q = (p + 20_000 + int(rng.integers(0, 50_000))) % (G - L)
            b = gsym[q:q + L].copy()
        if orientation == "fr":
            x, y = a, revcomp(b)
        else:
            x, y = revcomp(a), b
        if i % 2:
            x, y = y, x
        m1.append(x); m2.append(y)
    r = np.stack(m1 + m2).astype(np.uint8)
    r = np.where(rng.random(r.shape) < 0.01, (r + 1) & 3, r).astype(np.uint8)
    if n_frac:
        r[rng.random(r.shape) < n_frac] = 4
    return r


def names_for(k, rng, tag):
    out = []
    for i in range(k):
        ln = (1, 254, 300, 12)[i % 4] if i % 5 == 0 else 8
        out.append(("%s%d_" % (tag, i) + "x" * ln)[:ln] if ln != 8 else "%s%05d" % (tag, i))
    return out


class Case:
    def __init__(self, paired, typ, qual, bits, lengths, policy="fr", overlap=True, mixed=True, discordant=False):
        self.paired, self.typ, self.qual, self.bits, self.lengths = paired, typ, qual, bits, lengths
        self.pair = nb.PairParams(min_frag=0, max_frag=330 if policy == "rf" else 500, min_mate_score=50, rescue_capacity=4096,
                                  policy=policy, overlap=overlap, mixed=mixed, discordant=discordant) if paired else None

    def params(self, quals=None):
        if self.qual:
            scheme = aln.QualityGotohScheme(2 if self.typ == aln.LOCAL else 0, 2, 6, 5, 3, 5, 3)
        else:
            scheme = aln.SimpleGotohScheme(2, -2, -5, -3) if self.typ == aln.LOCAL else aln.SimpleGotohScheme(0, -6, -5, -3)
        return nb.SeedExtendParams(seed_len=20, seed_interval=10, band_len=31, type=self.typ, both_strands=True, max_seed_hits=50,
                                   scheme=scheme, read_quals=quals)

    def mapq(self):
        return MapqParams.local(L) if self.typ == aln.LOCAL else MapqParams.end_to_end(L)


CASES = {
    "se-local-2bit": Case(False, aln.LOCAL, False, 2, True),
    "se-semiglobal-qual-4bit": Case(False, aln.SEMI_GLOBAL, True, 4, False),
    "pe-fr-local": Case(True, aln.LOCAL, False, 2, False),
    "pe-rf-nooverlap-nomixed-discordant-qual-4bit": Case(True, aln.LOCAL, True, 4, True, policy="rf", overlap=False, mixed=False, discordant=True),
}


def make_batches(w, case, rng, max_reads, n_batches):
    """(symbols, lengths, quals, names) per batch: a first batch that aligns nowhere, full batches, a short last batch"""
    out = []
    for b in range(n_batches):
        n = max_reads if b < n_batches - 1 else max_reads // 2 + 2
        if case.paired:
            sym = pe_reads(w["gsym"], n // 2, rng, case.pair.policy, 0.004 if case.bits == 4 else 0.0)
        else:
            sym = se_reads(w["gsym"], n, rng, 0.004 if case.bits == 4 else 0.0)
        if b == 0:
            sym = np.zeros_like(sym)                                        # poly-A: no seed occurs in the random genome, nothing aligns
        lens = rng.integers(60, L + 1, n).astype(np.uint32) if case.lengths else None
        if lens is not None:
            lens[::5] = L
        k = n // 2 if case.paired else n
        out.append(dict(n=n, sym=sym, lens=lens, names=names_for(k, rng, "b%d_" % b)))
    return out


def direct(w, case, bt, words, stride, quals_host, max_reads):
    """the Python chain on one batch: (records bytes, BGZF bytes, counts, n_hits, n_rescue, pair flags)"""
    n = bt["n"]
    dw = torch.from_numpy(np.ascontiguousarray(words)).cuda()
    lens = torch.from_numpy(bt["lens"].view(np.int32)).cuda() if bt["lens"] is not None else None
    rs = PackedStringSet(words=dw.reshape(-1), bits=case.bits, big_endian=True, offsets=None, lengths=lens, stride=stride, length=L, count=n)
    q = torch.from_numpy(quals_host.reshape(-1)).cuda() if case.qual else None
    params = case.params(q)
    hc = 32 * max_reads + 1024
    names = [nm[:254] for nm in bt["names"]]                            # nvb_bam_records cuts longer names there
    if case.paired:
        ws = nb.seed_extend_paired(w["fmi"], w["gw"], rs, params, case.pair, mapq=case.mapq(), traceback=True, hit_capacity=hc)
        f = nb.finish_alignments(w["gw"], rs, ws.mate_ops, ws.mate_n_ops, ws.mate_begin, ws.mate_strand, genome_len=G)
    else:
        ws = nb.seed_extend(w["fmi"], w["gw"], rs, params, traceback=True, mapq=case.mapq(), hit_capacity=hc)
        f = nb.finish_alignments(w["gw"], rs, ws.best_ops, ws.best_n_ops, ws.best_begin, ws.best_strand, genome_len=G)
    recs = nb.bam_records(ws, f, rs, w["contigs"], names, quals=q)
    z = nb.bgzf_compress(recs)
    torch.cuda.synchronize()
    raw = recs.to_bytes()
    assert recs.stored() == recs.offsets.numel() - 1
    return dict(raw=raw, z=z.to_bytes(), counts=tuple(int(v) for v in recs.counts.cpu()), n_hits=tuple(int(v) for v in ws.n_hits.cpu()[:3]),
                n_rescue=tuple(int(v) for v in ws.n_rescue.cpu()) if case.paired else None,
                flags=ws.pair_flags.cpu().numpy() if case.paired else None)


def check_batch(got, want, compress):
    assert got.compressed == compress
    assert got.counts == want["counts"] and got.n_records == want["counts"][0]
    assert got.n_hits == want["n_hits"] and got.n_rescue == want["n_rescue"]
    assert got.record_bytes == len(want["raw"])
    pay = got.to_bytes()
    if compress:
        assert pay == want["z"]
        assert gzip.decompress(pay) == want["raw"]
        assert got.n_blocks == -(-len(want["raw"]) // 0xFF00)
    else:
        assert pay == want["raw"] and got.n_blocks == 0


@pytest.mark.parametrize("compress", [True, False])
@pytest.mark.parametrize("name", list(CASES))
def test_pipeline_equals_direct_chain(world, name, compress, tmp_path, monkeypatch):
    w, case = world, CASES[name]
    rng = np.random.default_rng(zlib.crc32(name.encode()) % 1000 + compress)
    max_reads = 480
    depth = {"se-local-2bit": 2, "se-semiglobal-qual-4bit": 3, "pe-fr-local": 1}.get(name, 3)
    if name.startswith("pe-rf"):
        monkeypatch.setenv("NVB_PIPELINE_COMPUTE_STREAMS", "2")
    batches = make_batches(w, case, rng, max_reads, 2 * depth + 2)     # batch 2 * depth reuses the unwaited slot
    spw = 32 // case.bits
    wpr = -(-L // spw)
    stride = wpr * spw
    words = [pack_rows(bt["sym"], case.bits) for bt in batches]
    quals = [rng.integers(2, 41, (bt["n"], stride)).astype(np.uint8) for bt in batches]
    st = nb.StreamingBam(w["fmi"], w["gw"], case.params(), max_reads, L, wpr, w["contigs"], case.mapq(), pair=case.pair, quals=case.qual,
                         lengths=case.lengths, compress=compress, depth=depth, bits=case.bits, max_name_bytes=max_reads * 300)
    assert st.slot_bytes > 0

    def submit(i):
        bt = batches[i]
        return st.submit(torch.from_numpy(words[i]).pin_memory() if i % 2 else words[i], bt["names"],
                         quals=quals[i] if case.qual else None, lengths=bt["lens"], n=bt["n"])

    got = {}
    # depth batches in flight, waited newest first; then a slot reused without a wait (the batch's payload is fetched by that submit)
    tickets = [submit(i) for i in range(depth)]
    for i in reversed(range(depth)):
        got[i] = st.result(tickets[i])
        want = direct(w, case, batches[i], words[i], stride, quals[i], max_reads)
        check_batch(got[i], want, compress)
        got[i] = (got[i], want)
    skipped = submit(depth)                       # never waited for
    for i in range(depth + 1, len(batches)):
        t = submit(i)
        r = st.result(t)
        want = direct(w, case, batches[i], words[i], stride, quals[i], max_reads)
        check_batch(r, want, compress)
        got[i] = (r, want)
        if i == depth + 1:
            got[i] = (nb.BamBatch(**{**r.__dict__, "payload": r.payload.clone()}), want)    # outlives later submits
    assert skipped is not None
    empty = [g for i, g in got.items() if i == 0]
    assert empty and empty[0][0].counts[1] == 0                      # the random batch: nothing aligned
    counts = np.sum([g[0].counts for i, g in got.items() if i != 0], axis=0)
    assert counts[1] > 0.5 * counts[0] and counts[2] > 0, counts      # mapped records; spans cut by a contig boundary
    if case.paired:
        flags = np.concatenate([g[1]["flags"] for g in got.values()])
        assert ((flags & 6) != 0).sum() > 0, "no rescued mate"
        if case.pair.discordant:
            assert (flags == 8).sum() > 0, "no discordant pair"
    # the batches waited last written by write_bam: gzip (and htslib) read back the records of every batch in order
    keep = [got[i] for i in sorted(got) if i >= depth + 1]
    p = str(tmp_path / "out.bam")
    hdr = nb.bam_header(w["contigs"])
    nb.write_bam(p, hdr, [keep[0][0]])
    assert gzip.open(p).read() == hdr + keep[0][1]["raw"]
    if RefBam.available():
        text = RefBam().format(p)
        assert text.count("\n") == keep[0][1]["counts"][0]
    st.close()


def test_depth_and_out_of_order_single_stream(world):
    """single end at depth 1, 2 and 3 over depth + 2 batches each, waited in reverse order: every payload equals the direct chain's"""
    w, case = world, CASES["se-local-2bit"]
    rng = np.random.default_rng(99)
    wpr, stride = -(-L // 16), -(-L // 16) * 16
    for depth in (1, 2, 3):
        batches = make_batches(w, case, rng, 200, depth + 2)
        words = [pack_rows(bt["sym"], 2) for bt in batches]
        st = nb.StreamingBam(w["fmi"], w["gw"], case.params(), 200, L, wpr, w["contigs"], case.mapq(), lengths=True, depth=depth,
                             max_name_bytes=200 * 300)
        pending = []
        for i, bt in enumerate(batches):
            if len(pending) == depth:
                for j, t in reversed(pending):
                    check_batch(st.result(t), direct(w, case, batches[j], words[j], stride, None, 200), True)
                pending = []
            pending.append((i, st.submit(words[i], bt["names"], lengths=bt["lens"], n=bt["n"])))
        for j, t in reversed(pending):
            check_batch(st.result(t), direct(w, case, batches[j], words[j], stride, None, 200), True)
        st.close()


def _dc_bgzf(data, count, bound):
    d_n = torch.tensor([count], dtype=torch.int64, device="cuda")
    nbk = -(-bound // 0xFF00)
    out = torch.empty(max(65311 * nbk, 16), dtype=torch.uint8, device="cuda")
    offs = torch.full((nbk + 1,), -1, dtype=torch.int64, device="cuda")
    o = BgzfOutStruct(); o.d_out, o.capacity, o.d_block_offsets = out.data_ptr(), 65311 * nbk, offs.data_ptr()
    tb = C.c_size_t(0)
    f = lib().nvb_debug_bgzf_compress_device_count
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    r = f(C.c_void_p(data.data_ptr()), C.c_void_p(d_n.data_ptr()), C.c_uint64(bound), C.byref(o), None, C.byref(tb), st)
    assert r == -2
    temp = torch.empty(max(tb.value, 1), dtype=torch.uint8, device="cuda")
    check(f(C.c_void_p(data.data_ptr()), C.c_void_p(d_n.data_ptr()), C.c_uint64(bound), C.byref(o), C.c_void_p(temp.data_ptr()), C.byref(tb), st),
          "nvb_debug_bgzf_compress_device_count")
    torch.cuda.synchronize()
    off = offs.cpu().numpy()
    return out, off


@pytest.mark.parametrize("count", [0, 1, 0xFF00 - 1, 0xFF00, 0xFF00 + 1, 10_000_000])
def test_device_count_bgzf_equals_host_count(count):
    require_gpu()
    rng = np.random.default_rng(count % 997)
    bound = count + 5 * 0xFF00 + 12345
    host = np.frombuffer(bytes(range(256)) * (bound // 256 + 1), np.uint8)[:bound].copy()
    host[::7] = rng.integers(0, 256, host[::7].size)                  # part compressible, part noise
    data = torch.from_numpy(host).cuda()
    out, off = _dc_bgzf(data, count, bound)
    want = nb.bgzf_compress(data[:count]) if count else None
    nbk = -(-count // 0xFF00)
    if count:
        wo = want.offsets.cpu().numpy()
        assert np.array_equal(off[:nbk + 1], wo)
        assert out[:int(wo[-1])].cpu().numpy().tobytes() == want.to_bytes()
        assert gzip.decompress(want.to_bytes()) == host[:count].tobytes()
    total = off[nbk]
    assert (off[nbk:] == total).all() and (total == 0) == (count == 0)
    # a device count above the bound is taken as the bound
    if count == 1:
        out2, off2 = _dc_bgzf(data[:0xFF00 + 7].clone(), 10 ** 9, 0xFF00 + 7)
        ref = nb.bgzf_compress(data[:0xFF00 + 7].clone())
        assert np.array_equal(off2, ref.offsets.cpu().numpy()) and out2[:int(off2[-1])].cpu().numpy().tobytes() == ref.to_bytes()
