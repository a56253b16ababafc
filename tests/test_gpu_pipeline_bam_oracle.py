"""-m gpu: the BAM mode of nvb_pipeline (StreamingBam) against the host oracle chain (tests/stream_oracle.py), which builds every record
from the batch's host reads, qualities, lengths and names through the stage oracles alone.  tests/test_gpu_pipeline_bam.py compares the
pipeline with the direct device chain, which shares each stage hand-off with it; here each batch is also held to records no device
stage touched, and the direct chain is still compared so that a failure shows which side moved.

  1. small worlds (the 400 kbp genome of test_gpu_pipeline_bam.py, a contig shorter than a read added): single end LOCAL / SEMI_GLOBAL,
     the constant and the quality-table scheme, 2- and 4-bit reads with N, lengths 20 .. read_len, reads past the genome's end; paired
     FR, RF with --no-overlap, FF with discordant pairs and --no-mixed, rescued mates and mates of unequal lengths; batches of 1 (2),
     max_reads - 1 (- 2) and max_reads reads; names that fill max_name_bytes exactly;
  2. the slot layout: a record bound R below the traceback ops O (small max_cigar / max_md, short names), read from the layout itself,
     where nearly every record is unmapped by truncation, and a mix of truncated and whole records; the per-slot pinned payload buffer
     growing under a slot whose other neighbour is unread, results read in reverse and twice; the device-count BGZF with a bound of
     40,000 blocks over 1 and 2 real ones;
  3. bench.py's shape on its 1.9 Gbp index: 4 single-end batches of 250 K reads with qualities and names and 2 batches of 250 K pairs at
     depth 3 on two compute streams, each equal to the direct chain and, on a sample of 2,000 reads (pairs), to the host chain; the
     device memory create takes against depth x slot_bytes; the stream written by write_bam read back through gzip and htslib.

Every case prints its coverage counts (rescued mates, discordant pairs, off-contig and truncated records) and asserts the ones it is
there for."""
import ctypes as C
import gc
import gzip
import struct
import time
import zlib

import numpy as np
import pytest
import torch

import bench
import nvbio_b200 as nb
from nvbio_b200 import aln, synth
from nvbio_b200._lib import lib, check
from nvbio_b200.pipeline import MapqParams
from nvbio_b200.strings import PackedStringSet
from oracle import orc
from oracle.ref_bam import RefBam
from tests import stream_oracle
from tests.gpu_util import require_gpu
from tests.test_gpu_pipeline_bam import world, Case, direct, pack_rows, revcomp, names_for, _dc_bgzf, G, L   # noqa: F401 (fixture)
from tests.test_gpu_headline_chain import H, params as bench_params, contig_table, unpack_rows, N   # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu

BAND = 31
MAX_OPS = 2 * L + BAND                         # StreamingBam's defaults: nothing truncates
SHORT_CONTIG = (200_000, 200_060)              # a contig shorter than a read


# ---------------------------------------------------------------------------------------------------------------------------------------
# records: split, compare field by field
# ---------------------------------------------------------------------------------------------------------------------------------------
def split(raw):
    """the records of a BAM record stream (block_size first)"""
    out, o = [], 0
    while o < len(raw):
        bs = int.from_bytes(raw[o:o + 4], "little")
        out.append(raw[o:o + 4 + bs])
        o += 4 + bs
    assert o == len(raw)
    return out


def _tags(b):
    out, o = [], 0
    size = dict(c=1, C=1, s=2, S=2, i=4, I=4, A=1, f=4)
    while o < len(b):
        name, t = b[o:o + 2].decode(), chr(b[o + 2])
        o += 3
        if t == "Z":
            e = b.index(0, o)
            out.append((name, b[o:e])); o = e + 1
        else:
            out.append((name, b[o:o + size[t]])); o += size[t]
    return out


def fields(rec):
    """(field, value) of a record, in the order a mismatch is reported"""
    bs, ref, pos, lname, mapq, bin_, ncig, flag, lseq, nref, npos, tlen = struct.unpack_from("<iiiBBHHHiiii", rec, 0)
    o = 36
    name = rec[o:o + lname]; o += lname
    cig = rec[o:o + 4 * ncig]; o += 4 * ncig
    seq = rec[o:o + (lseq + 1) // 2]; o += (lseq + 1) // 2
    qual = rec[o:o + lseq]; o += lseq
    tags = _tags(rec[o:])
    return ([("flag", flag), ("refID", ref), ("pos", pos), ("mapq", mapq), ("CIGAR", cig)] + [("tag " + k, v) for k, v in tags] +
            [("tag set", [k for k, _ in tags]), ("SEQ", seq), ("QUAL", qual), ("mate", (nref, npos)), ("TLEN", tlen), ("name", name),
             ("bin", bin_), ("block_size", bs)])


def first_diff(got, want):
    g, w = dict(fields(got)), fields(want)
    for k, v in w:
        if g.get(k) != v:
            return k, g.get(k), v
    return "bytes", got, want


def assert_records(got, want, index, what):
    """got / want: record lists; index[i]: the read (pair) of record i"""
    assert len(got) == len(want), (what, len(got), len(want))
    for i, (g, w) in enumerate(zip(got, want)):
        if g != w:
            k, gv, wv = first_diff(g, w)
            pytest.fail("%s: record %d (read %d) differs first in %s: pipeline %r, host chain %r" % (what, i, int(index[i]), k, gv, wv))


def coverage(o):
    """rescued mates, discordant pairs, off-contig and truncated records of a host chain result"""
    fl = o["pair_flags"]
    return dict(records=o["counts"][0], mapped=o["counts"][1], rescued=len(o["rescued"]),
                discordant=int((fl == 8).sum()) if fl is not None else 0, off_contig=o["counts"][2], truncated=o["counts"][3])


def payload_records(batch):
    pay = batch.to_bytes()
    return split(gzip.decompress(pay) if batch.compressed else pay)


def layout(st):
    v = (C.c_uint64 * 8)()
    check(lib().nvb_debug_pipeline_bam_layout(st._h, v, C.c_uint32(8)), "nvb_debug_pipeline_bam_layout")
    return dict(zip(("O", "R", "x_fin", "x_btemp", "z_blocks", "z_cap", "o_x", "slot_bytes"), (int(x) for x in v)))


def align256(x):
    return -(-x // 256) * 256


# ---------------------------------------------------------------------------------------------------------------------------------------
# small worlds
# ---------------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ow(world):
    """the world with the oracle's index, and its contigs plus one shorter than a read"""
    O = orc.Oracle()
    idx = O.build_index(world["gsym"])
    cb = np.unique(np.concatenate([world["contigs"].begin, SHORT_CONTIG]))
    contigs = nb.ContigTable(["c%d" % i for i in range(len(cb) - 1)], np.diff(cb))
    return dict(world, O=O, idx=idx, contigs=contigs)


def se_batch(gsym, n, rng, bits, lengths):
    """n reads, odd ones reverse complemented, 2 % substitutions; every 23rd runs past the genome's end by 1-60 symbols, every 29th
    ends on it, every 31st spans the short contig; lengths 20 .. L (every 5th whole)"""
    pos = rng.integers(0, G - L, n)
    r = np.stack([gsym[p:p + L] for p in pos])
    r = np.where(rng.random(r.shape) < 0.02, (r + rng.integers(1, 4, r.shape)) & 3, r).astype(np.uint8)
    for i in range(n):
        if i % 23 == 7:
            k = int(rng.integers(1, 61))
            r[i] = np.concatenate([gsym[G - L + k:], rng.integers(0, 4, k)])
        elif i % 29 == 11:
            r[i] = gsym[G - L:]
        elif i % 31 == 13:
            r[i] = gsym[SHORT_CONTIG[0] - 50:SHORT_CONTIG[0] - 50 + L]
        if i % 2:
            r[i] = revcomp(r[i])
    if bits == 4:
        r[rng.random(r.shape) < 0.004] = 4
    lens = None
    if lengths:
        lens = rng.integers(20, L + 1, n).astype(np.uint32)
        lens[::5] = L
    return r, lens


def pe_batch(gsym, n_pairs, rng, policy, bits, lengths):
    """n_pairs pairs in policy's orientation, fragments 250-420 bp (mate 1 of every pair, then mate 2): every 7th pair's second mate
    15 % substituted (rescue material), every 11th pair's mates 20-70 kbp apart (discordant material); with lengths, mate 2 of every
    third pair 60 .. L long"""
    m1, m2 = [], []
    for i in range(n_pairs):
        frag = int(rng.integers(250, 420))
        p = int(rng.integers(0, G - frag))
        a, b = gsym[p:p + L].copy(), gsym[p + frag - L:p + frag].copy()
        if i % 7 == 3:
            b = np.where(rng.random(L) < 0.15, (b + 1) & 3, b).astype(np.uint8)
        elif i % 11 == 5:
            q = (p + 20_000 + int(rng.integers(0, 50_000))) % (G - L)
            b = gsym[q:q + L].copy()
        if policy == "fr":
            x, y = (a, revcomp(b)) if i % 2 == 0 else (revcomp(b), a)
        elif policy == "rf":
            x, y = (revcomp(a), b) if i % 2 == 0 else (b, revcomp(a))
        else:                                                        # ff: both forward, or both reverse with mate 2 on the left
            x, y = (a, b) if i % 2 == 0 else (revcomp(b), revcomp(a))
        m1.append(x); m2.append(y)
    r = np.stack(m1 + m2).astype(np.uint8)
    r = np.where(rng.random(r.shape) < 0.01, (r + 1) & 3, r).astype(np.uint8)
    if bits == 4:
        r[rng.random(r.shape) < 0.004] = 4
    lens = None
    if lengths:
        lens = np.full(2 * n_pairs, L, np.uint32)
        third = np.arange(0, n_pairs, 3)
        lens[n_pairs + third] = rng.integers(60, L + 1, len(third))
    return r, lens


class Stream:
    """one StreamingBam over a world and the batches it gets; .check(i, batch) holds batch i to the direct chain and the host chain"""

    def __init__(self, w, case, max_reads, compress, depth=2, max_cigar=0, max_md=0, max_name_bytes=None):
        self.w, self.case, self.max_reads, self.compress = w, case, max_reads, compress
        self.max_cigar, self.max_md = max_cigar or MAX_OPS + 2, max_md or 3 * MAX_OPS + 1
        spw = 32 // case.bits
        self.wpr = -(-L // spw)
        self.stride = self.wpr * spw
        self.batches = []
        self.max_name_bytes = max_name_bytes
        self.st = None
        self.depth, self.raw_max = depth, (max_cigar, max_md)

    def add(self, n, rng, names=None):
        c = self.case
        if c.paired:
            sym, lens = pe_batch(self.w["gsym"], n // 2, rng, c.pair.policy, c.bits, c.lengths)
        else:
            sym, lens = se_batch(self.w["gsym"], n, rng, c.bits, c.lengths)
        if names is None:
            names = names_for(n // 2 if c.paired else n, rng, "b%d_" % len(self.batches))
        quals = rng.integers(2, 41, (n, self.stride)).astype(np.uint8)
        self.batches.append(dict(n=n, sym=sym, lens=lens, names=names, words=pack_rows(sym, c.bits), quals=quals))
        return len(self.batches) - 1

    def open(self):
        c = self.case
        nbytes = max(len(nb.pack_names(bt["names"])[0]) for bt in self.batches)
        self.max_name_bytes = self.max_name_bytes or nbytes
        self.st = nb.StreamingBam(self.w["fmi"], self.w["gw"], c.params(), self.max_reads, L, self.wpr, self.w["contigs"], c.mapq(),
                                  pair=c.pair, quals=c.qual, lengths=c.lengths, compress=self.compress, depth=self.depth, bits=c.bits,
                                  max_name_bytes=self.max_name_bytes, max_cigar=self.raw_max[0], max_md=self.raw_max[1])
        return self.st

    def submit(self, i):
        bt = self.batches[i]
        return self.st.submit(bt["words"], bt["names"], quals=bt["quals"] if self.case.qual else None, lengths=bt["lens"], n=bt["n"])

    def host_chain(self, i, sel=None):
        """the host chain on batch i, or on its reads (pairs) sel"""
        bt, c = self.batches[i], self.case
        n = bt["n"]
        k = n // 2 if c.paired else n
        sel = np.arange(k) if sel is None else np.asarray(sel)
        rows = np.concatenate([sel, k + sel]) if c.paired else sel
        lens = bt["lens"][rows] if bt["lens"] is not None else None
        return stream_oracle.chain(self.w["O"], self.w["idx"], self.w["gsym"], bt["sym"][rows], lens,
                                   bt["quals"][rows] if c.qual else None, [bt["names"][j] for j in sel], c.params(), c.mapq(),
                                   c.pair, self.w["contigs"], MAX_OPS, self.max_cigar, self.max_md)

    def check(self, i, batch, sel=None, with_direct=True):
        """batch i's payload == the direct chain's (when the maxima are the defaults) and record for record the host chain's"""
        bt, c = self.batches[i], self.case
        what = "batch %d (n=%d)" % (i, bt["n"])
        got = payload_records(batch)
        assert batch.counts[0] == len(got) and batch.n_hits[0] == batch.n_hits[1], (what, batch.counts, batch.n_hits)
        if with_direct:
            want = direct(self.w, c, bt, bt["words"], self.stride, bt["quals"], self.max_reads)
            assert batch.counts == want["counts"] and batch.n_hits == want["n_hits"], what
            assert b"".join(got) == want["raw"], (what, "the pipeline and the direct chain differ")
            if self.compress:
                assert batch.to_bytes() == want["z"], what
        o = self.host_chain(i, sel)
        if sel is None:
            assert_records(got, o["records"], np.arange(len(got)) // (2 if c.paired else 1), what)
            assert tuple(batch.counts) == tuple(o["counts"]), (what, batch.counts, o["counts"])
        else:
            rec = np.stack([2 * sel, 2 * sel + 1], 1).reshape(-1) if c.paired else np.asarray(sel)
            assert_records([got[k] for k in rec], o["records"], rec // (2 if c.paired else 1), what + " sample")
        return o


SMALL = {
    "se-local-const-2bit": (Case(False, aln.LOCAL, False, 2, True), True),
    "se-semiglobal-qual-4bit": (Case(False, aln.SEMI_GLOBAL, True, 4, True), False),
    "pe-fr-local-const-2bit": (Case(True, aln.LOCAL, False, 2, True, policy="fr"), True),
    "pe-rf-nooverlap-qual-4bit": (Case(True, aln.LOCAL, True, 4, False, policy="rf", overlap=False), False),
    "pe-ff-discordant-nomixed": (Case(True, aln.LOCAL, False, 2, True, policy="ff", mixed=False, discordant=True), True),
}


@pytest.mark.parametrize("name", list(SMALL))
def test_small_world_equals_host_chain(ow, name):
    """batches of max_reads, 1 (paired: 2) and max_reads - 1 (- 2) reads at depth 2: the second is waited before the first, the third
    reuses the first's slot with other lengths; every record equals the host chain's"""
    case, compress = SMALL[name]
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    max_reads = 200
    s = Stream(ow, case, max_reads, compress)
    small = 2 if case.paired else 1
    for n in (max_reads, small, max_reads - small):
        s.add(n, rng)
    st = s.open()
    assert max(len(nb.pack_names(bt["names"])[0]) for bt in s.batches) == s.max_name_bytes    # the largest batch fills it exactly
    t0, t1 = s.submit(0), s.submit(1)
    outs = [None] * 3
    outs[1] = s.check(1, st.result(t1))
    outs[0] = s.check(0, st.result(t0))
    outs[2] = s.check(2, st.result(s.submit(2)))
    st.close()
    cov = {k: sum(coverage(o)[k] for o in outs) for k in coverage(outs[0])}
    print("\n%s: %s" % (name, cov), flush=True)
    assert cov["mapped"] > 0.5 * cov["records"] and cov["off_contig"] > 0, cov
    if case.paired:
        assert cov["rescued"] > 0, cov
    if case.pair is not None and case.pair.discordant:
        assert cov["discordant"] > 0, cov
    assert cov["truncated"] == 0, cov


# ---------------------------------------------------------------------------------------------------------------------------------------
# slot layout and host buffer edges
# ---------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("max_cigar,max_md", [(1, 1), (3, 12)])
def test_truncating_maxima(ow, max_cigar, max_md):
    """max_cigar = max_md = 1 with names of at most 8 bytes puts the record bound R below the traceback ops O, so the finish outputs sit
    at O; nearly every record is unmapped by truncation.  (3, 12): R above O, some records truncated and some whole.  Every record equals
    the host chain run with the same maxima"""
    case = Case(False, aln.LOCAL, False, 2, True)
    rng = np.random.default_rng(max_cigar * 100 + max_md)
    max_reads = 200
    s = Stream(ow, case, max_reads, True, max_cigar=max_cigar, max_md=max_md)
    for n in (max_reads, max_reads - 1):
        s.add(n, rng, names=["t%05d" % i for i in range(n)])
    st = s.open()
    lay = layout(st)
    print("\nlayout %s" % lay, flush=True)
    assert lay["O"] == align256(max_reads * MAX_OPS)
    assert lay["x_fin"] == align256(max(lay["O"], lay["R"]))
    if max_cigar == 1:
        assert lay["O"] > lay["R"] and lay["x_fin"] == lay["O"]
    cov = []
    for i in range(2):
        cov.append(coverage(s.check(i, st.result(s.submit(i)), with_direct=False)))
    st.close()
    tr, mp = sum(c["truncated"] for c in cov), sum(c["mapped"] for c in cov)
    print("maxima (%d, %d): %s" % (max_cigar, max_md, cov), flush=True)
    assert tr > 0
    if max_cigar == 1:
        assert tr > 10 * mp
    else:
        assert mp > 0


def test_payload_growth(ow):
    """depth 2, raw records: two small batches (each slot's pinned payload buffer at its first size), then two full ones -- the second
    submitted while the other slot's payload is unread -- whose payloads outgrow both buffers; results read in reverse and one twice.
    Payloads equal the direct chain whole and the host chain on a sample"""
    case = Case(False, aln.LOCAL, False, 2, True)
    rng = np.random.default_rng(77)
    max_reads = 6000
    s = Stream(ow, case, max_reads, False)
    for n in (100, 150, max_reads, max_reads - 17):
        s.add(n, rng)
    st = s.open()
    t0, t1 = s.submit(0), s.submit(1)
    s.check(1, st.result(t1))
    s.check(0, st.result(t0))
    small = max(len(st.result(t).payload) for t in (t0, t1))
    t2 = s.submit(2)
    t3 = s.submit(3)                                                   # slot of batch 2 still unread
    sizes = []
    for i, t in ((3, t3), (2, t2), (3, t3)):
        b = st.result(t)
        sizes.append(b.record_bytes)
        s.check(i, b, sel=np.sort(rng.choice(s.batches[i]["n"], 300, replace=False)))
    st.close()
    print("\npayloads: small batches up to %d bytes, full ones %s" % (small, sizes), flush=True)
    assert min(sizes) > (1 << 20) + small                             # past the first buffer of each slot (1 MiB granules)


@pytest.mark.parametrize("blocks", [1, 2])
def test_device_count_bgzf_large_gap(blocks):
    """a host bound of 40,000 BGZF blocks over 1 and 2 real ones: members and offsets equal nvb_bgzf_compress of the real bytes,
    every entry past the real blocks holds the total (d_block_offsets[z_blocks] is the payload size the pipeline reads), and the members
    inflate to the bytes"""
    require_gpu()
    bound = 40_000 * 0xFF00
    count = blocks * 0xFF00 - 4321
    rng = np.random.default_rng(blocks)
    host = rng.integers(0, 256, count, dtype=np.uint8)
    host[::3] = 0                                                     # a little compressible
    data = torch.empty(bound, dtype=torch.uint8, device="cuda")
    data[:count] = torch.from_numpy(host).cuda()
    data[count:count + (1 << 20)] = 0x5A                              # bytes past the count that must not be read
    out, off = _dc_bgzf(data, count, bound)
    want = nb.bgzf_compress(data[:count])
    wz = want.to_bytes()
    wo = want.offsets.cpu().numpy()
    assert len(off) == 40_000 + 1 and want.n_blocks == blocks
    assert np.array_equal(off[:blocks + 1], wo)
    assert (off[blocks:] == len(wz)).all() and int(off[-1]) == len(wz)
    assert out[:len(wz)].cpu().numpy().tobytes() == wz
    assert gzip.decompress(wz) == host.tobytes()
    del data, out
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------------------------------
# bench.py's shape on the headline index
# ---------------------------------------------------------------------------------------------------------------------------------------
SAMPLE = 2000


def _direct_headline(H, words, quals, names, contigs, mq, pair=None):
    """the direct chain on a whole batch: (records bytes, BGZF bytes, counts, n_hits, n_rescue)"""
    n = words.shape[0]
    dw = words.cuda()
    rs = PackedStringSet.fixed(dw.reshape(-1), n, L, stride=words.shape[1] * 16)
    q = torch.from_numpy(quals.reshape(-1)).cuda()
    hc = 32 * n + 1024
    if pair is None:
        ws = nb.seed_extend(H.fmi, H.genome, rs, bench_params(), traceback=True, mapq=mq, hit_capacity=hc)
        f = nb.finish_alignments(H.genome, rs, ws.best_ops, ws.best_n_ops, ws.best_begin, ws.best_strand, genome_len=N)
    else:
        ws = nb.seed_extend_paired(H.fmi, H.genome, rs, bench_params(), pair, mapq=mq, traceback=True, hit_capacity=hc)
        f = nb.finish_alignments(H.genome, rs, ws.mate_ops, ws.mate_n_ops, ws.mate_begin, ws.mate_strand, genome_len=N)
    recs = nb.bam_records(ws, f, rs, contigs, names, quals=q)
    z = nb.bgzf_compress(recs)
    torch.cuda.synchronize()
    out = dict(raw=recs.to_bytes(), z=z.to_bytes(), counts=tuple(int(v) for v in recs.counts.cpu()),
               n_hits=tuple(int(v) for v in ws.n_hits.cpu()[:3]), n_rescue=tuple(int(v) for v in ws.n_rescue.cpu()) if pair else None)
    del ws, f, recs, z, dw, q
    gc.collect(); torch.cuda.empty_cache()
    return out


def _run_headline(H, batches, pair, tmp_path, what):
    """batches: (host words [n, wpr], quals, names); depth 3 on two compute streams.  Returns the coverage of the samples"""
    mq = MapqParams.local(L)
    contigs = contig_table([])
    max_reads = batches[0][0].shape[0]
    wpr = batches[0][0].shape[1]
    gc.collect(); torch.cuda.empty_cache()
    free0 = torch.cuda.mem_get_info()[0]
    st = nb.StreamingBam(H.fmi, H.genome, bench_params(), max_reads, L, wpr, contigs, mq, pair=pair, quals=True, depth=3,
                         max_name_bytes=max(len(nb.pack_names(b[2])[0]) for b in batches))
    free1 = torch.cuda.mem_get_info()[0]
    print("\n%s: create took %.2f GB of device memory for depth 3 x %.2f GB slots (%.1f GB free before)" %
          (what, (free0 - free1) / 1e9, st.slot_bytes / 1e9, free0 / 1e9), flush=True)
    assert free0 - free1 >= 3 * st.slot_bytes
    got, t0 = [], time.perf_counter()
    tickets = [st.submit(b[0], b[2], quals=b[1]) for b in batches[:3]]
    for i in range(len(batches)):
        r = st.result(tickets[i])
        got.append(nb.BamBatch(**{**r.__dict__, "payload": r.payload.clone()}))    # outlives later submits
        if i + 3 < len(batches):
            tickets.append(st.submit(batches[i + 3][0], batches[i + 3][2], quals=batches[i + 3][1]))
    st.close()
    print("%s: %d batches through the pipeline in %.1f s" % (what, len(batches), time.perf_counter() - t0), flush=True)
    O = orc.Oracle()
    rng = np.random.default_rng(len(batches))
    cov = []
    raws = []
    for i, ((words, quals, names), b) in enumerate(zip(batches, got)):
        want = _direct_headline(H, words, quals, names, contigs, mq, pair)
        kept, found, _ = b.n_hits
        assert kept == found, (what, i, b.n_hits)                     # hit_capacity: nothing truncated
        if pair is not None:
            assert b.n_rescue[0] == b.n_rescue[1] and b.n_rescue == want["n_rescue"], (what, i)
        assert b.counts == want["counts"] and b.n_hits == want["n_hits"], (what, i)
        pay = b.to_bytes()
        assert pay == want["z"], (what, i, "the pipeline and the direct chain differ")
        raw = gzip.decompress(pay)
        assert raw == want["raw"], (what, i)
        raws.append(raw)
        # the host chain on a sample: every read (pair) depends on itself alone once nothing truncates
        k = max_reads // 2 if pair is not None else max_reads
        sel = np.sort(rng.choice(k, SAMPLE, replace=False))
        rows = np.concatenate([sel, k + sel]) if pair is not None else sel
        hw = words.numpy()
        reads = unpack_rows(hw[rows])
        t1 = time.perf_counter()
        o = stream_oracle.chain(O, H.idx, H.g, reads, None, quals[rows], [names[j] for j in sel], bench_params(), mq, pair, contigs,
                                MAX_OPS, MAX_OPS + 2, 3 * MAX_OPS + 1)
        recs = split(raw)
        rec = np.stack([2 * sel, 2 * sel + 1], 1).reshape(-1) if pair is not None else sel
        assert_records([recs[j] for j in rec], o["records"], rec // (2 if pair is not None else 1), "%s batch %d" % (what, i))
        cov.append(coverage(o))
        print("%s batch %d: %d records, payload %.1f MB; sample %s; host chain %.0f s" %
              (what, i, b.counts[0], len(pay) / 1e6, cov[-1], time.perf_counter() - t1), flush=True)
    # the whole stream through write_bam: gzip and htslib read every record back
    p = str(tmp_path / "stream.bam")
    hdr = nb.bam_header(contigs)
    nb.write_bam(p, hdr, got)
    assert gzip.open(p).read() == hdr + b"".join(raws)
    if RefBam.available():
        text = RefBam().format(p, cap=1 << 31)                       # about 400 bytes of SAM text per record
        assert text.count("\n") == sum(b.counts[0] for b in got)
    return cov


def test_headline_single_end(H, monkeypatch, tmp_path):
    """bench's batch generator, 4 batches of 250 K x 150 bp reads with qualities and names, depth 3, two compute streams"""
    monkeypatch.setenv("NVB_PIPELINE_COMPUTE_STREAMS", "2")
    rng = np.random.default_rng(250)
    n = 250_000
    batches = []
    for b in range(4):
        w = bench.make_reads(H.genome, N, n, b, H.genome.device).cpu()
        batches.append((w.pin_memory(), rng.integers(2, 41, (n, w.shape[1] * 16)).astype(np.uint8), nb.numbered_names(n, "s%d_" % b)))
    cov = _run_headline(H, batches, None, tmp_path, "single end")
    assert sum(c["mapped"] for c in cov) > 0.9 * len(cov) * SAMPLE


def test_headline_paired(H, monkeypatch, tmp_path):
    """2 batches of 250 K FR pairs (bench's pair generator), depth 3, two compute streams"""
    monkeypatch.setenv("NVB_PIPELINE_COMPUTE_STREAMS", "2")
    rng = np.random.default_rng(500)
    np_ = 250_000
    batches = []
    for b in range(2):
        w, _, _ = synth.sample_pairs(H.genome, N, np_, L, frag_mean=350.0, frag_sd=30.0, sub_rate=0.01, hard_frac=0.05,
                                     hard_sub_rate=0.2, device=H.genome.device, seed=0x51ED + b, mut_seed=0xC0FFEE + b)
        w = w.cpu()
        batches.append((w.pin_memory(), rng.integers(2, 41, (2 * np_, w.shape[1] * 16)).astype(np.uint8),
                        nb.numbered_names(np_, "p%d_" % b)))
    pair = nb.PairParams(min_frag=0, max_frag=500, min_mate_score=80)
    cov = _run_headline(H, batches, pair, tmp_path, "paired")
    assert sum(c["rescued"] for c in cov) > 0
