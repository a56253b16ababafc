"""CPU: the argument rules of the pipeline's BAM mode (nvb_pipeline_create_bam / submit_bam / wait_bam) and of the device-count BGZF hook,
which all answer before any CUDA call, and the exports that go with them."""
import ctypes as C
import pytest
from nvbio_b200 import _lib
from nvbio_b200._lib import (FmIndexStruct, SeedExtendParamsStruct, GotohSchemeStruct, PairParamsStruct, MapqParamsStruct,
                             PipelineBamParamsStruct, PipelineBamResultStruct, BgzfOutStruct)
from tests.test_cabi_exports import declared_symbols

INVALID, UNSUPPORTED = -1, -4
NAMES = ("nvb_pipeline_create_bam", "nvb_pipeline_submit_bam", "nvb_pipeline_wait_bam", "nvb_pipeline_slot_bytes")


@pytest.fixture(scope="module")
def L():
    return _lib.lib()


def test_exports():
    assert set(NAMES) <= set(_lib.EXPORTS) and set(NAMES) <= set(declared_symbols())
    hooks = {"nvb_debug_bgzf_compress_device_count", "nvb_debug_pipeline_bam_submit_check"}
    assert hooks <= set(_lib.DEBUG_EXPORTS) and hooks <= set(declared_symbols("nvbio_b200_debug.h"))
    assert not hooks & set(declared_symbols())                       # no new public BGZF or pipeline hook


def _args():
    fm = FmIndexStruct(); fm.d_bwt_occ = 32; fm.d_ssa = 32; fm.length = 1000; fm.primary = 5; fm.sa_interval = 16
    sch = GotohSchemeStruct(); sch.match, sch.mismatch, sch.pattern_gap_open, sch.pattern_gap_ext, sch.text_gap_open, sch.text_gap_ext = 2, -2, -5, -3, -5, -3
    sp = SeedExtendParamsStruct(); sp.seed_len, sp.seed_interval, sp.band_len, sp.type, sp.both_strands, sp.max_seed_hits, sp.dedup_jobs = 20, 10, 31, 1, 1, 100, 1
    sp.scheme = sch
    mp = MapqParamsStruct(); mp.d_min_score = 256; mp.max_read_len = 150; mp.match_bonus = 2
    bp = PipelineBamParamsStruct(); bp.mapq = C.addressof(mp); bp.d_contig_begin = 256; bp.n_contigs = 1; bp.max_name_bytes = 1000; bp.compress = 1
    pp = PairParamsStruct(); pp.min_frag, pp.max_frag, pp.min_mate_score, pp.rescue_capacity = 0, 500, 60, 100
    return dict(fm=fm, sp=sp, mp=mp, bp=bp, pp=pp)


def _create(L, a, paired=False, bam=True, max_reads=64, read_len=150, wpr=10, bits=2, depth=2, out=True, genome=True):
    h = C.c_void_p()
    return L.nvb_pipeline_create_bam(C.byref(a["fm"]), C.c_void_p(16) if genome else None, C.byref(a["sp"]),
                                     C.byref(a["pp"]) if paired else None, C.byref(a["bp"]) if bam else None,
                                     C.c_uint32(max_reads), C.c_uint32(read_len), C.c_uint32(wpr), C.c_uint32(bits), C.c_uint32(1000),
                                     C.c_uint32(depth), C.byref(h) if out else None)


def test_create_rules(L):
    # the checks nvb_pipeline_create makes
    for kw in (dict(bam=False), dict(out=False), dict(genome=False), dict(max_reads=0), dict(depth=0), dict(depth=17), dict(bits=3),
               dict(bits=8), dict(wpr=9), dict(paired=True, max_reads=63)):
        assert _create(L, _args(), **kw) == INVALID, kw
    a = _args(); a["pp"].policy = 4
    assert _create(L, a, paired=True) == INVALID
    a = _args(); a["pp"].flags = 8
    assert _create(L, a, paired=True) == INVALID
    # the BAM parameters
    a = _args(); a["bp"].mapq = None
    assert _create(L, a) == INVALID
    a = _args(); a["mp"].d_min_score = None
    assert _create(L, a) == INVALID
    a = _args(); a["bp"].d_contig_begin = None
    assert _create(L, a) == INVALID
    a = _args(); a["bp"].n_contigs = 0
    assert _create(L, a) == INVALID
    a = _args(); a["bp"].max_name_bytes = 0
    assert _create(L, a) == INVALID
    a = _args(); a["sp"].d_read_quals = 256                          # qualities come with every batch
    assert _create(L, a) == INVALID
    a = _args(); a["sp"].scheme.d_qual_table = 256                   # a quality table needs has_quals
    assert _create(L, a) == INVALID
    a = _args(); a["mp"].max_read_len = 149
    assert _create(L, a) == INVALID
    # read_len above the traceback calls' 512; an INVALID rule wins over it
    a = _args(); a["mp"].max_read_len = 600
    assert _create(L, a, read_len=513, wpr=33) == UNSUPPORTED and _create(L, a, read_len=513, wpr=32) == INVALID
    assert _create(L, _args(), read_len=513, wpr=33) == INVALID        # max_read_len 150 < read_len


def test_discordant_accepted_by_the_bam_mode_only(L):
    """NVB_PE_DISCORDANT is refused by nvb_pipeline_create and passes the BAM mode's checks (which then reach the device; here the
    first CUDA call fails, with a CUDA error rather than NVB_E_INVALID)"""
    a = _args(); a["pp"].flags = 2
    h = C.c_void_p()
    assert L.nvb_pipeline_create(C.byref(a["fm"]), C.c_void_p(16), C.byref(a["sp"]), C.byref(a["pp"]), C.c_uint32(64), C.c_uint32(150),
                                 C.c_uint32(10), C.c_uint32(2), C.c_uint32(1000), C.c_uint32(2), C.byref(h)) == INVALID
    try:
        import torch
        if torch.cuda.is_available():
            pytest.skip("with a device the create goes through (tests/test_gpu_pipeline_bam.py)")
    except ImportError:
        pass
    assert _create(L, a, paired=True) not in (INVALID, UNSUPPORTED, 0)


def _check(L, bp, paired=False, max_reads=8, read_len=150, n=8, words=True, quals=None, lengths=None, names=b"abcdefgh", offsets=None):
    n_names = n // 2 if paired else n
    if offsets is None:
        offsets = list(range(n_names + 1))
    off = (C.c_uint32 * max(len(offsets), 1))(*offsets)
    w = (C.c_uint32 * 160)()
    q = (C.c_uint8 * (8 * 160))(*([30] * 8 * 160)) if quals else None
    ln = (C.c_uint32 * len(lengths))(*lengths) if lengths is not None else None
    nm = C.create_string_buffer(names) if names is not None else None
    return L.nvb_debug_pipeline_bam_submit_check(C.byref(bp), C.c_uint32(paired), C.c_uint32(max_reads), C.c_uint32(read_len), C.c_uint32(n),
                                                 w if words else None, q, ln, nm, off if offsets != [] else None)


def test_submit_rules(L):
    bp = _args()["bp"]
    assert _check(L, bp) == 0
    assert _check(L, bp, n=5) == 0                                   # a short batch
    assert _check(L, bp, n=0) == INVALID and _check(L, bp, n=9) == INVALID
    assert _check(L, bp, paired=True) == 0 and _check(L, bp, paired=True, n=6) == 0
    assert _check(L, bp, paired=True, n=7, offsets=[0, 1, 2, 3]) == INVALID          # odd when paired
    assert _check(L, bp, words=False) == INVALID and _check(L, bp, names=None) == INVALID and _check(L, bp, offsets=[]) == INVALID
    # name offsets: from 0, increasing (no empty name), ending within max_name_bytes
    assert _check(L, bp, offsets=[1, 2, 3, 4, 5, 6, 7, 8, 9]) == INVALID
    assert _check(L, bp, offsets=[0, 1, 2, 2, 4, 5, 6, 7, 8]) == INVALID
    assert _check(L, bp, offsets=[0, 1, 3, 2, 4, 5, 6, 7, 8]) == INVALID
    assert _check(L, bp, n=1, offsets=[0, 1000]) == 0 and _check(L, bp, n=1, offsets=[0, 1001]) == INVALID
    # quals and lengths when the create flags ask for them
    bp.has_quals = 1
    assert _check(L, bp) == INVALID and _check(L, bp, quals=True) == 0
    bp.has_quals = 0
    bp.has_lengths = 1
    assert _check(L, bp) == INVALID
    assert _check(L, bp, lengths=[150, 1, 2, 3, 4, 5, 6, 7]) == 0
    assert _check(L, bp, lengths=[150, 0, 2, 3, 4, 5, 6, 7]) == INVALID
    assert _check(L, bp, lengths=[151, 1, 2, 3, 4, 5, 6, 7]) == INVALID
    assert _check(L, bp, read_len=100, lengths=[100] * 8) == 0 and _check(L, bp, read_len=100, lengths=[101] + [100] * 7) == INVALID


def test_submit_and_wait_without_a_bam_pipeline(L):
    r = PipelineBamResultStruct()
    t = C.c_uint32(0)
    w = (C.c_uint32 * 16)()
    nm, off = C.create_string_buffer(b"a"), (C.c_uint32 * 2)(0, 1)
    assert L.nvb_pipeline_submit_bam(None, C.c_uint32(1), w, None, None, nm, off, C.byref(t)) == INVALID
    assert L.nvb_pipeline_wait_bam(None, C.c_uint32(0), C.byref(r)) == INVALID
    L.nvb_pipeline_slot_bytes.restype = C.c_size_t
    assert L.nvb_pipeline_slot_bytes(None) == 0


def test_device_count_bgzf_rules(L):
    o = BgzfOutStruct(); o.d_block_offsets = 256
    tb = C.c_size_t(0)
    f = L.nvb_debug_bgzf_compress_device_count
    assert f(C.c_void_p(256), None, C.c_uint64(100), C.byref(o), None, C.byref(tb), None) == INVALID            # no device count
    assert f(None, C.c_void_p(256), C.c_uint64(100), C.byref(o), None, C.byref(tb), None) == INVALID            # no input
    assert f(C.c_void_p(256), C.c_void_p(256), C.c_uint64(100), None, None, C.byref(tb), None) == INVALID
    assert f(C.c_void_p(256), C.c_void_p(256), C.c_uint64(100), C.byref(o), None, None, None) == INVALID
    o.capacity = 10
    assert f(C.c_void_p(256), C.c_void_p(256), C.c_uint64(100), C.byref(o), None, C.byref(tb), None) == INVALID  # capacity without d_out
    o.capacity = 0
    assert f(C.c_void_p(256), C.c_void_p(256), C.c_uint64(0xFF00 << 32), C.byref(o), None, C.byref(tb), None) == INVALID   # 2^32 blocks


def test_write_bam_accepts_a_batch(tmp_path):
    """write_bam: a compressed BamBatch verbatim, an uncompressed one framed like BamRecords"""
    import gzip
    import torch
    from nvbio_b200.bam import BamBatch, write_bam, _bgzf_block, _BGZF_EOF
    recs = bytes(range(256)) * 300
    z = _bgzf_block(recs)
    mk = lambda payload, comp: BamBatch(payload=torch.frombuffer(bytearray(payload), dtype=torch.uint8), compressed=comp, n_records=1,   # noqa: E731
                                        counts=(1, 1, 0, 0), n_hits=(0, 0, 0), n_rescue=None, record_bytes=len(recs),
                                        n_blocks=1 if comp else 0, device_ms=0.0)
    p1, p2 = str(tmp_path / "a.bam"), str(tmp_path / "b.bam")
    write_bam(p1, b"HDR", [mk(z, True), mk(recs, False)])
    write_bam(p2, b"HDR", [recs, recs])
    assert gzip.open(p1).read() == gzip.open(p2).read() == b"HDR" + recs + recs
    raw = open(p1, "rb").read()
    assert raw.endswith(_BGZF_EOF) and z in raw
