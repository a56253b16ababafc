"""The device-count forms of the Gotoh score entry points, nvb_banded_gotoh_score_indirect and nvb_gotoh_score_indirect: the count
lives on the device (`d_n`, written on the stream right before the call, as seed + extend writes its DP list's length) and `n_max` is
only a capacity.  Under a device count the banded call runs the ticket form of gotoh_pair_kernel (a resident grid whose warps claim
32 pairs at a time from a per-call ticket) and the full-matrix call keeps the warp kernel up to four times the exact-count threshold.

The edges and kernel variants that tests/test_gpu_gotoh_limits.py pins through the exact-count calls run here through the device-count
calls: every result equals the int32 oracle exactly (score, sink.x, sink.y), the route (nvb_debug_gotoh_last_route) says which kernel
took the batch and how many alignments went to the int32 todo list, and no entry at or past the count -- up to a pad past the
capacity -- is written."""
import ctypes as C
import numpy as np
import pytest
import torch
from oracle import orc
import nvbio_b200 as nb
from nvbio_b200 import aln, synth
from nvbio_b200.strings import PackedStringSet, unpack_symbols
from tests.gpu_util import require_gpu, host_u32
from tests.test_gpu_gotoh_limits import (BANDS, GLOBAL, LOCAL, SEMI, FULL_S, Scheme6, assert_route, assert_same, banded_cases, case_id,
                                         case_problems, debug_knobs, edge_table, full_batch, full_cases, last_route)
from tests.test_host_core import fixed_problems

pytestmark = pytest.mark.gpu

NVB_OK, NVB_E_TEMP_SIZE = 0, -2
PAD = 37                     # output entries past the capacity: no call may write them
SENT = -7                    # what the outputs hold before a call (a sink of (-7, -7) is never a result)
S4 = (2, -2, -5, -3)
COUNTS = (0, 1, 2, 63, 64, 65, 127, 128, 129, 1001)     # whole 32-pair claims +- 1 alignment, and an odd tail
MIX_CAP = 1200


@pytest.fixture(scope="module")
def O():
    require_gpu()
    return orc.Oracle()


# --------------------------------------------------------------------------------------------------------------------------------------
# the device-count call
# --------------------------------------------------------------------------------------------------------------------------------------
def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


class Indirect:
    """one device-count entry point on one batch of capacity n_max, with one temp buffer for all its launches.  launch(count) writes
    the count to d_n with a device op on the current stream and enqueues the call right behind it, with no host sync in between;
    the outputs it returns hold n_max + PAD entries, all `sentinel` before the call."""

    def __init__(self, lead, scheme, P, T, n_max, qual=None, full=False):
        L = nb.lib()
        self.fn = L.nvb_gotoh_score_indirect if full else L.nvb_banded_gotoh_score_indirect
        self.lead = lead                                   # (band, type) or (type,)
        self.keep = (scheme, P, T, qual)
        self.sch, self.ps, self.ts = scheme.struct(), P.struct(), T.struct()
        self.qp = C.c_void_p(qual.data_ptr()) if qual is not None else None
        self.n_max = n_max
        self.d_n = torch.empty(1, dtype=torch.int32, device="cuda")
        tb = C.c_size_t(0)
        assert self._call(None, None, None, tb) == NVB_E_TEMP_SIZE
        self.temp = torch.empty(max(tb.value, 1), dtype=torch.uint8, device="cuda")

    def _call(self, score, sink, temp, tb):
        return self.fn(*(C.c_int(v) for v in self.lead), C.byref(self.sch), C.byref(self.ps), self.qp, C.byref(self.ts),
                       C.c_void_p(self.d_n.data_ptr()), C.c_uint32(self.n_max), score, sink, temp, C.byref(tb), _stream())

    def launch(self, count, sentinel=SENT):
        """count None: d_n is left as allocated, never written"""
        score = torch.full((self.n_max + PAD,), sentinel, dtype=torch.int32, device="cuda")
        sink = torch.full((self.n_max + PAD, 2), sentinel, dtype=torch.int32, device="cuda")
        if count is not None:
            self.d_n.fill_(count)
        tb = C.c_size_t(self.temp.numel())
        assert self._call(C.c_void_p(score.data_ptr()), C.c_void_p(sink.data_ptr()), C.c_void_p(self.temp.data_ptr()), tb) == NVB_OK
        return score, sink


def indirect_banded(band, typ, scheme, P, T, count, n_max, sentinel=SENT, qual=None):
    """(score, sink) of n_max + PAD entries and the route of one nvb_banded_gotoh_score_indirect call"""
    out = Indirect((band, typ), scheme, P, T, n_max, qual).launch(count, sentinel)
    return out, last_route()


def indirect_full(typ, scheme, P, T, count, n_max, sentinel=SENT, qual=None):
    """(score, sink) of n_max + PAD entries and the route of one nvb_gotoh_score_indirect call"""
    out = Indirect((typ,), scheme, P, T, n_max, qual, full=True).launch(count, sentinel)
    return out, last_route()


def check(out, want, count, what, sentinel=SENT):
    """the first `count` entries == want, every entry from `count` to the end of the pad still `sentinel`"""
    score, sink = out
    s, k = score.cpu().numpy(), host_u32(sink)
    assert_same((s[:count], k[:count, 0], k[:count, 1]), [w[:count] for w in want[:3]], what)
    bad = np.flatnonzero((s[count:] != sentinel) | (k[count:].view(np.int32) != sentinel).any(axis=1))
    assert len(bad) == 0, "%s: %d entries at or past the count %d were written, first %d" % (what, len(bad), count, count + bad[0])


# --------------------------------------------------------------------------------------------------------------------------------------
# batches
# --------------------------------------------------------------------------------------------------------------------------------------
def tile(pr, n_max):
    """the batch's alignments repeated up to the capacity: every slot up to n_max holds a real problem (that no call may score
    past its count)"""
    pat, p_off, p_len, txt, t_off, t_len = pr
    return pat, np.resize(p_off, n_max), np.resize(p_len, n_max), txt, np.resize(t_off, n_max), np.resize(t_len, n_max)


def head(pr, n):
    pat, p_off, p_len, txt, t_off, t_len = pr
    return pat, p_off[:n], p_len[:n], txt, t_off[:n], t_len[:n]


def string_sets(pr, max_m, pbits=2, pbe=True, tbe=True):
    pat, p_off, p_len, txt, t_off, t_len = pr
    P = PackedStringSet.from_symbols(pat, p_off, p_len, bits=pbits, big_endian=pbe)
    P.length = max_m
    return P, PackedStringSet.from_symbols(txt, t_off, t_len, bits=2, big_endian=tbe)


def mixed_banded(rng, band, m, n):
    """n alignments of m symbols in full windows (fixed_problems), some of them broken: a window one symbol short of
    m + band - 1, an empty pattern, a pattern 3 symbols shorter (which only LOCAL admits beside a longer one)"""
    pat, p_off, p_len, txt, t_off, t_len = fixed_problems(rng, n, band, m)
    p_len, t_len = p_len.copy(), t_len.copy()
    kind = rng.integers(0, 10, n)
    t_len[kind == 1] = m + band - 2
    p_len[kind == 2] = 0
    p_len[kind == 3] = m - 3
    return pat, p_off, p_len, txt, t_off, t_len


def refused_banded(pr, band, typ, count):
    """alignments the pair kernel must send to the int32 list among the first `count`: both of a pair whose pattern is empty, whose
    window is shorter than M + band - 1, or (GLOBAL / SEMI_GLOBAL) whose pattern lengths differ; the tail alignment alone"""
    p_len, t_len = pr[2].astype(np.int64), pr[5].astype(np.int64)
    total = 0
    for a0 in range(0, count, 2):
        a1 = min(a0 + 1, count - 1)
        M0, M1, N0, N1 = p_len[a0], p_len[a1], t_len[a0], t_len[a1]
        if M0 == 0 or M1 == 0 or N0 < M0 + band - 1 or N1 < M1 + band - 1 or (typ != LOCAL and M0 != M1):
            total += a1 - a0 + 1
    return total


def window_batch(rng, n, band, m):
    """n patterns of m symbols against full windows of m + band - 1 random text symbols, vectorised: the window's symbols on a random
    diagonal with 4% substitutions, or (one in ten) a random pattern"""
    N = m + band - 1
    txt = rng.integers(0, 4, (n, N), dtype=np.uint8)
    j = rng.integers(0, band, n)
    pat = np.take_along_axis(txt, j[:, None] + np.arange(m)[None, :], axis=1)
    sub = rng.integers(0, 25, (n, m), dtype=np.uint8) == 0
    pat = np.where(sub, (pat + rng.integers(1, 4, (n, m), dtype=np.uint8)) % 4, pat)
    rnd = rng.integers(0, 10, n) == 0
    pat[rnd] = rng.integers(0, 4, (int(rnd.sum()), m), dtype=np.uint8)
    return (pat.astype(np.uint8).reshape(-1), np.arange(n, dtype=np.uint32) * m, np.full(n, m, np.uint32),
            txt.reshape(-1), np.arange(n, dtype=np.uint32) * N, np.full(n, N, np.uint32))


def warp_slots():
    """(SMs, thread slots per SM): a grid resident on this device never holds more than their product in threads"""
    p = torch.cuda.get_device_properties(torch.cuda.current_device())
    return p.multi_processor_count, p.max_threads_per_multi_processor


# --------------------------------------------------------------------------------------------------------------------------------------
# banded: the ticket kernels
# --------------------------------------------------------------------------------------------------------------------------------------
EDGE_COUNT, EDGE_CAP = 61, 256          # an odd count (a tail pair) far below the capacity
# (pattern bits, pattern big-endian, text big-endian, pair_format, pair_rows2): the compile-time pattern readers (PFMT 2 / 4) and the
# run-time one (PFMT 0), both row schedules; little-endian patterns (PFMT 0) and little-endian 2-bit texts (the selector staging's
# !be branch)
VARIANTS = [(2, 1, 1, 1, 1), (2, 1, 1, 1, 0), (2, 1, 1, 0, 1), (2, 1, 1, 0, 0), (4, 1, 1, 1, 1), (4, 1, 1, 1, 0), (4, 1, 1, 0, 1),
            (4, 1, 1, 0, 0), (2, 0, 0, 1, 1), (4, 0, 0, 1, 0), (2, 1, 0, 1, 1), (4, 1, 0, 1, 0)]
QTAB_VARIANTS = [(4, 1, 1, 1, 1), (4, 1, 1, 1, 0), (2, 0, 0, 1, 1)]        # a quality table always takes PFMT 0


@pytest.mark.parametrize("band", BANDS)
def test_banded_ticket_kernels_at_every_edge(O, band):
    """every admission edge of test_gpu_gotoh_limits through the device-count call, in every ticket-kernel variant: the count far
    below the capacity, the packed kernel alone on the admitted side of each edge, the int32 kernel on the refused side"""
    require_gpu()
    for c in banded_cases(band):
        name, _, typ, s6, m, ok, qtab = c
        pr, qual = case_problems(c, n=EDGE_COUNT)
        want = O.banded_gotoh(band, typ, s6, *pr, qual=qual, qtab=qtab)
        assert want[3].all()
        pr = tile(pr, EDGE_CAP)
        sch = Scheme6(s6, qtab)
        q = torch.from_numpy(qual).cuda() if qual is not None else None
        for pbits, pbe, tbe, fmt, rows2 in (VARIANTS if qtab is None else QTAB_VARIANTS):
            P, T = string_sets(pr, m, pbits, pbe, tbe)
            with debug_knobs(pair_format=fmt, pair_rows2=rows2):
                out, route = indirect_banded(band, typ, sch, P, T, EDGE_COUNT, EDGE_CAP, qual=q)
            what = "%s pbits=%d pbe=%d tbe=%d fmt=%d rows2=%d" % (case_id(c), pbits, pbe, tbe, fmt, rows2)
            check(out, want, EDGE_COUNT, what)
            assert_route(route, ok, what)
        P, T = string_sets(pr, m, 4)
        with debug_knobs(force_gotoh_path=1):
            out, route = indirect_banded(band, typ, sch, P, T, EDGE_COUNT, EDGE_CAP, qual=q)
        check(out, want, EDGE_COUNT, case_id(c) + " int32")
        assert route == (0, 0)


@pytest.mark.parametrize("band", (3, 5, 63))
def test_banded_generic_bands_under_a_device_count(O, band):
    """bands without a pair kernel: gotoh_generic_kernel reads the count from the device, for every type, a constant and a quality
    scheme, ragged patterns; a count past the capacity scores exactly the capacity"""
    require_gpu()
    rng = np.random.default_rng(4100 + band)
    pr = fixed_problems(rng, EDGE_COUNT, band, 90, ragged=True)
    qual = rng.integers(0, 8, len(pr[0])).astype(np.uint8)
    q = torch.from_numpy(qual).cuda()
    prt = tile(pr, EDGE_CAP)
    P, T = string_sets(prt, int(pr[2].max()), 4)
    for typ in (GLOBAL, LOCAL, SEMI):
        for s6, qtab in ((S4, None), ((0, 0, -8, -3, -7, -2), edge_table(-12, 6))):
            want = O.banded_gotoh(band, typ, s6, *prt, qual=qual if qtab is not None else None, qtab=qtab)
            for count in (EDGE_COUNT, EDGE_CAP + 5):
                out, route = indirect_banded(band, typ, Scheme6(s6, qtab), P, T, count, EDGE_CAP, qual=q if qtab is not None else None)
                what = "B%d t%d %s count=%d" % (band, typ, "qtab" if qtab is not None else "const", count)
                check(out, want, min(count, EDGE_CAP), what)
                assert route == (0, 0), what


@pytest.mark.parametrize("band", (7, 31))
@pytest.mark.parametrize("typ", (GLOBAL, LOCAL, SEMI))
def test_banded_refused_pairs_and_count_shapes(O, band, typ):
    """pairs the ticket kernel refuses (short window, empty pattern, unequal lengths outside LOCAL) go to the todo list whole and
    are scored by the int32 kernel under the same count; refused pairs past the count are never listed.  Counts of whole 32-pair
    claims +- 1 alignment, an odd tail, the capacity, and past it (which scores exactly the capacity)"""
    require_gpu()
    rng = np.random.default_rng(4200 + 10 * band + typ)
    m = 60
    pr = mixed_banded(rng, band, m, MIX_CAP)
    qual = rng.integers(0, 8, len(pr[0])).astype(np.uint8)
    q = torch.from_numpy(qual).cuda()
    assert 0 < refused_banded(pr, band, typ, 1001) < refused_banded(pr, band, typ, MIX_CAP)     # refused pairs on both sides of a count
    s6q, qtab = (0, 0, -8, -3, -7, -2), edge_table(-12, 6)
    # (pattern bits, knobs, quality table): PFMT 2 / two rows, PFMT 0 / one row, PFMT 0 with a quality table
    for pbits, knobs, with_q in ((2, {}, False), (4, dict(pair_format=0, pair_rows2=0), False), (4, {}, True)):
        want = O.banded_gotoh(band, typ, s6q, *pr, qual=qual, qtab=qtab) if with_q else O.banded_gotoh(band, typ, S4, *pr)
        sch = Scheme6(s6q, qtab) if with_q else Scheme6(S4)
        P, T = string_sets(pr, m, pbits)
        for count in COUNTS + (MIX_CAP, MIX_CAP + 5):
            n = min(count, MIX_CAP)
            with debug_knobs(**knobs):
                out, route = indirect_banded(band, typ, sch, P, T, count, MIX_CAP, qual=q if with_q else None)
            what = "B%d t%d pbits=%d %s qtab=%d count=%d" % (band, typ, pbits, knobs, with_q, count)
            check(out, want, n, what)
            assert route == (1, refused_banded(pr, band, typ, n)), what


def test_zero_capacity_with_an_unwritten_count():
    """n_max == 0: both calls return NVB_OK without reading d_n (never written here) or writing any output"""
    require_gpu()
    pr = fixed_problems(np.random.default_rng(4300), 4, 31, 40)
    P, T = string_sets(pr, 40)
    for full in (False, True):
        call = Indirect((LOCAL,) if full else (31, LOCAL), Scheme6(S4), P, T, 0, full=full)
        out = call.launch(None)
        torch.cuda.synchronize()
        check(out, [np.zeros(0)] * 3, 0, "full=%d n_max=0" % full)


def test_banded_temp_reuse_in_stream_order(O):
    """three calls back to back on one temp buffer and one stream, no sync between them (the todo list's length and the pair ticket
    are zeroed by each): each call's results are its own, and the first count repeated gives the identical result"""
    require_gpu()
    band, typ, m = 15, SEMI, 60
    pr = mixed_banded(np.random.default_rng(4400), band, m, MIX_CAP)
    want = O.banded_gotoh(band, typ, S4, *pr)
    P, T = string_sets(pr, m)
    call = Indirect((band, typ), Scheme6(S4), P, T, MIX_CAP)
    a = call.launch(1001, -7)
    b = call.launch(129, -9)
    c = call.launch(1001, -11)
    route = last_route()                                   # of the third call
    check(a, want, 1001, "first", -7)
    check(b, want, 129, "second", -9)
    check(c, want, 1001, "third", -11)
    assert route == (1, refused_banded(pr, band, typ, 1001))
    assert torch.equal(a[0][:1001], c[0][:1001]) and torch.equal(a[1][:1001], c[1][:1001])


# --------------------------------------------------------------------------------------------------------------------------------------
# banded: several resident rounds (each warp comes back to the ticket)
# --------------------------------------------------------------------------------------------------------------------------------------
def test_banded_ticket_rounds_cheap_shape(O):
    """band 7, m = 24, at a count that gives the warps of ANY resident grid on this device at least three claims each (3 x the SMs'
    thread slots, in pairs): every alignment == the oracle, for every type"""
    require_gpu()
    sms, slots = warp_slots()
    count = 2 * 3 * sms * slots + 1
    n_max = count + 999
    band, m = 7, 24
    pr = window_batch(np.random.default_rng(4500), n_max, band, m)
    P, T = string_sets(pr, m)
    for typ in (GLOBAL, LOCAL, SEMI):
        want = O.banded_gotoh(band, typ, S4, *head(pr, count))
        out, route = indirect_banded(band, typ, Scheme6(S4), P, T, count, n_max)
        check(out, want, count, "rounds B7 t%d count=%d" % (typ, count))
        assert route == (1, 0)


def reads_batch(n_max, band, m, seed):
    """n_max reads of m bp sampled from a 2 Mbp genome on the device (synth.sample_reads) against windows of m + band - 1 symbols
    starting band // 2 before them, 2-bit big-endian; quality values 0..7 per pattern symbol"""
    n_gen = 2_000_000
    gw = synth.random_genome_words(n_gen, seed=seed)
    rw, pos, _ = synth.sample_reads(gw, n_gen, n_max, m, rc_half=False, seed=seed + 1, mut_seed=seed + 2)
    begin = (pos - band // 2).clamp_(0).to(torch.int32)
    stride = rw.shape[1] * 16
    g = torch.Generator(device="cuda"); g.manual_seed(seed)
    quals = torch.randint(0, 8, (n_max * stride,), dtype=torch.uint8, device="cuda", generator=g)
    return gw, n_gen, rw, begin, stride, quals


def check_rounds_on_reads(O, band, m, count, n_max, runs, seed):
    """runs = [(type, Scheme6, with quality)]: the device-count call at `count` == the exact-count call on the same jobs (all of them),
    == the oracle on a stride sample and on the last 256 alignments; nothing past the count written"""
    gw, n_gen, rw, begin, stride, quals = reads_batch(n_max, band, m, seed)
    P = PackedStringSet.fixed(rw.reshape(-1), n_max, m, stride=stride)
    T = PackedStringSet(words=gw, bits=2, big_endian=True, offsets=begin, lengths=None, stride=0, length=m + band - 1, count=n_max)
    Pc = PackedStringSet.fixed(rw.reshape(-1), count, m, stride=stride)
    Tc = PackedStringSet(words=gw, bits=2, big_endian=True, offsets=begin[:count], lengths=None, stride=0, length=m + band - 1, count=count)
    sample = np.unique(np.concatenate([np.arange(0, count, 997), np.arange(count - 256, count)]))
    gsym = unpack_symbols(host_u32(gw), n_gen)
    ps = unpack_symbols(host_u32(rw[torch.from_numpy(sample).cuda()]).reshape(-1), len(sample) * stride).reshape(len(sample), stride)[:, :m]
    qs = quals.view(n_max, stride)[torch.from_numpy(sample).cuda(), :m].cpu().numpy()
    k = len(sample)
    spr = (ps.reshape(-1), np.arange(k, dtype=np.uint32) * m, np.full(k, m, np.uint32), gsym, host_u32(begin)[sample], np.full(k, m + band - 1, np.uint32))
    for typ, sch, with_q in runs:
        what = "B%d m%d t%d %s count=%d" % (band, m, typ, sch.s6 if sch.qtab is None else "qtab", count)
        q = quals if with_q else None
        score, sink = Indirect((band, typ), sch, P, T, n_max, q).launch(count)
        assert last_route() == (1, 0), what
        ws, wk = aln.batch_banded_alignment_score(band, aln.make_gotoh_aligner(typ, sch), Pc, Tc, quals=q)
        assert last_route() == (1, 0), what
        assert torch.equal(score[:count], ws) and torch.equal(sink[:count], wk), what + ": differs from the exact-count call"
        assert bool((score[count:] == SENT).all()) and bool((sink[count:] == SENT).all()), what + ": written past the count"
        want = O.banded_gotoh(band, typ, sch.s6, *spr, qual=qs.reshape(-1) if with_q else None, qtab=sch.qtab)
        s, kk = score.cpu().numpy()[sample], host_u32(sink)[sample]
        assert_same((s, kk[:, 0], kk[:, 1]), want, what + " vs the oracle")


def test_banded_ticket_rounds_pipeline_shape(O):
    """band 31, m = 150, LOCAL (the seed + extend DP shape), 2-bit patterns (PFMT 2) and a quality table (PFMT 0), at three claims
    per warp of any resident grid"""
    require_gpu()
    sms, slots = warp_slots()
    count = 2 * 3 * sms * slots + 1
    runs = [(LOCAL, Scheme6(S4), False), (LOCAL, Scheme6((0, 0, -5, -3, -5, -3), edge_table(-6, 2)), True)]
    check_rounds_on_reads(O, 31, 150, count, count + 4096, runs, 4600)


def test_banded_ticket_rounds_at_the_selector_cap(O):
    """m = 801 - band: 200 KB of selectors, one CTA per SM, so 3 x SMs x 128 pairs already give every warp three claims"""
    require_gpu()
    sms, _ = warp_slots()
    count = 2 * 3 * sms * 128 + 1
    band = 31
    check_rounds_on_reads(O, band, 801 - band, count, count + 1000, [(t, Scheme6(S4), False) for t in (GLOBAL, LOCAL, SEMI)], 4700)


# --------------------------------------------------------------------------------------------------------------------------------------
# full matrix
# --------------------------------------------------------------------------------------------------------------------------------------
def full_sets(pr):
    pat, p_off, p_len, txt, t_off, t_len = pr
    return (PackedStringSet.from_symbols(pat, p_off, p_len, bits=2, big_endian=True),
            PackedStringSet.from_symbols(txt, t_off, t_len, bits=2, big_endian=True))


def test_full_device_count_at_every_edge(O):
    """every full_cases() edge through nvb_gotoh_score_indirect: the pair kernel at minb 2 / 3 / 4, its quality-table form and
    gotoh_full_kernel, the count far below the capacity"""
    require_gpu()
    count, n_max = 7, 32
    for name, typ, s4, m, n, ok in full_cases():
        rng = np.random.default_rng(7000 + 10 * typ + m + n)
        pr = full_batch(rng, 4, m, n)
        want = O.gotoh_full(typ, s4, *pr)
        P, T = full_sets(tile(pr, n_max))
        what = "%s t%d m%d n%d" % (name, typ, m, n)
        for minb in (2, 3, 4):
            with debug_knobs(full_warp=2, full_minb=minb):
                out, route = indirect_full(typ, Scheme6(s4), P, T, count, n_max)
            check(out, want, count, what + " minb=%d" % minb)
            assert_route(route, ok, what)
            assert not ok or route[0] == 1
        with debug_knobs(force_gotoh_path=1):
            out, route = indirect_full(typ, Scheme6(s4), P, T, count, n_max)
        check(out, want, count, what + " int32")
        assert route == (0, 0)
        qtab = edge_table(-3, s4[0])
        qual = rng.integers(0, 8, len(pr[0])).astype(np.uint8)
        s6 = (0, 0, -5, -5, -5, -5)
        want_q = O.gotoh_full(typ, s6, *pr, qual=qual, qtab=qtab)
        out, route = indirect_full(typ, Scheme6(s6, qtab), P, T, count, n_max, qual=torch.from_numpy(qual).cuda())
        check(out, want_q, count, what + " qtab")
        assert_route(route, ok, what + " qtab")


@pytest.mark.parametrize("W", range(1, 9))
def test_full_warp_kernel_edges_under_a_device_count(O, W):
    """the W = 1..8 edges of test_full_warp_kernel_at_its_limits through the device-count call"""
    require_gpu()
    count, n_max = 5, 24
    m = 256 if W == 8 else 32 * W - 3
    cases = [(typ, FULL_S, m, 5996 - m, True) for typ in (GLOBAL, LOCAL, SEMI)] + [(GLOBAL, FULL_S, m, 7400 - m, False)] + \
        [(typ, FULL_S, m, 5997 - m, False) for typ in (GLOBAL, LOCAL, SEMI)]
    if W == 8:
        cases += [(LOCAL, (8, -3, -5, -5), 255, 600, True), (LOCAL, (8, -3, -5, -5), 256, 600, False)]
    for typ, s4, mm, n, ok in cases:
        rng = np.random.default_rng(8000 + 10 * W + typ + n)
        pr = full_batch(rng, 3, mm, n)
        want = O.gotoh_full(typ, s4, *pr)
        P, T = full_sets(tile(pr, n_max))
        with debug_knobs(full_warp=1):
            out, route = indirect_full(typ, Scheme6(s4), P, T, count, n_max)
        what = "W%d t%d m%d n%d" % (W, typ, mm, n)
        check(out, want, count, what)
        assert_route(route, ok, what)
        assert not ok or route[0] == 2


def test_full_warp_threshold_under_a_device_count(O):
    """default knobs: with a device count the warp kernel takes up to 4 x 30,000 pairs of capacity (240,000 alignments), one
    alignment more goes to the pair kernel; exact on both sides, whatever the (small) count"""
    require_gpu()
    n_big, m, n, count = 240_001, 40, 64, 1001
    g = torch.Generator(device="cuda"); g.manual_seed(4800)

    def words(k):
        return torch.randint(-(1 << 31), 1 << 31, (k,), dtype=torch.int64, device="cuda", generator=g).to(torch.int32)
    tw = words(n_big * n // 16 + 8)
    pw = tw ^ (words(len(tw)) & words(len(tw)) & words(len(tw)))        # the text with one symbol in ~3 changed
    T = PackedStringSet.fixed(tw, n_big, n, stride=n)
    P = PackedStringSet(words=pw, bits=2, big_endian=True, offsets=(torch.arange(n_big, device="cuda", dtype=torch.int32) * n + 12),
                        lengths=None, stride=0, length=m, count=n_big)
    k = count * n
    tsym, psym = unpack_symbols(host_u32(tw[:k // 16]), k), unpack_symbols(host_u32(pw[:k // 16]), k)
    pr = (psym, np.arange(count, dtype=np.uint32) * n + 12, np.full(count, m, np.uint32), tsym, np.arange(count, dtype=np.uint32) * n,
          np.full(count, n, np.uint32))
    for typ in (GLOBAL, LOCAL, SEMI):
        want = O.gotoh_full(typ, S4, *pr)
        for n_max, packed in ((240_000, 2), (240_001, 1)):
            out, route = indirect_full(typ, Scheme6(S4), P, T, count, n_max)
            what = "t%d n_max=%d" % (typ, n_max)
            check(out, want, count, what)
            assert route == (packed, 0), what


def mixed_full(rng, n_pairs, max_m=100, max_n=160):
    """pairs of equal (m, n) (which the packed kernels admit) and pairs whose second alignment differs in m or in n (which they
    refuse): patterns that are substrings of their text with a few substitutions, or random"""
    pats, txts, pl, tl = [], [], [], []
    for _ in range(n_pairs):
        M = int(rng.integers(1, max_m + 1)); N = int(rng.integers(1, max_n + 1))
        kind = int(rng.integers(0, 4))
        for k in range(2):
            Mk = M if kind != 2 or k == 0 else max(1, M - int(rng.integers(1, 4)))
            Nk = N if kind != 3 or k == 0 else N + int(rng.integers(1, 4))
            t = rng.integers(0, 4, Nk).astype(np.uint8)
            if Nk > Mk and rng.random() < 0.7:
                st = int(rng.integers(0, Nk - Mk + 1)); p = t[st:st + Mk].copy()
                p[rng.integers(0, Mk, 3)] = rng.integers(0, 4, 3)
            else:
                p = rng.integers(0, 4, Mk).astype(np.uint8)
            pats.append(p); txts.append(t); pl.append(Mk); tl.append(Nk)
    pl, tl = np.array(pl, np.uint32), np.array(tl, np.uint32)
    po = np.concatenate([[0], np.cumsum(pl)[:-1]]).astype(np.uint32)
    to = np.concatenate([[0], np.cumsum(tl)[:-1]]).astype(np.uint32)
    return np.concatenate(pats), po, pl, np.concatenate(txts), to, tl


def refused_full(pr, count):
    """alignments the packed full-matrix kernels send to the int32 list among the first `count`: both of a pair whose (m, n) differ"""
    p_len, t_len = pr[2], pr[5]
    total = 0
    for a0 in range(0, count - 1, 2):
        if p_len[a0] != p_len[a0 + 1] or t_len[a0] != t_len[a0 + 1]:
            total += 2
    return total


@pytest.mark.parametrize("typ", (GLOBAL, LOCAL, SEMI))
def test_full_refused_pairs_and_count_shapes(O, typ):
    """pairs with unequal (m, n) go through the todo list and gotoh_full_todo_kernel under the device count, from the warp kernel,
    the pair kernel and its quality-table form; the count shapes of the banded test, the capacity and past it"""
    require_gpu()
    rng = np.random.default_rng(4900 + typ)
    pr = mixed_full(rng, MIX_CAP // 2)
    assert 0 < refused_full(pr, 1001) < refused_full(pr, MIX_CAP)
    qual = rng.integers(0, 8, len(pr[0])).astype(np.uint8)
    P, T = full_sets(pr)
    s6q, qtab = (0, 0, -5, -3, -5, -3), edge_table(-4, 3)
    want_c, want_q = O.gotoh_full(typ, S4, *pr), O.gotoh_full(typ, s6q, *pr, qual=qual, qtab=qtab)
    # (knobs, quality table, route): the warp kernel (the default at this capacity), the pair kernel, the pair kernel's quality form
    for knobs, with_q, packed in (({}, False, 2), (dict(full_warp=2), False, 1), ({}, True, 1)):
        for count in COUNTS + (MIX_CAP, MIX_CAP + 5):
            nn = min(count, MIX_CAP)
            with debug_knobs(**knobs):
                out, route = indirect_full(typ, Scheme6(s6q, qtab) if with_q else Scheme6(S4), P, T, count, MIX_CAP,
                                           qual=torch.from_numpy(qual).cuda() if with_q else None)
            what = "t%d %s qtab=%d count=%d" % (typ, knobs, with_q, count)
            check(out, want_q if with_q else want_c, nn, what)
            assert route == (packed, refused_full(pr, nn)), what


def test_full_temp_reuse_in_stream_order(O):
    """three full-matrix calls back to back on one temp buffer and one stream, no sync between them"""
    require_gpu()
    pr = mixed_full(np.random.default_rng(5000), MIX_CAP // 2)
    want = O.gotoh_full(LOCAL, S4, *pr)
    P, T = full_sets(pr)
    call = Indirect((LOCAL,), Scheme6(S4), P, T, MIX_CAP, full=True)
    a = call.launch(1001, -7)
    b = call.launch(129, -9)
    c = call.launch(1001, -11)
    route = last_route()
    check(a, want, 1001, "first", -7)
    check(b, want, 129, "second", -9)
    check(c, want, 1001, "third", -11)
    assert route == (2, refused_full(pr, 1001))
    assert torch.equal(a[0][:1001], c[0][:1001]) and torch.equal(a[1][:1001], c[1][:1001])
