"""nvb_banded_gotoh_score_indirect: the packed DP under a device-side count far below the batch capacity (the seed + extend DP list) gives
exactly what nvb_banded_gotoh_score gives on the same count, leaves every entry past the count untouched, and can be called again on
the same temp buffer (its pair ticket is zeroed per call)."""
import ctypes as C
import pytest
import torch
import nvbio_b200 as nb
from nvbio_b200 import aln, synth
from nvbio_b200.strings import PackedStringSet
from tests.gpu_util import require_gpu

pytestmark = pytest.mark.gpu

BAND, M, CAPACITY = 31, 150, 200_000


def test_indirect_count_below_capacity_equals_exact_count():
    require_gpu()
    L = nb.lib()
    n_gen = 2_000_000
    gw = synth.random_genome_words(n_gen, seed=11)
    n_max_jobs = 20_001
    rw, pos, _ = synth.sample_reads(gw, n_gen, n_max_jobs, M, rc_half=False)
    begin = (pos - BAND // 2).clamp_(0).to(torch.int32)
    P = PackedStringSet.fixed(rw.reshape(-1), n_max_jobs, M, stride=rw.shape[1] * 16)
    T = PackedStringSet(words=gw, bits=2, big_endian=True, offsets=begin, lengths=None, stride=0, length=M + BAND - 1, count=n_max_jobs)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    ps, ts = P.struct(), T.struct()
    for typ in (aln.LOCAL, aln.GLOBAL, aln.SEMI_GLOBAL):
        sch = aln.make_gotoh_aligner(typ, aln.SimpleGotohScheme(2, -2, -5, -3)).scheme.struct()
        tb = C.c_size_t(0)
        L.nvb_banded_gotoh_score_indirect(C.c_int(BAND), C.c_int(typ), C.byref(sch), C.byref(ps), None, C.byref(ts),
                                          C.c_void_p(16), C.c_uint32(CAPACITY), None, None, None, C.byref(tb), stream)
        temp = torch.empty(tb.value, dtype=torch.uint8, device="cuda")
        for n in (0, 1, 2, 255, 256, 257, 4097, n_max_jobs):
            want = aln.batch_banded_alignment_score(BAND, aln.make_gotoh_aligner(typ, aln.SimpleGotohScheme(2, -2, -5, -3)),
                                                    PackedStringSet.fixed(rw.reshape(-1), max(n, 1), M, stride=rw.shape[1] * 16),
                                                    PackedStringSet(words=gw, bits=2, big_endian=True, offsets=begin[:max(n, 1)], lengths=None,
                                                                    stride=0, length=M + BAND - 1, count=max(n, 1)))
            score = torch.full((CAPACITY,), -7, dtype=torch.int32, device="cuda")
            sink = torch.full((CAPACITY, 2), -7, dtype=torch.int32, device="cuda")
            d_n = torch.tensor([n], dtype=torch.int32, device="cuda")
            for _ in range(2):                                  # the same temp twice: the ticket must start from zero each call
                t = C.c_size_t(temp.numel())
                assert L.nvb_banded_gotoh_score_indirect(C.c_int(BAND), C.c_int(typ), C.byref(sch), C.byref(ps), None, C.byref(ts),
                                                         C.c_void_p(d_n.data_ptr()), C.c_uint32(CAPACITY), C.c_void_p(score.data_ptr()),
                                                         C.c_void_p(sink.data_ptr()), C.c_void_p(temp.data_ptr()), C.byref(t), stream) == 0
                torch.cuda.synchronize()
                assert torch.equal(score[:n], want[0][:n]) and torch.equal(sink[:n], want[1][:n]), (typ, n)
                assert bool((score[n:] == -7).all()) and bool((sink[n:] == -7).all()), (typ, n)
                score[:n] = -7; sink[:n] = -7
