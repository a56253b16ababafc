"""Cost of the coordinate sort (nvb_bam_sort) and the BAI index (nvb_bam_index) on the device, on tools/bench_bgzf.py's workload: bench.py's
paired-end reads (500k FR pairs of 2 x 150 bp, 1.9 Gbp genome, 25 contigs), paired traceback, finish_alignments and nvb_bam_records once,
no base qualities.  Each call is timed with device events over repeated calls (median, min, max); a separate torch.profiler run gives
the device time of each kernel of one call, and the gather kernel's 2 x record bytes over its time as a share of 3.35 TB/s.  Also the wall
time of write_sorted_bam next to write_bam's device path (bgzf_compress).  Prints one JSON line with the card and its power limit.

    python tools/bench_bam_sort.py [--steps 20] [--warmup 3]
"""
import argparse
import ctypes as C
import json
import os
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench  # noqa: E402
from tools.bench_mapq import power_limit_w  # noqa: E402
from tools.bench_bam import contig_table  # noqa: E402

HBM_TBPS = 3.35


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--pairs", type=int, default=500_000)
    ap.add_argument("--genome-mbp", type=float, default=1900.0)
    a = ap.parse_args()
    import nvbio_b200 as nb
    from nvbio_b200 import aln, synth
    from nvbio_b200.bam import BamCall
    from nvbio_b200.bam_sort import _bgzf_block, _BGZF_DATA
    from nvbio_b200._lib import lib, check, BaiOutStruct, BamSortOutStruct
    from nvbio_b200.strings import PackedStringSet
    from nvbio_b200.pipeline import PairedWorkspace

    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    idx_args = argparse.Namespace(genome_mbp=a.genome_mbp, sa_interval=1, ktab_k=15, ktab_located=2, impl="ours")
    n, genome, fmi, _, _ = bench.build_index(idx_args, 0, 1, device)
    params = nb.SeedExtendParams(seed_len=bench.SEED_LEN, seed_interval=bench.SEED_INTERVAL, band_len=bench.BAND, type=aln.LOCAL,
                                 both_strands=True, max_seed_hits=100, scheme=aln.SimpleGotohScheme(*bench.SCHEME))
    R = bench.READ_LEN
    n_pairs = a.pairs
    words, _, _ = synth.sample_pairs(genome, n, n_pairs, R, frag_mean=350.0, frag_sd=30.0, sub_rate=0.01, hard_frac=0.05,
                                     hard_sub_rate=0.2, device=device, seed=0x51ED, mut_seed=0xC0FFEE)
    reads = PackedStringSet.fixed(words.reshape(-1), 2 * n_pairs, R, stride=words.shape[1] * 16)
    pair = nb.PairParams(min_frag=0, max_frag=500, min_mate_score=80, rescue_capacity=max(n_pairs // 4, 1024))
    ws = nb.seed_extend_paired(fmi, genome, reads, params, pair,
                               workspace=PairedWorkspace(fmi, genome, reads, params, pair, 24 * 2 * n_pairs, traceback=True))
    f = nb.finish_alignments(genome, reads, ws.mate_ops, ws.mate_n_ops, ws.mate_begin, ws.mate_strand, genome_len=n)
    table = contig_table(nb, n, 25, 1)
    names = nb.numbered_names(n_pairs, "pair")
    recs = BamCall(ws, f, reads, table, names, None).run()
    torch.cuda.synchronize()
    n_rec = recs.offsets.numel() - 1
    total = int(recs.offsets[-1])

    # the sort call with its buffers made once
    src, src_off = recs.data[:total], recs.offsets
    s_data = torch.empty(total, dtype=torch.uint8, device=device)
    s_off = torch.empty(n_rec + 1, dtype=torch.int64, device=device)
    s_order = torch.empty(n_rec, dtype=torch.int32, device=device)
    so = BamSortOutStruct()
    so.d_records, so.capacity, so.d_offsets, so.d_order = s_data.data_ptr(), total, s_off.data_ptr(), s_order.data_ptr()
    sargs = (C.c_void_p(src.data_ptr()), C.c_void_p(src_off.data_ptr()), C.c_uint32(n_rec), C.byref(so))
    tb = C.c_size_t(0)
    lib().nvb_bam_sort(*sargs, None, C.byref(tb), None)
    s_temp = torch.empty(tb.value, dtype=torch.uint8, device=device)
    s_tb = tb.value

    def sort_call():
        t = C.c_size_t(s_tb)
        check(lib().nvb_bam_sort(*sargs, C.c_void_p(s_temp.data_ptr()), C.byref(t), C.c_void_p(torch.cuda.current_stream().cuda_stream)),
              "nvb_bam_sort")

    sort_call()
    blocks = nb.bgzf_compress(s_data)
    header = nb.bam_header(table, sort_order="coordinate")
    hb = sum(len(_bgzf_block(header[i:i + _BGZF_DATA])) for i in range(0, len(header), _BGZF_DATA))
    sorted_recs = nb.SortedBamRecords(data=s_data, offsets=s_off, order=s_order)
    bai_len = len(nb.bam_index(sorted_recs, blocks, hb, table))
    bai = torch.empty(bai_len, dtype=torch.uint8, device=device)
    size = torch.zeros(1, dtype=torch.int64, device=device)
    status = torch.zeros(1, dtype=torch.int32, device=device)
    bo = BaiOutStruct()
    bo.d_bai, bo.capacity, bo.d_size, bo.d_status = bai.data_ptr(), bai_len, size.data_ptr(), status.data_ptr()
    iargs = (C.c_void_p(s_data.data_ptr()), C.c_void_p(s_off.data_ptr()), C.c_uint32(n_rec), C.c_void_p(blocks.offsets.data_ptr()),
             C.c_uint64(hb), C.c_uint32(len(table.names)), C.c_uint32(int(table.lengths.max())), C.byref(bo))
    lib().nvb_bam_index(*iargs, None, C.byref(tb), None)
    i_temp = torch.empty(tb.value, dtype=torch.uint8, device=device)
    i_tb = tb.value

    def index_call():
        t = C.c_size_t(i_tb)
        check(lib().nvb_bam_index(*iargs, C.c_void_p(i_temp.data_ptr()), C.byref(t), C.c_void_p(torch.cuda.current_stream().cuda_stream)),
              "nvb_bam_index")

    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(fn):
        for _ in range(a.warmup):
            fn()
        times = []
        for _ in range(a.steps):
            ev0.record(); fn(); ev1.record()
            torch.cuda.synchronize()
            times.append(ev0.elapsed_time(ev1))
        times.sort()
        return {"ms_median": round(times[len(times) // 2], 4), "ms_min": round(times[0], 4), "ms_max": round(times[-1], 4)}

    result = {"workload": "nvb_bam_sort + nvb_bam_index of nvb_bam_records after seed_extend_paired_traceback + finish_alignments",
              "pairs": n_pairs, "records": n_rec, "record_bytes": total, "bai_bytes": bai_len, "card": torch.cuda.get_device_name(device),
              "power_limit_w": power_limit_w()}
    result["sort"] = timed(sort_call)
    result["index"] = timed(index_call)
    assert int(status) == 0

    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        sort_call(); index_call(); torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        if e.device_time_total > 0:
            kern[e.key[:80]] = round(e.device_time_total / 1e3, 4)
    result["kernels_ms"] = kern
    gather_ms = sum(v for k, v in kern.items() if "bam_gather_kernel" in k)
    if gather_ms:
        result["gather_tbps"] = round(2 * total / (gather_ms * 1e-3) / 1e12, 3)
        result["gather_share_of_hbm"] = round(result["gather_tbps"] / HBM_TBPS, 3)

    with tempfile.TemporaryDirectory() as td:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        nb.write_bam(os.path.join(td, "u.bam"), nb.bam_header(table), [nb.bgzf_compress(recs)])
        result["write_bam_device_path_s"] = round(time.perf_counter() - t0, 3)
        t0 = time.perf_counter()
        nb.write_sorted_bam(os.path.join(td, "s.bam"), table, recs)
        result["write_sorted_bam_s"] = round(time.perf_counter() - t0, 3)
    result.update(steps=a.steps, warmup=a.warmup)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
