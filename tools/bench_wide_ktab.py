"""Seed-match split on bench.py's headline workload (1M x 150 bp reads, 1.9 Gbp genome, full suffix array, 15-mer context table, per-row
array) with the 16-byte and the 32-byte (wide) k-mer table, alternating over the rounds on the same index: the table is rebuilt in
place for each configuration (both do not fit the card together).  Reports per configuration the step and seed_match times from device
events, the per-kernel device time of the two seed-match passes from torch.profiler, and checks that the per-read results are identical.
Prints one JSON line with the card, its power limit and the device memory resident after the index build and at its peak
afterwards (the steps and the table rebuilds).

    python tools/bench_wide_ktab.py [--rounds 3] [--steps 10] [--warmup 3]
"""
import argparse
import ctypes as C
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench  # noqa: E402
from tools.bench_mapq import power_limit_w  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reads", type=int, default=1_000_000)
    ap.add_argument("--genome-mbp", type=float, default=1900.0)
    a = ap.parse_args()
    import nvbio_b200 as nb
    from nvbio_b200 import aln
    from nvbio_b200._lib import lib, check
    from nvbio_b200.fmindex import _stream
    from nvbio_b200.strings import PackedStringSet
    from nvbio_b200.pipeline import SeedExtendWorkspace, last_stage_ms
    from torch.profiler import profile, ProfilerActivity

    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    nb.lib()
    idx_args = argparse.Namespace(genome_mbp=a.genome_mbp, sa_interval=1, ktab_k=15, ktab_located=2, impl="ours")
    n, genome, fmi, t_build, _ = bench.build_index(idx_args, 0, 1, device)
    torch.cuda.synchronize()
    resident_after_build = torch.cuda.memory_allocated(device)
    peak_during_build = torch.cuda.max_memory_allocated(device)
    torch.cuda.reset_peak_memory_stats(device)
    built_wide = bool(fmi.ktab_wide)
    k = fmi.ktab_k

    def use(cfg):
        if bool(fmi.ktab_wide) == (cfg == "wide"):
            return
        fmi.ktab = None
        torch.cuda.empty_cache()
        tab = torch.empty((4 ** k, 8 if cfg == "wide" else 4), dtype=torch.int32, device=device)
        s = fmi.struct()
        fn = lib().nvb_fm_build_ktab_wide if cfg == "wide" else lib().nvb_fm_build_ktab_context
        check(fn(C.byref(s), C.c_uint32(k), C.c_void_p(genome.data_ptr()), C.c_void_p(tab.data_ptr()), _stream()), cfg)
        torch.cuda.synchronize()
        fmi.ktab, fmi.ktab_wide = tab, cfg == "wide"

    params = nb.SeedExtendParams(seed_len=bench.SEED_LEN, seed_interval=bench.SEED_INTERVAL, band_len=bench.BAND, type=aln.LOCAL,
                                 both_strands=True, max_seed_hits=100, scheme=aln.SimpleGotohScheme(*bench.SCHEME))
    batches = [bench.make_reads(genome, n, a.reads, b, device) for b in range(2)]
    wpr = batches[0].shape[1]

    def as_set(words):
        return PackedStringSet.fixed(words.reshape(-1), a.reads, bench.READ_LEN, stride=wpr * 16)
    ws = SeedExtendWorkspace(fmi, genome, as_set(batches[0]), params, 24 * a.reads, keep_hits=False)
    flush = torch.empty(512 << 20, dtype=torch.uint8, device=device)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def step(i):
        nb.seed_extend(fmi, genome, as_set(batches[i % 2]), params, workspace=ws)

    def timed():
        for i in range(a.warmup):
            flush.zero_(); step(i)
        total, seed = 0.0, 0.0
        for i in range(a.steps):
            flush.zero_()
            ev0.record(); step(i); ev1.record()
            torch.cuda.synchronize()
            total += ev0.elapsed_time(ev1)
            seed += last_stage_ms()["seed_match"]
        return total / a.steps, seed / a.steps

    def kernel_split():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for i in range(a.steps):
                flush.zero_(); step(i)
            torch.cuda.synchronize()
        out = {}
        for e in prof.key_averages():
            if "pipe_seed_match" in e.key:
                us = getattr(e, "device_time_total", None)
                if us is None:
                    us = e.cuda_time_total
                out[e.key] = {"ms_per_step": us / 1e3 / a.steps, "calls": e.count}
        return out

    configs = ["narrow", "wide"]
    results = {c: [] for c in configs}
    outputs, split = {}, {}
    for r in range(a.rounds):
        for c in configs:
            use(c)
            ms, seed_ms = timed()
            results[c].append({"step_ms": ms, "mreads_s": a.reads / (ms * 1e-3) / 1e6, "seed_match_ms": seed_ms})
            if r == 0:
                outputs[c] = (ws.best_score.clone(), ws.best_pos.clone(), ws.n_hits.clone())
                split[c] = kernel_split()
    same = all(torch.equal(x, y) for x, y in zip(outputs["narrow"], outputs["wide"]))
    print(json.dumps({"workload": "seed_extend seed-match split, 16- vs 32-byte k-mer table", "reads": a.reads, "read_len": bench.READ_LEN,
                      "genome_bp": n, "card": torch.cuda.get_device_name(device), "power_limit_w": power_limit_w(), "steps": a.steps,
                      "warmup": a.warmup, "index_build_s": t_build, "built_wide": built_wide, "rows": fmi.rows is not None,
                      "bytes_resident_after_index_build": resident_after_build,
                      "peak_bytes_during_index_build": peak_during_build, "peak_bytes_after_index_build": torch.cuda.max_memory_allocated(device),
                      "index_bytes_wide": fmi.nbytes(), "rounds": results, "kernels": split, "outputs_identical": same}))
    assert same, "per-read results differ between the 16- and 32-byte tables"


if __name__ == "__main__":
    main()
