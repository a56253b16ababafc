"""Extension split on bench.py's headline workload (1M x 150 bp reads, 1.9 Gbp genome, band 31 LOCAL, (2, -2, -5, -3)) with the exact
shortcut's one-gap check on and off (nvb_debug_perfect_shortcut 1 / 2), alternating over the rounds in one process on the same index.
Reports per rule the step and extension-stage times from device events, the jobs left to the DP per step (nvb_debug_dp_jobs), the
per-kernel device time of the kernel that runs the shortcut (pipe_resolve_reads_kernel), the banded DP kernels, the scatter and the finalize from torch.profiler, and checks that the per-read
results are identical.  Prints one JSON line with the card and its power limit.

    python tools/bench_shortcut.py [--rounds 3] [--steps 10] [--warmup 3]
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

KERNELS = ("pipe_resolve_reads_kernel", "gotoh_pair_kernel", "gotoh_generic_kernel", "pipe_scatter_dp_kernel", "pipe_finalize_dp_kernel")
RULES = {"one_gap": 1, "gap_free": 2}


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
    from nvbio_b200.strings import PackedStringSet
    from nvbio_b200.pipeline import SeedExtendWorkspace, last_stage_ms
    from torch.profiler import profile, ProfilerActivity

    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    L_ = nb.lib()
    idx_args = argparse.Namespace(genome_mbp=a.genome_mbp, sa_interval=1, ktab_k=15, ktab_located=2, impl="ours")
    n, genome, fmi, t_build, _ = bench.build_index(idx_args, 0, 1, device)
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

    def dp_jobs():
        v = C.c_uint32(0)
        assert L_.nvb_debug_dp_jobs(C.byref(v)) == 0
        return v.value

    def timed():
        for i in range(a.warmup):
            flush.zero_(); step(i)
        total, ext, dp = 0.0, 0.0, 0
        for i in range(a.steps):
            flush.zero_()
            ev0.record(); step(i); ev1.record()
            torch.cuda.synchronize()
            total += ev0.elapsed_time(ev1)
            ext += last_stage_ms()["extend"]
            dp += dp_jobs()
        return total / a.steps, ext / a.steps, dp / a.steps

    def kernel_split():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for i in range(a.steps):
                flush.zero_(); step(i)
            torch.cuda.synchronize()
        out = {}
        for e in prof.key_averages():
            if any(k in e.key for k in KERNELS):
                us = getattr(e, "device_time_total", None)
                if us is None:
                    us = e.cuda_time_total
                out[e.key] = {"ms_per_step": us / 1e3 / a.steps, "calls": e.count}
        return out

    results = {c: [] for c in RULES}
    outputs, split = {}, {}
    try:
        for r in range(a.rounds):
            for c, rule in RULES.items():
                L_.nvb_debug_perfect_shortcut(C.c_int(rule))
                ms, ext_ms, dp = timed()
                results[c].append({"step_ms": ms, "mreads_s": a.reads / (ms * 1e-3) / 1e6, "extend_ms": ext_ms, "dp_jobs_per_step": dp})
                if r == 0:
                    outputs[c] = (ws.best_score.clone(), ws.best_pos.clone(), ws.n_hits.clone())
                    split[c] = kernel_split()
    finally:
        L_.nvb_debug_perfect_shortcut(C.c_int(1))
    same = all(torch.equal(x, y) for x, y in zip(outputs["one_gap"], outputs["gap_free"]))
    print(json.dumps({"workload": "seed_extend extension split, exact shortcut with / without the one-gap check", "reads": a.reads,
                      "read_len": bench.READ_LEN, "genome_bp": n, "card": torch.cuda.get_device_name(device), "power_limit_w": power_limit_w(),
                      "steps": a.steps, "warmup": a.warmup, "index_build_s": t_build, "rounds": results, "kernels": split,
                      "outputs_identical": same}))
    assert same, "per-read results differ between the two rules"


if __name__ == "__main__":
    main()
