"""Per-kernel split of one seed + extend step on bench.py's headline workload (1M x 150 bp reads, 1.9 Gbp genome, band 31 LOCAL,
(2, -2, -5, -3), hit capacity 24 per read, per-read path).  Reports the device time of every kernel the step launches (torch.profiler,
nothing filtered: the L2 flush between steps is listed too, under its own name), the step time from device events, the stage split
(last_stage_ms), the jobs left to the DP (nvb_debug_dp_jobs) and n_hits, with the card and its power limit, as one JSON line.  Only public
API is used, so the same file measures any build of the library.  --type global runs the same reads end to end, where the exact
shortcut does not apply and every job goes through the DP list.

    python tools/bench_resolve.py [--steps 10] [--warmup 3] [--type local|global] [--out DIR]
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

# kernels that are not the glue between the seed match and the DP: the [fw, rc] strings, the seed match, the banded DP, the flush
NOT_GLUE = ("pipe_make_strings", "pipe_seed_match", "gotoh_", "elementwise_kernel")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reads", type=int, default=1_000_000)
    ap.add_argument("--genome-mbp", type=float, default=1900.0)
    ap.add_argument("--type", default="local", choices=["local", "global"])
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/bench_resolve_<type>.json")
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
    params = nb.SeedExtendParams(seed_len=bench.SEED_LEN, seed_interval=bench.SEED_INTERVAL, band_len=bench.BAND,
                                 type=aln.LOCAL if a.type == "local" else aln.GLOBAL,
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

    for i in range(a.warmup):
        flush.zero_(); step(i)
    total, stages, dp = 0.0, None, 0
    for i in range(a.steps):
        flush.zero_()
        ev0.record(); step(i); ev1.record()
        torch.cuda.synchronize()
        total += ev0.elapsed_time(ev1)
        st = last_stage_ms()
        stages = st if stages is None else {k: stages[k] + st[k] for k in st}
        v = C.c_uint32(0)
        if dp is not None and L_.nvb_debug_dp_jobs(C.byref(v)) == 0:
            dp += v.value
        else:
            dp = None                                      # a build that only counts the DP list when the shortcut runs
    n_hits = [int(x) for x in ws.n_hits.cpu()]

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(a.steps):
            flush.zero_(); step(i)
        torch.cuda.synchronize()
    kernels = {}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        if us <= 0:
            continue
        kernels[e.key] = {"ms_per_step": us / 1e3 / a.steps, "calls_per_step": e.count / a.steps}
    kernels = dict(sorted(kernels.items(), key=lambda kv: -kv[1]["ms_per_step"]))
    glue = sum(v["ms_per_step"] for k, v in kernels.items() if not any(p in k for p in NOT_GLUE))
    line = {"workload": "seed_extend per-kernel split (headline, per-read path)", "reads": a.reads, "read_len": bench.READ_LEN, "genome_bp": n,
            "type": a.type, "temp_bytes": ws.temp_bytes, "card": torch.cuda.get_device_name(device), "power_limit_w": power_limit_w(), "steps": a.steps, "warmup": a.warmup,
            "index_build_s": t_build, "step_ms": total / a.steps, "mreads_s": a.reads / (total / a.steps * 1e-3) / 1e6,
            "stage_ms": {k: v / a.steps for k, v in stages.items()}, "dp_jobs_per_step": None if dp is None else dp / a.steps, "n_hits": n_hits,
            "glue_ms": glue, "glue_note": "every kernel except the strings, the seed match, the banded DP and the L2 flush",
            "kernels": kernels}
    s = json.dumps(line)
    print(s, flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_resolve_%s.json" % a.type), "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
