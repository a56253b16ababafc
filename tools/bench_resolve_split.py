"""Where the time between the seed match and the DP goes, on bench.py's headline workload (1M x 150 bp reads, 1.9 Gbp genome, band 31
LOCAL, (2, -2, -5, -3), hit capacity 24 per read, per-read path).  One process, one index, three measurements, one JSON line:

  * `resolve`: device time per step of pipe_resolve_reads_kernel and gotoh_pair_kernel (torch.profiler) with the exact shortcut on
    (nvb_debug_perfect_shortcut 1), without its one-gap check (2) and off (0), with the jobs left to the DP.  Off, phase B only copies
    every job into the DP list, so 1 - 0 is the shortcut's own time in the kernel and 0 is the ranges, hit slots, look-back and phase A
    (plus the DP-list copy); the DP's time at 0 and 1 prices its job count.
  * `dp_launch`: gotoh_pair_kernel alone on the step's DP job count (the 1 above; synthetic 150 bp reads against 180-symbol windows of
    the same genome), called with the exact count (nvb_banded_gotoh_score) and with a device-side count under the pipeline's capacity of
    24 M jobs (nvb_banded_gotoh_score_indirect).  The difference is what the packed launch costs beyond its jobs.
  * the card and its power limit.

    python tools/bench_resolve_split.py [--steps 10] [--warmup 3] [--out DIR]
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

KERNELS = ("pipe_resolve_reads_kernel", "gotoh_pair_kernel")


def profiled_ms(fn, steps, names):
    """device ms per call of every kernel whose name contains one of `names` (fn is called `steps` times under the profiler)"""
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(steps):
            fn(i)
        torch.cuda.synchronize()
    out = {n: 0.0 for n in names}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        for n in names:
            if n in e.key:
                out[n] += us / 1e3 / steps
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reads", type=int, default=1_000_000)
    ap.add_argument("--genome-mbp", type=float, default=1900.0)
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/bench_resolve_split.json")
    a = ap.parse_args()
    import nvbio_b200 as nb
    from nvbio_b200 import aln
    from nvbio_b200.strings import PackedStringSet
    from nvbio_b200.pipeline import SeedExtendWorkspace

    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    L_ = nb.lib()
    idx_args = argparse.Namespace(genome_mbp=a.genome_mbp, sa_interval=1, ktab_k=15, ktab_located=2, impl="ours")
    n, genome, fmi, _, _ = bench.build_index(idx_args, 0, 1, device)
    params = nb.SeedExtendParams(seed_len=bench.SEED_LEN, seed_interval=bench.SEED_INTERVAL, band_len=bench.BAND, type=aln.LOCAL,
                                 both_strands=True, max_seed_hits=100, scheme=aln.SimpleGotohScheme(*bench.SCHEME))
    batches = [bench.make_reads(genome, n, a.reads, b, device) for b in range(2)]
    wpr = batches[0].shape[1]
    capacity = 24 * a.reads

    def as_set(words):
        return PackedStringSet.fixed(words.reshape(-1), a.reads, bench.READ_LEN, stride=wpr * 16)
    ws = SeedExtendWorkspace(fmi, genome, as_set(batches[0]), params, capacity, keep_hits=False)
    flush = torch.empty(512 << 20, dtype=torch.uint8, device=device)

    def step(i):
        flush.zero_()
        nb.seed_extend(fmi, genome, as_set(batches[i % 2]), params, workspace=ws)

    resolve = {}
    for mode in (1, 2, 0):
        L_.nvb_debug_perfect_shortcut(C.c_int(mode))
        for i in range(a.warmup):
            step(i)
        ms = profiled_ms(step, a.steps, KERNELS)
        v = C.c_uint32(0)
        L_.nvb_debug_dp_jobs(C.byref(v))
        resolve[str(mode)] = {"kernels_ms": ms, "dp_jobs": v.value, "n_hits": [int(x) for x in ws.n_hits.cpu()]}
    L_.nvb_debug_perfect_shortcut(C.c_int(1))

    # the DP alone on the step's job count: exact count against a device-side count under the pipeline's capacity
    jobs = resolve["1"]["dp_jobs"]
    g = torch.Generator(device="cpu").manual_seed(7)
    pos = torch.randint(16, n - 400, (jobs,), generator=g).to(torch.int32)
    rw = bench.make_reads(genome, n, jobs, 3, device)
    P = PackedStringSet.fixed(rw.reshape(-1), jobs, bench.READ_LEN, stride=rw.shape[1] * 16)
    T = PackedStringSet(words=genome, bits=2, big_endian=True, offsets=pos.to(device), lengths=None, stride=0,
                        length=bench.READ_LEN + bench.BAND - 1, count=jobs)
    aligner = aln.make_gotoh_aligner(aln.LOCAL, aln.SimpleGotohScheme(*bench.SCHEME))
    sch, ps, ts = aligner.scheme.struct(), P.struct(), T.struct()
    score = torch.empty(capacity, dtype=torch.int32, device=device)
    sink = torch.empty((capacity, 2), dtype=torch.int32, device=device)
    d_n = torch.tensor([jobs], dtype=torch.int32, device=device)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    tb = C.c_size_t(0)
    L_.nvb_banded_gotoh_score_indirect(C.c_int(bench.BAND), C.c_int(aln.LOCAL), C.byref(sch), C.byref(ps), None, C.byref(ts),
                                       C.c_void_p(d_n.data_ptr()), C.c_uint32(capacity), None, None, None, C.byref(tb), stream)
    temp = torch.empty(max(tb.value, 1), dtype=torch.uint8, device=device)

    def direct(_):
        t = C.c_size_t(temp.numel())
        assert L_.nvb_banded_gotoh_score(C.c_int(bench.BAND), C.c_int(aln.LOCAL), C.byref(sch), C.byref(ps), None, C.byref(ts),
                                         C.c_uint32(jobs), C.c_void_p(score.data_ptr()), C.c_void_p(sink.data_ptr()),
                                         C.c_void_p(temp.data_ptr()), C.byref(t), stream) == 0

    def indirect(_):
        t = C.c_size_t(temp.numel())
        assert L_.nvb_banded_gotoh_score_indirect(C.c_int(bench.BAND), C.c_int(aln.LOCAL), C.byref(sch), C.byref(ps), None, C.byref(ts),
                                                  C.c_void_p(d_n.data_ptr()), C.c_uint32(capacity), C.c_void_p(score.data_ptr()),
                                                  C.c_void_p(sink.data_ptr()), C.c_void_p(temp.data_ptr()), C.byref(t), stream) == 0
    dp_launch = {}
    for name, fn in (("direct", direct), ("indirect", indirect), ("direct_again", direct)):
        for i in range(a.warmup):
            fn(i)
        dp_launch[name] = profiled_ms(fn, a.steps, ("gotoh_pair_kernel",))["gotoh_pair_kernel"]
    direct(0)
    ref = (score[:jobs].clone(), sink[:jobs].clone())
    indirect(0)
    dp_launch["identical"] = bool(torch.equal(ref[0], score[:jobs]) and torch.equal(ref[1], sink[:jobs]))
    dp_launch["jobs"] = jobs
    dp_launch["capacity"] = capacity

    line = {"workload": "resolve / DP split (headline, per-read path)", "reads": a.reads, "genome_bp": n, "steps": a.steps,
            "card": torch.cuda.get_device_name(device), "power_limit_w": power_limit_w(),
            "resolve_by_shortcut_mode": resolve, "dp_launch_ms": dp_launch}
    s = json.dumps(line)
    print(s, flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_resolve_split.json"), "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
