"""The two seed-match passes on bench.py's headline workload (1M x 150 bp reads, 1.9 Gbp genome, full suffix array, wide 15-mer table and
per-row array, the per-read path), for the in-tree library and optionally a second build of it (--other-lib, e.g. one built from an
earlier commit), alternating over the rounds on one index in one process.  Reports per build the step and seed_match times from device
events, the per-kernel device time of pipe_seed_match_kernel (first pass) and pipe_seed_match_wide_kernel (second pass) from
torch.profiler in a run of its own, and the seeds the first pass handed to the second per step (nvb_debug_seed_todo, read from the
device after the step; null for a build without that hook), and checks that both builds give identical per-read results.  Prints one
JSON line with the card and its power limit.

    python tools/bench_seed_passes.py [--other-lib PATH] [--rounds 3] [--steps 10] [--warmup 3]
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
from tools.bench_resolve_split import profiled_ms  # noqa: E402

KERNELS = ("pipe_seed_match_kernel", "pipe_seed_match_wide_kernel")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--other-lib", default=None, help="a second build of libnvbio_b200.so to compare with the in-tree one")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reads", type=int, default=1_000_000)
    ap.add_argument("--genome-mbp", type=float, default=1900.0)
    a = ap.parse_args()
    import nvbio_b200 as nb
    from nvbio_b200 import _lib, aln
    from nvbio_b200.strings import PackedStringSet
    from nvbio_b200.pipeline import SeedExtendWorkspace, last_stage_ms

    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    libs = {"tree": nb.lib()}
    if a.other_lib:
        # the wrappers call _lib.lib(): the module's handle is switched between the builds
        libs["other"] = C.CDLL(os.path.abspath(a.other_lib))
        libs["other"].nvb_error_string.restype = C.c_char_p
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
        flush.zero_()
        nb.seed_extend(fmi, genome, as_set(batches[i % 2]), params, workspace=ws)

    def todo_count():
        try:
            hook = _lib._lib.nvb_debug_seed_todo
        except AttributeError:
            return None
        v = C.c_uint32(0)
        return v.value if hook(C.byref(v)) == 0 else None

    def timed():
        for i in range(a.warmup):
            step(i)
        total = seed = 0.0
        todo = []
        for i in range(a.steps):
            flush.zero_()
            ev0.record(); nb.seed_extend(fmi, genome, as_set(batches[i % 2]), params, workspace=ws); ev1.record()
            torch.cuda.synchronize()
            total += ev0.elapsed_time(ev1)
            seed += last_stage_ms()["seed_match"]
            todo.append(todo_count())
        return total / a.steps, seed / a.steps, todo

    results = {c: [] for c in libs}
    outputs, kernels, todo = {}, {}, {}
    for r in range(a.rounds):
        for c, handle in libs.items():
            _lib._lib = handle
            ms, seed_ms, t = timed()
            results[c].append({"step_ms": ms, "mreads_s": a.reads / (ms * 1e-3) / 1e6, "seed_match_ms": seed_ms})
            if r == 0:
                outputs[c] = (ws.best_score.clone(), ws.best_pos.clone(), ws.n_hits.clone())
                todo[c] = None if None in t else sum(t) / len(t)
                kernels[c] = profiled_ms(step, a.steps, KERNELS)
    _lib._lib = libs["tree"]
    same = all(torch.equal(x, y) for c in libs for x, y in zip(outputs[c], outputs["tree"]))
    print(json.dumps({"workload": "seed_extend seed-match passes", "reads": a.reads, "read_len": bench.READ_LEN, "genome_bp": n,
                      "card": torch.cuda.get_device_name(device), "power_limit_w": power_limit_w(), "steps": a.steps, "warmup": a.warmup,
                      "index_build_s": t_build, "ktab_wide": bool(fmi.ktab_wide), "rows": fmi.rows is not None,
                      "other_lib": a.other_lib, "rounds": results, "kernels_ms_per_step": kernels,
                      "seeds_to_second_pass_per_step": todo,
                      "outputs_identical": same}))
    assert same, "per-read results differ between the two builds"


if __name__ == "__main__":
    main()
