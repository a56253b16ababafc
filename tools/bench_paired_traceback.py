"""Cost of the alignment of both mates: nvb_seed_extend_paired against nvb_seed_extend_paired_traceback (and, in a second pair of
workspaces, nvb_seed_extend_paired_mapq against the traceback with mapq) on bench.py's paired-end workload (500k FR pairs of 2 x 150 bp
from synth.sample_pairs, 1.9 Gbp genome, full suffix array, 15-mer table with text context, PairParams(0, 500, 80, n/4)), alternated in
one process over several rounds and timed with device events.  Asserts that the pair outputs are equal.  Also times the single-end
nvb_seed_extend_traceback over the 2n mates on the per-read path against the per-hit path (nvb_debug_pipeline_path(1)) and checks that
both give the same outputs.  Prints one JSON line with the card and its power limit, ms per step, the added ms, the rescued mates traced
and every workspace's temp bytes.  When the workspaces do not fit beside the index the tool says so and halves the pairs.
--profile: instead, one torch.profiler run of each call (CUDA activities) and the per-kernel device times of the traceback's kernels.

    python tools/bench_paired_traceback.py [--rounds 3] [--steps 10] [--warmup 3] [--profile]
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

PAIR_OUTPUTS = ("pair_score", "pair_flags", "mate_score", "mate_pos", "mate_strand", "n_rescue", "n_hits")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--pairs", type=int, default=500_000)
    ap.add_argument("--genome-mbp", type=float, default=1900.0)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    import nvbio_b200 as nb
    from nvbio_b200 import aln, synth
    from nvbio_b200.strings import PackedStringSet
    from nvbio_b200.pipeline import PairedWorkspace, SeedExtendWorkspace, MapqParams

    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    L = nb.lib()
    idx_args = argparse.Namespace(genome_mbp=a.genome_mbp, sa_interval=1, ktab_k=15, ktab_located=2, impl="ours")
    n, genome, fmi, _, _ = bench.build_index(idx_args, 0, 1, device)
    params = nb.SeedExtendParams(seed_len=bench.SEED_LEN, seed_interval=bench.SEED_INTERVAL, band_len=bench.BAND, type=aln.LOCAL,
                                 both_strands=True, max_seed_hits=100, scheme=aln.SimpleGotohScheme(*bench.SCHEME))
    R = bench.READ_LEN
    mq = MapqParams.local(R, device=device)
    n_pairs, note = a.pairs, None
    while True:
        try:
            batches = []
            for seed, mut in ((0x51ED, 0xC0FFEE), (0x61ED, 0xD0FFEE)):          # bench.py's two batches (rank 0)
                words, _, _ = synth.sample_pairs(genome, n, n_pairs, R, frag_mean=350.0, frag_sd=30.0, sub_rate=0.01, hard_frac=0.05,
                                                 hard_sub_rate=0.2, device=device, seed=seed, mut_seed=mut)
                batches.append(PackedStringSet.fixed(words.reshape(-1), 2 * n_pairs, R, stride=words.shape[1] * 16))
            pair = nb.PairParams(min_frag=0, max_frag=500, min_mate_score=80, rescue_capacity=max(n_pairs // 4, 1024))
            cap = 24 * 2 * n_pairs
            ws = {"paired": PairedWorkspace(fmi, genome, batches[0], params, pair, cap),
                  "paired_traceback": PairedWorkspace(fmi, genome, batches[0], params, pair, cap, traceback=True),
                  "paired_mapq": PairedWorkspace(fmi, genome, batches[0], params, pair, cap, mapq=mq),
                  "paired_traceback_mapq": PairedWorkspace(fmi, genome, batches[0], params, pair, cap, mapq=mq, traceback=True)}
            break
        except torch.cuda.OutOfMemoryError:
            ws = batches = None
            torch.cuda.empty_cache()
            if n_pairs <= 1024:
                raise
            note = "the workspaces did not fit beside the index at %d pairs" % n_pairs
            n_pairs //= 2
    flush = torch.empty(512 << 20, dtype=torch.uint8, device=device)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def call(name, i):
        if name.startswith("single"):
            L.nvb_debug_pipeline_path(C.c_int(1 if name == "single_per_hit" else 0))
            nb.seed_extend(fmi, genome, batches[i % 2], params, workspace=se_hit if name == "single_per_hit" else se, traceback=True)
            L.nvb_debug_pipeline_path(C.c_int(0))
        else:
            nb.seed_extend_paired(fmi, genome, batches[i % 2], params, pair, workspace=ws[name])

    def timed(name):
        for i in range(a.warmup):
            flush.zero_(); call(name, i)
        total = 0.0
        for i in range(a.steps):
            flush.zero_()
            ev0.record(); call(name, i); ev1.record()
            torch.cuda.synchronize()
            total += ev0.elapsed_time(ev1)
        call(name, 0)                                        # leave batch 0's results for the checks
        torch.cuda.synchronize()
        return total / a.steps

    def single_end():
        """the single-end workspaces, once the paired ones are gone"""
        for k in list(ws):
            ws[k] = None
        torch.cuda.empty_cache()
        se = SeedExtendWorkspace(fmi, genome, batches[0], params, cap, traceback=True)
        L.nvb_debug_pipeline_path(C.c_int(1))
        se_hit = SeedExtendWorkspace(fmi, genome, batches[0], params, cap, traceback=True)
        L.nvb_debug_pipeline_path(C.c_int(0))
        return se, se_hit

    paired_names = ("paired", "paired_traceback", "paired_mapq", "paired_traceback_mapq")
    single_names = ("single_per_read", "single_per_hit")
    se = se_hit = None
    if a.profile:
        from torch.profiler import profile, ProfilerActivity
        per = {}
        for names in (paired_names, single_names):
            if names is single_names:
                se, se_hit = single_end()
            for nm in names:
                call(nm, 0)
            torch.cuda.synchronize()
            for nm in names:
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    call(nm, 0); torch.cuda.synchronize()
                per[nm] = {e.key: round(e.device_time_total / 1e3, 4) for e in prof.key_averages() if e.device_time_total > 0}
        print(json.dumps({"profile": "device ms per kernel, one call each", "pairs": n_pairs, "card": torch.cuda.get_device_name(device),
                          "power_limit_w": power_limit_w(), "kernels": per}))
        return

    rounds = []
    for r in range(a.rounds):
        t = {nm: timed(nm) for nm in paired_names}
        for k in PAIR_OUTPUTS:
            assert torch.equal(getattr(ws["paired"], k), getattr(ws["paired_traceback"], k)), k
            assert torch.equal(getattr(ws["paired_mapq"], k), getattr(ws["paired_traceback_mapq"], k)), k
        for k in ("mate_ops", "mate_n_ops", "mate_begin"):
            assert torch.equal(getattr(ws["paired_traceback"], k), getattr(ws["paired_traceback_mapq"], k)), k
        rounds.append(dict(t, added_ms=t["paired_traceback"] - t["paired"], added_mapq_ms=t["paired_traceback_mapq"] - t["paired_mapq"]))
    flags = ws["paired_traceback"].pair_flags
    rescued = int(((flags == 2) | (flags == 4)).sum().item())
    temp = {k: w.temp_bytes for k, w in ws.items()}
    se, se_hit = single_end()
    single = []
    for r in range(a.rounds):
        t = {nm: timed(nm) for nm in single_names}
        for k in ("best_score", "best_pos", "best_ops", "best_n_ops", "best_begin", "best_strand"):
            assert torch.equal(getattr(se, k), getattr(se_hit, k)), k
        single.append(dict(t, per_hit_minus_per_read_ms=t["single_per_hit"] - t["single_per_read"]))
    added = sorted(x["added_ms"] for x in rounds)
    print(json.dumps({"workload": "seed_extend_paired vs seed_extend_paired_traceback", "pairs": n_pairs, "note": note, "read_len": R,
                      "genome_bp": n, "card": torch.cuda.get_device_name(device), "power_limit_w": power_limit_w(), "steps": a.steps,
                      "warmup": a.warmup, "rounds": rounds, "added_ms_median": added[len(added) // 2], "rescued_mates_traced": rescued,
                      "single_end_traceback_2n_mates": single,
                      "temp_bytes": dict(temp, single_per_read=se.temp_bytes, single_per_hit=se_hit.temp_bytes)}))


if __name__ == "__main__":
    main()
