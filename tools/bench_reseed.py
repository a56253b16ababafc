"""Cost of the reseeding rounds: nvb_seed_extend_mapq against nvb_seed_extend_reseed at max_reseed 0 and 2 on bench.py's headline
workload (1M x 150 bp reads, 1.9 Gbp genome, full suffix array, 15-mer table with text context, LOCAL, ReseedParams.local), alternated
in one process over several rounds and timed with device events.  Asserts that max_reseed = 0 gives nvb_seed_extend_mapq's outputs.
Prints one JSON line: the card and its power limit, ms per step of each call, the added ms, the reads seeded in each round and how many
reads changed their best alignment or became aligned.  --profile DIR: instead, one max_reseed = 2 step under torch.profiler, its CUDA
kernels' total times as JSON (a separate run: tracing slows the host).

    python tools/bench_reseed.py [--rounds 3] [--steps 10] [--warmup 3] [--profile DIR]
"""
import argparse
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
    ap.add_argument("--profile", default=None)
    a = ap.parse_args()
    import nvbio_b200 as nb
    from nvbio_b200 import aln
    from nvbio_b200.strings import PackedStringSet
    from nvbio_b200.pipeline import SeedExtendWorkspace, MapqParams, ReseedParams, ReseedWorkspace

    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    nb.lib()
    idx_args = argparse.Namespace(genome_mbp=a.genome_mbp, sa_interval=1, ktab_k=15, ktab_located=2, impl="ours")
    n, genome, fmi, _, _ = bench.build_index(idx_args, 0, 1, device)
    params = nb.SeedExtendParams(seed_len=bench.SEED_LEN, seed_interval=bench.SEED_INTERVAL, band_len=bench.BAND, type=aln.LOCAL,
                                 both_strands=True, max_seed_hits=100, scheme=aln.SimpleGotohScheme(*bench.SCHEME))
    batches = [bench.make_reads(genome, n, a.reads, b, device) for b in range(2)]
    wpr = batches[0].shape[1]

    def as_set(words):
        return PackedStringSet.fixed(words.reshape(-1), a.reads, bench.READ_LEN, stride=wpr * 16)
    cap = 24 * a.reads
    mq = MapqParams.local(bench.READ_LEN, device=device)
    rp = {k: ReseedParams.local(bench.READ_LEN, max_reseed=k, device=device) for k in (0, 2)}
    ws = {"mapq": SeedExtendWorkspace(fmi, genome, as_set(batches[0]), params, cap, mapq=mq)}
    for k in (0, 2):
        ws[k] = ReseedWorkspace(fmi, genome, as_set(batches[0]), params, cap, rp[k], mapq=mq)

    def step(which, i):
        if which == "mapq":
            nb.seed_extend(fmi, genome, as_set(batches[i % 2]), params, workspace=ws["mapq"])
        else:
            nb.seed_extend_reseed(fmi, genome, as_set(batches[i % 2]), params, rp[which], workspace=ws[which])

    if a.profile:
        from torch.profiler import profile, ProfilerActivity
        for i in range(a.warmup):
            step(2, i)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            step(2, 0)
            torch.cuda.synchronize()
        kern = {}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
            if t:
                kern[e.key[:90]] = {"ms": t / 1e3, "calls": e.count}
        os.makedirs(a.profile, exist_ok=True)
        out = {"workload": "seed_extend_reseed max_reseed=2, one step", "card": torch.cuda.get_device_name(device), "power_limit_w": power_limit_w(),
               "kernels": dict(sorted(kern.items(), key=lambda kv: -kv[1]["ms"]))}
        with open(os.path.join(a.profile, "reseed_kernels.json"), "w") as f:
            json.dump(out, f, indent=1)
        print(json.dumps(out))
        return

    flush = torch.empty(512 << 20, dtype=torch.uint8, device=device)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(which):
        for i in range(a.warmup):
            flush.zero_(); step(which, i)
        total = 0.0
        for i in range(a.steps):
            flush.zero_()
            ev0.record(); step(which, i); ev1.record()
            torch.cuda.synchronize()
            total += ev0.elapsed_time(ev1)
        return total / a.steps

    rounds = []
    for r in range(a.rounds):
        ms = {w: timed(w) for w in ("mapq", 0, 2)}
        # the same last batch in all three: max_reseed = 0 is seed_extend_mapq
        for k in ("best_score", "best_pos", "second_score", "second_pos", "second_strand", "mapq", "n_hits"):
            assert torch.equal(getattr(ws["mapq"], k), getattr(ws[0], k)), k
        rounds.append({"seed_extend_mapq_ms": ms["mapq"], "reseed0_ms": ms[0], "reseed2_ms": ms[2], "added_ms": ms[2] - ms["mapq"]})
    b0, b2 = ws[0], ws[2]
    aligned0 = b0.best_score >= mq.min_score[bench.READ_LEN]
    aligned2 = b2.best_score >= mq.min_score[bench.READ_LEN]
    changed = (b0.best_score != b2.best_score) | (b0.best_pos != b2.best_pos)
    print(json.dumps({"workload": "seed_extend_mapq vs seed_extend_reseed (max_reseed 0, 2)", "reads": a.reads, "read_len": bench.READ_LEN,
                      "genome_bp": n, "card": torch.cuda.get_device_name(device), "power_limit_w": power_limit_w(), "steps": a.steps,
                      "warmup": a.warmup, "rounds": rounds, "added_ms_median": sorted(x["added_ms"] for x in rounds)[len(rounds) // 2],
                      "active_per_round": b2.active.cpu().tolist(), "reads_best_changed": int(changed.sum()),
                      "reads_newly_aligned": int((aligned2 & ~aligned0).sum()), "reads_aligned_0": int(aligned0.sum()),
                      "reads_aligned_2": int(aligned2.sum())}))


if __name__ == "__main__":
    main()
