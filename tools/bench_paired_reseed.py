"""Cost and effect of the paired reseeding rounds: nvb_seed_extend_paired_mapq against nvb_seed_extend_paired_reseed (with MAPQ) at
max_reseed 0 and 2 on bench.py's paired workload (500 k pairs of 2 x 150 bp from synth.sample_pairs as paired_end_config draws them,
5 % of second mates heavily mutated, 1.9 Gbp genome, full suffix array, 15-mer table with text context, LOCAL,
PairParams(0, 500, 80, n / 4), ReseedParams.local(150)), alternated in one process over several rounds and timed with device events.
Asserts that max_reseed = 0 gives nvb_seed_extend_paired_mapq's outputs.  Prints one JSON line: the card and its power limit, ms per
step of each call, the mates seeded in each round, the pairs whose flags changed, and the fraction of pairs with both mates at the
generator's locus (alignment end within --tolerance bp of the mate's true end) with and without reseeding.  --profile DIR: instead,
one max_reseed = 2 step under torch.profiler, its CUDA kernels' total times as JSON (a separate run: tracing slows the host).

    python tools/bench_paired_reseed.py [--rounds 3] [--steps 10] [--warmup 3] [--profile DIR]
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
    ap.add_argument("--pairs", type=int, default=500_000)
    ap.add_argument("--genome-mbp", type=float, default=1900.0)
    ap.add_argument("--tolerance", type=int, default=20)
    ap.add_argument("--profile", default=None)
    a = ap.parse_args()
    import nvbio_b200 as nb
    from nvbio_b200 import aln, synth
    from nvbio_b200.strings import PackedStringSet
    from nvbio_b200.pipeline import MapqParams, ReseedParams, PairedWorkspace, PairedReseedWorkspace

    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    nb.lib()
    idx_args = argparse.Namespace(genome_mbp=a.genome_mbp, sa_interval=1, ktab_k=15, ktab_located=2, impl="ours")
    n, genome, fmi, _, _ = bench.build_index(idx_args, 0, 1, device)
    params = nb.SeedExtendParams(seed_len=bench.SEED_LEN, seed_interval=bench.SEED_INTERVAL, band_len=bench.BAND, type=aln.LOCAL,
                                 both_strands=True, max_seed_hits=100, scheme=aln.SimpleGotohScheme(*bench.SCHEME))
    n_pairs, RL = a.pairs, bench.READ_LEN
    batches = []
    for seed, mut in ((0x51ED, 0xC0FFEE), (0x61ED, 0xD0FFEE)):          # paired_end_config's two batches (rank 0)
        words, left, frag = synth.sample_pairs(genome, n, n_pairs, RL, frag_mean=350.0, frag_sd=30.0, sub_rate=0.01, hard_frac=0.05,
                                               hard_sub_rate=0.2, device=device, seed=seed, mut_seed=mut)
        rs = PackedStringSet.fixed(words.reshape(-1), 2 * n_pairs, RL, stride=words.shape[1] * 16)
        batches.append((rs, left, frag))
    pair = nb.PairParams(min_frag=0, max_frag=500, min_mate_score=80, rescue_capacity=max(n_pairs // 4, 1024))
    cap = 24 * 2 * n_pairs
    mq = MapqParams.local(RL, device=device)
    rp = {k: ReseedParams.local(RL, max_reseed=k, device=device) for k in (0, 2)}
    rs0 = batches[0][0]
    ws = {"mapq": PairedWorkspace(fmi, genome, rs0, params, pair, cap, mapq=mq)}
    for k in (0, 2):
        ws[k] = PairedReseedWorkspace(fmi, genome, rs0, params, pair, cap, rp[k], mapq=mq)

    def step(which, i):
        rs = batches[i % 2][0]
        if which == "mapq":
            nb.seed_extend_paired(fmi, genome, rs, params, pair, workspace=ws["mapq"], mapq=mq)
        else:
            nb.seed_extend_paired_reseed(fmi, genome, rs, params, pair, rp[which], mapq=mq, workspace=ws[which])

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
        out = {"workload": "seed_extend_paired_reseed max_reseed=2 with MAPQ, one step", "card": torch.cuda.get_device_name(device),
               "power_limit_w": power_limit_w(), "active_per_round": ws[2].active.cpu().tolist(),
               "kernels": dict(sorted(kern.items(), key=lambda kv: -kv[1]["ms"]))}
        with open(os.path.join(a.profile, "paired_reseed_kernels.json"), "w") as f:
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

    keys = ("pair_score", "pair_flags", "mate_score", "mate_pos", "mate_strand", "n_rescue", "n_hits", "second_pair_score",
            "second_mate_pos", "second_mate_strand", "mate_second_score", "mate_mapq")
    rounds = []
    for r in range(a.rounds):
        ms = {w: timed(w) for w in ("mapq", 0, 2)}
        # the same last batch in all three: max_reseed = 0 is seed_extend_paired_mapq
        for k in keys:
            assert torch.equal(getattr(ws["mapq"], k), getattr(ws[0], k)), k
        rounds.append({"paired_mapq_ms": ms["mapq"], "reseed0_ms": ms[0], "reseed2_ms": ms[2], "added_ms": ms[2] - ms["mapq"]})

    # the effect on the last timed batch
    last = batches[(a.steps - 1) % 2]
    left, frag = last[1], last[2]
    odd = (torch.arange(n_pairs, device=device) & 1).bool()
    fw_end, rv_end = left + RL, left + frag
    true_end = torch.stack([torch.where(odd, rv_end, fw_end), torch.where(odd, fw_end, rv_end)])      # [2, n]: mate 1, mate 2

    def at_locus(w):
        pos = w.mate_pos.to(torch.int64) & 0xFFFFFFFF
        return ((pos - true_end).abs() <= a.tolerance).all(dim=0)

    f0, f2 = ws[0].pair_flags, ws[2].pair_flags
    resc = lambda f: (f == nb.pipeline.PAIR_RESCUED_MATE1) | (f == nb.pipeline.PAIR_RESCUED_MATE2)     # noqa: E731
    conc2 = f2 == nb.pipeline.PAIR_CONCORDANT
    print(json.dumps({"workload": "seed_extend_paired_mapq vs seed_extend_paired_reseed with MAPQ (max_reseed 0, 2)", "pairs": n_pairs,
                      "read_len": RL, "genome_bp": n, "card": torch.cuda.get_device_name(device), "power_limit_w": power_limit_w(),
                      "steps": a.steps, "warmup": a.warmup, "rounds": rounds,
                      "added_ms_median": sorted(x["added_ms"] for x in rounds)[len(rounds) // 2],
                      "active_per_round": ws[2].active.cpu().tolist(), "pairs_flags_changed": int((f0 != f2).sum()),
                      "unpaired_to_concordant": int(((f0 == nb.pipeline.PAIR_UNPAIRED) & conc2).sum()),
                      "rescued_to_concordant": int((resc(f0) & conc2).sum()), "tolerance_bp": a.tolerance,
                      "both_at_locus_0": float(at_locus(ws[0]).double().mean()), "both_at_locus_2": float(at_locus(ws[2]).double().mean())}))


if __name__ == "__main__":
    main()
