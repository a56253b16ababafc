"""Per-step time of nvb_seed_extend_paired_mapq under each pairing policy (FR, RF, FF, RR) on bench.py's paired workload generated in
that orientation (500 k pairs of 2 x 150 bp from synth.sample_pairs as paired_end_config draws them, 5 % of second mates heavily
mutated, 1.9 Gbp genome, full suffix array, 15-mer table with text context, LOCAL, PairParams(0, 500, 80, n / 4, policy)), alternated
over several rounds and timed with device events.  The policy only changes the per-pair kernels after the extension, so every policy is
expected near FR's time.  Prints one JSON line: the card and its power limit, ms per step of each policy per round, and each policy's
concordant and rescued fractions.

    python tools/bench_pair_policy.py [--rounds 3] [--steps 10] [--warmup 3]
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

POLICIES = ("fr", "rf", "ff", "rr")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--pairs", type=int, default=500_000)
    ap.add_argument("--genome-mbp", type=float, default=1900.0)
    a = ap.parse_args()
    import nvbio_b200 as nb
    from nvbio_b200 import aln, synth
    from nvbio_b200.strings import PackedStringSet
    from nvbio_b200.pipeline import MapqParams, PairedWorkspace

    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    nb.lib()
    idx_args = argparse.Namespace(genome_mbp=a.genome_mbp, sa_interval=1, ktab_k=15, ktab_located=2, impl="ours")
    n, genome, fmi, _, _ = bench.build_index(idx_args, 0, 1, device)
    params = nb.SeedExtendParams(seed_len=bench.SEED_LEN, seed_interval=bench.SEED_INTERVAL, band_len=bench.BAND, type=aln.LOCAL,
                                 both_strands=True, max_seed_hits=100, scheme=aln.SimpleGotohScheme(*bench.SCHEME))
    n_pairs, RL = a.pairs, bench.READ_LEN
    mq = MapqParams.local(RL, device=device)
    cap = 24 * 2 * n_pairs
    batches, pairs, ws = {}, {}, {}
    for pol in POLICIES:
        batches[pol] = []
        for seed, mut in ((0x51ED, 0xC0FFEE), (0x61ED, 0xD0FFEE)):      # paired_end_config's two batches (rank 0), in this orientation
            words, _, _ = synth.sample_pairs(genome, n, n_pairs, RL, frag_mean=350.0, frag_sd=30.0, sub_rate=0.01, hard_frac=0.05,
                                             hard_sub_rate=0.2, device=device, seed=seed, mut_seed=mut, orientation=pol)
            batches[pol].append(PackedStringSet.fixed(words.reshape(-1), 2 * n_pairs, RL, stride=words.shape[1] * 16))
        pairs[pol] = nb.PairParams(min_frag=0, max_frag=500, min_mate_score=80, rescue_capacity=max(n_pairs // 4, 1024), policy=pol)
        ws[pol] = PairedWorkspace(fmi, genome, batches[pol][0], params, pairs[pol], cap, mapq=mq)

    flush = torch.empty(512 << 20, dtype=torch.uint8, device=device)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def step(pol, i):
        nb.seed_extend_paired(fmi, genome, batches[pol][i % 2], params, pairs[pol], workspace=ws[pol], mapq=mq)

    def timed(pol):
        for i in range(a.warmup):
            flush.zero_(); step(pol, i)
        total = 0.0
        for i in range(a.steps):
            flush.zero_()
            ev0.record(); step(pol, i); ev1.record()
            torch.cuda.synchronize()
            total += ev0.elapsed_time(ev1)
        return total / a.steps

    rounds = [{pol: timed(pol) for pol in POLICIES} for _ in range(a.rounds)]
    frac = {}
    for pol in POLICIES:                                                 # the last timed batch of each policy
        f = ws[pol].pair_flags
        frac[pol] = {"concordant": float((f == nb.PAIR_CONCORDANT).double().mean()),
                     "rescued": float(((f == nb.PAIR_RESCUED_MATE1) | (f == nb.PAIR_RESCUED_MATE2)).double().mean()),
                     "rescue_jobs": ws[pol].n_rescue.cpu().tolist()}
    print(json.dumps({"workload": "seed_extend_paired_mapq per policy, pairs generated in that orientation", "pairs": n_pairs,
                      "read_len": RL, "genome_bp": n, "card": torch.cuda.get_device_name(device), "power_limit_w": power_limit_w(),
                      "steps": a.steps, "warmup": a.warmup, "ms_per_step": rounds, "fractions": frac}))


if __name__ == "__main__":
    main()
