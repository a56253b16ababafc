"""Cost of the second-best pair / paired MAPQ stage: nvb_seed_extend_paired against nvb_seed_extend_paired_mapq on bench.py's paired-end
workload (500k FR pairs of 2 x 150 bp from synth.sample_pairs, 1.9 Gbp genome, full suffix array, 15-mer table with text context,
PairParams(0, 500, 80, n/4)), alternated in one process over several rounds and timed with device events.  Asserts that both calls return
the same pair outputs.  Prints one JSON line: the card and its power limit, ms per step of both calls per round and the added
milliseconds, the share of pairs with a second pair, how many second pairs score above the reported pair, and the MAPQ histogram of the
mates split by whether their pair was placed at the generator's truth.

    python tools/bench_pair_mapq.py [--rounds 3] [--steps 10] [--warmup 3]
"""
import argparse
import json
import os
import sys

import numpy as np
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
    a = ap.parse_args()
    import nvbio_b200 as nb
    from nvbio_b200 import aln, synth
    from nvbio_b200.strings import PackedStringSet
    from nvbio_b200.pipeline import PairedWorkspace, MapqParams

    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    nb.lib()
    idx_args = argparse.Namespace(genome_mbp=a.genome_mbp, sa_interval=1, ktab_k=15, ktab_located=2, impl="ours")
    n, genome, fmi, _, _ = bench.build_index(idx_args, 0, 1, device)
    params = nb.SeedExtendParams(seed_len=bench.SEED_LEN, seed_interval=bench.SEED_INTERVAL, band_len=bench.BAND, type=aln.LOCAL,
                                 both_strands=True, max_seed_hits=100, scheme=aln.SimpleGotohScheme(*bench.SCHEME))
    n_pairs, R = a.pairs, bench.READ_LEN
    batches = []
    for seed, mut in ((0x51ED, 0xC0FFEE), (0x61ED, 0xD0FFEE)):          # bench.py's two batches (rank 0)
        words, left, frag = synth.sample_pairs(genome, n, n_pairs, R, frag_mean=350.0, frag_sd=30.0, sub_rate=0.01, hard_frac=0.05,
                                               hard_sub_rate=0.2, device=device, seed=seed, mut_seed=mut)
        batches.append((PackedStringSet.fixed(words.reshape(-1), 2 * n_pairs, R, stride=words.shape[1] * 16), left, frag))
    pair = nb.PairParams(min_frag=0, max_frag=500, min_mate_score=80, rescue_capacity=max(n_pairs // 4, 1024))
    cap = 24 * 2 * n_pairs
    mq = MapqParams.local(R, device=device)
    ws_plain = PairedWorkspace(fmi, genome, batches[0][0], params, pair, cap)
    ws_mapq = PairedWorkspace(fmi, genome, batches[0][0], params, pair, cap, mapq=mq)
    flush = torch.empty(512 << 20, dtype=torch.uint8, device=device)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(ws):
        for i in range(a.warmup):
            flush.zero_(); nb.seed_extend_paired(fmi, genome, batches[i % 2][0], params, pair, workspace=ws)
        total = 0.0
        for i in range(a.steps):
            flush.zero_()
            ev0.record(); nb.seed_extend_paired(fmi, genome, batches[i % 2][0], params, pair, workspace=ws); ev1.record()
            torch.cuda.synchronize()
            total += ev0.elapsed_time(ev1)
        nb.seed_extend_paired(fmi, genome, batches[0][0], params, pair, workspace=ws)     # leave batch 0's results for the checks
        torch.cuda.synchronize()
        kept, found, _ = [int(v) for v in ws.n_hits.cpu()]
        assert kept == found, "hit capacity exceeded"
        return total / a.steps

    rounds = []
    for r in range(a.rounds):
        ms_p = timed(ws_plain)
        ms_m = timed(ws_mapq)
        for k in PAIR_OUTPUTS:
            assert torch.equal(getattr(ws_plain, k), getattr(ws_mapq, k)), k
        rounds.append({"paired_ms": ms_p, "paired_mapq_ms": ms_m, "added_ms": ms_m - ms_p,
                       "paired_mreads_s": 2 * n_pairs / (ms_p * 1e-3) / 1e6, "paired_mapq_mreads_s": 2 * n_pairs / (ms_m * 1e-3) / 1e6})
    # placement against the generator's truth, as bench.py checks it: the forward mate ends at left + R, the reverse one at left + frag
    flags = ws_mapq.pair_flags.cpu().numpy()
    pos = ws_mapq.mate_pos.cpu().numpy().view(np.uint32).astype(np.int64)
    strand = ws_mapq.mate_strand.cpu().numpy()
    left, frag = batches[0][1].cpu().numpy(), batches[0][2].cpu().numpy()
    truth = np.where(strand == 0, left[None, :] + R, (left + frag)[None, :])
    at_truth = (np.abs(pos - truth) <= 8).all(axis=0)
    mapq = ws_mapq.mate_mapq.cpu().numpy()
    s2 = ws_mapq.second_pair_score.cpu().numpy()
    ps = ws_mapq.pair_score.cpu().numpy()
    paired = flags != 0
    has2 = s2 != -2**31
    hist = lambda m: np.bincount(m.reshape(-1), minlength=45).tolist()      # noqa: E731
    added = sorted(x["added_ms"] for x in rounds)
    print(json.dumps({"workload": "seed_extend_paired vs seed_extend_paired_mapq", "pairs": n_pairs, "read_len": R, "genome_bp": n,
                      "card": torch.cuda.get_device_name(device), "power_limit_w": power_limit_w(), "steps": a.steps, "warmup": a.warmup,
                      "rounds": rounds, "added_ms_median": added[len(added) // 2], "added_ms_min": added[0], "added_ms_max": added[-1],
                      "pairs_paired_frac": float(paired.mean()), "pairs_with_second_frac": float(has2.mean()),
                      "paired_pairs_with_second_frac": float(has2[paired].mean()) if paired.any() else None,
                      "second_above_reported": int((has2 & paired & (s2 > ps)).sum()),
                      "pairs_at_truth_frac": float(at_truth.mean()),
                      "mapq_histogram_at_truth": hist(mapq[:, at_truth]), "mapq_histogram_not_at_truth": hist(mapq[:, ~at_truth])}))


if __name__ == "__main__":
    main()
