"""Cost of finishing traced alignments on the device (nvb_finish_alignments: CIGAR, MD, NM / XM / XO / XG) on bench.py's paired-end workload
(500k FR pairs of 2 x 150 bp from synth.sample_pairs, 1.9 Gbp genome, full suffix array, 15-mer table with text context, PairParams(0, 500,
80, n/4)): nvb_seed_extend_paired_traceback with and without nvb_finish_alignments over the 2n mates after it, alternated in one process
over several rounds and timed with device events; then the same single end (nvb_seed_extend_traceback over the 2n mates).  Also reports
the bytes the finishing kernel moves (ops, op counts, begins, strands, the reads' words, the genome words under every span, and the
outputs it writes) so that they can be set against the kernel time and the H100's 3.35 TB/s.  Prints one JSON line with the card and its
power limit.
--profile: instead, one torch.profiler run of each (CUDA activities): the finishing kernel's device time and its achieved bandwidth.

    python tools/bench_finish.py [--rounds 3] [--steps 10] [--warmup 3] [--profile]
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

HBM_TBPS = 3.35


def bytes_moved(f, ops, n_ops, reads):
    """bytes the finishing kernel reads and writes for these alignments (from the shapes and the counts it produced)"""
    max_ops = ops.shape[-1]
    n = ops.numel() // max_ops
    k = n_ops.reshape(-1).to(torch.int64)
    words_per_read = reads.words.numel() // max(reads.count, 1)
    rd = int(k.clamp(max=max_ops).sum()) + 4 * n + 8 * n + n               # ops actually read (bounded by n_ops), n_ops, begin, strand
    rd += 4 * words_per_read * n                                           # the reads' words
    rd += int((4 * (k // 16 + 2) * (k > 0)).sum())                        # genome words under every span (M + D <= n_ops)
    wr = 4 * int(f.n_cigar.to(torch.int64).clamp(max=f.cigar.shape[1]).sum()) + int(f.md_len.to(torch.int64).clamp(max=f.md.shape[1]).sum())
    wr += 4 * n * 2 + 16 * n                                               # n_cigar, md_len, edits
    return rd, wr


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
    from nvbio_b200.pipeline import PairedWorkspace, SeedExtendWorkspace

    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    idx_args = argparse.Namespace(genome_mbp=a.genome_mbp, sa_interval=1, ktab_k=15, ktab_located=2, impl="ours")
    n, genome, fmi, _, _ = bench.build_index(idx_args, 0, 1, device)
    params = nb.SeedExtendParams(seed_len=bench.SEED_LEN, seed_interval=bench.SEED_INTERVAL, band_len=bench.BAND, type=aln.LOCAL,
                                 both_strands=True, max_seed_hits=100, scheme=aln.SimpleGotohScheme(*bench.SCHEME))
    R = bench.READ_LEN
    n_pairs = a.pairs
    batches = []
    for seed, mut in ((0x51ED, 0xC0FFEE), (0x61ED, 0xD0FFEE)):          # bench.py's two batches (rank 0)
        words, _, _ = synth.sample_pairs(genome, n, n_pairs, R, frag_mean=350.0, frag_sd=30.0, sub_rate=0.01, hard_frac=0.05,
                                         hard_sub_rate=0.2, device=device, seed=seed, mut_seed=mut)
        batches.append(PackedStringSet.fixed(words.reshape(-1), 2 * n_pairs, R, stride=words.shape[1] * 16))
    pair = nb.PairParams(min_frag=0, max_frag=500, min_mate_score=80, rescue_capacity=max(n_pairs // 4, 1024))
    cap = 24 * 2 * n_pairs
    flush = torch.empty(512 << 20, dtype=torch.uint8, device=device)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    state = {}

    def traced(mode, i):
        if mode == "paired":
            ws = nb.seed_extend_paired(fmi, genome, batches[i % 2], params, pair, workspace=state["pw"])
            return ws, (ws.mate_ops, ws.mate_n_ops, ws.mate_begin, ws.mate_strand)
        ws = nb.seed_extend(fmi, genome, batches[i % 2], params, workspace=state["sw"], traceback=True)
        return ws, (ws.best_ops, ws.best_n_ops, ws.best_begin, ws.best_strand)

    def call(mode, finish, i):
        ws, t = traced(mode, i)
        f = nb.finish_alignments(genome, batches[i % 2], *t, genome_len=n) if finish else None
        return t, f

    def timed(mode, finish):
        for i in range(a.warmup):
            flush.zero_(); call(mode, finish, i)
        total = 0.0
        for i in range(a.steps):
            flush.zero_()
            ev0.record(); call(mode, finish, i); ev1.record()
            torch.cuda.synchronize()
            total += ev0.elapsed_time(ev1)
        return total / a.steps

    result = {"workload": "seed_extend[_paired]_traceback with and without finish_alignments", "pairs": n_pairs, "read_len": R, "genome_bp": n,
              "card": torch.cuda.get_device_name(device), "power_limit_w": power_limit_w()}
    for mode in ("paired", "single"):
        if mode == "paired":
            state["pw"] = PairedWorkspace(fmi, genome, batches[0], params, pair, cap, traceback=True)
        else:
            state["pw"] = None
            torch.cuda.empty_cache()
            state["sw"] = SeedExtendWorkspace(fmi, genome, batches[0], params, cap, traceback=True)
        t, f = call(mode, True, 0)
        torch.cuda.synchronize()
        rd, wr = bytes_moved(f, t[0], t[1], batches[0])
        if a.profile:
            from torch.profiler import profile, ProfilerActivity
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                call(mode, True, 0); torch.cuda.synchronize()
            k = [e for e in prof.key_averages() if "finish_alignments_kernel" in e.key]
            ms = sum(e.device_time_total for e in k) / 1e3
            result[mode] = {"finish_kernel_ms": round(ms, 4), "bytes_read": rd, "bytes_written": wr,
                            "achieved_tbps": round((rd + wr) / (ms * 1e-3) / 1e12, 3) if ms else None, "of_hbm_peak": HBM_TBPS,
                            "alignments": int(t[1].numel())}
            continue
        rounds = []
        for r in range(a.rounds):
            base, fin = timed(mode, False), timed(mode, True)
            rounds.append({"traceback_ms": round(base, 4), "traceback_finish_ms": round(fin, 4), "added_ms": round(fin - base, 4)})
        added = sorted(x["added_ms"] for x in rounds)
        result[mode] = {"rounds": rounds, "added_ms_median": added[len(added) // 2], "bytes_read": rd, "bytes_written": wr,
                        "alignments": int(t[1].numel())}
    result.update(steps=a.steps, warmup=a.warmup, profile=a.profile)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
