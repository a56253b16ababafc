"""Cost of reporting up to k distinct alignments per read: nvb_seed_extend_mapq with the best-alignment traceback against
nvb_seed_extend_all at k = 1 and k = 8, alternated in one process over several rounds on bench.py's headline workload (1M x 150 bp reads,
1.9 Gbp genome, full suffix array, 15-mer table with text context) and timed with device events; then one run on a genome with a planted
16-copy repeat family, where reads average several alignments, and a torch.profiler run of each workload for the time of the selection
kernels (all_*, the segmented sort, the candidate scatter) and of the traceback kernels.  Prints one JSON line with per-step ms, stage
times, alignments per read, the card and its power limit.  Asserts that rank 0 equals the best-alignment call's alignment.

    python tools/bench_all.py [--rounds 3] [--steps 10] [--warmup 3] [--out DIR]
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

SELECT = ("all_select", "all_count", "all_emit", "all_begin", "pair_cand_scatter", "DeviceSegmentedSort", "DeviceScan", "SegmentedSort")
TRACE = ("traceback", "gotoh", "banded", "pair_")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reads", type=int, default=1_000_000)
    ap.add_argument("--genome-mbp", type=float, default=1900.0)
    ap.add_argument("--out", default=None, help="directory for the profiler's kernel table")
    a = ap.parse_args()
    import nvbio_b200 as nb
    from nvbio_b200 import aln
    from nvbio_b200.strings import PackedStringSet, pack_symbols
    from nvbio_b200.pipeline import SeedExtendWorkspace, MapqParams, AllAlignments

    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    nb.lib()
    params = nb.SeedExtendParams(seed_len=bench.SEED_LEN, seed_interval=bench.SEED_INTERVAL, band_len=bench.BAND, type=aln.LOCAL,
                                 both_strands=True, max_seed_hits=100, scheme=aln.SimpleGotohScheme(*bench.SCHEME))
    mq = MapqParams.local(bench.READ_LEN, device=device)
    flush = torch.empty(512 << 20, dtype=torch.uint8, device=device)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(step, sets):
        for i in range(a.warmup):
            flush.zero_(); step(sets[i % len(sets)])
        total = 0.0
        for i in range(a.steps):
            flush.zero_()
            ev0.record(); step(sets[i % len(sets)]); ev1.record()
            torch.cuda.synchronize()
            total += ev0.elapsed_time(ev1)
        return total / a.steps

    def profiled(step, s):
        from torch.profiler import profile, ProfilerActivity
        step(s); torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            step(s); torch.cuda.synchronize()
        sel = tb = 0.0
        for e in prof.key_averages():
            us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
            if any(k in e.key for k in SELECT):
                sel += us
            elif any(k in e.key for k in TRACE) and "score" not in e.key:
                tb += us
        if a.out:
            os.makedirs(a.out, exist_ok=True)
            with open(os.path.join(a.out, "bench_all_kernels.txt"), "a") as f:
                f.write(prof.key_averages().table(sort_by="cuda_time_total", row_limit=40) + "\n")
        return sel / 1e3, tb / 1e3

    def check_rank0(ws, al):
        torch.cuda.synchronize()
        first = al.first[:-1].long()
        has = al.first[1:] > al.first[:-1]
        rows = torch.nonzero(has).flatten()
        f0 = first[rows]
        for k_ws, k_al in (("best_score", "score"), ("best_pos", "pos"), ("best_strand", "strand"), ("best_n_ops", "n_ops"), ("best_begin", "begin")):
            assert torch.equal(getattr(ws, k_ws)[rows], getattr(al, k_al)[f0]), k_ws
        return float(al.count[1]) / al.n_reads, float(has.float().mean())

    def workload(name, fmi, genome, sets, n_reads, cap):
        ws = SeedExtendWorkspace(fmi, genome, sets[0], params, cap, traceback=True, mapq=mq)
        als = {k: AllAlignments(fmi, genome, sets[0], params, mq, k, k * n_reads, cap) for k in (1, 8)}
        base = lambda s: nb.seed_extend(fmi, genome, s, params, workspace=ws)            # noqa: E731
        runs = {k: (lambda s, al=al: al.run(fmi, genome, s, params)) for k, al in als.items()}
        rounds = []
        for r in range(a.rounds):
            row = {"mapq_traceback_ms": timed(base, sets)}
            for k, f in runs.items():
                row["all_k%d_ms" % k] = timed(f, sets)
            rounds.append(row)
        out = {"workload": name, "reads": n_reads, "rounds": rounds}
        for k in runs:
            out["all_k%d_over_mapq_traceback_median" % k] = sorted(x["all_k%d_ms" % k] / x["mapq_traceback_ms"] for x in rounds)[len(rounds) // 2]
        base(sets[0])
        for k, al in als.items():
            al.run(fmi, genome, sets[0], params)
            per_read, aligned = check_rank0(ws, al)
            assert int(al.count[0]) == int(al.count[1]), "alignment capacity exceeded"
            assert int(al.n_hits[0]) == int(al.n_hits[1]), "hit capacity exceeded"
            out["k%d_alignments_per_read" % k] = per_read
            out["k%d_reads_with_alignment" % k] = aligned
        out["profile_ms"] = {"mapq_traceback": dict(zip(("selection", "traceback"), profiled(base, sets[0])))}
        for k, f in runs.items():
            out["profile_ms"]["all_k%d" % k] = dict(zip(("selection", "traceback"), profiled(f, sets[0])))
        return out

    # bench.py's headline workload
    idx_args = argparse.Namespace(genome_mbp=a.genome_mbp, sa_interval=1, ktab_k=15, ktab_located=2, impl="ours")
    n, genome, fmi, _, _ = bench.build_index(idx_args, 0, 1, device)
    batches = [bench.make_reads(genome, n, a.reads, b, device) for b in range(2)]
    wpr = batches[0].shape[1]
    sets = [PackedStringSet.fixed(w.reshape(-1), a.reads, bench.READ_LEN, stride=wpr * 16) for w in batches]
    results = [workload("headline", fmi, genome, sets, a.reads, 24 * a.reads)]
    del fmi, genome, batches, sets
    torch.cuda.empty_cache()

    # planted repeats: a 32 Mbp random genome with one 2 kbp segment copied 16 times (4 of them reverse-complemented, 3 with 1-3
    # substitutions per 100 bp); half of the reads come from the family
    rng = np.random.default_rng(1)
    G = 32_000_000
    g = rng.integers(0, 4, G).astype(np.uint8)
    seg = g[1_000_000:1_002_000].copy()
    for c in range(1, 16):
        s = seg.copy()
        if c % 4 == 0:
            s = np.where(s < 4, 3 - s, s)[::-1].astype(np.uint8)
        if c % 5 == 1:
            s[50::100 // (c % 3 + 1)] = (s[50::100 // (c % 3 + 1)] + 1) % 4
        g[1_000_000 + c * 1_900_000: 1_000_000 + c * 1_900_000 + 2000] = s
    gw = torch.from_numpy(np.concatenate([pack_symbols(g, 2, True).view(np.int32), np.zeros(4, np.int32)])).to(device)   # readable past the end
    rfmi = nb.FMIndexDevice.from_text(gw, G, sa_interval=1)[0]
    rfmi.build_ktab(15, located=True, text=gw)
    nr = a.reads // 4
    L = bench.READ_LEN
    starts = np.where(np.arange(nr) % 2 == 0, 1_000_000 + rng.integers(0, 2000 - L, nr), rng.integers(0, G - L, nr))
    reads = np.stack([g[p:p + L] for p in starts])
    rcm = rng.random(nr) < 0.5
    reads[rcm] = np.where(reads[rcm] < 4, 3 - reads[rcm], reads[rcm])[:, ::-1]
    offs = (np.arange(nr) * L).astype(np.uint32)
    rs = PackedStringSet.from_symbols(reads.reshape(-1), offs, np.full(nr, L, np.uint32), bits=2, big_endian=True, device=device)
    results.append(workload("planted_repeats_16_copies", rfmi, gw, [rs], nr, 400 * nr))
    print(json.dumps({"card": torch.cuda.get_device_name(device), "power_limit_w": power_limit_w(), "steps": a.steps, "warmup": a.warmup,
                      "results": results}))


if __name__ == "__main__":
    main()
