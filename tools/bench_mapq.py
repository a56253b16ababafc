"""Cost of the second-best / MAPQ stage: nvb_seed_extend against nvb_seed_extend_mapq on bench.py's headline workload (1M x 150 bp
reads, 1.9 Gbp genome, full suffix array, 15-mer table with text context), alternated in one process over several rounds and timed with
device events.  Prints one JSON line: Mreads/s of both calls per round, the added milliseconds per step, the card and its power limit.
Asserts that both calls return the same best score and position for every read.

    python tools/bench_mapq.py [--rounds 3] [--steps 10] [--warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench  # noqa: E402


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reads", type=int, default=1_000_000)
    ap.add_argument("--genome-mbp", type=float, default=1900.0)
    a = ap.parse_args()
    import nvbio_b200 as nb
    from nvbio_b200 import aln
    from nvbio_b200.strings import PackedStringSet
    from nvbio_b200.pipeline import SeedExtendWorkspace, MapqParams

    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    nb.lib()
    # bench.py's index and reads: its defaults (full suffix array, 15-mer table with text context)
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
    ws_plain = SeedExtendWorkspace(fmi, genome, as_set(batches[0]), params, cap)
    ws_mapq = SeedExtendWorkspace(fmi, genome, as_set(batches[0]), params, cap, mapq=mq)
    flush = torch.empty(512 << 20, dtype=torch.uint8, device=device)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(ws):
        for i in range(a.warmup):
            flush.zero_(); nb.seed_extend(fmi, genome, as_set(batches[i % 2]), params, workspace=ws)
        total = 0.0
        for i in range(a.steps):
            flush.zero_()
            ev0.record(); nb.seed_extend(fmi, genome, as_set(batches[i % 2]), params, workspace=ws); ev1.record()
            torch.cuda.synchronize()
            total += ev0.elapsed_time(ev1)
        kept, found, jobs = [int(v) for v in ws.n_hits.cpu()]
        assert kept == found, "hit capacity exceeded"
        return total / a.steps, jobs

    rounds = []
    for r in range(a.rounds):
        ms_p, jobs = timed(ws_plain)
        ms_m, _ = timed(ws_mapq)
        # same last batch in both: the best alignment is unchanged by the extra stage
        assert torch.equal(ws_plain.best_score, ws_mapq.best_score) and torch.equal(ws_plain.best_pos, ws_mapq.best_pos)
        rounds.append({"seed_extend_ms": ms_p, "seed_extend_mapq_ms": ms_m, "added_ms": ms_m - ms_p,
                       "seed_extend_mreads_s": a.reads / (ms_p * 1e-3) / 1e6, "seed_extend_mapq_mreads_s": a.reads / (ms_m * 1e-3) / 1e6,
                       "jobs": jobs})
    has2 = float((ws_mapq.second_score != -2**31).float().mean())
    mapq_hist = torch.bincount(ws_mapq.mapq.long(), minlength=45).cpu().tolist()
    print(json.dumps({"workload": "seed_extend vs seed_extend_mapq", "reads": a.reads, "read_len": bench.READ_LEN, "genome_bp": n,
                      "card": torch.cuda.get_device_name(device), "power_limit_w": power_limit_w(), "steps": a.steps, "warmup": a.warmup,
                      "rounds": rounds, "added_ms_median": sorted(x["added_ms"] for x in rounds)[len(rounds) // 2],
                      "reads_with_second": has2, "mapq_histogram": mapq_hist}))


if __name__ == "__main__":
    main()
