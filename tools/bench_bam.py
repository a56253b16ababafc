"""Cost of building BAM records on the device (nvb_bam_records) on bench.py's paired-end workload (500k FR pairs of 2 x 150 bp from
synth.sample_pairs, 1.9 Gbp genome, full suffix array, 15-mer table with text context, PairParams(0, 500, 80, n/4)).  The paired
traceback and finish_alignments run once; then nvb_bam_records alone is timed with device events over repeated calls, with the genome
cut into a 25-contig and into a 3,000-contig table, paired (records of both mates) and single end (the 2n mates traced single end).
Reports ms per call, the bytes the three steps read and write (computed from the shapes and the sizes the call produced, not measured),
and their share of the H100's 3.35 TB/s data-sheet bandwidth, with the card and its power limit.  Prints one JSON line.
--profile: instead, one torch.profiler run per case: the device time of the plan kernel, the scan and the write kernel.

    python tools/bench_bam.py [--steps 20] [--warmup 3] [--profile]
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

HBM_TBPS = 3.35


def contig_table(nb, n, k, seed):
    """k contigs of random lengths tiling the n-symbol genome"""
    rng = np.random.default_rng(seed)
    cuts = np.unique(rng.integers(1, n, k - 1))
    lens = np.diff(np.concatenate([[0], cuts, [n]]))
    return nb.ContigTable(["chr%d" % i for i in range(len(lens))], lens)


def bytes_moved(call, f, reads, n_contigs):
    """bytes the plan kernel, the scan and the write kernel read and write (from shapes and the record sizes)"""
    n = call.n
    total = int(call.offsets[-1])
    n_cigar = f.n_cigar.to(torch.int64).clamp(max=f.cigar.shape[1])
    md = f.md_len.to(torch.int64).clamp(max=f.md.shape[1])
    words_per_read = reads.words.numel() // max(reads.count, 1)
    # plan: n_ops, begin, strand, n_cigar, md_len, edits, score, mapq, second, the CIGAR rows, names' offsets, ~log2(contigs) probes
    plan_rd = n * (4 + 8 + 1 + 4 + 4 + 16 + 4 + 1 + 4 + 4) + 4 * int(n_cigar.sum()) + 4 * n * int(np.ceil(np.log2(max(n_contigs, 2))))
    plan_wr = 32 * n + 8 * n
    scan = 2 * 8 * (n + 1)
    # write: cores, offsets, the reads' words, quals (none here), names, CIGAR rows, MD rows, edits; the records
    write_rd = 32 * n + 8 * (n + 1) + 4 * words_per_read * n + 4 * int(n_cigar.sum()) + int(md.sum()) + 16 * n
    write_rd += int(call.name_bytes)
    return plan_rd + scan + write_rd, plan_wr + scan + total, total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--pairs", type=int, default=500_000)
    ap.add_argument("--genome-mbp", type=float, default=1900.0)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    import nvbio_b200 as nb
    from nvbio_b200 import aln, synth
    from nvbio_b200.bam import BamCall
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
    words, _, _ = synth.sample_pairs(genome, n, n_pairs, R, frag_mean=350.0, frag_sd=30.0, sub_rate=0.01, hard_frac=0.05,
                                     hard_sub_rate=0.2, device=device, seed=0x51ED, mut_seed=0xC0FFEE)
    reads = PackedStringSet.fixed(words.reshape(-1), 2 * n_pairs, R, stride=words.shape[1] * 16)
    pair = nb.PairParams(min_frag=0, max_frag=500, min_mate_score=80, rescue_capacity=max(n_pairs // 4, 1024))
    cap = 24 * 2 * n_pairs
    flush = torch.empty(512 << 20, dtype=torch.uint8, device=device)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    result = {"workload": "nvb_bam_records after seed_extend[_paired]_traceback + finish_alignments", "pairs": n_pairs, "read_len": R,
              "genome_bp": n, "card": torch.cuda.get_device_name(device), "power_limit_w": power_limit_w()}
    tables = {25: contig_table(nb, n, 25, 1), 3000: contig_table(nb, n, 3000, 2)}
    for mode in ("paired", "single"):
        if mode == "paired":
            ws = nb.seed_extend_paired(fmi, genome, reads, params, pair, workspace=PairedWorkspace(fmi, genome, reads, params, pair, cap, traceback=True))
            t = (ws.mate_ops, ws.mate_n_ops, ws.mate_begin, ws.mate_strand)
            names = nb.numbered_names(n_pairs, "pair")
        else:
            ws = None
            torch.cuda.empty_cache()
            ws = nb.seed_extend(fmi, genome, reads, params, workspace=SeedExtendWorkspace(fmi, genome, reads, params, cap, traceback=True),
                                traceback=True)
            t = (ws.best_ops, ws.best_n_ops, ws.best_begin, ws.best_strand)
            names = nb.numbered_names(2 * n_pairs, "read")
        f = nb.finish_alignments(genome, reads, *t, genome_len=n)
        torch.cuda.synchronize()
        for k, table in tables.items():
            call = BamCall(ws, f, reads, table, names)
            call.run(); torch.cuda.synchronize()
            rd, wr, total = bytes_moved(call, f, reads, k)
            counts = call.counts.cpu().tolist()
            key = "%s_%d_contigs" % (mode, k)
            if a.profile:
                from torch.profiler import profile, ProfilerActivity
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    call.run(); torch.cuda.synchronize()
                ev = prof.key_averages()
                ms = lambda s: round(sum(e.device_time_total for e in ev if s in e.key) / 1e3, 4)  # noqa: E731
                result[key] = {"plan_ms": ms("bam_plan_kernel"), "scan_ms": ms("DeviceScan"), "write_ms": ms("bam_write_kernel"),
                               "record_bytes": total, "counts": counts}
                continue
            for i in range(a.warmup):
                flush.zero_(); call.run()
            times = []
            for i in range(a.steps):
                flush.zero_()
                ev0.record(); call.run(); ev1.record()
                torch.cuda.synchronize()
                times.append(ev0.elapsed_time(ev1))
            times.sort()
            med = times[len(times) // 2]
            result[key] = {"ms_median": round(med, 4), "ms_min": round(times[0], 4), "ms_max": round(times[-1], 4), "bytes_read": rd,
                           "bytes_written": wr, "record_bytes": total, "bytes_per_record": round(total / call.n, 1), "counts": counts,
                           "achieved_tbps": round((rd + wr) / (med * 1e-3) / 1e12, 3), "share_of_3_35_tbps": round((rd + wr) / (med * 1e-3) / 1e12 / HBM_TBPS, 3)}
        del f
    result.update(steps=a.steps, warmup=a.warmup, profile=a.profile)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
