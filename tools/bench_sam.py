"""Cost of formatting BAM records as SAM text on the device (nvb_sam_format) on bench.py's paired-end workload (500k FR pairs of 2 x 150 bp
from synth.sample_pairs, 1.9 Gbp genome cut into 25 contigs, full suffix array, 15-mer table with text context, PairParams(0, 500, 80,
n/4)).  The paired traceback, finish_alignments and nvb_bam_records run once; then nvb_sam_format and nvb_bam_records on the same
records are timed alternately in three rounds, with device events after warm-up, and nvb_sam_format on the coordinate-sorted records
(nvb_bam_sort) to show that the input order does not matter.  Reports ms per call, the bytes each call reads and writes (computed from
the sizes it produced, not measured) and their share of the H100's 3.35 TB/s data-sheet bandwidth, with the card and its power limit.
Prints one JSON line.  --profile: instead, one torch.profiler run per call: the size kernel, the scan and the write kernel.

    python tools/bench_sam.py [--steps 20] [--warmup 3] [--profile]
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
from tools.bench_bam import contig_table, bytes_moved as bam_bytes  # noqa: E402

HBM_TBPS = 3.35


def sam_bytes(call):
    """bytes nvb_sam_format reads and writes: the size kernel reads the offsets and each record's fixed fields, CIGAR and tags (bounded
    here by the whole record), the scan reads and writes 8 bytes per record twice, the write kernel reads the offsets and the records and
    writes the text"""
    n = call.n
    offsets = call._keep[1]
    rec = int(offsets[-1])
    text = int(call.offsets[-1])
    rd = 8 * (n + 1) + rec + 2 * 8 * (n + 1) + 2 * 8 * (n + 1) + rec
    wr = 8 * (n + 1) + 8 * (n + 1) + text
    return rd, wr, rec, text


def timed(fn, steps, warmup, flush):
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(warmup):
        flush.zero_(); fn()
    times = []
    for _ in range(steps):
        flush.zero_()
        ev0.record(); fn(); ev1.record()
        torch.cuda.synchronize()
        times.append(ev0.elapsed_time(ev1))
    times.sort()
    return times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--pairs", type=int, default=500_000)
    ap.add_argument("--genome-mbp", type=float, default=1900.0)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    import nvbio_b200 as nb
    from nvbio_b200 import aln, synth
    from nvbio_b200.bam import BamCall
    from nvbio_b200.sam import SamCall
    from nvbio_b200.strings import PackedStringSet
    from nvbio_b200.pipeline import PairedWorkspace

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
    ws = nb.seed_extend_paired(fmi, genome, reads, params, pair, workspace=PairedWorkspace(fmi, genome, reads, params, pair, cap, traceback=True))
    f = nb.finish_alignments(genome, reads, ws.mate_ops, ws.mate_n_ops, ws.mate_begin, ws.mate_strand, genome_len=n)
    contigs = contig_table(nb, n, 25, 1)
    bam = BamCall(ws, f, reads, contigs, nb.numbered_names(n_pairs, "pair"))
    recs = bam.run()
    torch.cuda.synchronize()
    srt = nb.sort_bam_records(recs)
    sam = SamCall(recs, contigs)
    sam_sorted = SamCall(srt, contigs)
    sam.run(); sam_sorted.run(); torch.cuda.synchronize()
    assert int(sam.rejected[0]) == 0 and int(sam_sorted.rejected[0]) == 0
    assert int(sam.offsets[-1]) == int(sam_sorted.offsets[-1])
    result = {"workload": "nvb_sam_format vs nvb_bam_records on the records of seed_extend_paired_traceback + finish_alignments",
              "pairs": n_pairs, "records": bam.n, "read_len": R, "genome_bp": n, "contigs": 25,
              "card": torch.cuda.get_device_name(device), "power_limit_w": power_limit_w()}
    b_rd, b_wr, rec_bytes = bam_bytes(bam, f, reads, 25)
    s_rd, s_wr, _, text_bytes = sam_bytes(sam)
    result.update(record_bytes=rec_bytes, text_bytes=text_bytes, text_over_record_bytes=round(text_bytes / rec_bytes, 3))
    if a.profile:
        from torch.profiler import profile, ProfilerActivity
        for key, call in (("sam", sam), ("sam_sorted", sam_sorted), ("bam", bam)):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                call.run(); torch.cuda.synchronize()
            ev = prof.key_averages()
            ms = lambda s: round(sum(e.device_time_total for e in ev if s in e.key) / 1e3, 4)  # noqa: E731
            if key == "bam":
                result[key] = {"plan_ms": ms("bam_plan_kernel"), "scan_ms": ms("DeviceScan"), "write_ms": ms("bam_write_kernel")}
            else:
                result[key] = {"size_ms": ms("sam_size_kernel"), "scan_ms": ms("DeviceScan"), "write_ms": ms("sam_write_kernel")}
    else:
        rounds = {"sam": [], "bam": [], "sam_sorted": []}
        for _ in range(a.rounds):
            for key, call in (("sam", sam), ("bam", bam), ("sam_sorted", sam_sorted)):
                rounds[key].append(timed(call.run, a.steps, a.warmup, flush))
        for key, (rd, wr) in (("sam", (s_rd, s_wr)), ("sam_sorted", (s_rd, s_wr)), ("bam", (b_rd, b_wr))):
            meds = [t[len(t) // 2] for t in rounds[key]]
            med = float(np.median(meds))
            result[key] = {"ms_median_per_round": [round(m, 4) for m in meds], "ms_median": round(med, 4),
                           "ms_per_1m_records": round(med / bam.n * 1e6, 4), "bytes_read": rd, "bytes_written": wr,
                           "achieved_tbps": round((rd + wr) / (med * 1e-3) / 1e12, 3),
                           "share_of_3_35_tbps": round((rd + wr) / (med * 1e-3) / 1e12 / HBM_TBPS, 3)}
        result["sam_over_bam"] = round(result["sam"]["ms_median"] / result["bam"]["ms_median"], 3)
    result.update(steps=a.steps, warmup=a.warmup, rounds=a.rounds, profile=a.profile)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
