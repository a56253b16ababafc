"""Cost and ratio of BGZF compression on the device (nvb_bgzf_compress) on bench.py's paired-end workload, as tools/bench_bam.py builds it
(500k FR pairs of 2 x 150 bp, 1.9 Gbp genome, paired traceback, finish_alignments and nvb_bam_records once, 25 contigs).  Two batches of
records: without base qualities (QUAL all 0xFF) and with seeded Illumina-like qualities.  For each, bgzf_compress alone is timed with
device events over repeated calls (median, min, max) and reported as input GB/s; on the same bytes, the compressed size against host zlib
levels 1 and 6 over the same 0xFF00-byte blocks (with their single-thread host-CPU MB/s), and the wall time of write_bam for the batch on
the host path (D2H + zlib level 6 + file write) against the device path (compression + D2H of the members + file write).  Prints one JSON
line with the card and its power limit.
--profile: instead, one torch.profiler run per batch: the device time of each kernel of one call.

    python tools/bench_bgzf.py [--steps 20] [--warmup 3] [--profile]
"""
import argparse
import json
import os
import sys
import tempfile
import time
import zlib

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench  # noqa: E402
from tools.bench_mapq import power_limit_w  # noqa: E402
from tools.bench_bam import contig_table  # noqa: E402

BLOCK = 0xFF00


def illumina_quals(n_reads, read_len, device, seed):
    """phred values per base: high in the first cycles, declining and noisier toward the 3' end, with runs of Q2 at some read ends"""
    rng = np.random.default_rng(seed)
    pos = np.arange(read_len)[None, :]
    mean = 37.0 - 10.0 * (pos / read_len) ** 2
    q = np.rint(mean + rng.normal(0, 1.0 + 3.0 * pos / read_len, (n_reads, read_len)))
    q = np.clip(q, 2, 41)
    q = np.where(rng.random((n_reads, read_len)) < 0.6, np.round(q / 4) * 4 - 1, q)       # binned values dominate, as on recent instruments
    tail = rng.random(n_reads) < 0.1
    start = rng.integers(read_len // 2, read_len, n_reads)
    q[tail[:, None] & (pos >= start[:, None])] = 2
    return torch.from_numpy(np.clip(q, 2, 41).astype(np.uint8).reshape(-1)).to(device)


def host_zlib(raw, level):
    t0 = time.perf_counter()
    size = 0
    for i in range(0, len(raw), BLOCK):
        c = zlib.compressobj(level, zlib.DEFLATED, -15)
        size += len(c.compress(raw[i:i + BLOCK]) + c.flush()) + 26
    return size, time.perf_counter() - t0


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
    from nvbio_b200.bgzf import BgzfCall
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
    ws = nb.seed_extend_paired(fmi, genome, reads, params, pair,
                               workspace=PairedWorkspace(fmi, genome, reads, params, pair, 24 * 2 * n_pairs, traceback=True))
    f = nb.finish_alignments(genome, reads, ws.mate_ops, ws.mate_n_ops, ws.mate_begin, ws.mate_strand, genome_len=n)
    table = contig_table(nb, n, 25, 1)
    names = nb.numbered_names(n_pairs, "pair")
    header = nb.bam_header(table)
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    result = {"workload": "nvb_bgzf_compress of nvb_bam_records after seed_extend_paired_traceback + finish_alignments", "pairs": n_pairs,
              "read_len": R, "genome_bp": n, "card": torch.cuda.get_device_name(device), "power_limit_w": power_limit_w()}
    for key, quals in (("no_quals", None), ("illumina_quals", illumina_quals(2 * n_pairs, R, device, 7))):
        recs = BamCall(ws, f, reads, table, names, quals).run()
        raw_t = recs.data[:int(recs.offsets[-1])]
        call = BgzfCall(raw_t)
        blocks = call.run()
        torch.cuda.synchronize()
        n_in = raw_t.numel()
        if a.profile:
            from torch.profiler import profile, ProfilerActivity
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                call.run(); torch.cuda.synchronize()
            ev = prof.key_averages()
            ms = lambda s: round(sum(e.device_time_total for e in ev if s in e.key) / 1e3, 4)  # noqa: E731
            result[key] = {"compress_ms": ms("bgzf_compress_kernel"), "scan_ms": ms("bgzf_scan_kernel"), "copy_ms": ms("bgzf_copy_kernel"),
                           "input_bytes": n_in}
            continue
        for _ in range(a.warmup):
            call.run()
        times = []
        for _ in range(a.steps):
            ev0.record(); call.run(); ev1.record()
            torch.cuda.synchronize()
            times.append(ev0.elapsed_time(ev1))
        times.sort()
        med = times[len(times) // 2]
        out_bytes = int(blocks.offsets[-1])
        raw = raw_t.cpu().numpy().tobytes()
        z1, t1 = host_zlib(raw, 1)
        z6, t6 = host_zlib(raw, 6)
        with tempfile.TemporaryDirectory() as td:
            t0 = time.perf_counter()
            nb.write_bam(os.path.join(td, "host.bam"), header, [recs])
            host_wall = time.perf_counter() - t0
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            nb.write_bam(os.path.join(td, "dev.bam"), header, [call.run()])
            dev_wall = time.perf_counter() - t0
        result[key] = {"input_bytes": n_in, "blocks": blocks.n_blocks, "output_bytes": out_bytes,
                       "ms_median": round(med, 4), "ms_min": round(times[0], 4), "ms_max": round(times[-1], 4),
                       "input_gbps": round(n_in / (med * 1e-3) / 1e9, 2),
                       "ratio": round(n_in / out_bytes, 4), "host_cpu_zlib1_ratio": round(n_in / z1, 4), "host_cpu_zlib6_ratio": round(n_in / z6, 4),
                       "ratio_vs_zlib1": round(z1 / out_bytes, 4), "ratio_vs_zlib6": round(z6 / out_bytes, 4),
                       "host_cpu_zlib1_mbps_1thread": round(n_in / t1 / 1e6, 1), "host_cpu_zlib6_mbps_1thread": round(n_in / t6 / 1e6, 1),
                       "write_bam_host_path_s": round(host_wall, 3), "write_bam_device_path_s": round(dev_wall, 3)}
    result.update(steps=a.steps, warmup=a.warmup, profile=a.profile)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
