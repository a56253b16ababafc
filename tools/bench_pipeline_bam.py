"""Host-to-host BAM output through the pipeline's BAM mode (StreamingBam, nvb_pipeline_create_bam) on bench.py's workloads: 1 M single-end
reads and 500 k pairs of 2 x 150 bp (the draws of bench.py's make_reads / paired_end_config), on its 1.9 Gbp genome with the full suffix
array and the 15-mer table with text context, LOCAL (2, -2, -5, -3), band 31, nvBowtie's --local MAPQ, 64 contigs, numbered names.

For each mode (single end, paired), compression on and off, depth 1 / 2 / 3 and 1 / 2 compute streams (NVB_PIPELINE_COMPUTE_STREAMS), it
times `steps` batches submitted with `depth` in flight, two input batches alternated, and reports host-to-host Mreads/s (submit of the
first batch to the payload of the last on the host), device ms per batch (the compute stream's events), the slot size (the library's and
cudaMemGetInfo around the create) and the payload per batch.  The same batches through the synchronous Python chain (seed_extend with
traceback and MAPQ -> finish_alignments -> bam_records -> bgzf_compress -> host bytes) give the comparison.  A case whose slots do not fit
beside the index is reported as such.  Prints one JSON line.

    python tools/bench_pipeline_bam.py [--steps 6] [--modes se,pe] [--depths 1,2,3]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench  # noqa: E402
from tools.bench_mapq import power_limit_w  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--reads", type=int, default=1_000_000)
    ap.add_argument("--pairs", type=int, default=500_000)
    ap.add_argument("--genome-mbp", type=float, default=1900.0)
    ap.add_argument("--modes", default="se,pe")
    ap.add_argument("--depths", default="1,2,3")
    ap.add_argument("--streams", default="1,2")
    a = ap.parse_args()
    import nvbio_b200 as nb
    from nvbio_b200 import aln, synth
    from nvbio_b200.strings import PackedStringSet
    from nvbio_b200.pipeline import MapqParams, SeedExtendWorkspace, PairedWorkspace
    from nvbio_b200.bam import BamCall, pack_names
    from nvbio_b200.bgzf import BgzfCall

    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    nb.lib()
    idx_args = argparse.Namespace(genome_mbp=a.genome_mbp, sa_interval=1, ktab_k=15, ktab_located=2, impl="ours")
    n, genome, fmi, _, _ = bench.build_index(idx_args, 0, 1, device)
    params = nb.SeedExtendParams(seed_len=bench.SEED_LEN, seed_interval=bench.SEED_INTERVAL, band_len=bench.BAND, type=aln.LOCAL,
                                 both_strands=True, max_seed_hits=100, scheme=aln.SimpleGotohScheme(*bench.SCHEME))
    RL = bench.READ_LEN
    mq = MapqParams.local(RL, device=device)
    k = 64
    contigs = nb.ContigTable(["chr%d" % i for i in range(k)], [n // k] * (k - 1) + [n - (k - 1) * (n // k)])
    out = {"workload": "StreamingBam on bench.py's single-end and paired batches", "genome_bp": n, "read_len": RL,
           "card": torch.cuda.get_device_name(device), "power_limit_w": power_limit_w(), "steps": a.steps, "cases": [], "chain": {}}

    for mode in a.modes.split(","):
        paired = mode == "pe"
        if paired:
            n_reads = 2 * a.pairs
            pair = nb.PairParams(min_frag=0, max_frag=500, min_mate_score=80, rescue_capacity=max(a.pairs // 4, 1024))
            words = []
            for seed, mut in ((0x51ED, 0xC0FFEE), (0x61ED, 0xD0FFEE)):
                w, _, _ = synth.sample_pairs(genome, n, a.pairs, RL, frag_mean=350.0, frag_sd=30.0, sub_rate=0.01, hard_frac=0.05,
                                             hard_sub_rate=0.2, device=device, seed=seed, mut_seed=mut)
                words.append(w.contiguous())
        else:
            n_reads, pair = a.reads, None
            words = [bench.make_reads(genome, n, n_reads, b, device) for b in range(2)]
        wpr = words[0].shape[1]
        hc = 24 * n_reads
        host = [w.cpu().pin_memory() for w in words]
        names = pack_names(nb.numbered_names(n_reads // 2 if paired else n_reads, "r"))
        torch.cuda.synchronize()
        for compress in (True, False):
            for depth in [int(x) for x in a.depths.split(",")]:
                for streams in [int(x) for x in a.streams.split(",")]:
                    if streams > depth:
                        continue
                    case = {"mode": mode, "reads": n_reads, "compress": compress, "depth": depth, "compute_streams": streams}
                    os.environ["NVB_PIPELINE_COMPUTE_STREAMS"] = str(streams)
                    torch.cuda.empty_cache()
                    free0, _ = torch.cuda.mem_get_info(device)
                    try:
                        st = nb.StreamingBam(fmi, genome, params, n_reads, RL, wpr, contigs, mq, pair=pair, compress=compress, depth=depth,
                                             hit_capacity=hc, max_name_bytes=int(names[1][-1]))
                    except nb.NvbError as e:
                        case["error"] = str(e)
                        out["cases"].append(case)
                        continue
                    free1, _ = torch.cuda.mem_get_info(device)
                    case["slot_bytes"] = st.slot_bytes
                    case["mem_get_info_bytes_per_slot"] = (free0 - free1) / depth
                    for i in range(depth):                                # warm-up: every slot once
                        st.result(st.submit(host[i % 2], names))
                    dev_ms, pay = [], []
                    t0 = time.perf_counter()
                    pending = []
                    for i in range(a.steps):
                        if len(pending) == depth:
                            r = st.result(pending.pop(0)); dev_ms.append(r.device_ms); pay.append(r.payload.numel())
                        pending.append(st.submit(host[i % 2], names))
                    for t in pending:
                        r = st.result(t); dev_ms.append(r.device_ms); pay.append(r.payload.numel())
                    wall = time.perf_counter() - t0
                    case.update(Mreads_per_s=a.steps * n_reads / wall / 1e6, wall_ms_per_batch=wall * 1e3 / a.steps,
                                device_ms_per_batch=[round(x, 2) for x in dev_ms], payload_bytes=int(np.mean(pay)),
                                records=r.n_records, mapped=r.counts[1])
                    st.close()
                    del st
                    out["cases"].append(case)
                    print(json.dumps(case), file=sys.stderr, flush=True)
        # the synchronous Python chain on the same batches
        os.environ.pop("NVB_PIPELINE_COMPUTE_STREAMS", None)
        torch.cuda.empty_cache()
        sets = [PackedStringSet.fixed(w.reshape(-1), n_reads, RL, stride=wpr * 16) for w in words]
        name_list = nb.numbered_names(n_reads // 2 if paired else n_reads, "r")
        try:
            if paired:
                ws = PairedWorkspace(fmi, genome, sets[0], params, pair, hc, mapq=mq, traceback=True)
                al = lambda ws: (ws.mate_ops, ws.mate_n_ops, ws.mate_begin, ws.mate_strand)        # noqa: E731
            else:
                ws = SeedExtendWorkspace(fmi, genome, sets[0], params, hc, traceback=True, mapq=mq)
                al = lambda ws: (ws.best_ops, ws.best_n_ops, ws.best_begin, ws.best_strand)        # noqa: E731
            bc = None
            res = {}
            for compress in (True, False):
                times = []
                for i in range(a.steps + 1):
                    torch.cuda.synchronize(); t0 = time.perf_counter()
                    hs = host[i % 2].cuda(non_blocking=True)
                    rs = PackedStringSet.fixed(hs.reshape(-1), n_reads, RL, stride=wpr * 16)
                    if paired:
                        nb.seed_extend_paired(fmi, genome, rs, params, pair, workspace=ws, mapq=mq, traceback=True)
                    else:
                        nb.seed_extend(fmi, genome, rs, params, workspace=ws, mapq=mq)
                    f = nb.finish_alignments(genome, rs, *al(ws), genome_len=n)
                    if bc is None:
                        bc = BamCall(ws, f, rs, contigs, name_list)
                    else:
                        bc._keep = (ws, f, rs) + bc._keep[3:]
                        fo = bc.a.finish
                        fo.d_cigar, fo.d_n_cigar, fo.d_md = f.cigar.data_ptr(), f.n_cigar.data_ptr(), f.md.data_ptr()
                        fo.d_md_len, fo.d_edits = f.md_len.data_ptr(), f.edits.data_ptr()
                        bc.a.reads = rs.struct()
                    recs = bc.run()
                    payload = BgzfCall(recs).run().to_bytes() if compress else recs.to_bytes()
                    if i:
                        times.append(time.perf_counter() - t0)
                    del f
                res["compress" if compress else "raw"] = {"Mreads_per_s": n_reads / np.mean(times) / 1e6, "ms_per_batch": 1e3 * np.mean(times),
                                                          "payload_bytes": len(payload)}
            out["chain"][mode] = res
            del ws, bc
        except (torch.cuda.OutOfMemoryError, nb.NvbError) as e:
            out["chain"][mode] = {"error": str(e)[:200]}
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
