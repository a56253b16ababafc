"""-m gpu: the drop-in boundary (include/nvbio_b200/shim, DESIGN B-A1 / B-B1 / B-A2 / B-B2) against the reference's own kernels.

tests/shim/*.cu are programs written against nvbio's own types -- io::FMIndexDataDevice::fm_index_type, FMIndexFilterDevice::rank/locate
over an InfixSet of 4-bit reads, aln::batch_banded_alignment_score<B>, BatchedBandedAlignmentScore<...>::enact on a user-defined stream,
aln::batch_alignment_score, nvBowtie's map_* entry points and its best-score extension.  oracle/ref_shim.mk compiles each twice into
oracle/_ref/shim: as is (`_ref`: the reference's templates and kernels) and with include/nvbio_b200/shim/*.h + libnvbio_b200.so
(`_b200`).  Both builds run on the same seeded inputs; every result array they dump must be byte-identical, and the call counters must
show that the `_b200` build ran the nvbio_b200 kernels exactly where the shim claims to and the reference's own code everywhere else.

The `edges` program runs the batch classes where a forwarding layer goes wrong: bands 3 / 5 / 7 / 15 / 31 / 63 x GLOBAL / LOCAL /
SEMI_GLOBAL, BestSink<int16> and <int32>, 2- and 4-bit patterns of either endianness with N's, pattern lengths 0..830 in one batch
(past the packed kernels' 801 - band cap, so one call takes both routes), windows of M + B - 1 symbols, one short, shorter than the
pattern and empty, scores outside the int16 range under both schedulers, a user stream's min_score under both schedulers, deliberate
fall-backs (band 9) and the scratch arenas growing and shrinking.  Windows the reference's kernel reads past are left out; tests/shim/shim_harness.cu says which and why.

The binaries are built only where an nvbio source tree is at hand; elsewhere these tests skip, naming the missing file."""
import filecmp
import json
import os
import subprocess

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "oracle", "_ref", "shim")

# calls the `edges` program makes (tests/shim/shim_harness.cu run_edges).  Accelerated: 6 bands x (3 types + BestSink<int16>), 2 more
# int16, 3 packings, 3 staged, 6 scratch sizes, 4 thread-scheduler wide-score calls, 4 user-stream batches enacted 3 times each.  Run by
# the reference's kernel: band 9 once through priv::AlignmentStream and 3 times through the user stream; the LOCAL and SEMI_GLOBAL
# wide-score calls into BestSink<int16> (their scores leave int16); the 3 staged wide-score calls (their H wraps in the short2
# checkpoints); the staged user stream with a min_score in reach, 3 times.  6 full-matrix calls.
EDGE_CALLS = {"banded": 6 * 4 + 2 + 3 + 3 + 6 + 4 + 4 * 3, "full": 6, "fallbacks": 1 + 3 + 2 + 3 + 3}
# map_* calls of the mapping harness: 13 configurations, of which approx_s34 (seed length 34: 3 * 34 + 1 > NVB_MAP_MAX_PUSHES) falls back
MAPPING_CONFIGS = ("exact_r0", "exact_r1", "exact_fw", "approx_r0", "approx_rc", "map_sub", "map_nosub", "exact_tiny",
                   "exact_h1", "exact_min70", "approx_s33", "approx_s34", "approx_h1")
MAPPING_CALLS = {"mapped": 12, "fallbacks": 1}
SCORE_CONFIGS = ("local_b31", "local_b15", "e2e_b31", "e2e_b7", "local_b3", "local_b7", "e2e_b15")


def pair(name):
    """(reference build, shim build) of a harness; skips naming the first missing file"""
    paths = tuple(os.path.join(BIN, name + s) for s in ("_ref", "_b200"))
    for p in paths:
        if not os.path.exists(p):
            pytest.skip("%s not built (oracle/ref_shim.mk builds it where an nvbio source tree is at hand)" % os.path.relpath(p, ROOT))
    return paths


def run(binary, args, out):
    """run one build with `out` as its dump directory (the argument OUT); returns its JSON line"""
    os.makedirs(out, exist_ok=True)
    r = subprocess.run([binary] + [out if a == "OUT" else a for a in args], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, "%s failed: %s" % (os.path.basename(binary), (r.stderr or r.stdout)[-800:])
    return json.loads(r.stdout.strip().splitlines()[-1])


def same_dumps(a, b):
    fa, fb = sorted(os.listdir(a)), sorted(os.listdir(b))
    assert fa == fb and fa, (fa, fb)
    diff = [f for f in fa if not filecmp.cmp(os.path.join(a, f), os.path.join(b, f), shallow=False)]
    assert not diff, "arrays differ between the reference build and the shim build: %s" % diff
    return fa


def run_pair(name, args, tmp):
    ref, b2 = pair(name)
    out = {}
    for tag, binary in (("ref", ref), ("b200", b2)):
        out[tag] = run(binary, args, os.path.join(str(tmp), tag))
    files = same_dumps(os.path.join(str(tmp), "ref"), os.path.join(str(tmp), "b200"))
    assert out["ref"]["shim"] == 0 and out["b200"]["shim"] == 1
    return out["ref"], out["b200"], files


def check_fmmap(tmp):
    """B-A1: nvbio's fmmap loop (rank, locate, banded DP with BestSink<int16> and <int32>)"""
    ref, b2, files = run_pair("shim_harness", ["fmmap", "OUT", "3000000", "40000", "100"], tmp)
    assert {"fmmap_ranges.bin", "fmmap_slots.bin", "fmmap_hits.bin", "fmmap_scores_i16.bin", "fmmap_sinks_i32.bin", "fmmap_best_i32.bin"} <= set(files)
    assert ref["hits"] == b2["hits"] and ref["hits"] > ref["reads"]
    assert b2["b200_calls"] == {"fm_rank": 3, "fm_locate": 6, "banded": 6, "full": 0, "fallbacks": 0}, b2["b200_calls"]
    return ref, b2


def check_batch(tmp):
    """B-B1: BatchedBandedAlignmentScore on a user stream (thread and staged schedulers) and aln::batch_alignment_score"""
    ref, b2, files = run_pair("shim_harness", ["batch", "OUT", "65536"], tmp)
    assert len(files) == 7 + 6
    assert b2["b200_calls"] == {"banded": 21, "full": 9, "fallbacks": 0}, b2["b200_calls"]
    return ref, b2


def check_edges(tmp):
    ref, b2, files = run_pair("shim_harness", ["edges", "OUT", "20000"], tmp)
    assert ref["planned"] == b2["planned"] == EDGE_CALLS, ref["planned"]
    assert b2["b200_calls"] == EDGE_CALLS, b2["b200_calls"]
    # the batch holds every case it is there for
    for k in ("empty_patterns", "long_patterns", "patterns_with_n", "full_windows", "short1_windows", "random_windows", "below_windows", "empty_windows"):
        assert ref[k] > 20, (k, ref[k])
    d = os.path.join(str(tmp), "ref")
    ld = lambda f, t: np.fromfile(os.path.join(d, f), t)
    # windows shorter than the pattern keep the sink's defaults; int16 scores really left the int16 range in the int32 sinks
    for b in (3, 63):
        sinks = ld("b%d_local_sinks.bin" % b, np.uint32).reshape(-1, 2)
        assert (sinks[:, 0] == 0xFFFFFFFF).sum() >= ref["below_windows"] + ref["empty_windows"]
    wide = ld("wide_b15_global_scores.bin", np.int32)
    assert (wide > 32767).sum() > 1000
    # ... and the reference's staged passes really differ from one pass there (its short2 checkpoints wrap), which is why the shim
    # hands those batches back to the reference's kernel
    for t in ("global", "local", "semi"):
        assert not np.array_equal(ld("wide_b15_%s_staged_scores.bin" % t, np.int32), ld("wide_b15_%s_scores.bin" % t, np.int32)), t
    return ref, b2


def check_mapping(tmp):
    """B-A2: nvBowtie's non-template map_exact / map_approx / map / gather_ranges on nvBowtie's own PODs, linked once against nvBowtie's
    mapping.cu and once against tests/shim/nvbowtie_mapping_b200.cu: deque sizes, the SeedHits of every read (canonical order), the range
    sizes in pop_top() order, reseed flags, gather_ranges totals and the deque index of every read left without hits are identical"""
    ref, b2, files = run_pair("nvbowtie_harness", ["OUT", "400000", "4000"], tmp)
    assert "exact_r0_hits.bin" in files and "approx_r0_hits.bin" in files and "exact_tiny_sizes.bin" in files
    for cfg in MAPPING_CONFIGS:
        a, b = ref[cfg], b2[cfg]
        assert a["hits"] == b["hits"] > 0 and a["range_total"] == b["range_total"] and a["full_deques"] == b["full_deques"], (cfg, a, b)
        assert a["pop_order_ok"] == 1 and b["pop_order_ok"] == 1, cfg
    assert ref["exact_tiny"]["full_deques"] > 100 and ref["exact_h1"]["full_deques"] > 1000 and ref["approx_h1"]["full_deques"] > 1000
    assert ref["reads_below_20"] > 100
    # min_read_len = 70 drops reads of 60..69 bp that exact_fw (seed length 16, min_read_len 20) maps
    d = os.path.join(str(tmp), "ref")
    assert (np.fromfile(os.path.join(d, "exact_min70_empty_index.bin"), np.uint32) == 0xFFFFFFFF).sum() > \
           (np.fromfile(os.path.join(d, "exact_fw_empty_index.bin"), np.uint32) == 0xFFFFFFFF).sum()
    assert b2["b200_calls"] == MAPPING_CALLS, b2["b200_calls"]
    return ref, b2


def check_score_best(tmp):
    """B-B2: nvBowtie's best-score extension (detail::banded_score_best) with the shim's SmithWatermanScoringScheme binding: hit.score
    (the worst_score clamp included) and hit.sink of every hit, bands 3 / 7 / 15 / 31, --local and end-to-end"""
    ref, b2, files = run_pair("nvbowtie_score_harness", ["OUT", "2000000", "20000", "200000"], tmp)
    assert len(files) == 2 * len(SCORE_CONFIGS)
    sc = np.fromfile(os.path.join(str(tmp), "ref", "local_b31_score.bin"), np.int32)
    assert (sc > 60).mean() > 0.5 and (sc != 12345).all()
    for c in SCORE_CONFIGS:
        assert ref[c + "_clamped"] == b2[c + "_clamped"] > 0, c
    assert b2["b200_calls"] == {"banded": 3 * len(SCORE_CONFIGS), "fallbacks": 0}, b2["b200_calls"]
    return ref, b2


CHECKS = (check_fmmap, check_batch, check_edges, check_mapping, check_score_best)


@pytest.mark.parametrize("check", CHECKS, ids=[c.__name__[len("check_"):] for c in CHECKS])
def test_shim_build_identical_to_reference_build(check, tmp_path):
    from tests.gpu_util import require_gpu
    require_gpu()
    check(tmp_path)
