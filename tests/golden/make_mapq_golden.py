"""Generate tests/golden/mapq.npz by RUNNING THE REFERENCE ITSELF: nvBowtie's own BowtieMapq2 (mapq.h:142-331, unpaired) and SimpleFunc
(func.h:39-51), compiled from an nvbio source tree by oracle/ref_mapq.mk into oracle/_ref/libnvbio_ref_mapq.so.

Run in the dev container only (needs the nvbio tree to have built oracle/_ref):
    make -C oracle -f ref_mapq.mk && python tests/golden/make_mapq_golden.py

The grid of every fixture point is mapq_grid(); the tests rebuild it from `cfg` instead of storing it.
"""
import os
import sys
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

OUT = os.path.dirname(os.path.abspath(__file__))

# MAPQ fixture: read lengths x match bonus x --score-min functions (end-to-end ones for bonus 0, local ones otherwise)
MAPQ_LENGTHS = (1, 20, 50, 100, 150, 151, 250, 1000)
MAPQ_BONUS = (0, 2, 3)
MAPQ_MIN_E2E = (("L", -0.6, -0.6), ("L", 0.0, -0.2), ("S", -4.0, -1.5), ("L", -3.0, 0.0))      # the first: nvBowtie's end-to-end preset
MAPQ_MIN_LOCAL = (("G", 0.0, 10.0), ("G", 20.0, 8.0), ("L", 0.0, 1.2), ("S", 10.0, 3.0))       # nvBowtie's --local preset, bowtie2's default
# SimpleFunc fixture: the presets above, nvBowtie's seed intervals (S,1,0.75 local / S,1,1.15 end-to-end) and a few more
SIMPLE_FUNCS = MAPQ_MIN_E2E + MAPQ_MIN_LOCAL + (("S", 1.0, 0.75), ("S", 1.0, 1.15), ("G", -5.0, 3.3), ("L", 0.5, 0.37), ("G", 1.5, -2.25))


def mapq_grid(length, bonus, min_score):
    """(best, has_second, second) points of the MAPQ fixture for one (read length, match bonus, min score): every best score from
    min - 2 to max(perfect, min) + 3, each with no second (second = INT_MIN) and with every second score from min - 2 to best"""
    lo = int(min_score) - 2
    bests = np.arange(lo, max(int(length) * int(bonus), int(min_score)) + 4, dtype=np.int64)
    counts = bests - lo + 2
    best = np.repeat(bests, counts)
    k = np.arange(len(best)) - np.repeat(np.cumsum(counts) - counts, counts)        # 0: no second, k >= 1: second = lo + k - 1
    has = k > 0
    second = np.where(has, lo + k - 1, -2**31)
    return best.astype(np.int32), has.astype(np.uint8), second.astype(np.int32)


def make_mapq(ref):
    """cfg[c] = (read length, match bonus, min score, index of its function in SIMPLE_FUNCS); the MAPQ of the points
    mapq_grid(*cfg[c, :3]) is mapq[offsets[c]:offsets[c + 1]].  sf_vals[f] = SimpleFunc sf_funcs[f] = (type L/G/S as 0/1/2, const, coeff)
    over sf_x = 1..4096."""
    out = {}
    out["sf_funcs"] = np.array([("LGS".index(t), k, m) for t, k, m in SIMPLE_FUNCS], np.float64)
    out["sf_x"] = np.arange(1, 4097, dtype=np.int32)
    out["sf_vals"] = np.stack([ref.simple_func(t, k, m, out["sf_x"]) for t, k, m in SIMPLE_FUNCS])
    cfg, mapq, offsets = [], [], [0]
    for length in MAPQ_LENGTHS:
        for bonus in MAPQ_BONUS:
            for t, k, m in (MAPQ_MIN_E2E if bonus == 0 else MAPQ_MIN_LOCAL):
                ms = int(ref.simple_func(t, k, m, [length])[0])
                best, has, second = mapq_grid(length, bonus, ms)
                mapq.append(ref.mapq(best, has, second, length, bonus, ms))
                cfg.append((length, bonus, ms, SIMPLE_FUNCS.index((t, k, m))))
                offsets.append(offsets[-1] + len(best))
    out["cfg"] = np.array(cfg, np.int32)
    out["offsets"] = np.array(offsets, np.int64)
    out["mapq"] = np.concatenate(mapq)
    np.savez_compressed(os.path.join(OUT, "mapq.npz"), **out)


def main():
    from oracle.ref_mapq import RefMapq
    assert RefMapq.available(), "build oracle/_ref first: make -C oracle -f ref_mapq.mk"
    make_mapq(RefMapq())
    print("wrote mapq.npz")


if __name__ == "__main__":
    main()
