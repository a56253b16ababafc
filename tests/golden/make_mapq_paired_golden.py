"""Generate tests/golden/mapq_paired.npz by RUNNING THE REFERENCE ITSELF: nvBowtie's own BowtieMapq2 on paired best alignments
(mapq.h:155-170, as MapqFunctorPE runs it, aligner_best_approx_paired.h:50-96), compiled from an nvbio source tree by
oracle/ref_mapq_paired.mk into oracle/_ref/libnvbio_ref_mapq_paired.so; the --score-min values come from nvBowtie's SimpleFunc through
oracle/ref_mapq.mk's oracle/_ref/libnvbio_ref_mapq.so.

Run in the dev container only (needs the nvbio tree to have built oracle/_ref):
    make -C oracle -f ref_mapq.mk && make -C oracle -f ref_mapq_paired.mk && python tests/golden/make_mapq_paired_golden.py

The points of every fixture configuration are pair_grid(); the tests rebuild them from `cfg` instead of storing them.
"""
import os
import sys
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests.golden.make_mapq_golden import MAPQ_BONUS, MAPQ_MIN_E2E, MAPQ_MIN_LOCAL, SIMPLE_FUNCS  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))

# mate read lengths: every pair l1 <= l2 of these
PAIR_LENGTHS = (1, 50, 100, 150, 151, 250, 1000)
# the fractions of the score range where BowtieMapq2 changes its answer (mapq.h:180-327)
THRESHOLDS = (0.1, 0.2, 0.3, 0.4, 0.5, 0.6, 0.67, 0.68, 0.7, 0.8, 0.84, 0.88, 0.9)
KIND_NONE, KIND_PAIRED, KIND_UNPAIRED = 0, 1, 2


def split(s):
    """a pair score as two mate scores (what the reference sums): floor half and the rest"""
    s = np.asarray(s, np.int64)
    a = np.floor_divide(s, 2)
    return a, s - a


def pair_grid(len1, len2, bonus, min1, min2):
    """(s1, s2, kind, t1, t2) points of one configuration.  Pair scores `best` from min - 2 to max(perfect, min) + 3: every one when the
    range is short, else a stride plus every score within 2 of a threshold.  Per best: no second; an unpaired second (scores best and
    min - 2: the reference must ignore it); paired seconds at distances 0..3 and within 2 of every threshold distance, below AND above best."""
    lo = int(min1) + int(min2) - 2
    perfect = (int(len1) + int(len2)) * int(bonus)
    hi = max(perfect, int(min1) + int(min2)) + 3
    diff = perfect - (int(min1) + int(min2))
    near = np.array([int(round(abs(diff) * c)) + d for c in THRESHOLDS for d in range(-2, 3)], np.int64)
    if hi - lo <= 160:
        bests = np.arange(lo, hi + 1, dtype=np.int64)
    else:
        bests = np.unique(np.concatenate([np.arange(lo, hi + 1, max(1, (hi - lo) // 60)), lo + 2 + near, [lo, lo + 1, hi, perfect, perfect - 1]]))
        bests = bests[(bests >= lo) & (bests <= hi)]
    dist = np.unique(np.concatenate([np.arange(0, 4), near[near > 0]]))
    dist = np.concatenate([dist, -dist[dist > 0]])
    best, kind, second = [], [], []
    for b in bests:
        sec = b - dist
        sec = sec[sec >= lo]
        best.append(np.full(3 + len(sec), b)); kind.append(np.r_[KIND_NONE, KIND_UNPAIRED, KIND_UNPAIRED, np.full(len(sec), KIND_PAIRED)])
        second.append(np.r_[0, b, lo, sec])
    best, kind, second = np.concatenate(best), np.concatenate(kind), np.concatenate(second)
    s1, s2 = split(best)
    t1, t2 = split(second)
    t1 = np.where(kind == KIND_PAIRED, t1, second)                   # an unpaired second is one alignment of the whole score
    t2 = np.where(kind == KIND_PAIRED, t2, 0)
    return (s1.astype(np.int32), s2.astype(np.int32), kind.astype(np.uint8), t1.astype(np.int32), t2.astype(np.int32))


def configs(simple_func):
    """cfg rows (len1, len2, match bonus, min1, min2, index of the --score-min function in SIMPLE_FUNCS); simple_func(kind, k, m, x)"""
    out = []
    for i, l1 in enumerate(PAIR_LENGTHS):
        for l2 in PAIR_LENGTHS[i:]:
            for bonus in MAPQ_BONUS:
                for t, k, m in (MAPQ_MIN_E2E if bonus == 0 else MAPQ_MIN_LOCAL):
                    m1, m2 = (int(v) for v in simple_func(t, k, m, [l1, l2]))
                    out.append((l1, l2, bonus, m1, m2, SIMPLE_FUNCS.index((t, k, m))))
    return np.array(out, np.int32)


def make_mapq_paired(ref, simple_func):
    """cfg[c] as configs(simple_func); the MAPQ of the points pair_grid(*cfg[c, :5]) is mapq[offsets[c]:offsets[c + 1]]"""
    cfg = configs(simple_func)
    mapq, offsets = [], [0]
    for l1, l2, bonus, m1, m2, _ in cfg:
        s1, s2, kind, t1, t2 = pair_grid(l1, l2, bonus, m1, m2)
        mapq.append(ref.mapq_paired(s1, s2, kind, t1, t2, l1, l2, bonus, m1, m2))
        offsets.append(offsets[-1] + len(s1))
    np.savez_compressed(os.path.join(OUT, "mapq_paired.npz"), cfg=cfg, offsets=np.array(offsets, np.int64), mapq=np.concatenate(mapq))
    return offsets[-1]


def main():
    from oracle.ref_mapq import RefMapq
    from oracle.ref_mapq_paired import RefMapqPaired
    assert RefMapq.available() and RefMapqPaired.available(), "build oracle/_ref first: make -C oracle -f ref_mapq.mk && make -C oracle -f ref_mapq_paired.mk"
    print("wrote mapq_paired.npz: %d points" % make_mapq_paired(RefMapqPaired(), RefMapq().simple_func))


if __name__ == "__main__":
    main()
