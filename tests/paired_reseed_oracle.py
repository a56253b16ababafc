"""Oracle composition of nvb_seed_extend_paired_reseed (test infrastructure): the mates' rounds from seed_extend_reseed_oracle under the
paired flag rule (its reseed_flag with the alignment term held true: seed statistics only), and the pairing of seed_extend_paired_oracle
/ pair_mapq_oracle run once on the union of every round's hits (their single-end stage, seed_extend_oracle, answered by that union).
The pinned oracles run as they are; only the two names they look up are substituted for the duration of one call."""
from unittest import mock
import numpy as np
from tests import reseed_oracle, pipeline_oracle, pair_mapq_oracle as pmo


def union_se(rs):
    """seed_extend_reseed_oracle's kept hits of all rounds (round-major, so hit index order is (round, tie)) as a single-end result"""
    return dict(hit_string=rs["hit_string"], hit_window=rs["hit_window"], hit_score=rs["hit_score"], hit_sink=rs["hit_sink"])


_reseed_flag = reseed_oracle.reseed_flag


def stats_only_flag(range_sum, range_count, rep_seeds, aligned):
    """the paired flag rule: reseed_oracle.reseed_flag without the alignment term"""
    return _reseed_flag(range_sum, range_count, rep_seeds, True)


def seed_extend_paired_reseed_oracle(O, idx, genome_sym, reads, params, pair, n_pairs, max_reseed, rep_seeds, hit_capacity,
                                     min_score=None, match_bonus=None, quals=None):
    """reads: mate 1 of every pair, then mate 2.  Returns the outputs of seed_extend_paired_oracle (or, with min_score and match_bonus,
    pair_mapq_oracle) over the union, plus rounds[2, n_pairs], active (per round), n_hits = (kept, found) and the mates' per-round
    stats / flags."""
    unused = np.zeros(max(len(r) for r in reads) + 1, np.int64)        # a min-score table the stats-only flag never reads
    with mock.patch.object(reseed_oracle, "reseed_flag", stats_only_flag):
        rs = reseed_oracle.seed_extend_reseed_oracle(O, idx, genome_sym, reads, params, max_reseed, rep_seeds, unused, hit_capacity,
                                                     quals=quals)
    se = union_se(rs)
    union = lambda *a, **k: se                                           # noqa: E731
    with mock.patch.object(pipeline_oracle, "seed_extend_oracle", union), mock.patch.object(pmo, "seed_extend_oracle", union):
        if match_bonus is None:
            out = pipeline_oracle.seed_extend_paired_oracle(O, idx, genome_sym, reads, params, pair, n_pairs, quals=quals)
        else:
            out = pmo.pair_mapq_oracle(O, idx, genome_sym, reads, params, pair, n_pairs, min_score, match_bonus, quals=quals)
    out.update(rounds=np.asarray(rs["rounds"]).reshape(2, n_pairs), active=rs["active"], n_hits=rs["n_hits"], stats=rs["stats"],
               flags=rs["flags"], hit_round=rs["hit_round"])
    return out


# The test world of tests/test_paired_reseed_oracle.py and tests/test_gpu_paired_reseed.py: a random genome with a planted 16-copy family
# and pairs in these classes, mate 1 of every pair first, then mate 2 (the reads as sequenced).  With both strands, round 0's seeds of a
# 90 bp read (L 16, I 24) leave read positions [18, 24), [42, 48), [66, 72) uncovered.
RL, L, I = 90, 16, 24
UNIT, COPIES = 600, 16
SUBST = [2, 26, 50, 74]        # under every round-0 seed of both strings, under no forward seed at offset 8 (max_reseed 2, round 1)
CLASSES = ("sub2", "sub1", "family", "ordinary", "mutated", "short", "swapped", "nowhere")


def rc(s):
    return np.where(s < 4, 3 - s, s)[::-1].astype(np.uint8)


def planted_pairs(G=320_000, per_class=(24, 24, 32, 40, 24, 16, 24, 8), seed=21):
    """returns (genome, reads, cls[n_pairs] index into CLASSES, truth[n_pairs, 2] = (genome begin of mate 1's locus, of mate 2's)).
    sub2: both mates carry a substitution under every round-0 seed; sub1: mate 1 does, mate 2 is clean; family: the fragment lies
    inside copy c, and each mate carries copy c's private variant at read position 20 (copy c: mate 1's at unit offset 30 + 15c,
    mate 2's at 309 + 15c); ordinary / mutated (6 % substitutions) / short (mate 2 shorter, some below L) pairs in FR orientation;
    swapped: mate 1 on the reverse strand; nowhere: random mates."""
    rng = np.random.default_rng(seed)
    g = rng.integers(0, 4, G).astype(np.uint8)
    unit = rng.integers(0, 4, UNIT).astype(np.uint8)
    starts = [5_000 + 17_000 * c for c in range(COPIES)]
    for c, st in enumerate(starts):
        u = unit.copy()
        for v in (30 + 15 * c, 309 + 15 * c):
            u[v] = (u[v] + 1) % 4
        g[st:st + UNIT] = u
    m1, m2, cls, truth = [], [], [], []

    def fr(p, frag, ln2=RL):
        return g[p:p + RL].copy(), rc(g[p + frag - ln2:p + frag]), (p, p + frag - ln2)

    def sub(r):
        r[SUBST] = (r[SUBST] + 1 + rng.integers(0, 3, len(SUBST))) % 4
        return r

    k = 0
    for ci, n in enumerate(per_class):
        for i in range(n):
            name = CLASSES[ci]
            if name in ("sub2", "sub1"):
                a, b, t = fr(285_000 + 700 * k, int(rng.integers(200, 400))); k += 1
                a = sub(a)
                if name == "sub2":
                    b = sub(b)
            elif name == "family":
                c = i % COPIES
                a, b, t = fr(starts[c] + 10 + 15 * c, 320)
            elif name == "nowhere":
                a, b, t = rng.integers(0, 4, RL).astype(np.uint8), rng.integers(0, 4, RL).astype(np.uint8), (-1, -1)
            else:
                ln2 = int(rng.integers(14, RL)) if name == "short" else RL
                p = int(rng.integers(0, 280_000 - 500))
                a, b, t = fr(p, int(rng.integers(200, 400)), ln2)
                if name == "mutated":
                    for r in (a, b):
                        mm = rng.random(len(r)) < 0.06
                        r[mm] = (r[mm] + 1) % 4
                if name == "swapped":
                    a, b, t = b, a, (t[1], t[0])
            m1.append(a); m2.append(b); cls.append(ci); truth.append(t)
    return g, m1 + m2, np.array(cls), np.array(truth, np.int64)
