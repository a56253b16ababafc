"""CPU: the composed oracle of nvb_seed_extend_paired_reseed (tests/paired_reseed_oracle.py) against the pinned pieces it is built from:
at max_reseed 0 it is seed_extend_paired_oracle / pair_mapq_oracle output for output; with rounds its flags are the mates' range
statistics under nvb_map_seeds' rule without the alignment term; and a pair's outputs depend only on its own two mates."""
import numpy as np
import pytest
from oracle import orc
from nvbio_b200 import aln
from nvbio_b200.pipeline import SeedExtendParams, PairParams, simple_func
from tests.paired_reseed_oracle import seed_extend_paired_reseed_oracle, planted_pairs, RL, L, I
from tests.reseed_oracle import seed_extend_reseed_oracle
from tests.pipeline_oracle import seed_extend_paired_oracle
from tests.pair_mapq_oracle import pair_mapq_oracle

REP = 8
BIG = 10**9
PAIR = PairParams(min_frag=0, max_frag=500, min_mate_score=60)
PAIR_KEYS = ("pair_score", "pair_flags", "mate_score", "mate_pos", "mate_strand")
MAPQ_KEYS = ("second_pair_score", "second_mate_pos", "second_mate_strand", "mate_second_score", "mate_mapq")


@pytest.fixture(scope="module")
def world():
    O = orc.Oracle()
    g, reads, cls, truth = planted_pairs(per_class=(6, 6, 16, 10, 6, 4, 6, 2))
    return dict(O=O, g=g, idx=O.build_index(g), reads=reads, n_pairs=len(reads) // 2,
                min_score=simple_func("G", 0.0, 10.0, np.arange(RL + 1)))


def params():
    return SeedExtendParams(seed_len=L, seed_interval=I, band_len=15, type=aln.LOCAL, both_strands=True, max_seed_hits=4,
                            scheme=aln.SimpleGotohScheme(2, -2, -5, -3))


def composed(w, max_reseed, reads=None, mapq=True):
    reads = w["reads"] if reads is None else reads
    return seed_extend_paired_reseed_oracle(w["O"], w["idx"], w["g"], reads, params(), PAIR, len(reads) // 2, max_reseed, REP, BIG,
                                            min_score=w["min_score"] if mapq else None, match_bonus=2 if mapq else None)


def test_max_reseed_zero_is_the_paired_oracles(world):
    w = world
    n = w["n_pairs"]
    pe = seed_extend_paired_oracle(w["O"], w["idx"], w["g"], w["reads"], params(), PAIR, n)
    got = composed(w, 0, mapq=False)
    for k in PAIR_KEYS + ("n_rescue",):
        assert np.array_equal(np.asarray(got[k]), np.asarray(pe[k])), k
    pm = pair_mapq_oracle(w["O"], w["idx"], w["g"], w["reads"], params(), PAIR, n, w["min_score"], 2)
    got = composed(w, 0)
    for k in PAIR_KEYS + MAPQ_KEYS + ("n_rescue",):
        assert np.array_equal(np.asarray(got[k]), np.asarray(pm[k])), k
    assert (got["rounds"] == 1).all() and got["active"].tolist() == [2 * n]
    # the composition leaves the pinned oracles' names as they were
    from tests import reseed_oracle, pipeline_oracle, pair_mapq_oracle as pmo
    assert reseed_oracle.reseed_flag.__module__ == "tests.reseed_oracle"
    assert pipeline_oracle.seed_extend_oracle is pmo.seed_extend_oracle and pmo.seed_extend_oracle.__module__ == "tests.pipeline_oracle"


@pytest.mark.parametrize("max_reseed", [1, 2, 3])
def test_flags_are_the_seed_statistics(world, max_reseed):
    w = world
    got = composed(w, max_reseed)
    single = seed_extend_reseed_oracle(w["O"], w["idx"], w["g"], w["reads"], params(), max_reseed, REP, w["min_score"], BIG)
    assert got["stats"][0] == single["stats"][0]                   # round 0 seeds every mate alike
    for r, flags in enumerate(got["flags"]):
        st = got["stats"][r]
        assert sorted(flags) == sorted(st)
        for m, f in flags.items():
            s, c = st[m]
            assert f == (c == 0 or s >= ((REP * c) & 0xFFFFFFFF)), (r, m)
        assert got["active"][r + 1] == sum(flags.values())
    rounds = got["rounds"].reshape(-1)
    for r in range(max_reseed + 1):
        assert (rounds > r).sum() == got["active"][r]
    assert got["active"][1] > 0


def test_pair_depends_only_on_its_own_mates(world):
    """with the default rescue capacity and no hit cap, every third pair run alone gives what it gets in the whole batch"""
    w = world
    n = w["n_pairs"]
    full = composed(w, 2)
    sub = np.arange(0, n, 3)
    reads = [w["reads"][p] for p in sub] + [w["reads"][n + p] for p in sub]
    part = composed(w, 2, reads)
    for k in PAIR_KEYS + MAPQ_KEYS + ("rounds",):
        a, b = np.asarray(full[k]), np.asarray(part[k])
        assert np.array_equal(a[..., sub], b), k
