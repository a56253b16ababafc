"""CPU: paired BAM records under every pair flag, discordant (8) included, and mates laid out as every pairing policy places them.
nvb_bam_records' per-record routines (bam_core.cuh, built for the host by tests/host/bam_harness.cu) against tests/bam_oracle.py byte
for byte, and against htslib's encoding of the oracle's SAM lines where oracle/_ref is built:

  * traced and finished pairs (test_bam_host.traced_inputs) with pair flags drawn from {0, 1, 2, 4, 8};
  * hand-built pairs: FR, RF (the reverse mate left of the forward one), FF and RR (both mates on one strand, either mate left), equal
    begins on equal and on opposite strands, mates of unequal length, mates on different contigs, one mate unaligned and one mate off
    its contig, each under every pair flag.

FLAG 0x2 (proper pair) is set only on concordant and rescued pairs (1, 2, 4) whose two mates are placed; a discordant pair's records
carry 0x1, 0x40 / 0x80, 0x20 and the mate fields, never 0x2."""
import struct
import numpy as np
import pytest
from oracle.ref_bam import RefBam
from tests import bam_oracle as bo
from tests.golden.make_bam_golden import fixture_inputs
from tests.test_bam_host import H, HF, genome, run_host, check_against_oracle, traced_inputs, LIVE   # noqa: F401 (fixtures)

PROPER = (1, 2, 4)
FLAGS = (0, 1, 2, 4, 8)


def live_encode(inp, want):
    if LIVE:
        hdr = bo.header_text(inp["contig_names"], inp["contig_lengths"])
        assert RefBam().encode(hdr, [s for _, s in want]) == [w for w, _ in want]


def fields(rec):
    """(flag, refID, pos, next refID, next pos, tlen) of one BAM record's fixed part"""
    ref, pos, _, flag_nc, _, nref, npos, tlen = struct.unpack("<iiIIiiii", rec[4:36])
    return flag_nc >> 16, ref, pos, nref, npos, tlen


@pytest.mark.parametrize("bits", [2, 4])
def test_traced_pairs_every_flag(H, HF, genome, bits):
    """traced pairs with discordant flags among the draws: the routine equals the oracle, and a discordant pair with both mates placed
    has neither record marked proper"""
    rng = np.random.default_rng(800 + bits)
    seen = dict(discordant=0, proper=0, improper=0)
    for i, (typ, band) in enumerate([(1, 31), (2, 15), (0, 63)]):
        inp = traced_inputs(HF, rng, genome, bits, True, band=band, typ=typ, quals=i % 2 == 0, mapq=i != 2)
        inp["pair_flags"] = rng.choice(FLAGS, len(inp["n_ops"]) // 2).astype(np.uint32)
        want, _ = check_against_oracle(H, inp, bits)
        live_encode(inp, want)
        for p, pf in enumerate(inp["pair_flags"]):
            f = [fields(want[2 * p + m][0])[0] for m in (0, 1)]
            if any(x & 0xC for x in f):
                continue
            proper = [bool(x & 0x2) for x in f]
            assert proper == [int(pf) in PROPER] * 2, (p, pf, f)
            seen["discordant" if pf == 8 else ("proper" if pf in PROPER else "improper")] += 1
    assert min(seen.values()) >= 10, seen


# ---- hand-built pairs --------------------------------------------------------------------------------------------------------------------

def layouts(cb):
    """(name, mate 1, mate 2) with a mate (global begin, strand, length) or None for an unaligned mate; cb: the contig begins"""
    c3 = int(cb[2])
    return [("fr", (1_000, 0, 100), (1_250, 1, 80)),
            ("rf", (1_000, 1, 100), (1_300, 0, 100)),                   # the reverse mate left of the forward one
            ("rf_swapped", (1_300, 0, 90), (1_000, 1, 110)),
            ("ff", (2_000, 0, 100), (2_250, 0, 100)),
            ("ff_m2_left", (2_250, 0, 120), (2_000, 0, 60)),
            ("rr", (3_000, 1, 100), (3_400, 1, 100)),
            ("rr_m2_left", (3_400, 1, 50), (3_000, 1, 150)),
            ("equal_same_strand", (5_000, 0, 100), (5_000, 0, 100)),
            ("equal_opposite", (5_000, 1, 100), (5_000, 0, 70)),       # equal begins, unequal lengths: TLEN from the longer mate
            ("contigs", (100, 0, 100), (c3 + 500, 1, 100)),           # chr1 and c3
            ("contigs_rr", (c3 + 500, 1, 100), (100, 1, 100)),
            ("mate2_unaligned", (7_000, 1, 100), None),
            ("mate1_unaligned", None, (7_000, 0, 100)),
            ("mate2_off_contig", (39_500, 0, 100), (int(cb[1]) - 40, 1, 100))]   # mate 2 runs 60 bases past chr1's end


def hand_inputs():
    """every layout under every pair flag, pairs in layout-major order"""
    L = layouts(fixture_inputs(True, 5, n=2)["contig_begin"])
    cases = [(nm, m1, m2, pf) for nm, m1, m2 in L for pf in FLAGS]
    h = len(cases)
    inp = fixture_inputs(True, 5, n=2 * h)
    inp["quals"] = None
    for p, (_, m1, m2, pf) in enumerate(cases):
        inp["pair_flags"][p] = pf
        for a, m in ((p, m1), (h + p, m2)):
            ln = 100 if m is None else m[2]
            inp["reads"][a] = np.arange(ln, dtype=np.uint8) % 4
            inp["n_ops"][a] = 0 if m is None else ln
            inp["n_cigar"][a] = 1; inp["cigar"][a] = 0; inp["cigar"][a, 0] = ln << 4
            md = str(ln).encode()
            inp["md_len"][a] = len(md); inp["md"][a] = 0; inp["md"][a, :len(md)] = np.frombuffer(md, np.uint8)
            inp["edits"][a] = (0, 0, 0, 0)
            inp["begin"][a] = (0, 0) if m is None else (m[0], 0)
            inp["strand"][a] = 0 if m is None else m[1]
    return inp, cases


def test_hand_built_layouts(H):
    inp, cases = hand_inputs()
    want, cnt = check_against_oracle(H, inp, 2)
    live_encode(inp, want)
    cb = inp["contig_begin"]
    got, _, _, _ = run_host(H, inp, 2)
    seen = set()
    for p, (nm, m1, m2, pf) in enumerate(cases):
        placed = [m is not None and not (k == 1 and nm.endswith("off_contig")) for k, m in enumerate((m1, m2))]
        for k, (me, mate) in enumerate(((m1, m2), (m2, m1))):
            flag, ref, pos, nref, npos, tlen = fields(got[2 * p + k])
            assert flag & 0x1 and flag & (0x80 if k else 0x40), (nm, pf, k, flag)
            both = placed[0] and placed[1]
            assert bool(flag & 0x2) == (both and pf in PROPER), (nm, pf, k, flag)
            assert bool(flag & 0x4) == (not placed[k]) and bool(flag & 0x8) == (not placed[1 - k]), (nm, pf, k, flag)
            assert bool(flag & 0x20) == (placed[1 - k] and mate[1] == 1), (nm, pf, k, flag)
            if not both:
                assert tlen == 0, (nm, pf, k)
                continue
            r_me, r_mate = [int(np.searchsorted(cb, x[0], side="right")) - 1 for x in (me, mate)]
            assert (ref, pos, nref, npos) == (r_me, me[0] - int(cb[r_me]), r_mate, mate[0] - int(cb[r_mate])), (nm, pf, k)
            if r_me != r_mate:
                assert tlen == 0, (nm, pf, k)
                seen.add("contigs")
                continue
            span = max(me[0] + me[2], mate[0] + mate[2]) - min(me[0], mate[0])
            first = me[0] < mate[0] or (me[0] == mate[0] and k == 0)     # the leftmost mate, mate 1 on equal begins
            assert tlen == (span if first else -span), (nm, pf, k, tlen, span)
            seen.add("equal" if me[0] == mate[0] else ("same_strand" if me[1] == mate[1] else "opposite"))
            if pf == 8:
                seen.add("discordant")
    assert seen == {"contigs", "equal", "same_strand", "opposite", "discordant"}, seen
    assert cnt[2] == len(FLAGS)                                       # the off-contig mate 2 under every flag

