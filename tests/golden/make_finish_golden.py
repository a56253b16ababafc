"""Generate tests/golden/finish.npz by RUNNING THE REFERENCE ITSELF: nvbio's own io::analyze_md_string, count_symbols and
reference_cigar_length (nvbio/io/output/output_utils.h:42-121), compiled from an nvbio source tree by oracle/ref_finish.mk into
oracle/_ref/libnvbio_ref_finish.so, on the MDS vectors tests/finish_oracle.py restates from nvBowtie's finish_alignment_kernel
(traceback_inl.h:584-674) and on nvBowtie's io::Cigar runs of the same alignments.

Run in the dev container only (needs the nvbio tree to have built oracle/_ref):
    make -C oracle -f ref_finish.mk && python tests/golden/make_finish_golden.py

The alignments are fixture_alignments(): seeded scripts of match, mismatch, insertion, deletion and clip runs.  Match stretches stay at
most 255 long and indel runs at most 255: nvBowtie's MDS stores lengths in one byte, and analyze_md_string misreads a match stretch split
over several MDS tokens (it adds the next token's op code instead of its length and then parses that length as an op).
"""
import os
import sys
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

OUT = os.path.dirname(os.path.abspath(__file__))
N_ALIGNMENTS = 1500


def fixture_alignments():
    """(Batch, MDS vectors, io::Cigar (type, length) runs END -> START with soft clips as type 3, ours[i] = (NM, XM, XO, XG, genome span))"""
    from tests import finish_oracle as fo
    from tests.test_finish_host import Batch, build_case
    rng = np.random.default_rng(2024)
    genome = rng.integers(0, 4, 50_000).astype(np.uint8)
    b = Batch(genome, max_ops=1300)
    for _ in range(N_ALIGNMENTS):
        script = []
        if rng.random() < 0.5:
            script.append(("S", int(rng.integers(1, 20))))
        for _ in range(int(rng.integers(1, 12))):
            t = rng.choice(["M", "M", "X", "X", "I", "D"])
            if t == "M" and script and script[-1][0] == "M":
                t = "X"                                   # keeps every match stretch below 120
            script.append((str(t), int(rng.integers(1, 120)) if t == "M" else int(rng.integers(1, 4)) if t == "X" else int(rng.integers(1, 9))))
        if rng.random() < 0.5:
            script.append(("S", int(rng.integers(1, 20))))
        strand = int(rng.integers(0, 2))
        x = int(rng.integers(0, len(genome) - 2000))
        r, ops, beg = build_case(rng, genome, len(genome), x, script, strand)
        b.add(r, strand, ops, beg)
    mds, cig, ours = [], [], []
    for a in range(len(b)):
        cigar, md, ed = fo.finish(b.ops[a], b.n_ops[a], b.max_ops, b.begin[a], b.strand[a], b.reads[a], genome, len(genome))
        mds.append(fo.mds_vector(b.ops[a], b.n_ops[a], b.begin[a], b.strand[a], b.reads[a], genome, len(genome)))
        runs = [(3 if op == 4 else op, k) for k, op in cigar][::-1]           # io::Cigar types: 0 M, 1 I, 2 D, 3 S; stored END -> START
        cig.append(np.array(runs, np.uint16).reshape(-1, 2))
        ours.append(ed + (sum(k for k, op in cigar if op in (0, 2)),))
    return b, mds, cig, np.array(ours, np.int64)


def offsets(parts):
    return np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.uint64)


def main():
    from oracle.ref_finish import RefFinish
    assert RefFinish.available(), "build oracle/_ref first: make -C oracle -f ref_finish.mk"
    _, mds, cig, ours = fixture_alignments()
    out = dict(mds=np.concatenate(mds), mds_off=offsets(mds), cigar=np.concatenate(cig), cigar_off=offsets(cig))
    out["ref"] = RefFinish().analyze(out["mds"], out["mds_off"], out["cigar"], out["cigar_off"])
    assert np.array_equal(out["ref"][:, 0:3], ours[:, 1:4]), "the reference's XM / XO / XG differ from the restatement's"
    np.savez_compressed(os.path.join(OUT, "finish.npz"), **out)
    print("wrote finish.npz: %d alignments" % len(mds))


if __name__ == "__main__":
    main()
