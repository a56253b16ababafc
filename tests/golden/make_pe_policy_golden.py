"""Generate tests/golden/pe_policy.npz by RUNNING THE REFERENCE ITSELF: nvBowtie's own frame_opposite_mate
(nvBowtie/bowtie2/cuda/alignment_utils.h:61-98), compiled from an nvbio source tree by oracle/ref_pe_policy.mk into
oracle/_ref/libnvbio_ref_pe_policy.so, on all 16 inputs (4 policies x 2 anchors x 2 anchor orientations).

Run in the dev container only (needs the nvbio tree to have built oracle/_ref):
    make -C oracle -f ref_pe_policy.mk && python tests/golden/make_pe_policy_golden.py
"""
import os
import sys
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

OUT = os.path.dirname(os.path.abspath(__file__))


def inputs():
    """(policy in io::PE_POLICY_* numbering: FF 0, FR 1, RF 2, RR 3; anchor; anchor_fw) of all 16 inputs"""
    g = np.array([(pol, a, fw) for pol in range(4) for a in range(2) for fw in range(2)], np.int64)
    return g[:, 0].astype(np.int32), g[:, 1].astype(np.uint32), g[:, 2].astype(np.uint8)


def main():
    from oracle.ref_pe_policy import RefPePolicy
    policy, anchor, anchor_fw = inputs()
    left, fw = RefPePolicy().frame(policy, anchor, anchor_fw)
    np.savez_compressed(os.path.join(OUT, "pe_policy.npz"), policy=policy, anchor=anchor, anchor_fw=anchor_fw, left=left, fw=fw)
    print("pe_policy.npz: %d inputs" % len(policy))


if __name__ == "__main__":
    main()
