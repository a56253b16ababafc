"""ctypes binding of the TEST-ONLY paired-end framing checker oracle/_ref/libnvbio_ref_pe_policy.so (ref_pe_policy.cpp, built by
ref_pe_policy.mk): nvBowtie's own frame_opposite_mate.  Test infrastructure like orc.py: only tests/ may import it.  The product never
does."""
import ctypes as C
import os
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(_HERE, "_ref", "libnvbio_ref_pe_policy.so")


def _p(a):
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(C.c_void_p)


class RefPePolicy:
    @staticmethod
    def available():
        return os.path.exists(LIB)

    def __init__(self):
        self.lib = C.CDLL(LIB)

    def frame(self, policy, anchor, anchor_fw):
        """frame_opposite_mate over arrays (io::PE_POLICY_* numbering): (left, fw) uint8 per point"""
        policy = np.ascontiguousarray(policy, np.int32).reshape(-1)
        anchor = np.ascontiguousarray(anchor, np.uint32).reshape(-1)
        anchor_fw = np.ascontiguousarray(anchor_fw, np.uint8).reshape(-1)
        left, fw = np.zeros(len(policy), np.uint8), np.zeros(len(policy), np.uint8)
        self.lib.ref_frame_opposite_mate(_p(policy), _p(anchor), _p(anchor_fw), C.c_uint32(len(policy)), _p(left), _p(fw))
        return left, fw
