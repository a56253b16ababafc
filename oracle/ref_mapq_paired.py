"""ctypes binding of the TEST-ONLY paired MAPQ checker oracle/_ref/libnvbio_ref_mapq_paired.so (ref_mapq_paired.cpp, built by
ref_mapq_paired.mk): nvBowtie's own BowtieMapq2 on paired alignments.  Test infrastructure like orc.py: only tests/ may import it.  The
product never does."""
import ctypes as C
import os
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(_HERE, "_ref", "libnvbio_ref_mapq_paired.so")


def _p(a):
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(C.c_void_p)


class RefMapqPaired:
    @staticmethod
    def available():
        return os.path.exists(LIB)

    def __init__(self):
        self.lib = C.CDLL(LIB)

    def mapq_paired(self, s1, s2, kind, t1, t2, len1, len2, match_bonus, min1, min2):
        """BowtieMapq2 of paired best alignments (mapq.h:155-170, MapqFunctorPE) over arrays (broadcast to one length): best pair = mate
        scores (s1, s2), second = none (kind 0), paired (kind 1, mate scores t1, t2) or unpaired (kind 2, score t1); uint8 MAPQ per point"""
        a = np.broadcast_arrays(*[np.asarray(v) for v in (s1, s2, kind, t1, t2, len1, len2, match_bonus, min1, min2)])
        cols = [np.ascontiguousarray(v, dtype=t).reshape(-1) for v, t in
                zip(a, (np.int32, np.int32, np.uint8, np.int32, np.int32, np.uint32, np.uint32, np.int32, np.int32, np.int32))]
        out = np.zeros(len(cols[0]), np.uint8)
        self.lib.ref_nvbowtie_mapq_paired(*[_p(c) for c in cols], C.c_uint32(len(out)), _p(out))
        return out
