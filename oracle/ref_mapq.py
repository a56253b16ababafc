"""ctypes binding of the TEST-ONLY MAPQ checker oracle/_ref/libnvbio_ref_mapq.so (ref_mapq.cpp, built by ref_mapq.mk): nvBowtie's own
BowtieMapq2 and SimpleFunc.  Test infrastructure like orc.py: only tests/ may import it.  The product never does."""
import ctypes as C
import os
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(_HERE, "_ref", "libnvbio_ref_mapq.so")


def _p(a):
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(C.c_void_p)


class RefMapq:
    @staticmethod
    def available():
        return os.path.exists(LIB)

    def __init__(self):
        self.lib = C.CDLL(LIB)

    def mapq(self, best, has_second, second, length, match_bonus, min_score):
        """BowtieMapq2 (mapq.h:142-331) of unpaired reads over arrays (broadcast to one length): uint8 MAPQ per point"""
        a = np.broadcast_arrays(np.asarray(best), np.asarray(has_second), np.asarray(second), np.asarray(length), np.asarray(match_bonus),
                                np.asarray(min_score))
        best, has, sec, ln, mb, ms = [np.ascontiguousarray(v, dtype=t).reshape(-1) for v, t in
                                      zip(a, (np.int32, np.uint8, np.int32, np.uint32, np.int32, np.int32))]
        out = np.zeros(len(best), np.uint8)
        self.lib.ref_nvbowtie_mapq(_p(best), _p(has), _p(sec), _p(ln), _p(mb), _p(ms), C.c_uint32(len(best)), _p(out))
        return out

    def simple_func(self, kind, const, coeff, x):
        """SimpleFunc (func.h:39-51), kind 'L' / 'G' / 'S' (linear / log / sqrt): int32 f(x) per point"""
        x = np.ascontiguousarray(x, dtype=np.int32).reshape(-1)
        out = np.zeros(len(x), np.int32)
        self.lib.ref_nvbowtie_simple_func(C.c_int("LGS".index(kind)), C.c_float(const), C.c_float(coeff), _p(x), C.c_uint32(len(x)), _p(out))
        return out
