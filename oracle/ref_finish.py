"""ctypes binding of the TEST-ONLY finishing checker oracle/_ref/libnvbio_ref_finish.so (ref_finish.cpp, built by ref_finish.mk): nvbio's
own io::analyze_md_string, count_symbols and reference_cigar_length.  Test infrastructure like orc.py: only tests/ may import it."""
import ctypes as C
import os
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(_HERE, "_ref", "libnvbio_ref_finish.so")


def _p(a):
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(C.c_void_p)


class RefFinish:
    @staticmethod
    def available():
        return os.path.exists(LIB)

    def __init__(self):
        self.lib = C.CDLL(LIB)

    def analyze(self, mds, mds_off, cigar, cigar_off):
        """per alignment (n_mm, n_gapo, n_gape, inserted, deleted, reference length): analyze_md_string (output_utils.h:77-121) of MDS
        vector mds[mds_off[i]:mds_off[i + 1]], count_symbols / reference_cigar_length (output_utils.h:42-73) of the io::Cigar (type, length)
        pairs cigar[cigar_off[i]:cigar_off[i + 1]] (END -> START, nvBowtie's storage order)"""
        mds = np.ascontiguousarray(mds, np.uint8); mo = np.ascontiguousarray(mds_off, np.uint64)
        cig = np.ascontiguousarray(cigar, np.uint16).reshape(-1, 2); co = np.ascontiguousarray(cigar_off, np.uint64)
        n = len(mo) - 1
        out = np.zeros((n, 6), np.uint32)
        self.lib.ref_finish_analyze(_p(mds), _p(mo), _p(cig), _p(co), C.c_uint32(n), _p(out))
        return out
