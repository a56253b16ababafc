"""ctypes binding of the TEST-ONLY BAI checkers built by ref_bai.mk: htslib's bam_index_build and region queries through a given .bai
(oracle/_ref/libnvbio_ref_bai.so, ref_bai.c).  Test infrastructure like orc.py: only tests/ may import it."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(_HERE, "_ref", "libnvbio_ref_bai.so")


class RefBai:
    @staticmethod
    def available():
        return os.path.exists(LIB)

    def __init__(self):
        self.lib = C.CDLL(LIB)
        self.lib.ref_bam_index.restype = C.c_int
        self.lib.ref_bam_query.restype = C.c_longlong

    def index(self, path: str) -> bytes:
        """htslib's bam_index_build of a .bam file: writes path + ".bai" and returns its bytes"""
        r = self.lib.ref_bam_index(path.encode())
        if r != 0:
            raise ValueError("htslib could not index %s (%d)" % (path, r))
        with open(path + ".bai", "rb") as f:
            return f.read()

    def query(self, path: str, tid: int, beg: int, end: int, cap: int = 1 << 24):
        """the SAM lines of the records a region query [beg, end) on tid through path + ".bai" yields"""
        out = C.create_string_buffer(cap)
        n = self.lib.ref_bam_query(path.encode(), C.c_int(tid), C.c_int(beg), C.c_int(end), out, C.c_ulonglong(cap))
        if n < 0:
            raise ValueError("htslib region query on %s failed (%d)" % (path, n))
        return out.value.decode().splitlines()
