"""ctypes binding of the TEST-ONLY BAM checkers built by ref_bam.mk: htslib's sam_parse1 + bam_write1, sam_format1 and hts_reg2bin
(oracle/_ref/libnvbio_ref_bam.so, ref_bam.c) and nvbio's save_bns (oracle/_ref/libnvbio_ref_bns.so, ref_bns.cpp).  Test infrastructure
like orc.py: only tests/ may import it."""
import ctypes as C
import os
import tempfile
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(_HERE, "_ref", "libnvbio_ref_bam.so")
BNS_LIB = os.path.join(_HERE, "_ref", "libnvbio_ref_bns.so")


class RefBam:
    @staticmethod
    def available():
        return os.path.exists(LIB)

    def __init__(self):
        self.lib = C.CDLL(LIB)
        self.lib.ref_bam_encode.restype = C.c_longlong
        self.lib.ref_bam_format.restype = C.c_longlong
        self.lib.ref_reg2bin.restype = C.c_int

    def encode(self, header_text: str, lines):
        """htslib's BAM bytes of each SAM line (block_size included), as a list of bytes objects"""
        if not lines:
            return []
        body = "\n".join(lines).encode()
        cap = 4 * len(body) + 64 * len(lines) + 1024
        out = np.zeros(cap, np.uint8)
        with tempfile.TemporaryDirectory() as d:
            n = self.lib.ref_bam_encode(header_text.encode(), body, os.path.join(d, "r.bam").encode(), out.ctypes.data_as(C.c_void_p),
                                        C.c_ulonglong(cap))
        if n < 0:
            raise ValueError("htslib rejected SAM line %d: %r" % (-1 - n, lines[-1 - n]) if n > -100000 else "htslib I/O failure")
        raw, recs, o = out[:n].tobytes(), [], 0
        while o < len(raw):
            k = int.from_bytes(raw[o:o + 4], "little") + 4
            recs.append(raw[o:o + k]); o += k
        return recs

    def format(self, path: str, cap: int = 1 << 26) -> str:
        """the SAM text sam_format1 gives for every record of a .bam file, one line each"""
        out = C.create_string_buffer(cap)
        n = self.lib.ref_bam_format(path.encode(), out, C.c_ulonglong(cap))
        if n < 0:
            raise ValueError("htslib could not read %s (%d)" % (path, n))
        return out.value.decode()

    def reg2bin(self, beg: int, end: int) -> int:
        return self.lib.ref_reg2bin(C.c_longlong(beg), C.c_longlong(end))


def save_bns(prefix: str, names, annos, offsets, lengths, gis, l_pac: int, seed: int = 11):
    """nvbio's own save_bns: writes <prefix>.ann / <prefix>.amb"""
    lib = C.CDLL(BNS_LIB)
    n = len(names)
    r = lib.ref_save_bns(prefix.encode(), C.c_int(n), "\n".join(names).encode(), "\n".join(annos).encode(),
                         np.ascontiguousarray(offsets, np.int64).ctypes.data_as(C.c_void_p),
                         np.ascontiguousarray(lengths, np.int32).ctypes.data_as(C.c_void_p),
                         np.ascontiguousarray(gis, np.uint32).ctypes.data_as(C.c_void_p), C.c_longlong(l_pac), C.c_uint(seed))
    if r != 0:
        raise IOError("save_bns failed for %s" % prefix)
