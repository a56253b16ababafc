"""ctypes bindings for the TEST-ONLY checkers under oracle/.

  * ``Oracle``  -> oracle/liboracle.so      (plain-C restatement, nvb_oracle.c)
  * ``Ref``     -> oracle/_ref/libnvbio_ref.so (the unmodified reference templates, ref_shim.cpp)

Both expose the same numpy-level API so tests can pin one against the other.
This module is test infrastructure: only tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / ``--impl reference`` legs may import it.  The product never does.
"""
import ctypes as C
import os
import subprocess
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))

GLOBAL, LOCAL, SEMI_GLOBAL = 0, 1, 2   # nvbio/alignment/alignment_base.h:54


def _p(a, ty=None):
    if a is None:
        return None
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(C.c_void_p)


def seq_words(n):
    """BWT words, rounded up to whole 64-symbol blocks (4 words) as the loader requires
    (nvbio/io/fmindex/fmindex_impl.cu:289-303)."""
    return ((n + 63) // 64) * 4


class _Index(dict):
    __getattr__ = dict.__getitem__


class _Base:
    def _interleave(self, n, bwt, occ, cnt):
        sw = seq_words(n)
        bwt_occ = np.zeros(2 * sw, dtype=np.uint32)
        b = bwt_occ.reshape(-1, 8)
        b[:, 0:4] = bwt.reshape(-1, 4)
        b[:, 4:8] = occ.reshape(-1, 4)
        L2 = np.zeros(5, dtype=np.uint32)
        L2[1:] = np.cumsum(cnt.astype(np.uint64)).astype(np.uint32)
        return bwt_occ, L2


class Oracle(_Base):
    kind = "port"

    def __init__(self):
        path = os.path.join(_HERE, "liboracle.so")
        if not os.path.exists(path):
            subprocess.check_call(["make", "-C", _HERE, "liboracle.so"])
        self.lib = C.CDLL(path)
        self.lib.orc_match.restype = C.c_uint64
        self.lib.orc_match_from.restype = C.c_uint64
        self.lib.orc_locate.restype = C.c_uint64
        self.lib.orc_bwt_from_sa.restype = C.c_uint32
        self.lib.orc_dict_rank.restype = C.c_uint32

    def build_index(self, text):
        text = np.ascontiguousarray(text, dtype=np.uint8)
        n = len(text)
        sa = np.zeros(n + 1, dtype=np.int32)
        self.lib.orc_suffix_array(C.c_uint32(n), _p(text), _p(sa))
        return self.index_from_sa(text, sa)

    def index_from_sa(self, text, sa):
        n = len(text)
        sw = seq_words(n)
        bwt = np.zeros(sw, dtype=np.uint32)
        primary = self.lib.orc_bwt_from_sa(C.c_uint32(n), _p(text), _p(sa), _p(bwt), C.c_uint32(sw))
        occ = np.zeros(sw, dtype=np.uint32)
        cnt = np.zeros(4, dtype=np.uint32)
        self.lib.orc_build_occ(C.c_uint32(n), _p(bwt), _p(occ), _p(cnt))
        bwt_occ = np.zeros(2 * sw, dtype=np.uint32)
        L2 = np.zeros(5, dtype=np.uint32)
        self.lib.orc_interleave(C.c_uint32(sw), _p(bwt), _p(occ), _p(cnt), _p(bwt_occ), _p(L2))
        ssa = np.zeros((n + 16) // 16, dtype=np.uint32)
        self.lib.orc_build_ssa(C.c_uint32(n), _p(sa), _p(ssa))
        return _Index(n=n, primary=int(primary), sa=sa, bwt=bwt, occ=occ, bwt_occ=bwt_occ, L2=L2, ssa=ssa)

    def count_table(self):
        t = np.zeros(256, dtype=np.uint32)
        self.lib.orc_count_table(_p(t))
        return t

    def rank(self, idx, k, c):
        k = np.ascontiguousarray(k, dtype=np.uint32)
        c = np.ascontiguousarray(c, dtype=np.uint8)
        out = np.zeros(len(k), dtype=np.uint32)
        self.lib.orc_rank(_p(idx.bwt_occ), _p(idx.L2), C.c_uint32(idx.n), C.c_uint32(idx.primary),
                          _p(k), _p(c), C.c_uint32(len(k)), _p(out))
        return out

    def dict_rank(self, idx, i, c):
        return np.array([self.lib.orc_dict_rank(_p(idx.bwt_occ), C.c_uint32(int(a)), C.c_uint32(int(b)))
                         for a, b in zip(i, c)], dtype=np.uint32)

    def match(self, idx, q, off, ln, blocks_from_step=0):
        """returns (ranges[nq,2] inclusive, total 32-byte blocks touched by LF steps >= blocks_from_step)"""
        q = np.ascontiguousarray(q, dtype=np.uint8)
        off = np.ascontiguousarray(off, dtype=np.uint32)
        ln = np.ascontiguousarray(ln, dtype=np.uint32)
        out = np.zeros((len(off), 2), dtype=np.uint32)
        blocks = self.lib.orc_match_from(_p(idx.bwt_occ), _p(idx.L2), C.c_uint32(idx.n), C.c_uint32(idx.primary),
                                         _p(q), _p(off), _p(ln), C.c_uint32(len(off)), _p(out), C.c_uint32(blocks_from_step))
        return out, int(blocks)

    def locate(self, idx, rows):
        rows = np.ascontiguousarray(rows, dtype=np.uint32)
        out = np.zeros(len(rows), dtype=np.uint32)
        steps = self.lib.orc_locate(_p(idx.bwt_occ), _p(idx.ssa), _p(idx.L2), C.c_uint32(idx.n),
                                    C.c_uint32(idx.primary), _p(rows), C.c_uint32(len(rows)), _p(out))
        self.last_locate_steps = int(steps)
        return out

    def banded_gotoh_best2(self, band, typ, scheme, pat, p_off, p_len, txt, t_off, t_len, distinct_dist=0):
        """the plain-C banded DP feeding a restated aln::Best2Sink<int32>: int64 [n, 6]"""
        pat = np.ascontiguousarray(pat, dtype=np.uint8); txt = np.ascontiguousarray(txt, dtype=np.uint8)
        p_off = np.ascontiguousarray(p_off, dtype=np.uint32); p_len = np.ascontiguousarray(p_len, dtype=np.uint32)
        t_off = np.ascontiguousarray(t_off, dtype=np.uint32); t_len = np.ascontiguousarray(t_len, dtype=np.uint32)
        if len(scheme) == 4:
            scheme = (scheme[0], scheme[1], scheme[2], scheme[3], scheme[2], scheme[3])
        s6 = np.array(scheme, dtype=np.int32)
        out = np.zeros((len(p_off), 6), dtype=np.int64)
        self.lib.orc_banded_gotoh_best2(C.c_int(band), C.c_int(typ), _p(s6), _p(pat), _p(p_off), _p(p_len), _p(txt), _p(t_off), _p(t_len),
                                        C.c_uint32(len(p_off)), C.c_uint32(distinct_dist), _p(out))
        return out

    def banded_gotoh(self, band, typ, scheme, pat, p_off, p_len, txt, t_off, t_len, qual=None, qtab=None):
        """scheme = (match, mismatch, gap_open, gap_ext) or a 6-tuple
        (match, mismatch, pattern_gap_open, pattern_gap_ext, text_gap_open, text_gap_ext)."""
        if len(scheme) == 4:
            scheme = (scheme[0], scheme[1], scheme[2], scheme[3], scheme[2], scheme[3])
        s = np.array(scheme, dtype=np.int32)
        pat = np.ascontiguousarray(pat, dtype=np.uint8)
        txt = np.ascontiguousarray(txt, dtype=np.uint8)
        p_off = np.ascontiguousarray(p_off, dtype=np.uint32)
        p_len = np.ascontiguousarray(p_len, dtype=np.uint32)
        t_off = np.ascontiguousarray(t_off, dtype=np.uint32)
        t_len = np.ascontiguousarray(t_len, dtype=np.uint32)
        n = len(p_off)
        score = np.zeros(n, dtype=np.int32)
        sx = np.zeros(n, dtype=np.uint32)
        sy = np.zeros(n, dtype=np.uint32)
        ok = np.zeros(n, dtype=np.uint8)
        if qual is not None:
            qual = np.ascontiguousarray(qual, dtype=np.uint8)
        if qtab is not None:
            qtab = np.ascontiguousarray(qtab, dtype=np.int32)
        self.lib.orc_banded_gotoh(C.c_int(band), C.c_int(typ), _p(s), _p(qtab),
                                  _p(pat), _p(qual), _p(p_off), _p(p_len),
                                  _p(txt), _p(t_off), _p(t_len), C.c_uint32(n),
                                  _p(score), _p(sx), _p(sy), _p(ok))
        return score, sx, sy, ok


def _oracle_traceback(self, band, typ, scheme, pat, p_off, p_len, txt, t_off, t_len, max_ops=512, qual=None, qtab=None):
    """Oracle.banded_traceback: ops in END->START push order (0 M, 1 I, 2 D), clips = (M - sink.y, source.y); optional per-base
    qualities + 256x2 score table as in banded_gotoh"""
    pat, p_off, p_len, txt, t_off, t_len, n, o = _tb_args(pat, p_off, p_len, txt, t_off, t_len, max_ops)
    s = _scheme6(scheme)
    qual, qtab = _qual_args(qual, qtab)
    self.lib.orc_banded_traceback(C.c_int(band), C.c_int(typ), _p(s), _p(qtab), _p(pat), _p(qual), _p(p_off), _p(p_len), _p(txt), _p(t_off), _p(t_len),
                                  C.c_uint32(n), C.c_uint32(max_ops), _p(o["score"]), _p(o["sink"]), _p(o["source"]), _p(o["ops"]),
                                  _p(o["n_ops"]), _p(o["clips"]))
    return o


def _window_state(n, band):
    return dict(ckpt=np.zeros((n, band, 2), np.int16), score=np.zeros(n, np.int32), sx=np.zeros(n, np.uint32), sy=np.zeros(n, np.uint32),
                alive=np.zeros(n, np.uint8))


def _oracle_window(self, band, typ, scheme, pat, p_off, p_len, txt, t_off, t_len, wb, we, state, min_score=None, qual=None, qtab=None):
    """Oracle.banded_gotoh_window: one [wb, we) pass of the windowed banded score over a batch; `state` (from window_state) carries
    the checkpoints, BestSinks and alive flags between passes"""
    pat = np.ascontiguousarray(pat, dtype=np.uint8); txt = np.ascontiguousarray(txt, dtype=np.uint8)
    p_off = np.ascontiguousarray(p_off, dtype=np.uint32); p_len = np.ascontiguousarray(p_len, dtype=np.uint32)
    t_off = np.ascontiguousarray(t_off, dtype=np.uint32); t_len = np.ascontiguousarray(t_len, dtype=np.uint32)
    if len(scheme) == 4:
        scheme = (scheme[0], scheme[1], scheme[2], scheme[3], scheme[2], scheme[3])
    s = np.array(scheme, dtype=np.int32)
    ms = None if min_score is None else np.ascontiguousarray(min_score, dtype=np.int32)
    if qual is not None:
        qual = np.ascontiguousarray(qual, dtype=np.uint8)
    if qtab is not None:
        qtab = np.ascontiguousarray(qtab, dtype=np.int32)
    self.lib.orc_banded_gotoh_window(C.c_int(band), C.c_int(typ), _p(s), _p(qtab), _p(pat), _p(qual), _p(p_off), _p(p_len),
                                     _p(txt), _p(t_off), _p(t_len), C.c_uint32(len(p_off)), C.c_uint32(wb), C.c_uint32(we), _p(ms),
                                     _p(state["ckpt"]), _p(state["score"]), _p(state["sx"]), _p(state["sy"]), _p(state["alive"]))
    return state


def _oracle_full_traceback(self, typ, scheme, pat, p_off, p_len, txt, t_off, t_len, max_ops=1024, qual=None, qtab=None):
    """Oracle.gotoh_full_traceback: aln::alignment_traceback restated; ops END->START (0 M, 1 I, 2 D); optional qualities + table"""
    pat, p_off, p_len, txt, t_off, t_len, n, o = _tb_args(pat, p_off, p_len, txt, t_off, t_len, max_ops)
    s = _scheme6(scheme)
    qual, qtab = _qual_args(qual, qtab)
    self.lib.orc_gotoh_full_traceback(C.c_int(typ), _p(s), _p(qtab), _p(pat), _p(qual), _p(p_off), _p(p_len), _p(txt), _p(t_off), _p(t_len),
                                      C.c_uint32(n), C.c_uint32(max_ops), _p(o["score"]), _p(o["sink"]), _p(o["source"]), _p(o["ops"]),
                                      _p(o["n_ops"]), _p(o["clips"]))
    return o


def _scheme6(scheme):
    if len(scheme) == 4:
        scheme = (scheme[0], scheme[1], scheme[2], scheme[3], scheme[2], scheme[3])
    return np.array(scheme, dtype=np.int32)


def _qual_args(qual, qtab):
    return (None if qual is None else np.ascontiguousarray(qual, dtype=np.uint8),
            None if qtab is None else np.ascontiguousarray(qtab, dtype=np.int32))


def _tb_args(pat, p_off, p_len, txt, t_off, t_len, max_ops):
    pat = np.ascontiguousarray(pat, dtype=np.uint8); txt = np.ascontiguousarray(txt, dtype=np.uint8)
    p_off = np.ascontiguousarray(p_off, dtype=np.uint32); p_len = np.ascontiguousarray(p_len, dtype=np.uint32)
    t_off = np.ascontiguousarray(t_off, dtype=np.uint32); t_len = np.ascontiguousarray(t_len, dtype=np.uint32)
    n = len(p_off)
    out = dict(score=np.zeros(n, np.int32), sink=np.zeros((n, 2), np.uint32), source=np.zeros((n, 2), np.uint32),
               ops=np.zeros((n, max_ops), np.uint8), n_ops=np.zeros(n, np.uint32), clips=np.zeros((n, 2), np.uint32))
    return pat, p_off, p_len, txt, t_off, t_len, n, out


class Ref(_Base):
    """The reference's own templates (only where oracle/_ref/libnvbio_ref.so exists)."""
    kind = "reference"

    @staticmethod
    def available():
        return os.path.exists(os.path.join(_HERE, "_ref", "libnvbio_ref.so"))

    def __init__(self):
        self.lib = C.CDLL(os.path.join(_HERE, "_ref", "libnvbio_ref.so"))
        self.lib.ref_build_bwt.restype = C.c_uint32
        self.lib.ref_num_threads.restype = C.c_int

    def num_threads(self):
        return int(self.lib.ref_num_threads())

    def set_num_threads(self, t):
        self.lib.ref_set_num_threads(C.c_int(t))

    def build_index(self, text):
        text = np.ascontiguousarray(text, dtype=np.uint8)
        n = len(text)
        sw = seq_words(n)
        sa = np.zeros(n + 1, dtype=np.int32)
        bwt = np.zeros(sw, dtype=np.uint32)
        primary = self.lib.ref_build_bwt(C.c_uint32(n), _p(text), _p(sa), _p(bwt), C.c_uint32(sw))
        occ = np.zeros(sw, dtype=np.uint32)
        cnt = np.zeros(4, dtype=np.uint32)
        self.lib.ref_build_occ(C.c_uint32(n), _p(bwt), _p(occ), _p(cnt))
        bwt_occ, L2 = self._interleave(n, bwt, occ, cnt)
        ssa = np.zeros((n + 16) // 16, dtype=np.uint32)
        self.lib.ref_build_ssa(C.c_uint32(n), _p(sa), _p(ssa))
        return _Index(n=n, primary=int(primary), sa=sa, bwt=bwt, occ=occ, bwt_occ=bwt_occ, L2=L2, ssa=ssa)

    def count_table(self):
        t = np.zeros(256, dtype=np.uint32)
        self.lib.ref_count_table(_p(t))
        return t

    def rank(self, idx, k, c):
        k = np.ascontiguousarray(k, dtype=np.uint32)
        c = np.ascontiguousarray(c, dtype=np.uint8)
        out = np.zeros(len(k), dtype=np.uint32)
        self.lib.ref_rank(_p(idx.bwt_occ), _p(idx.L2), C.c_uint32(idx.n), C.c_uint32(idx.primary),
                          _p(k), _p(c), C.c_uint32(len(k)), _p(out))
        return out

    def dict_rank(self, idx, i, c):
        i = np.ascontiguousarray(i, dtype=np.uint32)
        c = np.ascontiguousarray(c, dtype=np.uint8)
        out = np.zeros(len(i), dtype=np.uint32)
        self.lib.ref_dict_rank(_p(idx.bwt_occ), _p(i), _p(c), C.c_uint32(len(i)), _p(out))
        return out

    def match(self, idx, q, off, ln):
        q = np.ascontiguousarray(q, dtype=np.uint8)
        off = np.ascontiguousarray(off, dtype=np.uint32)
        ln = np.ascontiguousarray(ln, dtype=np.uint32)
        out = np.zeros((len(off), 2), dtype=np.uint32)
        self.lib.ref_match(_p(idx.bwt_occ), _p(idx.L2), C.c_uint32(idx.n), C.c_uint32(idx.primary),
                           _p(q), _p(off), _p(ln), C.c_uint32(len(off)), _p(out))
        return out, None

    def locate(self, idx, rows):
        rows = np.ascontiguousarray(rows, dtype=np.uint32)
        out = np.zeros(len(rows), dtype=np.uint32)
        self.lib.ref_locate(_p(idx.bwt_occ), _p(idx.ssa), _p(idx.L2), C.c_uint32(idx.n),
                            C.c_uint32(idx.primary), _p(rows), C.c_uint32(len(rows)), _p(out))
        return out

    def banded_gotoh_window(self, band, typ, scheme, pat, p_off, p_len, txt, t_off, t_len, wb, we, state, min_score=None):
        """aln::banded_alignment_score<BAND>(..., window_begin, window_end, sink, checkpoint) over a batch (one pass)"""
        pat = np.ascontiguousarray(pat, dtype=np.uint8); txt = np.ascontiguousarray(txt, dtype=np.uint8)
        p_off = np.ascontiguousarray(p_off, dtype=np.uint32); p_len = np.ascontiguousarray(p_len, dtype=np.uint32)
        t_off = np.ascontiguousarray(t_off, dtype=np.uint32); t_len = np.ascontiguousarray(t_len, dtype=np.uint32)
        ms = None if min_score is None else np.ascontiguousarray(min_score, dtype=np.int32)
        r = self.lib.ref_banded_gotoh_window(C.c_int(band), C.c_int(typ), C.c_int(scheme[0]), C.c_int(scheme[1]), C.c_int(scheme[2]), C.c_int(scheme[3]),
                                             _p(pat), _p(p_off), _p(p_len), _p(txt), _p(t_off), _p(t_len), C.c_uint32(len(p_off)),
                                             C.c_uint32(wb), C.c_uint32(we), _p(ms), _p(state["ckpt"]), _p(state["score"]), _p(state["sx"]),
                                             _p(state["sy"]), _p(state["alive"]))
        assert r == 0, r
        return state

    def gotoh_full_traceback(self, typ, scheme, pat, p_off, p_len, txt, t_off, t_len, max_ops=1024):
        """aln::alignment_traceback<256,512,64>: ops in END->START push order (0 M, 1 I, 2 D)"""
        pat, p_off, p_len, txt, t_off, t_len, n, o = _tb_args(pat, p_off, p_len, txt, t_off, t_len, max_ops)
        r = self.lib.ref_gotoh_full_traceback(C.c_int(typ), C.c_int(scheme[0]), C.c_int(scheme[1]), C.c_int(scheme[2]), C.c_int(scheme[3]),
                                              _p(pat), _p(p_off), _p(p_len), _p(txt), _p(t_off), _p(t_len), C.c_uint32(n), C.c_uint32(max_ops),
                                              _p(o["score"]), _p(o["sink"]), _p(o["source"]), _p(o["ops"]), _p(o["n_ops"]), _p(o["clips"]))
        assert r == 0, r
        return o

    def banded_traceback(self, band, typ, scheme, pat, p_off, p_len, txt, t_off, t_len, max_ops=512):
        """aln::banded_alignment_traceback: ops in END->START push order (0 M, 1 I, 2 D)"""
        pat, p_off, p_len, txt, t_off, t_len, n, o = _tb_args(pat, p_off, p_len, txt, t_off, t_len, max_ops)
        r = self.lib.ref_banded_traceback(C.c_int(band), C.c_int(typ), C.c_int(scheme[0]), C.c_int(scheme[1]), C.c_int(scheme[2]), C.c_int(scheme[3]),
                                          _p(pat), _p(p_off), _p(p_len), _p(txt), _p(t_off), _p(t_len), C.c_uint32(n), C.c_uint32(max_ops),
                                          _p(o["score"]), _p(o["sink"]), _p(o["source"]), _p(o["ops"]), _p(o["n_ops"]), _p(o["clips"]))
        assert r == 0
        return o

    def banded_traceback_q(self, band, typ, scheme, pat, p_off, p_len, txt, t_off, t_len, qual, qtab, max_ops=512):
        """aln::banded_alignment_traceback<band,1024,32> with the table-driven scheme (TableGotohScheme in ref_shim.cpp) and per-base
        qualities; scheme as banded_gotoh (only its gap costs are used); bands 7 / 15 / 31"""
        pat, p_off, p_len, txt, t_off, t_len, n, o = _tb_args(pat, p_off, p_len, txt, t_off, t_len, max_ops)
        qual, qtab = _qual_args(qual, qtab)
        r = self.lib.ref_banded_traceback_q(C.c_int(band), C.c_int(typ), _p(_scheme6(scheme)), _p(qtab), _p(pat), _p(qual), _p(p_off), _p(p_len),
                                            _p(txt), _p(t_off), _p(t_len), C.c_uint32(n), C.c_uint32(max_ops),
                                            _p(o["score"]), _p(o["sink"]), _p(o["source"]), _p(o["ops"]), _p(o["n_ops"]), _p(o["clips"]))
        assert r == 0, r
        return o

    def gotoh_full_traceback_q(self, typ, scheme, pat, p_off, p_len, txt, t_off, t_len, qual, qtab, max_ops=1024):
        """aln::alignment_traceback<256,512,64> with the table-driven scheme and per-base qualities"""
        pat, p_off, p_len, txt, t_off, t_len, n, o = _tb_args(pat, p_off, p_len, txt, t_off, t_len, max_ops)
        qual, qtab = _qual_args(qual, qtab)
        r = self.lib.ref_gotoh_full_traceback_q(C.c_int(typ), _p(_scheme6(scheme)), _p(qtab), _p(pat), _p(qual), _p(p_off), _p(p_len),
                                                _p(txt), _p(t_off), _p(t_len), C.c_uint32(n), C.c_uint32(max_ops),
                                                _p(o["score"]), _p(o["sink"]), _p(o["source"]), _p(o["ops"]), _p(o["n_ops"]), _p(o["clips"]))
        assert r == 0, r
        return o

    def generic_rank(self, word_bits, K, text, qi, qc):
        """the reference's generic rank_dictionary (plain big-endian 2-bit PackedStream over 32- / 64-bit words, occ every K symbols;
        rank_dictionary_inl.h:243-422, build_occurrence_table :42-77): returns (words, occ, ranks)"""
        text = np.ascontiguousarray(text, dtype=np.uint8); n = len(text)
        wdt = np.uint32 if word_bits == 32 else np.uint64
        spw = word_bits // 2
        words = np.zeros((n + spw - 1) // spw + 4, dtype=wdt)
        occ = np.zeros(((n + K - 1) // K + 1) * 4, dtype=wdt)
        qi = np.ascontiguousarray(qi, dtype=np.uint64); qc = np.ascontiguousarray(qc, dtype=np.uint8)
        out = np.zeros(len(qi), dtype=np.uint64)
        r = self.lib.ref_generic_rank(C.c_int(word_bits), C.c_uint32(K), C.c_uint64(n), _p(text), _p(words), _p(occ), _p(qi), _p(qc), C.c_uint32(len(qi)), _p(out))
        assert r == 0, (word_bits, K)
        return words, occ[:((n + K - 1) // K) * 4], out

    def banded_gotoh_best2(self, band, typ, scheme, pat, p_off, p_len, txt, t_off, t_len, distinct_dist=0):
        """aln::banded_alignment_score<band> into aln::Best2Sink<int32>(distinct_dist): int64 [n, 6] (bands 7 / 15 / 31)"""
        pat = np.ascontiguousarray(pat, dtype=np.uint8); txt = np.ascontiguousarray(txt, dtype=np.uint8)
        p_off = np.ascontiguousarray(p_off, dtype=np.uint32); p_len = np.ascontiguousarray(p_len, dtype=np.uint32)
        t_off = np.ascontiguousarray(t_off, dtype=np.uint32); t_len = np.ascontiguousarray(t_len, dtype=np.uint32)
        out = np.zeros((len(p_off), 6), dtype=np.int64)
        r = self.lib.ref_banded_gotoh_best2(C.c_int(band), C.c_int(typ), C.c_int(scheme[0]), C.c_int(scheme[1]), C.c_int(scheme[2]), C.c_int(scheme[3]),
                                            _p(pat), _p(p_off), _p(p_len), _p(txt), _p(t_off), _p(t_len), C.c_uint32(len(p_off)), C.c_uint32(distinct_dist), _p(out))
        assert r == 0
        return out

    def nvbowtie_scheme(self, preset=0, match_bonus=0, mm_min=2, mm_max=6, read_gap=(5, 3), ref_gap=(5, 3)):
        """nvBowtie's own SmithWatermanScoringScheme<QualCost<int>,ConstantCost<int>> (scoring.h:203-317), compiled from the reference:
        (table[256,2] = substitution on match / mismatch per base quality, gaps = (pattern open, ext, text open, ext),
        (worst_score, perfect_score(100))).  preset 1 = scheme::local(), 2 = the default-constructed (end-to-end) scheme."""
        tab = np.zeros(512, np.int32); gaps = np.zeros(4, np.int32); lim = np.zeros(2, np.int32)
        self.lib.ref_nvbowtie_scheme(C.c_int(preset), C.c_int(match_bonus), C.c_int(mm_min), C.c_int(mm_max), C.c_int(read_gap[0]), C.c_int(read_gap[1]),
                                     C.c_int(ref_gap[0]), C.c_int(ref_gap[1]), _p(tab), _p(gaps), _p(lim))
        return tab.reshape(256, 2), tuple(int(v) for v in gaps), tuple(int(v) for v in lim)

    def nvbowtie_banded(self, band, typ, pat, qual, p_off, p_len, txt, t_off, t_len, preset=0, match_bonus=0, mm_min=2, mm_max=6,
                        read_gap=(5, 3), ref_gap=(5, 3)):
        """aln::banded_alignment_score<band> with nvBowtie's real scheme object and per-base qualities (band 15 / 31; LOCAL / SEMI_GLOBAL)"""
        pat = np.ascontiguousarray(pat, dtype=np.uint8); txt = np.ascontiguousarray(txt, dtype=np.uint8); qual = np.ascontiguousarray(qual, dtype=np.uint8)
        p_off = np.ascontiguousarray(p_off, dtype=np.uint32); p_len = np.ascontiguousarray(p_len, dtype=np.uint32)
        t_off = np.ascontiguousarray(t_off, dtype=np.uint32); t_len = np.ascontiguousarray(t_len, dtype=np.uint32)
        n = len(p_off)
        score = np.zeros(n, np.int32); sx = np.zeros(n, np.uint32); sy = np.zeros(n, np.uint32)
        r = self.lib.ref_nvbowtie_banded(C.c_int(band), C.c_int(typ), C.c_int(preset), C.c_int(match_bonus), C.c_int(mm_min), C.c_int(mm_max),
                                         C.c_int(read_gap[0]), C.c_int(read_gap[1]), C.c_int(ref_gap[0]), C.c_int(ref_gap[1]),
                                         _p(pat), _p(qual), _p(p_off), _p(p_len), _p(txt), _p(t_off), _p(t_len), C.c_uint32(n), _p(score), _p(sx), _p(sy))
        assert r == 0, r
        return score, sx, sy

    def banded_gotoh(self, band, typ, scheme, pat, p_off, p_len, txt, t_off, t_len, qual=None, qtab=None):
        if qtab is not None:
            # the reference templates with a table-driven scheme (TableGotohScheme in ref_shim.cpp); bands 7 / 15 / 31
            if len(scheme) == 4:
                scheme = (scheme[0], scheme[1], scheme[2], scheme[3], scheme[2], scheme[3])
            s6 = np.array(scheme, dtype=np.int32)
            pat = np.ascontiguousarray(pat, dtype=np.uint8); txt = np.ascontiguousarray(txt, dtype=np.uint8)
            qual = np.ascontiguousarray(qual, dtype=np.uint8); qtab = np.ascontiguousarray(qtab, dtype=np.int32)
            p_off = np.ascontiguousarray(p_off, dtype=np.uint32); p_len = np.ascontiguousarray(p_len, dtype=np.uint32)
            t_off = np.ascontiguousarray(t_off, dtype=np.uint32); t_len = np.ascontiguousarray(t_len, dtype=np.uint32)
            n = len(p_off)
            score = np.zeros(n, np.int32); sx = np.zeros(n, np.uint32); sy = np.zeros(n, np.uint32); ok = np.zeros(n, np.uint8)
            r = self.lib.ref_banded_gotoh_q(C.c_int(band), C.c_int(typ), _p(s6), _p(qtab), _p(pat), _p(qual), _p(p_off), _p(p_len),
                                            _p(txt), _p(t_off), _p(t_len), C.c_uint32(n), _p(score), _p(sx), _p(sy), _p(ok))
            assert r == 0
            return score, sx, sy, ok
        assert qual is None and len(scheme) == 4, "without a table the ref shim instantiates SimpleGotohScheme"
        pat = np.ascontiguousarray(pat, dtype=np.uint8)
        txt = np.ascontiguousarray(txt, dtype=np.uint8)
        p_off = np.ascontiguousarray(p_off, dtype=np.uint32)
        p_len = np.ascontiguousarray(p_len, dtype=np.uint32)
        t_off = np.ascontiguousarray(t_off, dtype=np.uint32)
        t_len = np.ascontiguousarray(t_len, dtype=np.uint32)
        n = len(p_off)
        score = np.zeros(n, dtype=np.int32)
        sx = np.zeros(n, dtype=np.uint32)
        sy = np.zeros(n, dtype=np.uint32)
        ok = np.zeros(n, dtype=np.uint8)
        r = self.lib.ref_banded_gotoh(C.c_int(band), C.c_int(typ), C.c_int(scheme[0]), C.c_int(scheme[1]),
                                      C.c_int(scheme[2]), C.c_int(scheme[3]),
                                      _p(pat), _p(p_off), _p(p_len), _p(txt), _p(t_off), _p(t_len),
                                      C.c_uint32(n), _p(score), _p(sx), _p(sy), _p(ok))
        assert r == 0
        return score, sx, sy, ok


def rle(ops):
    """run-length string of an op array in the given order, letters as TestBacktracker: 0 M, 1 I, 2 D"""
    out, prev, cnt = [], None, 0
    for o in ops:
        if o == prev:
            cnt += 1
        else:
            if prev is not None:
                out.append("%d%s" % (cnt, "MID"[prev]))
            prev, cnt = int(o), 1
    if prev is not None:
        out.append("%d%s" % (cnt, "MID"[prev]))
    return "".join(out)


def dna(s):
    """ASCII ACGT(N) -> symbols 0..3 (4)"""
    lut = np.full(256, 4, dtype=np.uint8)
    for i, ch in enumerate("ACGT"):
        lut[ord(ch)] = i
    return lut[np.frombuffer(s.encode(), dtype=np.uint8)]


Oracle.banded_traceback = _oracle_traceback
Oracle.gotoh_full_traceback = _oracle_full_traceback
Oracle.banded_gotoh_window = _oracle_window
window_state = _window_state


def _full_args(pat, p_off, p_len, txt, t_off, t_len):
    pat = np.ascontiguousarray(pat, dtype=np.uint8); txt = np.ascontiguousarray(txt, dtype=np.uint8)
    p_off = np.ascontiguousarray(p_off, dtype=np.uint32); p_len = np.ascontiguousarray(p_len, dtype=np.uint32)
    t_off = np.ascontiguousarray(t_off, dtype=np.uint32); t_len = np.ascontiguousarray(t_len, dtype=np.uint32)
    n = len(p_off)
    return pat, p_off, p_len, txt, t_off, t_len, n, np.zeros(n, np.int32), np.zeros(n, np.uint32), np.zeros(n, np.uint32)


def _oracle_full(self, typ, scheme, pat, p_off, p_len, txt, t_off, t_len, qual=None, qtab=None):
    """full-matrix Gotoh: (score, sink_x = text end, sink_y = pattern end); optional per-base qualities + 256x2 score table"""
    pat, p_off, p_len, txt, t_off, t_len, n, score, sx, sy = _full_args(pat, p_off, p_len, txt, t_off, t_len)
    if len(scheme) == 4:
        scheme = (scheme[0], scheme[1], scheme[2], scheme[3], scheme[2], scheme[3])
    s = np.array(scheme, dtype=np.int32)
    if qual is not None:
        qual = np.ascontiguousarray(qual, dtype=np.uint8)
    if qtab is not None:
        qtab = np.ascontiguousarray(qtab, dtype=np.int32)
    self.lib.orc_gotoh_full(C.c_int(typ), _p(s), _p(qtab), _p(pat), _p(qual), _p(p_off), _p(p_len), _p(txt), _p(t_off), _p(t_len), C.c_uint32(n),
                            _p(score), _p(sx), _p(sy))
    return score, sx, sy


def _ref_full_q(self, typ, scheme, pat, p_off, p_len, txt, t_off, t_len, qual, qtab):
    pat, p_off, p_len, txt, t_off, t_len, n, score, sx, sy = _full_args(pat, p_off, p_len, txt, t_off, t_len)
    if len(scheme) == 4:
        scheme = (scheme[0], scheme[1], scheme[2], scheme[3], scheme[2], scheme[3])
    s = np.array(scheme, dtype=np.int32)
    qual = np.ascontiguousarray(qual, dtype=np.uint8); qtab = np.ascontiguousarray(qtab, dtype=np.int32)
    r = self.lib.ref_gotoh_full_q(C.c_int(typ), _p(s), _p(qtab), _p(pat), _p(qual), _p(p_off), _p(p_len), _p(txt), _p(t_off), _p(t_len),
                                  C.c_uint32(n), _p(score), _p(sx), _p(sy))
    assert r == 0
    return score, sx, sy


def _ref_full(self, typ, scheme, pat, p_off, p_len, txt, t_off, t_len, qual=None, qtab=None):
    if qtab is not None:
        return _ref_full_q(self, typ, scheme, pat, p_off, p_len, txt, t_off, t_len, qual, qtab)
    pat, p_off, p_len, txt, t_off, t_len, n, score, sx, sy = _full_args(pat, p_off, p_len, txt, t_off, t_len)
    r = self.lib.ref_gotoh_full(C.c_int(typ), C.c_int(scheme[0]), C.c_int(scheme[1]), C.c_int(scheme[2]), C.c_int(scheme[3]),
                                _p(pat), _p(p_off), _p(p_len), _p(txt), _p(t_off), _p(t_len), C.c_uint32(n), _p(score), _p(sx), _p(sy))
    assert r == 0
    return score, sx, sy


Oracle.gotoh_full = _oracle_full
Ref.gotoh_full = _ref_full


def generic_rank_oracle(text, qi, qc, word_bits, K):
    """plain restatement of the generic rank dictionary (test infrastructure): words = text packed big-endian into word_bits-wide words,
    occ[4k + c] = #c in text[0, kK), rank(i, c) = #c in text[0, i] (i = all ones -> 0)"""
    text = np.asarray(text, dtype=np.uint8); n = len(text)
    spw = word_bits // 2
    wdt = np.uint32 if word_bits == 32 else np.uint64
    pad = np.zeros((-n) % spw, np.uint8)
    t = np.concatenate([text, pad]).reshape(-1, spw).astype(np.uint64)
    sh = (word_bits - 2 - 2 * np.arange(spw)).astype(np.uint64)
    words = np.bitwise_or.reduce(t << sh, axis=1).astype(wdt)
    onehot = (text[:, None] == np.arange(4)[None, :]).astype(np.uint64)
    pref = np.concatenate([np.zeros((1, 4), np.uint64), np.cumsum(onehot, axis=0)])          # pref[i] = counts in text[0, i)
    n_blocks = (n + K - 1) // K
    occ = pref[np.arange(n_blocks) * K].reshape(-1).astype(wdt)
    qi = np.asarray(qi, dtype=np.uint64)
    allones = qi == np.uint64(0xFFFFFFFFFFFFFFFF)
    idx = np.where(allones, 0, qi).astype(np.int64)
    ranks = np.where(allones, 0, pref[idx + 1, np.asarray(qc, dtype=np.int64)]).astype(np.uint64)
    return words, occ, ranks
