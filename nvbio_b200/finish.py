"""Finishing traced alignments on the device (nvb_finish_alignments): BAM CIGAR with soft clips, the MD:Z value and NM / XM / XO / XG of
every alignment nvb_seed_extend_traceback / nvb_seed_extend_paired_traceback reports (nvBowtie's finish_alignment_kernel,
nvBowtie/bowtie2/cuda/traceback_inl.h:520-723)."""
import ctypes as C
from dataclasses import dataclass
from typing import Optional
import torch
from ._lib import lib, check, BestAlignmentOutStruct, FinishOutStruct
from .strings import PackedStringSet

CIGAR_OPS = "MIDNSHP=X"          # BAM op codes 0..8; this stage writes 0 M, 1 I, 2 D, 4 S


@dataclass
class FinishedAlignments:
    """Device tensors over n alignments: cigar[n, max_cigar] (int32 bit patterns of BAM's run length << 4 | op, START -> END),
    n_cigar[n], md[n, max_md] (uint8, MD:Z bytes, not NUL-terminated), md_len[n] and edits[n, 4] = NM, XM, XO, XG (NM = -1 as int32,
    0xFFFFFFFF, for an alignment that could not be finished).  n_cigar / md_len are the full sizes, also when they exceed the capacity."""
    cigar: torch.Tensor
    n_cigar: torch.Tensor
    md: torch.Tensor
    md_len: torch.Tensor
    edits: torch.Tensor

    def cigar_string(self, i: int) -> str:
        """alignment i's CIGAR as SAM text ("" when it has none); raises when its runs exceeded max_cigar"""
        k = int(self.n_cigar[i])
        if k > self.cigar.shape[1]:
            raise ValueError("alignment %d has %d CIGAR runs, more than max_cigar = %d" % (i, k, self.cigar.shape[1]))
        runs = self.cigar[i, :k].cpu().tolist()
        return "".join("%d%s" % ((v & 0xFFFFFFFF) >> 4, CIGAR_OPS[v & 15]) for v in runs)

    def md_string(self, i: int) -> str:
        """alignment i's MD:Z value ("" when it has none); raises when it exceeded max_md"""
        k = int(self.md_len[i])
        if k > self.md.shape[1]:
            raise ValueError("alignment %d has an MD of %d bytes, more than max_md = %d" % (i, k, self.md.shape[1]))
        return bytes(self.md[i, :k].cpu().tolist()).decode("ascii")


def finish_alignments(genome: torch.Tensor, reads: PackedStringSet, ops: torch.Tensor, n_ops: torch.Tensor, begin: torch.Tensor,
                      strand: torch.Tensor, max_cigar: Optional[int] = None, max_md: Optional[int] = None, stream=None, *,
                      genome_len: int) -> FinishedAlignments:
    """CIGAR, MD and edit counts of traced alignments (nvb_finish_alignments).  genome: the packed 2-bit genome words the traceback ran on
    and genome_len its length in symbols (the words do not carry it); reads: the set passed to the traceback call; ops / n_ops / begin /
    strand: its outputs as they are -- SeedExtendWorkspace.best_ops / best_n_ops / best_begin / best_strand, or PairedWorkspace.mate_ops /
    mate_n_ops / mate_begin / mate_strand (the [2, n_pairs, ...] mate arrays are taken as 2 * n_pairs alignments, mate m of pair p at
    m * n_pairs + p, and so are the outputs).  Defaults: max_cigar = max_ops + 2, max_md = 3 * max_ops + 1, which never truncate.
    stream: a torch.cuda.Stream (default: the current one).  Runs asynchronously."""
    max_ops = ops.shape[-1]
    ops2 = ops.reshape(-1, max_ops)
    n = ops2.shape[0]
    n_ops1, begin2, strand1 = n_ops.reshape(-1), begin.reshape(-1, 2), strand.reshape(-1)
    if n_ops1.numel() != n or begin2.shape[0] != n or strand1.numel() != n:
        raise ValueError("finish_alignments: ops, n_ops, begin and strand describe different numbers of alignments")
    if reads.count != n:
        raise ValueError("finish_alignments: %d reads for %d alignments" % (reads.count, n))
    for t, dt, name in ((ops2, torch.uint8, "ops"), (n_ops1, torch.int32, "n_ops"), (begin2, torch.int32, "begin"),
                        (strand1, torch.uint8, "strand"), (genome, torch.int32, "genome")):
        if t.dtype != dt or not t.is_cuda or not t.is_contiguous():
            raise ValueError("finish_alignments: %s must be a contiguous %s tensor on the device" % (name, dt))
    max_cigar = max_ops + 2 if max_cigar is None else int(max_cigar)
    max_md = 3 * max_ops + 1 if max_md is None else int(max_md)
    dev = ops2.device
    out = FinishedAlignments(cigar=torch.empty((n, max_cigar), dtype=torch.int32, device=dev),
                             n_cigar=torch.empty(n, dtype=torch.int32, device=dev),
                             md=torch.empty((n, max_md), dtype=torch.uint8, device=dev),
                             md_len=torch.empty(n, dtype=torch.int32, device=dev),
                             edits=torch.empty((n, 4), dtype=torch.int32, device=dev))
    if n == 0:
        return out
    a = BestAlignmentOutStruct()
    a.d_ops, a.max_ops, a.d_n_ops = ops2.data_ptr(), max_ops, n_ops1.data_ptr()
    a.d_begin, a.d_strand = begin2.data_ptr(), strand1.data_ptr()
    o = FinishOutStruct()
    o.d_cigar, o.max_cigar, o.d_n_cigar = out.cigar.data_ptr(), max_cigar, out.n_cigar.data_ptr()
    o.d_md, o.max_md, o.d_md_len, o.d_edits = out.md.data_ptr(), max_md, out.md_len.data_ptr(), out.edits.data_ptr()
    rd = reads.struct()
    s = (stream if stream is not None else torch.cuda.current_stream(dev)).cuda_stream
    check(lib().nvb_finish_alignments(C.c_void_p(genome.data_ptr()), C.c_uint32(genome_len), C.byref(rd), C.c_uint32(n), C.byref(a), C.byref(o),
                                      C.c_void_p(s)), "nvb_finish_alignments")
    return out
