"""BGZF compression on the device (nvb_bgzf_compress): bytes in device memory, typically BAM records from bam_records, cut into 0xFF00-byte
blocks, each compressed by one CTA into a BGZF member (a dynamic-Huffman deflate block, or a stored block when that is not larger).  The
members are what write_bam writes for a batch; the format rules are stated once, in include/nvbio_b200.h."""
import ctypes as C
from dataclasses import dataclass
from typing import Optional, Union
import numpy as np
import torch
from ._lib import lib, check, BgzfOutStruct
from .bam import BamRecords

NVB_E_TEMP_SIZE = -2
BGZF_BLOCK = 0xFF00                           # input bytes per member, as write_bam's host path cuts them
BGZF_MAX_MEMBER = 18 + 5 + BGZF_BLOCK + 8     # a stored block of a full input block: the largest member


@dataclass
class BgzfBlocks:
    """data: uint8 device tensor of the members that fit, member i = data[offsets[i]:offsets[i + 1]]; offsets: int64 [n_blocks + 1],
    complete also past the capacity; n_input: the number of bytes compressed."""
    data: torch.Tensor
    offsets: torch.Tensor
    n_input: int

    @property
    def n_blocks(self) -> int:
        return self.offsets.numel() - 1

    def stored(self) -> int:
        """number of members stored whole in data"""
        off = self.offsets.cpu().numpy()
        return int(np.searchsorted(off[1:], self.data.numel(), side="right"))

    def to_bytes(self) -> bytes:
        """the stored members as one host byte string (a BGZF stream without the EOF block)"""
        off = self.offsets.cpu().numpy()
        k = int(np.searchsorted(off[1:], self.data.numel(), side="right"))
        return self.data[:int(off[k])].cpu().numpy().tobytes()


def _input(data) -> torch.Tensor:
    if isinstance(data, BamRecords):
        off = data.offsets.cpu().numpy()
        n = off.size - 1
        k = int(np.searchsorted(off[1:], data.data.numel(), side="right"))
        if k != n:
            raise ValueError("bgzf_compress: the BamRecords stored %d of %d records (capacity too small)" % (k, n))
        return data.data[:int(off[n])]
    if not isinstance(data, torch.Tensor) or data.dtype != torch.uint8 or not data.is_cuda:
        raise ValueError("bgzf_compress: data must be a uint8 CUDA tensor or BamRecords")
    if not data.is_contiguous():
        raise ValueError("bgzf_compress: data must be contiguous")
    return data.reshape(-1)


def bgzf_compress(data: Union[torch.Tensor, BamRecords], stream=None) -> BgzfBlocks:
    """BGZF members of `data` (a uint8 CUDA tensor, or BamRecords that stored all their records), one per 0xFF00 input bytes.  Runs
    asynchronously on `stream` (default: the current stream)."""
    return BgzfCall(data).run(stream)


class BgzfCall:
    """the arguments of one nvb_bgzf_compress call, built once (output and temp buffers), so that the call can be repeated; bgzf_compress is
    BgzfCall(data).run().  capacity: bytes of the output buffer; by default 65,311 per block, which never truncates."""

    def __init__(self, data: Union[torch.Tensor, BamRecords], capacity: Optional[int] = None):
        src = _input(data)
        self.src, self.n = src, src.numel()
        self.n_blocks = -(-self.n // BGZF_BLOCK)
        dev = src.device
        self.capacity = int(BGZF_MAX_MEMBER * self.n_blocks if capacity is None else capacity)
        self.data = torch.empty(max(self.capacity, 16), dtype=torch.uint8, device=dev)
        self.offsets = torch.empty(self.n_blocks + 1, dtype=torch.int64, device=dev)
        o = self.o = BgzfOutStruct()
        o.d_out, o.capacity, o.d_block_offsets = self.data.data_ptr(), self.capacity, self.offsets.data_ptr()
        tb = C.c_size_t(0)
        err = lib().nvb_bgzf_compress(C.c_void_p(self._in_ptr()), C.c_uint64(self.n), C.byref(o), None, C.byref(tb), None)
        if err not in (0, NVB_E_TEMP_SIZE):
            check(err, "nvb_bgzf_compress")
        self.temp = torch.empty(max(tb.value, 1), dtype=torch.uint8, device=dev)
        self.temp_bytes = tb.value

    def _in_ptr(self):
        return self.src.data_ptr() if self.n else None

    def run(self, stream=None) -> BgzfBlocks:
        st = stream if stream is not None else torch.cuda.current_stream(self.src.device)
        tb = C.c_size_t(self.temp_bytes)
        check(lib().nvb_bgzf_compress(C.c_void_p(self._in_ptr()), C.c_uint64(self.n), C.byref(self.o), C.c_void_p(self.temp.data_ptr()),
                                      C.byref(tb), C.c_void_p(st.cuda_stream)), "nvb_bgzf_compress")
        return BgzfBlocks(data=self.data[:self.capacity], offsets=self.offsets, n_input=self.n)
