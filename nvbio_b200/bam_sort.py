"""Coordinate-sorted, indexed BAM output on the device: nvb_bam_sort orders BAM records by (refID, pos), stably, with unplaced records last;
nvb_bam_index builds the BAI of the sorted records once nvbio_b200.bgzf has compressed them.  write_sorted_bam chains both with the BGZF
compression into a .bam and its .bai.  The order and the index rules are stated once, in include/nvbio_b200.h."""
import ctypes as C
from dataclasses import dataclass
from typing import List, Union
import numpy as np
import torch
from ._lib import lib, check, BamSortOutStruct, BaiOutStruct
from .bam import BamRecords, ContigTable, bam_header, _bgzf_block, _BGZF_DATA, _BGZF_EOF
from .bgzf import BgzfBlocks, bgzf_compress

NVB_E_TEMP_SIZE = -2
BAI_MAX_REF_LEN = 1 << 29
_STATUS = {1: "the records are not in coordinate order", 2: "a refID is not in the contig table", 3: "a record's span ends past 2^29"}


@dataclass
class SortedBamRecords:
    """data: uint8 device tensor of the sorted records, record j = data[offsets[j]:offsets[j + 1]]; offsets: int64 [n + 1]; order: int32 [n],
    output record j is input record order[j] (indices into the concatenated input)."""
    data: torch.Tensor
    offsets: torch.Tensor
    order: torch.Tensor

    @property
    def n(self) -> int:
        return self.offsets.numel() - 1

    def to_bytes(self) -> bytes:
        return self.data[:int(self.offsets[-1])].cpu().numpy().tobytes()


def _whole(r: BamRecords, what: str):
    k, n = r.stored(), r.offsets.numel() - 1
    if k != n:
        raise ValueError("%s: a batch stored %d of %d records (capacity too small)" % (what, k, n))
    return r.data[:int(r.offsets[-1])], r.offsets


def _concat(records: Union[BamRecords, List[BamRecords]]):
    """the records of one batch, or of a list of batches in order (offsets rebased), as one device byte stream"""
    if isinstance(records, BamRecords):
        return _whole(records, "sort_bam_records")
    if not records:
        raise ValueError("sort_bam_records: no batch")
    parts = [_whole(r, "sort_bam_records") for r in records]
    dev = parts[0][0].device
    data = torch.cat([d for d, _ in parts]) if any(d.numel() for d, _ in parts) else torch.empty(0, dtype=torch.uint8, device=dev)
    offs, base = [], 0
    for d, o in parts:
        offs.append(o[:-1] + base)
        base += d.numel()
    offs.append(torch.tensor([base], dtype=torch.int64, device=dev))
    return data, torch.cat(offs)


def _ptr(t: torch.Tensor):
    return C.c_void_p(t.data_ptr()) if t.numel() else None


def sort_bam_records(records: Union[BamRecords, List[BamRecords]], stream=None) -> SortedBamRecords:
    """the records in coordinate order: by (refID, pos) with unplaced records last, equal keys in input order.  A list of batches is
    concatenated in order first, so its order breaks ties.  Every batch must have stored all its records.  Runs asynchronously on
    `stream` (default: the current stream)."""
    data, offsets = _concat(records)
    dev = offsets.device
    n = offsets.numel() - 1
    st = stream if stream is not None else torch.cuda.current_stream(dev)
    out_data = torch.empty(max(data.numel(), 16), dtype=torch.uint8, device=dev)
    out_off = torch.empty(n + 1, dtype=torch.int64, device=dev)
    order = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
    o = BamSortOutStruct()
    o.d_records, o.capacity, o.d_offsets, o.d_order = out_data.data_ptr(), data.numel(), out_off.data_ptr(), order.data_ptr()
    tb = C.c_size_t(0)
    args = (_ptr(data), C.c_void_p(offsets.data_ptr()), C.c_uint32(n), C.byref(o))
    err = lib().nvb_bam_sort(*args, None, C.byref(tb), None)
    if err not in (0, NVB_E_TEMP_SIZE):
        check(err, "nvb_bam_sort")
    temp = torch.empty(max(tb.value, 1), dtype=torch.uint8, device=dev)
    check(lib().nvb_bam_sort(*args, C.c_void_p(temp.data_ptr()), C.byref(tb), C.c_void_p(st.cuda_stream)), "nvb_bam_sort")
    # the inputs and the temp buffer must outlive the asynchronous call
    for t in (data, offsets, temp):
        t.record_stream(st)
    return SortedBamRecords(data=out_data[:data.numel()], offsets=out_off, order=order[:n])


def bam_index(sorted_records: SortedBamRecords, blocks: BgzfBlocks, header_bytes: int, contigs: ContigTable, stream=None) -> bytes:
    """the .bai bytes of the file made of `header_bytes` compressed bytes of header members, the members `blocks` of bgzf_compress over
    exactly sorted_records' bytes, and the EOF block.  Raises when the records are not in coordinate order, name a refID past the
    contig table, or reach past 2^29, and (NvbError) when a contig is longer than BAI can index."""
    s = sorted_records
    n = s.n
    dev = s.offsets.device
    if blocks.n_input != int(s.offsets[-1]):
        raise ValueError("bam_index: the BGZF blocks hold %d bytes, the records %d" % (blocks.n_input, int(s.offsets[-1])))
    st = stream if stream is not None else torch.cuda.current_stream(dev)
    n_refs, max_len = len(contigs.names), int(contigs.lengths.max())
    size = torch.zeros(1, dtype=torch.int64, device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    # a capacity that holds every index whose records lie inside their contigs: 24 bytes per chunk and bin, the fixed part and the
    # linear index of every contig
    cap = 16 + 24 * n + sum(52 + 8 * ((int(ln) >> 14) + 1) for ln in contigs.lengths)
    tb = C.c_size_t(0)
    temp = None
    for _ in range(2):
        bai = torch.empty(max(cap, 16), dtype=torch.uint8, device=dev)
        o = BaiOutStruct()
        o.d_bai, o.capacity, o.d_size, o.d_status = bai.data_ptr(), cap, size.data_ptr(), status.data_ptr()
        args = (_ptr(s.data), C.c_void_p(s.offsets.data_ptr()), C.c_uint32(n), C.c_void_p(blocks.offsets.data_ptr()), C.c_uint64(header_bytes),
                C.c_uint32(n_refs), C.c_uint32(min(max_len, 0xFFFFFFFF)), C.byref(o))
        if temp is None:
            err = lib().nvb_bam_index(*args, None, C.byref(tb), None)
            if err not in (0, NVB_E_TEMP_SIZE):
                check(err, "nvb_bam_index")
            temp = torch.empty(max(tb.value, 1), dtype=torch.uint8, device=dev)
        check(lib().nvb_bam_index(*args, C.c_void_p(temp.data_ptr()), C.byref(tb), C.c_void_p(st.cuda_stream)), "nvb_bam_index")
        st.synchronize()
        code, need = int(status), int(size)
        if code:
            raise ValueError("bam_index: %s (status %d)" % (_STATUS.get(code, "?"), code))
        if need <= cap:
            return bai[:need].cpu().numpy().tobytes()
        cap = need
    raise RuntimeError("bam_index: the index did not fit its measured size")


def write_sorted_bam(path: str, contigs: ContigTable, records: Union[BamRecords, List[BamRecords]], program: str = "nvbio_b200") -> int:
    """write a coordinate-sorted .bam (header with SO:coordinate) and its index path + ".bai": sort_bam_records, bgzf_compress, header
    members compressed on the host, bam_index.  Raises on a batch that did not store all its records.  Returns the bytes of the .bam."""
    s = sort_bam_records(records)
    blocks = bgzf_compress(s.data[:int(s.offsets[-1])])
    header = bam_header(contigs, program, sort_order="coordinate")
    hz = b"".join(_bgzf_block(header[i:i + _BGZF_DATA]) for i in range(0, len(header), _BGZF_DATA))
    bai = bam_index(s, blocks, len(hz), contigs)
    if blocks.stored() != blocks.n_blocks:
        raise ValueError("write_sorted_bam: stored %d of %d BGZF members" % (blocks.stored(), blocks.n_blocks))
    z = blocks.to_bytes()
    with open(path, "wb") as f:
        f.write(hz); f.write(z); f.write(_BGZF_EOF)
    with open(path + ".bai", "wb") as f:
        f.write(bai)
    return len(hz) + len(z) + len(_BGZF_EOF)
