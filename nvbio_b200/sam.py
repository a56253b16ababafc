"""SAM text output (nvb_sam_format): BAM records in device memory -- from bam_records, bam_records_all or sort_bam_records -- formatted on
the device as the SAM lines htslib's sam_format1 prints for them, and a host-side writer that frames them as a .sam file.  The line rule
is stated once, in include/nvbio_b200.h."""
import ctypes as C
from dataclasses import dataclass
from typing import Iterable, Optional, Union
import numpy as np
import torch
from ._lib import lib, check, SamOutStruct
from .bam import BamRecords, ContigTable
from .bam_sort import SortedBamRecords

NVB_E_TEMP_SIZE = -2
SORT_ORDERS = ("unknown", "unsorted", "queryname", "coordinate")


def sam_header(contigs: ContigTable, program: str = "nvbio_b200", sort_order: str = "unsorted") -> str:
    """the SAM header text: @HD with SO:sort_order, one @SQ per contig, @PG"""
    if sort_order not in SORT_ORDERS:
        raise ValueError("sam_header: sort_order %r is not one of the SAM specification's" % sort_order)
    return "@HD\tVN:1.0\tSO:%s\n" % sort_order + "".join("@SQ\tSN:%s\tLN:%d\n" % (nm, ln) for nm, ln in zip(contigs.names, contigs.lengths)) + \
        "@PG\tID:%s\tPN:%s\n" % (program, program)


@dataclass
class SamText:
    """data: uint8 device tensor of the lines that fit, line i = data[offsets[i]:offsets[i + 1]] ('\\n' included, empty for a rejected
    record); offsets: int64 [n + 1], complete also past the capacity; rejected: int32 [2] = rejected records, index of the first (-1 when
    none)."""
    data: torch.Tensor
    offsets: torch.Tensor
    rejected: torch.Tensor

    @property
    def n(self) -> int:
        return self.offsets.numel() - 1

    def stored(self) -> int:
        """number of lines stored whole in data"""
        off = self.offsets.cpu().numpy()
        return int(np.searchsorted(off[1:], self.data.numel(), side="right"))

    def to_bytes(self) -> bytes:
        """the stored lines as one host byte string"""
        off = self.offsets.cpu().numpy()
        return self.data[:int(off[self.stored()])].cpu().numpy().tobytes()


def _records(records: Union[BamRecords, SortedBamRecords]):
    """(data, offsets) of a batch that holds all its records"""
    if isinstance(records, SortedBamRecords):
        return records.data, records.offsets
    if not isinstance(records, BamRecords):
        raise TypeError("sam_text: records must be BamRecords or SortedBamRecords, not %s" % type(records).__name__)
    k, n = records.stored(), records.offsets.numel() - 1
    if k != n:
        raise ValueError("sam_text: the batch stored %d of %d records (capacity too small)" % (k, n))
    return records.data, records.offsets


class SamCall:
    """the arguments of one nvb_sam_format call, built once (reference names on the device, output and temp buffers), so that the call
    can be repeated; sam_text is SamCall(...).run()"""

    def __init__(self, records: Union[BamRecords, SortedBamRecords], contigs: ContigTable, capacity: Optional[int] = None):
        data, offsets = _records(records)
        dev = offsets.device
        n = offsets.numel() - 1
        names, name_off = contigs.device_names(dev)
        if capacity is None:
            # a bound no line exceeds: 2.5 text bytes per record byte (a 4-byte CIGAR op or an integer tag prints at most 2.5x its
            # bytes, the rest less), plus the separators, both reference names and the integer fields of every core
            capacity = (5 * int(offsets[-1])) // 2 + n * (80 + 2 * max(len(nm.encode()) for nm in contigs.names))
        self.dev, self.n, self.capacity = dev, n, int(capacity)
        self.data = torch.empty(max(self.capacity, 16), dtype=torch.uint8, device=dev)
        self.offsets = torch.empty(n + 1, dtype=torch.int64, device=dev)
        self.rejected = torch.empty(2, dtype=torch.int32, device=dev)
        self._keep = (data, offsets, names, name_off)
        o = self.o = SamOutStruct()
        o.d_text, o.capacity, o.d_offsets, o.d_rejected = self.data.data_ptr(), self.capacity, self.offsets.data_ptr(), self.rejected.data_ptr()
        self.args = (C.c_void_p(data.data_ptr()) if data.numel() else None, C.c_void_p(offsets.data_ptr()), C.c_uint32(n),
                     C.c_void_p(names.data_ptr()), C.c_void_p(name_off.data_ptr()), C.c_uint32(len(contigs.names)), C.byref(o))
        tb = C.c_size_t(0)
        err = lib().nvb_sam_format(*self.args, None, C.byref(tb), None)
        if err not in (0, NVB_E_TEMP_SIZE):
            check(err, "nvb_sam_format")
        self.temp = torch.empty(max(tb.value, 1), dtype=torch.uint8, device=dev)
        self.temp_bytes = tb.value

    def run(self, stream=None) -> SamText:
        st = stream if stream is not None else torch.cuda.current_stream(self.dev)
        tb = C.c_size_t(self.temp_bytes)
        check(lib().nvb_sam_format(*self.args, C.c_void_p(self.temp.data_ptr()), C.byref(tb), C.c_void_p(st.cuda_stream)), "nvb_sam_format")
        return SamText(data=self.data[:self.capacity], offsets=self.offsets, rejected=self.rejected)


def sam_text(records: Union[BamRecords, SortedBamRecords], contigs: ContigTable, capacity: Optional[int] = None, stream=None) -> SamText:
    """the SAM line of every record: a BamRecords batch that stored all its records (raises otherwise) or a SortedBamRecords; contigs:
    the table the records were built on, whose order is the header's.  capacity: bytes of the text buffer; by default a bound that
    never truncates.  Runs asynchronously on `stream` (default: the current stream)."""
    return SamCall(records, contigs, capacity).run(stream)


def write_sam(path: str, header: Union[str, bytes], batches: Iterable) -> int:
    """write a .sam file: the header text (sam_header), then the lines of every batch (SamText, or bytes) verbatim.  Raises if a batch did
    not store all its lines or rejected a record.  Returns the bytes written."""
    total = 0
    with open(path, "wb") as f:
        h = header.encode() if isinstance(header, str) else bytes(header)
        f.write(h); total += len(h)
        for b in batches:
            if isinstance(b, SamText):
                k, n = b.stored(), b.n
                if k != n:
                    raise ValueError("write_sam: a batch stored %d of %d lines (capacity too small)" % (k, n))
                bad = b.rejected.cpu().tolist()
                if bad[0]:
                    raise ValueError("write_sam: a batch rejected %d records, the first is record %d" % (bad[0], bad[1]))
                b = b.to_bytes()
            b = bytes(b)
            f.write(b); total += len(b)
    return total
