"""BAM output of traced and finished alignments (nvb_bam_records): the records are built on the device in the bam1_t wire layout of the
SAM / BAM specification, with contig coordinates, the pair fields and TLEN; a small host-side writer frames them as a .bam file (BGZF
blocks compressed with zlib on the host, or members compressed on the device by nvbio_b200.bgzf).  The record rules are stated once,
in include/nvbio_b200.h."""
import ctypes as C
import struct
import zlib
from dataclasses import dataclass
from typing import Iterable, List, Optional, Sequence
import numpy as np
import torch
from ._lib import lib, check, BamInStruct, BamOutStruct, BamAllInStruct
from .finish import FinishedAlignments
from .fmindex import MAX_LENGTH
from .strings import PackedStringSet

NVB_E_TEMP_SIZE = -2
MAX_NAME = 254


class ContigTable:
    """Contig names and lengths of a genome that concatenates them (as nvBWT / BWA indices do); begin = the concatenated coordinate of
    every contig's first base plus the genome length.  The device copy is made on demand."""

    def __init__(self, names: Sequence[str], lengths: Sequence[int]):
        if len(names) == 0 or len(names) != len(lengths):
            raise ValueError("ContigTable: one length per name, at least one contig")
        for nm in names:
            if not nm or any(c.isspace() for c in nm) or "\0" in nm:
                raise ValueError("ContigTable: contig name %r is empty or holds white space" % nm)
        self.names = [str(nm) for nm in names]
        self.lengths = np.asarray(lengths, np.int64)
        if (self.lengths <= 0).any():
            raise ValueError("ContigTable: contig lengths must be positive")
        if (self.lengths >= 1 << 31).any():
            raise ValueError("ContigTable: a contig of 2^31 or more bases has no BAM position (l_ref and POS are int32)")
        self.begin = np.concatenate([[0], np.cumsum(self.lengths)]).astype(np.int64)
        if self.begin[-1] > MAX_LENGTH:
            raise ValueError("ContigTable: the genome is longer than 2^32 - 2 symbols (the longest FM-index text)")
        self._dev = {}

    @staticmethod
    def from_ann(path: str) -> "ContigTable":
        """the contigs of an nvBWT / BWA .ann file (nvbio_b200.io.read_ann); they must tile the genome"""
        from .io import read_ann
        a = read_ann(path)
        if not np.array_equal(np.asarray(a["offsets"], np.int64), np.concatenate([[0], np.cumsum(a["lengths"])[:-1]])):
            raise ValueError("%s: the contigs do not tile the concatenated genome" % path)
        return ContigTable(a["names"], a["lengths"])

    @property
    def genome_len(self) -> int:
        return int(self.begin[-1])

    def device(self, dev="cuda") -> torch.Tensor:
        dev = torch.device(dev)
        if dev not in self._dev:
            self._dev[dev] = torch.from_numpy(self.begin.astype(np.uint32).view(np.int32)).to(dev)
        return self._dev[dev]

    def device_names(self, dev="cuda"):
        """(bytes, offsets) of the names on the device: name j = bytes[offsets[j]:offsets[j + 1]], offsets uint32 [n + 1] (int32 tensor)"""
        dev = torch.device(dev)
        key = ("names", dev)
        if key not in self._dev:
            raw = [nm.encode() for nm in self.names]
            off = np.concatenate([[0], np.cumsum([len(b) for b in raw])]).astype(np.uint32)
            self._dev[key] = (torch.frombuffer(bytearray(b"".join(raw)), dtype=torch.uint8).to(dev), torch.from_numpy(off.view(np.int32)).to(dev))
        return self._dev[key]


def numbered_names(n: int, prefix: str = "r") -> List[str]:
    """read names prefix0, prefix1, ... for synthetic runs"""
    return ["%s%d" % (prefix, i) for i in range(n)]


def _names_tensors(names: Sequence, dev):
    raw = [nm.encode() if isinstance(nm, str) else bytes(nm) for nm in names]
    for nm in raw:
        if not 1 <= len(nm) <= MAX_NAME or any(c < 33 or c > 126 for c in nm):
            raise ValueError("bam_records: read name %r is not 1-%d printable bytes" % (nm, MAX_NAME))
    off = np.zeros(len(raw) + 1, np.int64)
    off[1:] = np.cumsum([len(nm) for nm in raw])
    buf = np.frombuffer(b"".join(raw) + b"\0", np.uint8)
    return (torch.from_numpy(buf.copy()).to(dev), torch.from_numpy(off.astype(np.uint32).view(np.int32)).to(dev), int(off[-1]))


@dataclass
class BamRecords:
    """data: uint8 device tensor of the records that fit, record i = data[offsets[i]:offsets[i + 1]] (block_size first); offsets: int64
    [n + 1], complete also past the capacity; counts: int32 [4] = records, mapped, unmapped by the contig rule, unmapped because finish
    could not write the alignment whole."""
    data: torch.Tensor
    offsets: torch.Tensor
    counts: torch.Tensor

    def stored(self) -> int:
        """number of records stored whole in data"""
        off = self.offsets.cpu().numpy()
        return int(np.searchsorted(off[1:], self.data.numel(), side="right"))

    def to_bytes(self) -> bytes:
        """the stored records as one host byte string"""
        off = self.offsets.cpu().numpy()
        k = self.stored()
        return self.data[:int(off[k])].cpu().numpy().tobytes()


def bam_records(ws, finished: FinishedAlignments, reads: PackedStringSet, contigs: ContigTable, names: Sequence,
                quals: Optional[torch.Tensor] = None, capacity: Optional[int] = None, stream=None) -> BamRecords:
    """BAM records of every read (single end: a SeedExtendWorkspace) or of both mates of every pair (a PairedWorkspace), record 2p + m
    for mate m of pair p; the workspace comes from a call with traceback=True and `finished` from finish_alignments on its outputs with
    the same `reads`.  names: one per read, or one per pair; quals: uint8 phred values indexed like the read symbols, or None.  MAPQ and
    XS come from the workspace when it was made with MAPQ parameters.  capacity: bytes of the output buffer; by default an upper bound
    that never truncates.  Runs asynchronously on `stream` (default: the current stream)."""
    call = BamCall(ws, finished, reads, contigs, names, quals, capacity)
    return call.run(stream)


class BamCall:
    """the arguments of one nvb_bam_records call, built once (names and the contig table on the device, output and temp buffers), so that
    the call can be repeated; bam_records is BamCall(...).run()"""

    def __init__(self, ws, finished, reads, contigs, names, quals=None, capacity=None):
        paired = hasattr(ws, "mate_ops")
        if paired:
            if ws.mate_ops is None:
                raise ValueError("bam_records: the PairedWorkspace was made without traceback=True")
            n = 2 * ws.n_pairs
            n_ops, begin, strand, score = ws.mate_n_ops, ws.mate_begin, ws.mate_strand, ws.mate_score
            mapq, second, pair_flags = ws.mate_mapq, ws.mate_second_score, ws.pair_flags
            n_names = ws.n_pairs
        else:
            if ws.best_ops is None:
                raise ValueError("bam_records: the SeedExtendWorkspace was made without traceback=True")
            n = ws.best_score.numel()
            n_ops, begin, strand, score = ws.best_n_ops, ws.best_begin, ws.best_strand, ws.best_score
            mapq, second, pair_flags = ws.mapq, ws.second_score, None
            n_names = n
        if reads.count != n or finished.n_cigar.numel() != n:
            raise ValueError("bam_records: %d reads and %d finished alignments for %d alignments" % (reads.count, finished.n_cigar.numel(), n))
        if len(names) != n_names:
            raise ValueError("bam_records: %d names for %d %s" % (len(names), n_names, "pairs" if paired else "reads"))
        if quals is not None and (quals.dtype != torch.uint8 or not quals.is_cuda):
            raise ValueError("bam_records: quals must be a uint8 device tensor")
        dev = score.device
        self.dev, self.n = dev, n
        d_names, d_name_off, name_bytes = _names_tensors(names, dev)
        self.name_bytes = name_bytes
        max_cigar, max_md = finished.cigar.shape[1], finished.md.shape[1]
        if capacity is None:
            per = 36 + 1 + 4 * max_cigar + (reads.length + 1) // 2 + reads.length + 6 * 7 + 4 + max_md
            capacity = n * per + name_bytes
        self.capacity = int(capacity)
        self.data = torch.empty(max(self.capacity, 16), dtype=torch.uint8, device=dev)
        self.offsets = torch.empty(n + 1, dtype=torch.int64, device=dev)
        self.counts = torch.empty(4, dtype=torch.int32, device=dev)

        def ptr(t):
            return None if t is None else t.data_ptr()

        # every tensor the structs point into stays referenced by this object
        self._keep = (ws, finished, reads, quals, d_names, d_name_off, contigs.device(dev))
        a = self.a = BamInStruct()
        a.reads = reads.struct()
        a.d_read_quals = ptr(quals)
        a.d_n_ops, a.d_begin, a.d_strand = ptr(n_ops), ptr(begin), ptr(strand)
        f = a.finish
        f.d_cigar, f.max_cigar, f.d_n_cigar = ptr(finished.cigar), max_cigar, ptr(finished.n_cigar)
        f.d_md, f.max_md, f.d_md_len, f.d_edits = ptr(finished.md), max_md, ptr(finished.md_len), ptr(finished.edits)
        a.d_score, a.d_mapq, a.d_second_score, a.d_pair_flags = ptr(score), ptr(mapq), ptr(second), ptr(pair_flags)
        a.d_contig_begin, a.n_contigs = ptr(contigs.device(dev)), len(contigs.names)
        a.d_names, a.d_name_offsets = ptr(d_names), ptr(d_name_off)
        o = self.o = BamOutStruct()
        o.d_records, o.capacity, o.d_offsets, o.d_counts = self.data.data_ptr(), self.capacity, self.offsets.data_ptr(), self.counts.data_ptr()
        tb = C.c_size_t(0)
        err = lib().nvb_bam_records(C.byref(a), C.c_uint32(n), C.byref(o), None, C.byref(tb), None)
        if err not in (0, NVB_E_TEMP_SIZE):
            check(err, "nvb_bam_records")
        self.temp = torch.empty(max(tb.value, 1), dtype=torch.uint8, device=dev)
        self.temp_bytes = tb.value

    def run(self, stream=None) -> BamRecords:
        st = stream if stream is not None else torch.cuda.current_stream(self.dev)
        tb = C.c_size_t(self.temp_bytes)
        check(lib().nvb_bam_records(C.byref(self.a), C.c_uint32(self.n), C.byref(self.o), C.c_void_p(self.temp.data_ptr()), C.byref(tb),
                                    C.c_void_p(st.cuda_stream)), "nvb_bam_records")
        return BamRecords(data=self.data[:self.capacity], offsets=self.offsets, counts=self.counts)


def bam_records_all(al, finished: FinishedAlignments, reads: PackedStringSet, contigs: ContigTable, names: Sequence,
                    quals: Optional[torch.Tensor] = None, capacity: Optional[int] = None, stream=None) -> BamRecords:
    """BAM records of seed_extend_all's alignments (nvb_bam_records_all): per read, its placeable alignments in rank order, the first
    primary (the read's MAPQ and XS), the others secondary (FLAG 0x100, MAPQ 255), each with NH; one unmapped record for a read without a
    placeable alignment.  al: an AllAlignments; finished: finish_alignments over al.strings(reads) and al's ops / n_ops / begin / strand;
    names: one per read; capacity: bytes of the output buffer (by default an upper bound that never truncates).  Waits for the record
    count, so that the result holds exactly the records."""
    n = al.n_reads
    if reads.count != n or len(names) != n:
        raise ValueError("bam_records_all: %d reads and %d names for %d reads" % (reads.count, len(names), n))
    if finished.n_cigar.numel() != al.capacity:
        raise ValueError("bam_records_all: %d finished alignments for %d alignment slots" % (finished.n_cigar.numel(), al.capacity))
    if quals is not None and (quals.dtype != torch.uint8 or not quals.is_cuda):
        raise ValueError("bam_records_all: quals must be a uint8 device tensor")
    dev = al.score.device
    d_names, d_name_off, name_bytes = _names_tensors(names, dev)
    max_cigar, max_md = finished.cigar.shape[1], finished.md.shape[1]
    slots = n + al.capacity
    if capacity is None:
        per = 36 + 1 + 4 * max_cigar + (reads.length + 1) // 2 + reads.length + 6 * 7 + 4 + max_md + 7
        capacity = slots * per + name_bytes * (1 + al.capacity)
    data = torch.empty(max(int(capacity), 16), dtype=torch.uint8, device=dev)
    offsets = torch.empty(slots + 1, dtype=torch.int64, device=dev)
    counts = torch.empty(4, dtype=torch.int32, device=dev)

    def ptr(t):
        return None if t is None else t.untyped_storage().data_ptr() + t.storage_offset() * t.element_size()
    cdev = contigs.device(dev)
    a = BamAllInStruct()
    b = a.base
    b.reads = reads.struct()
    b.d_read_quals = ptr(quals)
    b.d_n_ops, b.d_begin, b.d_strand = ptr(al.n_ops), ptr(al.begin), ptr(al.strand)
    f = b.finish
    f.d_cigar, f.max_cigar, f.d_n_cigar = ptr(finished.cigar), max_cigar, ptr(finished.n_cigar)
    f.d_md, f.max_md, f.d_md_len, f.d_edits = ptr(finished.md), max_md, ptr(finished.md_len), ptr(finished.edits)
    b.d_score, b.d_mapq, b.d_second_score, b.d_pair_flags = ptr(al.score), ptr(al.mapq), ptr(al.second_score), None
    b.d_contig_begin, b.n_contigs = ptr(cdev), len(contigs.names)
    b.d_names, b.d_name_offsets = ptr(d_names), ptr(d_name_off)
    a.d_first, a.capacity = ptr(al.first), al.capacity
    o = BamOutStruct()
    o.d_records, o.capacity, o.d_offsets, o.d_counts = data.data_ptr(), int(capacity), offsets.data_ptr(), counts.data_ptr()
    st = (stream if stream is not None else torch.cuda.current_stream(dev)).cuda_stream
    tb = C.c_size_t(0)
    err = lib().nvb_bam_records_all(C.byref(a), C.c_uint32(n), C.byref(o), None, C.byref(tb), C.c_void_p(st))
    if err not in (0, NVB_E_TEMP_SIZE):
        check(err, "nvb_bam_records_all")
    temp = torch.empty(max(tb.value, 1), dtype=torch.uint8, device=dev)
    check(lib().nvb_bam_records_all(C.byref(a), C.c_uint32(n), C.byref(o), C.c_void_p(temp.data_ptr()), C.byref(tb), C.c_void_p(st)),
          "nvb_bam_records_all")
    n_rec = int(counts[0])                                                 # (synchronises)
    return BamRecords(data=data[:int(capacity)], offsets=offsets[:n_rec + 1], counts=counts)


def pack_names(names: Sequence):
    """(bytes, offsets) of read names on the host, as nvb_pipeline_submit_bam takes them: a uint8 numpy array and uint32 offsets [n + 1]
    (name j = bytes[offsets[j]:offsets[j + 1]]).  Names are str or bytes of 1 or more bytes; nvb_bam_records cuts them at 254."""
    raw = [nm.encode() if isinstance(nm, str) else bytes(nm) for nm in names]
    off = np.zeros(len(raw) + 1, np.uint32)
    off[1:] = np.cumsum([len(nm) for nm in raw])
    return np.frombuffer(b"".join(raw) + b"\0", np.uint8), off


@dataclass
class BamBatch:
    """One batch of StreamingBam (nvb_pipeline_wait_bam): payload, a uint8 view of the pipeline's pinned host memory (valid until `depth`
    further submits) holding BGZF members when compressed, else the BAM records; n_records; counts = nvb_bam_records' tallies (records,
    mapped, unmapped by the contig rule, unfinished); n_hits = (kept, found, distinct jobs); n_rescue = (run, wanted) when paired, else None;
    record_bytes and n_blocks (BGZF members, 0 when not compressed); device_ms of the batch's kernels."""
    payload: torch.Tensor
    compressed: bool
    n_records: int
    counts: tuple
    n_hits: tuple
    n_rescue: Optional[tuple]
    record_bytes: int
    n_blocks: int
    device_ms: float

    def to_bytes(self) -> bytes:
        return self.payload.numpy().tobytes()


def bam_header(contigs: ContigTable, program: str = "nvbio_b200", sort_order: str = "unsorted") -> bytes:
    """BAM header bytes: magic, the SAM header text (@HD with SO:sort_order, one @SQ per contig, @PG) and the reference list"""
    from .sam import sam_header
    t = sam_header(contigs, program, sort_order).encode()
    out = [b"BAM\1", struct.pack("<i", len(t)), t, struct.pack("<i", len(contigs.names))]
    for nm, ln in zip(contigs.names, contigs.lengths):
        b = nm.encode() + b"\0"
        out += [struct.pack("<i", len(b)), b, struct.pack("<i", int(ln))]
    return b"".join(out)


def sam_header_text(header: bytes) -> str:
    """the SAM header text inside BAM header bytes"""
    (l_text,) = struct.unpack_from("<i", header, 4)
    return header[8:8 + l_text].decode()


_BGZF_EOF = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")
_BGZF_DATA = 0xFF00                    # uncompressed bytes per block: the compressed block stays within 64 KiB


def _bgzf_block(data: bytes) -> bytes:
    c = zlib.compressobj(6, zlib.DEFLATED, -15)
    z = c.compress(data) + c.flush()
    bsize = 18 + len(z) + 8
    return (b"\x1f\x8b\x08\x04\0\0\0\0\0\xff\x06\0BC\x02\0" + struct.pack("<H", bsize - 1) + z +
            struct.pack("<II", zlib.crc32(data) & 0xFFFFFFFF, len(data)))


def write_bam(path: str, header: bytes, batches: Iterable) -> int:
    """write a .bam file: header (bam_header) then the records of every batch (BamRecords, or bytes), BGZF-framed on the host with zlib
    (blocks of at most 64 KiB, then the 28-byte EOF block).  A BgzfBlocks batch (bgzf_compress on the device) is written verbatim, and so
    is a compressed BamBatch (StreamingBam); an uncompressed BamBatch is framed like BamRecords.  Raises if a batch did not store all its
    records or members.  Returns the bytes written."""
    from .bgzf import BgzfBlocks
    total = 0
    with open(path, "wb") as f:
        def emit(buf):
            nonlocal total
            for i in range(0, len(buf), _BGZF_DATA):
                blk = _bgzf_block(buf[i:i + _BGZF_DATA])
                f.write(blk); total += len(blk)
        emit(header)
        for b in batches:
            if isinstance(b, BgzfBlocks):
                if b.stored() != b.n_blocks:
                    raise ValueError("write_bam: a batch stored %d of %d BGZF members (capacity too small)" % (b.stored(), b.n_blocks))
                z = b.to_bytes()
                f.write(z); total += len(z)
                continue
            if isinstance(b, BamBatch):
                if b.compressed:
                    z = b.to_bytes()
                    f.write(z); total += len(z)
                    continue
                b = b.to_bytes()
            if isinstance(b, BamRecords):
                if b.stored() != b.offsets.numel() - 1:
                    raise ValueError("write_bam: a batch stored %d of %d records (capacity too small)" % (b.stored(), b.offsets.numel() - 1))
                b = b.to_bytes()
            emit(bytes(b))
        f.write(_BGZF_EOF); total += len(_BGZF_EOF)
    return total
