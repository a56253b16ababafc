"""FM-index files in the reference's (BWA-compatible) format, as written by nvBWT and read by
io::FMIndexDataHost::load (nvBWT/nvBWT.cu:314-351, nvbio/io/fmindex/fmindex_impl.cu:120-260):

  <prefix>.bwt : uint32 primary, uint32 cumFreq[4] (cumFreq[3] = text length), packed 2-bit big-endian BWT words
  <prefix>.sa  : uint32 primary, uint32 cumFreq[4], uint32 SA_INT, uint32 text length, uint32 ssa[1..]  (ssa[0] = -1 implied)

The loader hands the BWT words to the device, where the occurrence table is built and interleaved
(nvb_fm_build_occ) -- the reference does that serially on the host (fmindex_impl.cu:263-331)."""
import numpy as np
import torch
from .fmindex import FMIndexDevice


def save_index(prefix: str, bwt_occ: np.ndarray, ssa: np.ndarray, L2, length: int, primary: int, sa_interval: int = 16):
    """write <prefix>.bwt / <prefix>.sa from host arrays in the in-memory layout (32-byte {bwt,occ} blocks)"""
    L2 = np.asarray(L2, dtype=np.uint32)
    hdr = np.array([primary, L2[1], L2[2], L2[3], L2[4]], dtype=np.uint32)
    blocks = np.ascontiguousarray(bwt_occ, dtype=np.uint32).reshape(-1, 8)
    words = np.ascontiguousarray(blocks[:, :4]).reshape(-1)[:(length + 15) // 16]       # ceil(n / 16) words, as nvBWT writes (nvBWT.cu:394,514)
    with open(prefix + ".bwt", "wb") as f:
        hdr.tofile(f)
        words.tofile(f)
    with open(prefix + ".sa", "wb") as f:
        hdr.tofile(f)
        np.array([sa_interval, length], dtype=np.uint32).tofile(f)
        np.ascontiguousarray(ssa, dtype=np.uint32)[1:].tofile(f)


def read_index_files(prefix: str):
    """host-side parse of <prefix>.bwt (+ <prefix>.sa when present): dict(length, primary, cum[4], words (padded to whole 64-symbol
    blocks + 4), ssa (uint32, ssa[0] = 0xFFFFFFFF) or None, sa_interval).  Bytes 4..20 of a .sa file are not interpreted: nvBWT's
    save_ssa() writes the address of its cumFreq argument there (nvBWT.cu:348), not the counts."""
    raw = np.fromfile(prefix + ".bwt", dtype=np.uint32)
    primary, cum = int(raw[0]), raw[1:5].copy()
    n = int(cum[3])
    seq_words = ((n + 63) // 64) * 4                    # whole 64-symbol blocks, as the reference pads (align<4>)
    words = np.zeros(seq_words + 4, dtype=np.uint32)
    body = raw[5:5 + seq_words]
    if len(body) < (n + 15) // 16:
        raise IOError("%s.bwt is truncated" % prefix)
    words[:len(body)] = body
    ssa_h, interval = None, 16
    try:
        sa_raw = np.fromfile(prefix + ".sa", dtype=np.uint32)
    except FileNotFoundError:
        sa_raw = None
    if sa_raw is not None:
        if int(sa_raw[0]) != primary or int(sa_raw[6]) != n:
            raise IOError("SA file mismatch: primary/length differ from the .bwt")     # the reference throws file_mismatch
        interval = int(sa_raw[5])
        n_items = (n + interval) // interval
        if len(sa_raw) < 7 + n_items - 1:
            raise IOError("%s.sa is truncated" % prefix)
        ssa_h = np.empty(n_items, dtype=np.uint32)
        ssa_h[0] = 0xFFFFFFFF
        ssa_h[1:] = sa_raw[7:7 + n_items - 1]
    return dict(length=n, primary=primary, cum=cum, words=words, ssa=ssa_h, sa_interval=interval)


def load_index(prefix: str, device="cuda") -> FMIndexDevice:
    """read <prefix>.bwt (+ <prefix>.sa when present) and build the device index"""
    f = read_index_files(prefix)
    ssa = torch.from_numpy(f["ssa"].view(np.int32)).to(device) if f["ssa"] is not None else None
    d_words = torch.from_numpy(f["words"].view(np.int32)).to(device)
    fmi = FMIndexDevice.from_bwt(d_words, f["length"], f["primary"], ssa, sa_interval=f["sa_interval"])
    got = np.array(fmi.L2[1:], dtype=np.uint64)
    if not np.array_equal(got, f["cum"].astype(np.uint64)):
        raise IOError("cumulative symbol counts of %s.bwt do not match its header" % prefix)
    return fmi


def read_ann(path: str):
    """the contig annotations of an nvBWT / BWA .ann file (nvbio's save_bns / load_bns, nvbio/basic/bnt.cpp:37-160): a line
    "l_pac n_seqs seed", then per sequence "gi name [comment]" and "offset len n_ambs".  A name ends at the first white space.  Returns
    dict(l_pac, names, offsets, lengths)."""
    with open(path) as f:
        head = f.readline().split()
        if len(head) < 2:
            raise IOError("%s: missing the l_pac / n_seqs line" % path)
        l_pac, n_seqs = int(head[0]), int(head[1])
        names, offsets, lengths = [], [], []
        for i in range(n_seqs):
            a, b = f.readline().split(), f.readline().split()
            if len(a) < 2 or len(b) < 2:
                raise IOError("%s: sequence %d of %d is truncated" % (path, i, n_seqs))
            names.append(a[1]); offsets.append(int(b[0])); lengths.append(int(b[1]))
    return dict(l_pac=l_pac, names=names, offsets=np.array(offsets, np.int64), lengths=np.array(lengths, np.int64))
