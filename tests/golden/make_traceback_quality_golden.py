"""Generate tests/golden/traceback_quality.npz by RUNNING THE REFERENCE ITSELF: the banded (aln::banded_alignment_traceback<B,1024,32>)
and full-matrix (aln::alignment_traceback<256,512,64>) Gotoh tracebacks under a quality-table scheme (TableGotohScheme in
oracle/ref_shim.cpp) with per-base qualities.

Run where oracle/_ref/libnvbio_ref.so is built:
    python tests/golden/make_traceback_quality_golden.py

The fixture covers bands 7 / 15 / 31 and the full matrix, all three alignment types, two nvBowtie-like tables (QualityGotohScheme.host_table
with match bonus 2 and 0), text gap costs that differ from the pattern's, qualities 0..63 and 255, patterns with and without N's, texts with
N's, 1-2 % indels and low-quality mismatches beside the indels (where a gap and a mismatch compete).  The file is written with fixed zip
timestamps, so regenerating it reproduces it byte for byte.
"""
import os
import sys
import zipfile
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import orc  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "traceback_quality.npz")

# (match, mismatch, pattern gap open, pattern gap ext, text gap open, text gap ext): only the gap costs reach a table-driven scheme
SCHEME6 = (0, 0, -8, -3, -7, -2)


def quality_table(match_bonus, mm_min=2, mm_max=6):
    """QualityGotohScheme.host_table (nvbio_b200/aln.py), restated so that this file needs neither torch nor the extension"""
    q = np.arange(256)
    frac = (np.minimum(q, 40).astype(np.float32) / np.float32(40.0)).astype(np.float32)
    mmp = mm_min + np.trunc(frac * np.float32(mm_max - mm_min)).astype(np.int32)
    return np.ascontiguousarray(np.stack([np.full(256, match_bonus, np.int32), (-mmp).astype(np.int32)], axis=1))


def qualities(rng, n, profile):
    """base qualities: 'low' 2..8, 'high' 35..40, 'rand' 0..45, 'clamp' 41..63 and 255 (the table clamps them to 40), 'mixed' 0..63
    with 3 % at 255"""
    if profile == "low":
        return rng.integers(2, 9, n).astype(np.uint8)
    if profile == "high":
        return rng.integers(35, 41, n).astype(np.uint8)
    if profile == "rand":
        return rng.integers(0, 46, n).astype(np.uint8)
    if profile == "clamp":
        q = rng.integers(41, 64, n).astype(np.uint8)
        q[rng.random(n) < 0.2] = 255
        return q
    q = rng.integers(0, 64, n).astype(np.uint8)
    q[rng.random(n) < 0.03] = 255
    return q


def _mutate(rng, t, j, m, indel, sub, tie):
    """a read of m symbols copied from t from position j with substitutions and indels; returns (read, tie mask): after an indel, with
    probability `tie`, one or two substitutions follow (given a low quality by the caller, so that a gap and cheap mismatches compete)"""
    p, low = [], []
    N = len(t)
    pending = 0
    while len(p) < m:
        r = rng.random()
        if pending == 0 and j < N and r < indel / 2:
            p.append(int(rng.integers(0, 4))); low.append(False)                     # insertion
            pending = int(rng.integers(1, 3)) if rng.random() < tie else 0
        elif pending == 0 and j < N and r < indel:
            j += int(rng.integers(1, 3))                                             # deletion of 1-2 symbols
            pending = int(rng.integers(1, 3)) if rng.random() < tie else 0
        elif j >= N or pending or r < indel + sub:
            g = int(t[j]) & 3 if j < N else 0
            p.append((g + int(rng.integers(1, 4))) & 3); low.append(bool(pending)); j += 1
            pending = max(pending - 1, 0)
        else:
            p.append(int(t[j]) & 3); low.append(False); j += 1
    return np.array(p[:m], np.uint8), np.array(low[:m], bool)


def _text(rng, N, n_txt):
    if rng.random() < 0.2:                                                           # a low-complexity text: many equal-score paths
        unit = rng.integers(0, 4, int(rng.integers(1, 4)))
        t = np.resize(unit, N).astype(np.uint8)
        noise = rng.random(N) < 0.05
        t[noise] = rng.integers(0, 4, int(noise.sum()))
    else:
        t = rng.integers(0, 4, N).astype(np.uint8)
    if n_txt:
        t[rng.random(N) < n_txt] = 4
    return t


def _pack(items):
    pats, quals, txts = [x[0] for x in items], [x[1] for x in items], [x[2] for x in items]
    p_len = np.array([len(p) for p in pats], np.uint32); t_len = np.array([len(t) for t in txts], np.uint32)
    p_off = (np.cumsum(p_len) - p_len).astype(np.uint32); t_off = (np.cumsum(t_len) - t_len).astype(np.uint32)
    return (np.concatenate(pats), p_off, p_len, np.concatenate(txts), t_off, t_len), np.concatenate(quals)


def banded_problems(rng, n, band, max_m, min_m=None, extra_text=(0, 3), indel=0.015, sub=0.03, tie=0.5, n_pat=0.0, n_txt=0.0,
                    profile="mixed", ragged=True):
    """nvBowtie-shaped banded jobs (window = read + band + extra) with qualities: ((pat, p_off, p_len, txt, t_off, t_len), qual)"""
    min_m = max_m if not ragged else (min_m or max(1, max_m - 60))
    items = []
    for _ in range(n):
        m = int(rng.integers(min_m, max_m + 1))
        N = m + band + int(rng.integers(extra_text[0], extra_text[1] + 1))
        t = _text(rng, N, n_txt)
        p, low = _mutate(rng, t, int(rng.integers(0, band)), m, indel, sub, tie)
        if n_pat:
            p[rng.random(m) < n_pat] = 4
        q = qualities(rng, m, profile)
        q[low] = rng.integers(0, 12, int(low.sum()))
        items.append((p, q, t))
    return _pack(items)


def full_problems(rng, n, max_m, max_n, indel=0.015, sub=0.03, tie=0.5, n_pat=0.0, n_txt=0.0, profile="mixed"):
    """full-matrix jobs: patterns of 1..max_m symbols, texts of 1..max_n, the pattern mostly drawn from its text"""
    items = []
    for _ in range(n):
        m = int(rng.integers(1, max_m + 1)); N = int(rng.integers(max(1, m // 2), max_n + 1))
        t = _text(rng, N, n_txt)
        if N > m + 2 and rng.random() < 0.85:
            p, low = _mutate(rng, t, int(rng.integers(0, N - m - 1)), m, indel, sub, tie)
        else:
            p, low = rng.integers(0, 4, m).astype(np.uint8), np.zeros(m, bool)
        if n_pat:
            p[rng.random(m) < n_pat] = 4
        q = qualities(rng, m, profile)
        q[low] = rng.integers(0, 12, int(low.sum()))
        items.append((p, q, t))
    return _pack(items)


def savez_fixed(path, arrays):
    """np.savez_compressed with fixed zip timestamps (byte-reproducible)"""
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as z:
        for k in sorted(arrays):
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            with z.open(info, "w", force_zip64=True) as f:
                np.lib.format.write_array(f, np.asanyarray(arrays[k]), allow_pickle=False)


def cases():
    """(band (0 = full matrix), type, match bonus, keyword arguments of the problem generator) of every fixture case"""
    out = []
    for band in (7, 15, 31):
        for typ in (0, 1, 2):
            for mb in (2, 0):
                out.append((band, typ, mb, dict(n=24, max_m=120, n_pat=0.02, n_txt=0.02)))
                out.append((band, typ, mb, dict(n=16, max_m=150, indel=0.02)))                  # 2-bit patterns, no N's
    for typ in (0, 1, 2):
        for mb in (2, 0):
            out.append((0, typ, mb, dict(n=12, max_m=256, max_n=512, n_pat=0.02, n_txt=0.01)))
    return out


def main(path=OUT):
    ref = orc.Ref()
    rng = np.random.default_rng(20261017)
    out = {"qtab2": quality_table(2), "qtab0": quality_table(0), "scheme6": np.array(SCHEME6, np.int32)}
    meta = []
    for cid, (band, typ, mb, kw) in enumerate(cases()):
        pr, qual = banded_problems(rng, band=band, **kw) if band else full_problems(rng, **kw)
        qtab = out["qtab%d" % mb]
        max_ops = 2 * int(pr[2].max()) + band if band else int(pr[2].max()) + int(pr[5].max()) + 1
        if band:
            o = ref.banded_traceback_q(band, typ, SCHEME6, *pr, qual, qtab, max_ops=max_ops)
        else:
            o = ref.gotoh_full_traceback_q(typ, SCHEME6, *pr, qual, qtab, max_ops=max_ops)
        assert np.all(o["n_ops"] <= max_ops)
        for k, v in zip(("pat", "p_off", "p_len", "txt", "t_off", "t_len"), pr):
            out[f"c{cid}_{k}"] = v
        out[f"c{cid}_qual"] = qual
        out[f"c{cid}_res"] = np.stack([o["score"].astype(np.int64), o["sink"][:, 0].astype(np.int64), o["sink"][:, 1].astype(np.int64),
                                       o["source"][:, 0].astype(np.int64), o["source"][:, 1].astype(np.int64), o["n_ops"].astype(np.int64),
                                       o["clips"][:, 0].astype(np.int64), o["clips"][:, 1].astype(np.int64)])
        out[f"c{cid}_ops"] = np.concatenate([o["ops"][i][:o["n_ops"][i]] for i in range(len(o["n_ops"]))])
        meta.append((cid, band, typ, mb))
    out["cases"] = np.array(meta, np.int64)
    savez_fixed(path, out)
    return path


if __name__ == "__main__":
    print("wrote", main())
