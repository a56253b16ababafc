"""Synthetic workloads of BASELINE.json's configs (seeded; generated on the device).

Genome: uniform symbols in {0,1,2,3} (a uniform random uint32 word = 16 uniform symbols).
Reads: sampled at uniform positions, `sub_rate` substitutions and `indel_rate` single-base indels,
every other read reverse-complemented.  Seeds (SURVEY.md 8d): genome 0x9E3779B97F4A7C15,
queries 0xD1B54A32D192ED03, mutations 0x94D049BB133111EB (truncated to 63 bits for torch.Generator)."""
import numpy as np
import torch

SEED_GENOME = 0x9E3779B97F4A7C15 & 0x7FFFFFFFFFFFFFFF
SEED_QUERIES = 0xD1B54A32D192ED03 & 0x7FFFFFFFFFFFFFFF
SEED_MUT = 0x94D049BB133111EB & 0x7FFFFFFFFFFFFFFF


def _gen(seed, device):
    g = torch.Generator(device=device)
    g.manual_seed(seed)
    return g


def random_genome_words(n: int, device="cuda", seed=SEED_GENOME) -> torch.Tensor:
    """2-bit big-endian packed genome of n symbols as int32 words (+8 zero pad words); symbols past n are 0"""
    nw = (n + 15) // 16
    words = torch.zeros(nw + 8, dtype=torch.int32, device=device)
    g = _gen(seed, device)
    chunk = 1 << 28
    for s in range(0, nw, chunk):
        e = min(nw, s + chunk)
        words[s:e] = torch.randint(-(1 << 31), (1 << 31), (e - s,), dtype=torch.int64, device=device, generator=g).to(torch.int32)
    rem = n % 16
    if rem:
        mask = (0xFFFFFFFF << (32 - 2 * rem)) & 0xFFFFFFFF
        mask = mask - (1 << 32) if mask >= (1 << 31) else mask
        words[nw - 1] &= mask
    return words


def gather_symbols(words: torch.Tensor, pos: torch.Tensor) -> torch.Tensor:
    """symbols (int64 tensor) of a 2-bit big-endian stream at int64 positions `pos` (any shape)"""
    w = words[(pos >> 4)].to(torch.int64) & 0xFFFFFFFF
    sh = 30 - 2 * (pos & 15)
    return (w >> sh) & 3


def pack_2bit_be(sym: torch.Tensor) -> torch.Tensor:
    """[rows, L] symbols -> [rows, ceil(L/16)] int32 words (each row word-aligned)"""
    rows, L = sym.shape
    Lp = (L + 15) // 16 * 16
    if Lp != L:
        sym = torch.cat([sym, torch.zeros(rows, Lp - L, dtype=sym.dtype, device=sym.device)], dim=1)
    s = sym.view(rows, Lp // 16, 16).to(torch.int64)
    sh = (30 - 2 * torch.arange(16, device=sym.device, dtype=torch.int64))
    w = (s << sh).sum(dim=2)
    w = torch.where(w >= (1 << 31), w - (1 << 32), w)
    return w.to(torch.int32)


def sample_seeds(genome_words, n, n_seeds, seed_len, device="cuda", random_frac=0.0, seed=SEED_QUERIES):
    """C2: seeds of `seed_len` at uniform genome positions (all hit >= 1); a fraction may be random.
    Returns (words [n_seeds, ceil(len/16)] int32, positions)"""
    g = _gen(seed, device)
    pos = torch.randint(0, n - seed_len + 1, (n_seeds,), device=device, generator=g, dtype=torch.int64)
    idx = pos[:, None] + torch.arange(seed_len, device=device, dtype=torch.int64)[None, :]
    sym = gather_symbols(genome_words, idx)
    if random_frac > 0:
        k = int(n_seeds * random_frac)
        sym[:k] = torch.randint(0, 4, (k, seed_len), device=device, generator=g, dtype=torch.int64)
    return pack_2bit_be(sym), pos


def sample_reads(genome_words, n, n_reads, read_len, sub_rate=0.01, indel_rate=0.001, device="cuda",
                 seed=SEED_QUERIES, mut_seed=SEED_MUT, rc_half=True, chunk=1 << 18):
    """C3/C4 reads.  Returns (words [n_reads, ceil(read_len/16)] int32, pos int64[n_reads], strand uint8[n_reads])"""
    g, gm = _gen(seed, device), _gen(mut_seed, device)
    out, poss, strands = [], [], []
    margin = read_len + 64
    for s in range(0, n_reads, chunk):
        m = min(chunk, n_reads - s)
        pos = torch.randint(0, n - margin, (m,), device=device, generator=g, dtype=torch.int64)
        u = torch.rand((m, read_len), device=device, generator=gm)
        dele = (u < indel_rate / 2)
        ins = (u >= indel_rate / 2) & (u < indel_rate)
        delta = dele.to(torch.int64) - ins.to(torch.int64)
        shift = torch.cumsum(delta, dim=1)
        src = pos[:, None] + torch.arange(read_len, device=device, dtype=torch.int64)[None, :] + shift
        src = src.clamp_(0, n - 1)
        sym = gather_symbols(genome_words, src)
        rnd = torch.randint(0, 4, (m, read_len), device=device, generator=gm, dtype=torch.int64)
        sub = torch.rand((m, read_len), device=device, generator=gm) < sub_rate
        sym = torch.where(ins, rnd, sym)
        sym = torch.where(sub, (sym + 1 + (rnd % 3)) % 4, sym)
        strand = torch.zeros(m, dtype=torch.uint8, device=device)
        if rc_half:
            strand = (torch.arange(s, s + m, device=device) & 1).to(torch.uint8)
            rc = (3 - sym).flip(1)
            sym = torch.where(strand[:, None].bool(), rc, sym)
        out.append(pack_2bit_be(sym)); poss.append(pos); strands.append(strand)
    return torch.cat(out), torch.cat(poss), torch.cat(strands)


# (mate 1, mate 2) of a fragment sequenced in each orientation, from its left (L) and right (R) read_len bases, forward (fw) or reverse
# complemented (rv): (even pairs, odd pairs); an odd pair reads the fragment off the reverse strand (L <-> R, strands flipped)
_ORIENT = {"fr": (("fwL", "rvR"), ("rvR", "fwL")), "rf": (("rvL", "fwR"), ("fwR", "rvL")),
           "ff": (("fwL", "fwR"), ("rvR", "rvL")), "rr": (("fwR", "fwL"), ("rvL", "rvR"))}


def sample_pairs(genome_words, n, n_pairs, read_len, frag_mean=350.0, frag_sd=30.0, sub_rate=0.01, hard_frac=0.05, hard_sub_rate=0.2,
                 device="cuda", seed=SEED_QUERIES ^ 0x7777, mut_seed=SEED_MUT ^ 0x7777, chunk=1 << 18, orientation="fr"):
    """C5-shaped pairs of a fragment [p, p + frag) of the genome with L = its first read_len bases and R = its last read_len bases.
    orientation "fr" (the default): one mate = L forward, the other = the reverse complement of R; "rf": L reverse complemented, R
    forward; "ff": mate 1 = L, mate 2 = R, both forward; "rr": mate 1 = R, mate 2 = L, both forward.  Odd pairs read the fragment off
    the reverse strand (FR: which mate is which swaps).  A fraction `hard_frac` of the second mates carries `hard_sub_rate`
    substitutions (mostly no exact seed survives: the opposite-mate rescue has to place them).  The random draws do not depend on the
    orientation.  Returns (words [2*n_pairs, ceil(read_len/16)] int32 -- mate 1 of every pair, then mate 2 --, left int64[n_pairs],
    frag int64[n_pairs])"""
    if orientation not in _ORIENT:
        raise ValueError("sample_pairs: orientation must be one of %s, not %r" % (tuple(_ORIENT), orientation))
    g, gm = _gen(seed, device), _gen(mut_seed, device)
    m1, m2, lefts, frags = [], [], [], []
    ar = torch.arange(read_len, device=device, dtype=torch.int64)[None, :]
    for s in range(0, n_pairs, chunk):
        m = min(chunk, n_pairs - s)
        frag = (frag_mean + frag_sd * torch.randn(m, device=device, generator=g)).round().to(torch.int64).clamp_(read_len, int(frag_mean + 4 * frag_sd))
        left = torch.randint(0, n - int(frag_mean + 4 * frag_sd) - 64, (m,), device=device, generator=g, dtype=torch.int64)
        fwl = gather_symbols(genome_words, left[:, None] + ar)
        fwr = gather_symbols(genome_words, (left + frag - read_len)[:, None] + ar)
        seg = dict(fwL=fwl, rvR=(3 - fwr).flip(1), fwR=fwr, rvL=(3 - fwl).flip(1))
        (ea, eb), (oa, ob) = _ORIENT[orientation]
        swap = (torch.arange(s, s + m, device=device) & 1).bool()
        a = torch.where(swap[:, None], seg[oa], seg[ea])
        b = torch.where(swap[:, None], seg[ob], seg[eb])
        hard = torch.rand(m, device=device, generator=gm) < hard_frac
        for k, sym in enumerate((a, b)):
            rate = torch.full((m, 1), sub_rate, device=device)
            if k == 1:
                rate = torch.where(hard[:, None], torch.full_like(rate, hard_sub_rate), rate)
            rnd = torch.randint(0, 3, (m, read_len), device=device, generator=gm, dtype=torch.int64)
            sub = torch.rand((m, read_len), device=device, generator=gm) < rate
            sym = torch.where(sub, (sym + 1 + rnd) % 4, sym)
            (m1 if k == 0 else m2).append(pack_2bit_be(sym))
        lefts.append(left); frags.append(frag)
    return torch.cat(m1 + m2), torch.cat(lefts), torch.cat(frags)


def windows_for_reads(genome_len, pos, read_len, window_len, max_offset=15, device="cuda", seed=SEED_MUT ^ 0x5555):
    """C4: each read gets a `window_len` genome window containing it at offset <= max_offset"""
    g = _gen(seed, device)
    off = torch.randint(0, max_offset + 1, (pos.numel(),), device=device, generator=g, dtype=torch.int64)
    begin = (pos - off).clamp_(0, genome_len - window_len)
    return begin
