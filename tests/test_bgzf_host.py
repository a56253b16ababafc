"""CPU: nvb_bgzf_compress's per-block routines (bgzf_core.cuh), compiled for the host by tests/host/bgzf_harness.cu: the chunked CRC-32 and
its shift combine against zlib.crc32; length-limited code lengths on adversarial histograms against a package-merge restatement (limit,
completeness, optimal cost); whole members assembled from per-position matches (literal-only, one distance, stored, the host run of the
device's match finder) read back by zlib and gzip; argument validation of nvb_bgzf_compress without a GPU."""
import ctypes as C
import gzip
import heapq
import os
import struct
import subprocess
import zlib
import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
BLOCK = 0xFF00
MAX_MEMBER = 18 + 5 + BLOCK + 8
EOF_BLOCK = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")
HEADER = b"\x1f\x8b\x08\x04\0\0\0\0\0\xff\x06\0BC\x02\0"


@pytest.fixture(scope="module")
def H(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("bgzf_harness") / "libbgzf_harness.so")
    from nvbio_b200.build import NVCC
    subprocess.check_call([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "-Wno-deprecated-declarations",
                           "-Xcompiler", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "host", "bgzf_harness.cu")])
    h = C.CDLL(so)
    h.hh_crc32.restype = C.c_uint32
    h.hh_gf2_mulmod.restype = C.c_uint32
    h.hh_code_lengths.restype = C.c_uint32
    h.hh_member.restype = C.c_uint32
    return h


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


# ------------------------------------------------------------------------------------------------
# CRC-32
# ------------------------------------------------------------------------------------------------
def test_crc32_every_length(H):
    rng = np.random.default_rng(1)
    buf = rng.integers(0, 256, 4096, dtype=np.uint8).tobytes()
    for n in range(301):
        a = int(rng.integers(0, 4096 - n + 1))
        s = buf[a:a + n]
        for chunk in (1, 7, 128, 1 << 20):
            assert H.hh_crc32(s, C.c_uint64(n), C.c_uint32(chunk)) == zlib.crc32(s), (n, chunk)


@pytest.mark.parametrize("n", [BLOCK - 1, BLOCK, BLOCK + 1, 2 * BLOCK])
def test_crc32_block_sizes(H, n):
    rng = np.random.default_rng(n)
    s = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
    for chunk in (128, 4096, 1000):
        assert H.hh_crc32(s, C.c_uint64(n), C.c_uint32(chunk)) == zlib.crc32(s)
    z = bytes(n)
    assert H.hh_crc32(z, C.c_uint64(n), C.c_uint32(128)) == zlib.crc32(z)


def test_gf2_mulmod_identity(H):
    one = 0x80000000                                  # x^0, bit-reflected
    rng = np.random.default_rng(2)
    for a in rng.integers(0, 1 << 32, 50, dtype=np.uint64):
        assert H.hh_gf2_mulmod(C.c_uint32(int(a)), C.c_uint32(one)) == int(a)
        assert H.hh_gf2_mulmod(C.c_uint32(one), C.c_uint32(int(a))) == int(a)


# ------------------------------------------------------------------------------------------------
# code lengths
# ------------------------------------------------------------------------------------------------
def pm_cost(freqs, limit):
    """the optimal cost sum(f * len) of a code of at most `limit` bits (package-merge over the used symbols, at least two)"""
    w = sorted(f for f in freqs if f > 0)
    if len(w) < 2:
        return sum(w)                                   # one used symbol: one bit each
    level = list(w)                                    # a package's weight is the cost its leaves add
    for _ in range(limit - 1):
        level = sorted(w + [level[2 * k] + level[2 * k + 1] for k in range(len(level) // 2)])
    return sum(level[:2 * len(w) - 2])


def huffman_cost(freqs):
    w = [f for f in freqs if f > 0]
    if len(w) < 2:
        return sum(w)
    heapq.heapify(w)
    c = 0
    while len(w) > 1:
        a, b = heapq.heappop(w), heapq.heappop(w)
        c += a + b
        heapq.heappush(w, a + b)
    return c


def fib(n):
    a, b, out = 1, 1, []
    for _ in range(n):
        out.append(a)
        a, b = b, a + b
    return out


def histograms():
    rng = np.random.default_rng(3)
    yield "fibonacci_30", fib(30) + [0] * 256, 15
    yield "fibonacci_286", [min(x, 1 << 24) for x in fib(40)] + list(rng.integers(1, 5, 246)), 15
    yield "equal_286", [7] * 286, 15
    yield "one_symbol", [0] * 100 + [5] + [0] * 185, 15
    yield "one_symbol_at_0", [9] + [0] * 29, 15
    yield "two_symbols", [0] * 3 + [1] + [0] * 200 + [1000] + [0] * 82, 15
    yield "no_symbol", [0] * 30, 15
    yield "cl_fibonacci_19", fib(19), 7
    yield "cl_skewed_19", [60000, 1, 1, 2, 3, 5, 8, 13, 21, 34, 55, 89, 0, 0, 1, 0, 0, 1, 1], 7
    for k in range(10):
        f = (rng.pareto(0.7, 286) * rng.integers(0, 2, 286)).astype(np.int64).clip(0, 60000)
        yield "pareto_%d" % k, list(f), 15


@pytest.mark.parametrize("name,freqs,limit", list(histograms()), ids=[h[0] for h in histograms()])
def test_code_lengths(H, name, freqs, limit):
    f = np.array(freqs, np.uint32)
    n = f.size
    ln = np.zeros(n, np.uint8)
    used = H.hh_code_lengths(_p(f), C.c_uint32(n), C.c_uint32(limit), _p(ln))
    assert used == max(2, int((f > 0).sum()))
    assert ln.max() <= limit
    assert (ln[f > 0] > 0).all()                                     # every used symbol has a code
    # complete: Kraft sum exactly 1 (fewer than two used symbols get a second, never-sent code of length 1)
    assert sum(1 << (limit - int(x)) for x in ln if x) == 1 << limit
    cost = int((f.astype(np.int64) * ln).sum())
    assert cost == pm_cost(list(f), limit), name
    assert cost >= huffman_cost(list(f))
    if name == "fibonacci_30":
        assert pm_cost(list(f), 29) < cost                           # the limit binds


# ------------------------------------------------------------------------------------------------
# members
# ------------------------------------------------------------------------------------------------
def member(H, data, m, mode):
    n = len(data)
    out = np.zeros(65536, np.uint8)
    ntok = C.c_uint32(0)
    mm = np.ascontiguousarray(m, np.uint32) if n else np.zeros(1, np.uint32)
    sz = H.hh_member(data, C.c_uint32(n), _p(mm), C.c_int(mode), _p(out), C.byref(ntok))
    return out[:sz].tobytes(), ntok.value


def find_matches(H, data):
    m = np.zeros(max(len(data), 1), np.uint32)
    H.hh_find_matches(data, C.c_uint32(len(data)), C.c_uint32(512), _p(m))
    return m[:len(data)]


def check_member(z, data):
    assert len(z) <= MAX_MEMBER
    assert z[:16] == HEADER
    assert struct.unpack_from("<H", z, 16)[0] == len(z) - 1
    crc, isize = struct.unpack_from("<II", z, len(z) - 8)
    assert crc == zlib.crc32(data) and isize == len(data)
    assert zlib.decompress(z[18:-8], wbits=-15) == data
    assert gzip.decompress(z + EOF_BLOCK) == data


def one_distance(n, d):
    m = np.zeros(n, np.uint32)
    for p in range(d, n):
        ln = min(258, n - p)
        if ln >= 3:
            m[p] = ln << 16 | (d - 1)
    return m


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_member_literals(H, mode):
    rng = np.random.default_rng(4)
    cases = [b"", b"A", b"AB", bytes(1000), bytes(rng.integers(0, 4, 5000, dtype=np.uint8))]
    if mode != 2:                                     # a dynamic block of random bytes is larger than the stored one
        cases.append(bytes(rng.integers(0, 256, BLOCK, dtype=np.uint8)))
    for data in cases:
        z, ntok = member(H, data, np.zeros(len(data), np.uint32), mode)
        assert ntok == len(data)
        check_member(z, data)
        if mode == 1:
            assert len(z) == 18 + 5 + len(data) + 8


@pytest.mark.parametrize("d", [1, 2, 3, 7, 258, 4096, 32768])
def test_member_one_distance(H, d):
    rng = np.random.default_rng(d)
    n = BLOCK if d < 32768 else 32768 + 3000
    pat = rng.integers(0, 256, d, dtype=np.uint8)
    data = bytes(np.resize(pat, n))
    z, ntok = member(H, data, one_distance(n, d), 2)
    check_member(z, data)
    assert ntok <= d + (n - d) // 258 + 2
    assert len(z) < 18 + 5 + n + 8 if d < 32768 else True


def inputs():
    rng = np.random.default_rng(5)
    yield "zeros", bytes(BLOCK)
    yield "ff", b"\xff" * BLOCK
    yield "random", bytes(rng.integers(0, 256, BLOCK, dtype=np.uint8))
    yield "small_random", bytes(rng.integers(0, 256, 300, dtype=np.uint8))
    for p in (1, 2, 3, 4, 7, 258, 259, 32768, 32769):
        pat = rng.integers(0, 256, p, dtype=np.uint8)
        yield "period_%d" % p, bytes(np.resize(pat, BLOCK))
    # exactly-3-byte matches: every 6 bytes = one of 4 random triples + 3 fresh random bytes
    tri = rng.integers(0, 256, (4, 3), dtype=np.uint8)
    yield "three_byte_matches", bytes(np.concatenate([np.concatenate([tri[rng.integers(0, 4)], rng.integers(0, 256, 3, dtype=np.uint8)])
                                                      for _ in range(BLOCK // 6)]))
    fw = np.array(fib(20), np.float64)
    yield "fibonacci_bytes", bytes(rng.choice(20, BLOCK, p=fw / fw.sum()).astype(np.uint8) * 13)
    yield "single_byte", b"\x2a" * 777
    # no match at all: a de Bruijn-like sequence of distinct 3-byte windows
    yield "no_match", bytes(np.array([(i * 7) % 256 for i in range(256)] + [(i * 11 + 3) % 256 for i in range(256)], np.uint8))
    for n in (0, 1, 2, 3, 257, 258, 259, BLOCK - 1):
        yield "len_%d" % n, bytes(rng.integers(0, 3, n, dtype=np.uint8))


@pytest.mark.parametrize("name,data", list(inputs()), ids=[x[0] for x in inputs()])
def test_member_found_matches(H, name, data):
    """the device's match rule and greedy parse, run on the host: valid members, stored where random, matches within the window"""
    m = find_matches(H, data)
    dist = (m & 0xFFFF) + 1
    ln = m >> 16
    assert (dist[m != 0] <= 32768).all() and ((ln[m != 0] >= 3) & (ln[m != 0] <= 258)).all()
    for p in np.nonzero(m)[0][:2000]:
        p = int(p); L = int(ln[p]); D = int(dist[p])
        assert D <= p and data[p:p + L] == data[p - D:p - D + L]
    z, _ = member(H, data, m, 0)
    check_member(z, data)
    if name in ("random", "small_random"):
        assert len(z) == 18 + 5 + len(data) + 8
    if name in ("zeros", "ff", "period_1", "period_2", "period_258"):
        assert len(z) < 1000                          # the first chunk of 512 positions only sees distance 1
    if name == "period_32769":
        assert not ((dist > 32768) & (m != 0)).any()


# ------------------------------------------------------------------------------------------------
# argument validation of the entry point
# ------------------------------------------------------------------------------------------------
def test_argument_validation():
    from nvbio_b200 import _lib
    from nvbio_b200._lib import BgzfOutStruct
    L = _lib.lib()
    tb = C.c_size_t(0)
    o = BgzfOutStruct(); o.d_out, o.capacity, o.d_block_offsets = 16, 1 << 20, 16
    fake = C.c_void_p(16)
    assert L.nvb_bgzf_compress(fake, C.c_uint64(100), None, None, C.byref(tb), None) == -1
    assert L.nvb_bgzf_compress(fake, C.c_uint64(100), C.byref(o), None, None, None) == -1
    assert L.nvb_bgzf_compress(None, C.c_uint64(100), C.byref(o), None, C.byref(tb), None) == -1
    o2 = BgzfOutStruct(); o2.d_out, o2.capacity, o2.d_block_offsets = 16, 1 << 20, None
    assert L.nvb_bgzf_compress(fake, C.c_uint64(100), C.byref(o2), None, C.byref(tb), None) == -1
    o3 = BgzfOutStruct(); o3.d_out, o3.capacity, o3.d_block_offsets = None, 1, 16
    assert L.nvb_bgzf_compress(fake, C.c_uint64(100), C.byref(o3), None, C.byref(tb), None) == -1
    assert L.nvb_bgzf_compress(fake, C.c_uint64(BLOCK << 32), C.byref(o), None, C.byref(tb), None) == -1
    assert L.nvb_bgzf_compress(fake, C.c_uint64((BLOCK << 32) - BLOCK + 1), C.byref(o), None, C.byref(tb), None) == -1
    # size query: NVB_E_TEMP_SIZE with at least a 64 KiB slot per block; a sizing call (no output) is valid too
    for n in (1, BLOCK, 3 * BLOCK + 1):
        tb.value = 0
        assert L.nvb_bgzf_compress(fake, C.c_uint64(n), C.byref(o), None, C.byref(tb), None) == -2
        assert tb.value >= -(-n // BLOCK) * 65536
        o4 = BgzfOutStruct(); o4.d_out, o4.capacity, o4.d_block_offsets = None, 0, 16
        assert L.nvb_bgzf_compress(fake, C.c_uint64(n), C.byref(o4), None, C.byref(tb), None) == -2
