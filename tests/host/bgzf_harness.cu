// tests/host/bgzf_harness.cu -- TEST INFRASTRUCTURE.
// Runs the per-block routines of nvb_bgzf_compress (bgzf_core.cuh) serially on the CPU: the chunked CRC-32 with its shift combine,
// length-limited code construction, the match finder in the device's chunk order, and whole members assembled from per-position
// matches under the greedy parse (the parse the device's parallel walk converges to).  Built by tests/test_bgzf_host.py.
#include "../../nvbio_b200/csrc/bgzf_core.cuh"
#include <vector>

using namespace nvb;

static const uint32_t* crc_table()
{
    static uint32_t t[256];
    static bool init = false;
    if (!init) { for (uint32_t i = 0; i < 256; ++i) t[i] = crc32_table_entry(i); init = true; }
    return t;
}

// CRC-32 of p[0..n) computed chunk by chunk from zero-start registers and combined with crc32_shift
extern "C" uint32_t hh_crc32(const uint8_t* p, uint64_t n, uint32_t chunk)
{
    uint32_t c = crc32_shift(0xFFFFFFFFu, n);
    for (uint64_t a = 0; a < n; a += chunk) {
        const uint32_t len = (uint32_t)(n - a < chunk ? n - a : chunk);
        c ^= crc32_shift(crc32_raw(crc_table(), p + a, len, 0u), n - a - len);
    }
    return ~c;
}

extern "C" uint32_t hh_gf2_mulmod(uint32_t a, uint32_t b) { return gf2_mulmod(a, b); }

// code lengths of at most `limit` bits for f[0..n) (n <= 286); returns the number of used symbols after the bump to two
extern "C" uint32_t hh_code_lengths(const uint32_t* f, uint32_t n, uint32_t limit, uint8_t* len)
{
    std::vector<uint32_t> g(f, f + n);
    BgzfPm* pm = new BgzfPm;
    code_lengths(g.data(), n, limit, len, *pm);
    delete pm;
    uint32_t m = 0;
    for (uint32_t s = 0; s < n; ++s) m += g[s] != 0u;
    return m;
}

static std::vector<uint32_t> padded(const uint8_t* in, uint32_t n)
{
    std::vector<uint32_t> w((n + 16u) / 4u + 1u, 0u);
    memcpy(w.data(), in, n);
    return w;
}

// per-position matches as the device finds them: chunks of `chunk` positions look up the hash table as the earlier chunks left it,
// then insert their own positions (the latest position per hash wins, as atomicMax does)
extern "C" void hh_find_matches(const uint8_t* in, uint32_t n, uint32_t chunk, uint32_t* m)
{
    std::vector<uint32_t> w = padded(in, n);
    const uint8_t* s = (const uint8_t*)w.data();
    std::vector<uint32_t> table(1u << BGZF_HASH_BITS, 0u);
    for (uint32_t c0 = 0; c0 < n; c0 += chunk) {
        const uint32_t c1 = n - c0 < chunk ? n : c0 + chunk;
        for (uint32_t p = c0; p < c1; ++p) m[p] = find_match(s, n, p, p + 4u <= n ? table[bgzf_hash(s, p)] : 0u);
        for (uint32_t p = c0; p < c1; ++p)
            if (p + 4u <= n) { uint32_t& e = table[bgzf_hash(s, p)]; if (p + 1u > e) e = p + 1u; }
    }
}

// one member of the n <= 0xFF00 bytes `in` from per-position matches m (0, or (length << 16) | (distance - 1)) under the greedy parse.
// mode 0: the smaller of the dynamic and the stored block (stored on a tie), 1: stored, 2: dynamic.  out: BGZF_SLOT bytes.  Returns the
// member's size; *tokens = the number of tokens.
extern "C" uint32_t hh_member(const uint8_t* in, uint32_t n, const uint32_t* m, int mode, uint8_t* out, uint32_t* tokens)
{
    std::vector<uint32_t> w = padded(in, n);
    std::vector<uint8_t> mlen(n + 1u, 0u);
    std::vector<uint16_t> dist(n + 1u, 0u);
    std::vector<uint32_t> mbit(n / 32u + 1u, 0u);
    for (uint32_t p = 0; p < n; ++p)
        if (m[p]) { mlen[p] = (uint8_t)((m[p] >> 16) - 3u); dist[p] = (uint16_t)(m[p] & 0xFFFFu); mbit[p >> 5] |= 1u << (p & 31u); }
    BgzfParse v{ (const uint8_t*)w.data(), mlen.data(), mbit.data(), dist.data() };
    std::vector<uint32_t> tok;
    for (uint32_t p = 0; p < n; p += token_advance(v, p)) tok.push_back(p);
    *tokens = (uint32_t)tok.size();

    uint32_t hlit[BGZF_NLIT] = { 0 }, hdist[BGZF_NDIST] = { 0 };
    for (uint32_t p : tok) count_token(v, p, hlit, hdist);
    hlit[256] = 1u;
    BgzfCodes* c = new BgzfCodes;
    BgzfPm* pm = new BgzfPm;
    code_lengths(hlit, BGZF_NLIT, BGZF_MAX_BITS, c->lit_len, *pm);
    code_lengths(hdist, BGZF_NDIST, BGZF_MAX_BITS, c->dist_len, *pm);
    plan_header(*c, *pm);
    uint32_t bits = c->header_bits + c->lit_len[256];
    for (uint32_t p : tok) bits += put_token(v, *c, p, nullptr, 0u);
    const uint32_t dbytes = (bits + 7u) / 8u;
    const bool stored = mode == 1 || (mode == 0 && dbytes >= n + 5u);

    std::vector<uint32_t> o(BGZF_SLOT / 4u + 1u, 0u);
    uint8_t* o8 = (uint8_t*)o.data();
    uint32_t member;
    if (stored) {
        member = BGZF_HDR + 5u + n + BGZF_FTR;
        for (uint32_t k = 0; k < 5u; ++k) o8[BGZF_HDR + k] = stored_header_byte(k, n);
        memcpy(o8 + BGZF_HDR + 5u, in, n);
    } else {
        member = BGZF_HDR + dbytes + BGZF_FTR;
        uint32_t pos = 8u * BGZF_HDR;
        pos += write_header(o.data(), pos, *c);
        for (uint32_t p : tok) pos += put_token(v, *c, p, o.data(), pos);
        put_bits(o.data(), pos, c->lit_code[256], c->lit_len[256]);
    }
    for (uint32_t k = 0; k < BGZF_HDR; ++k) o8[k] = member_header_byte(k, member);
    const uint32_t crc = hh_crc32(in, n, 128u);
    for (uint32_t k = 0; k < BGZF_FTR; ++k) o8[member - BGZF_FTR + k] = member_footer_byte(k, crc, n);
    memcpy(out, o8, member);
    delete c; delete pm;
    return member;
}
