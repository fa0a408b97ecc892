// mortal_b200 — gzip members (RFC 1952) inflated (RFC 1951) on the device, straight into the text buffer k_mjai_decode reads, and
// a key count over that text (include/mjx_logio.h).
//
// Device: one warp per file (k_gunzip). DEFLATE cannot be split without speculation, so every lane walks the same bit stream:
// the lanes hold identical bit buffers and take identical branches, which keeps the warp converged without broadcasts. The
// lanes share the work that has width: filling the canonical-code lookup tables (in shared memory, per warp), copying matches
// (lane j writes byte j of every 32, read from the period `distance` before the match, so an overlapping copy needs no ordering
// inside the match), copying stored blocks, and the CRC-32 pass over the output (per-lane chunk CRCs combined with GF(2)
// multiplications by x^(8n)). Lane 0 writes the literals. -DMJX_HOST_EMUL builds the same code with one lane playing all 32 in
// turn for tests/host_emul/emul_inflate.cc.
//
// What is accepted is deliberately narrower than zlib where zlib is lenient: a literal/length or code-length code must be
// complete; a distance code may be complete, empty, or a single length-1 code (what zlib accepts). Everything Python's zlib
// writes is complete.
#pragma once
#include "../../include/mjx_logio.h"
#include "mjx_port.cuh"
#include "mjx_types.cuh"

namespace mjx {

constexpr int GZ_WARPS = 4;
constexpr int GZ_LIT_BITS = 10;   // the literal/length table's index width; longer codes take the canonical walk
constexpr int GZ_DIST_BITS = 8;   // the distance table's; the code-length code (7 bits at most) is built into the same space
constexpr int GZ_X8 = 48;         // x^(8 * 2^k) mod P for k < 48: outputs below 2^48 bytes
constexpr u32 GZ_POLY = 0xEDB88320u;  // CRC-32, bit-reflected

struct GzWarp {  // per-warp shared scratch
    u16 lit[1 << GZ_LIT_BITS];    // entry: symbol | code length << 9; 0 = not a short code
    u16 dist[1 << GZ_DIST_BITS];
    u16 codes[320];               // the canonical code of every symbol of the table being built
    u16 lit_sorted[288], dist_sorted[32];  // symbols ordered by (length, symbol), for the canonical walk
    u16 lit_cnt[16], dist_cnt[16];
    u8 lens[320];                 // literal/length lengths, then distance lengths
    u8 cl_lens[19];
    int build;                    // the table builder's verdict, for every lane
};

#ifdef MJX_HOST_EMUL
#define GZ_LANES(l) for (int l = 0; l < 32; l++)
#define GZ_LEAD if (true)
#else
#define GZ_LANES(l) for (int l = lane, l##_once_ = 1; l##_once_; l##_once_ = 0)
#define GZ_LEAD if (lane == 0)
#endif

MJX_CONST u16 GZ_LEN_BASE[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115,
                                 131, 163, 195, 227, 258};
MJX_CONST u8 GZ_LEN_EXTRA[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
MJX_CONST u16 GZ_DIST_BASE[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537,
                                  2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
MJX_CONST u8 GZ_DIST_EXTRA[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
MJX_CONST u8 GZ_CL_ORDER[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

// ---- CRC-32 -----------------------------------------------------------------------------------------------------------------
// Polynomials mod P in the reflected layout: the coefficient of x^i is bit 31 - i, so 1 = 0x80000000.
MJX_HD u32 gz_mulmod(u32 a, u32 b) {
    u32 p = 0;
    for (int i = 0; i < 32; i++) {
        if (a & (0x80000000u >> i)) p ^= b;
        b = (b >> 1) ^ ((b & 1) ? GZ_POLY : 0);  // b *= x
    }
    return p;
}

MJX_HD u32 gz_crc_entry(u32 c) {
    for (int k = 0; k < 8; k++) c = (c >> 1) ^ ((c & 1) ? GZ_POLY : 0);
    return c;
}

// x8[k] = x^(8 * 2^k) mod P; x^(8n) is the product of the x8[k] of n's set bits
MJX_HD void gz_x8_table(u32* x8) {
    x8[0] = 0x80000000u >> 8;
    for (int k = 1; k < GZ_X8; k++) x8[k] = gz_mulmod(x8[k - 1], x8[k - 1]);
}

MJX_HD u32 gz_shift(u32 c, long long n, const u32* x8) {  // c * x^(8n) mod P: the CRC register after n zero bytes
    for (int k = 0; n && k < GZ_X8; k++, n >>= 1)
        if (n & 1) c = gz_mulmod(c, x8[k]);
    return c;
}

// zlib.crc32 of p[0, n): lane l's chunk register (started at 0), shifted past the bytes after its chunk; the XOR of the lanes'
// terms is the register of the whole from 0, and the initial 0xFFFFFFFF's contribution is added by the same shift
MJX_D u32 gz_crc32(const u8* p, long long n, const u32* table, const u32* x8, int lane) {
    const long long chunk = (n + 31) / 32;
    u32 acc = 0;
    GZ_LANES(l) {
        const long long a = min(n, (long long)l * chunk), b = min(n, a + chunk);
        u32 r = 0;
        for (long long k = a; k < b; k++) r = table[(r ^ p[k]) & 0xFF] ^ (r >> 8);
        acc ^= gz_shift(r, n - b, x8);
    }
#ifndef MJX_HOST_EMUL
    for (int s = 16; s; s >>= 1) acc ^= __shfl_xor_sync(~0u, acc, s);
#endif
    return ~(acc ^ gz_shift(0xFFFFFFFFu, n, x8));
}

// ---- bit reader ---------------------------------------------------------------------------------------------------------------
// buf holds n >= 0 unread bits, LSB first; the next byte to load is p. Bytes at or past `end` read as zero, so a stream that runs
// past its file is caught by gz_overrun rather than by reading another file's bytes.
struct GzBits {
    const u8* g;
    long long n_gz, p, end;
    u64 buf;
    int n;
};

MJX_D u64 gz_load8(const GzBits& B, long long p) {
    if (p >= B.end) return 0;
    u64 v = 0;
#ifdef MJX_HOST_EMUL
    if (p + 8 <= B.end) std::memcpy(&v, B.g + p, 8);
    else for (long long k = 0; p + k < B.end; k++) v |= (u64)B.g[p + k] << (8 * k);
#else
    const long long a = p & ~7LL;  // gz is 8-byte aligned (mjx_gunzip_dev checks)
    if (a + 16 <= B.n_gz) {
        const u64 lo = __ldg(reinterpret_cast<const unsigned long long*>(B.g + a));
        const u64 hi = __ldg(reinterpret_cast<const unsigned long long*>(B.g + a + 8));
        const int s = (int)(p & 7) * 8;
        v = s ? (lo >> s) | (hi << (64 - s)) : lo;
    } else {
        for (int k = 0; k < 8 && p + k < B.n_gz; k++) v |= (u64)B.g[p + k] << (8 * k);
    }
    if (p + 8 > B.end) v &= (1ULL << (8 * (B.end - p))) - 1;
#endif
    return v;
}

MJX_D void gz_refill(GzBits& B) {  // afterwards n >= 56
    if (B.n <= 56) {
        B.buf |= gz_load8(B, B.p) << B.n;
        const int adv = (63 - B.n) >> 3;
        B.p += adv;
        B.n += 8 * adv;
    }
}

MJX_D u32 gz_take(GzBits& B, int k) {
    const u32 v = (u32)(B.buf & ((1ULL << k) - 1));
    B.buf >>= k;
    B.n -= k;
    return v;
}

MJX_D bool gz_overrun(const GzBits& B) { return B.p * 8 - B.n > B.end * 8; }

// ---- canonical codes ------------------------------------------------------------------------------------------------------------
enum : int { GZ_CODE_OK = 0, GZ_CODE_OVER = 1, GZ_CODE_INCOMPLETE = 2 };

MJX_D u32 gz_rev(u32 c, int len) {
#ifdef MJX_HOST_EMUL
    u32 r = 0;
    for (int k = 0; k < len; k++) r |= ((c >> k) & 1) << (len - 1 - k);
    return r;
#else
    return __brev(c) >> (32 - len);
#endif
}

// The decode table of the code with lengths lens[0, n): table[bits] (entries for codes of at most `bits` bits), cnt[len] and
// sorted[] for the canonical walk. Returns GZ_CODE_* | number of codes << 4 | the longest length << 16, the same for every lane.
MJX_D int gz_build(GzWarp& W, const u8* lens, int n, u16* table, int bits, u16* cnt, u16* sorted, int lane) {
    GZ_LEAD {
        for (int l = 0; l < 16; l++) cnt[l] = 0;
        for (int s = 0; s < n; s++) cnt[lens[s]]++;
        cnt[0] = 0;
        int left = 1, res = GZ_CODE_OK, codes = 0, longest = 0;
        u16 offs[16], next[16];
        u32 code = 0;
        offs[0] = next[0] = 0;
        for (int l = 1; l < 16; l++) {
            left = 2 * left - cnt[l];
            if (left < 0) res = GZ_CODE_OVER;
            codes += cnt[l];
            if (cnt[l]) longest = l;
            offs[l] = (u16)(l == 1 ? 0 : offs[l - 1] + cnt[l - 1]);
            code = (code + cnt[l - 1]) << 1;
            next[l] = (u16)code;
        }
        if (res == GZ_CODE_OK && left > 0) res = GZ_CODE_INCOMPLETE;
        if (res != GZ_CODE_OVER)
            for (int s = 0; s < n; s++)
                if (lens[s]) {
                    sorted[offs[lens[s]]++] = (u16)s;
                    W.codes[s] = next[lens[s]]++;
                }
        W.build = res | codes << 4 | longest << 16;
    }
    MJX_SYNCWARP();
    const int r = W.build;
    if ((r & 15) == GZ_CODE_OVER) return r;
    GZ_LANES(l) for (int k = l; k < (1 << bits); k += 32) table[k] = 0;
    MJX_SYNCWARP();
    GZ_LANES(l) for (int s = l; s < n; s += 32) {
        const int len = lens[s];
        if (len && len <= bits)
            for (u32 k = gz_rev(W.codes[s], len); k < (1u << bits); k += 1u << len) table[k] = (u16)(s | len << 9);
    }
    MJX_SYNCWARP();
    return r;
}

// the next symbol of a code (B.n >= 15), or -1 for a bit pattern no code has
MJX_D int gz_decode(GzBits& B, const u16* table, int bits, const u16* cnt, const u16* sorted) {
    const u16 e = table[B.buf & ((1u << bits) - 1)];
    if (e) {
        gz_take(B, e >> 9);
        return e & 511;
    }
    int code = 0, first = 0, index = 0;  // the canonical walk, one bit at a time
    for (int len = 1; len < 16; len++) {
        code |= (int)((B.buf >> (len - 1)) & 1);
        const int c = cnt[len];
        if (code - first < c) {
            gz_take(B, len);
            return sorted[index + code - first];
        }
        index += c;
        first = (first + c) << 1;
        code <<= 1;
    }
    return -1;
}

// ---- one member ---------------------------------------------------------------------------------------------------------------
// The deflate stream at B into out[0, cap): MJX_GZ_OK with *olen = the output length, or the status that declines it.
MJX_D int gz_inflate(GzWarp& W, GzBits& B, u8* out, long long cap, long long* olen, int lane) {
    long long o = 0;
    for (;;) {
        gz_refill(B);
        if (gz_overrun(B)) return MJX_GZ_TRUNCATED;
        const u32 final_ = gz_take(B, 1), type = gz_take(B, 2);
        if (type == 3) return MJX_GZ_BLOCK;
        if (type == 0) {  // stored: to the byte boundary, LEN, NLEN, LEN bytes
            gz_take(B, B.n & 7);
            gz_refill(B);
            const u32 len = gz_take(B, 16), nlen = gz_take(B, 16);
            if (gz_overrun(B)) return MJX_GZ_TRUNCATED;
            if (len != (~nlen & 0xFFFFu)) return MJX_GZ_BLOCK;
            const long long s = B.p - B.n / 8;
            if (s + len > B.end) return MJX_GZ_TRUNCATED;
            if (o + len > cap) return MJX_GZ_SIZE;
            GZ_LANES(l) for (long long k = l; k < len; k += 32) out[o + k] = B.g[s + k];
            o += len;
            B.p = s + len;
            B.n = 0;
            B.buf = 0;
        } else {
            if (type == 1) {  // fixed codes: 0-143 8 bits, 144-255 9, 256-279 7, 280-287 8; 32 distance codes of 5 bits
                GZ_LANES(l) for (int s = l; s < 320; s += 32)
                    W.lens[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : s < 288 ? 8 : 5;
                MJX_SYNCWARP();
                gz_build(W, W.lens, 288, W.lit, GZ_LIT_BITS, W.lit_cnt, W.lit_sorted, lane);
                gz_build(W, W.lens + 288, 32, W.dist, GZ_DIST_BITS, W.dist_cnt, W.dist_sorted, lane);
            } else {  // dynamic: HLIT, HDIST, HCLEN, the code-length code, then the lengths of both codes
                const int hlit = gz_take(B, 5) + 257, hdist = gz_take(B, 5) + 1, hclen = gz_take(B, 4) + 4;
                if (hlit > 286 || hdist > 30) return MJX_GZ_CODES;
                for (int k = 0; k < 19; k++) {
                    if (k % 8 == 0) gz_refill(B);
                    const int v = k < hclen ? (int)gz_take(B, 3) : 0;
                    GZ_LEAD W.cl_lens[GZ_CL_ORDER[k]] = (u8)v;
                }
                if (gz_overrun(B)) return MJX_GZ_TRUNCATED;
                MJX_SYNCWARP();
                if ((gz_build(W, W.cl_lens, 19, W.dist, 7, W.dist_cnt, W.dist_sorted, lane) & 15) != GZ_CODE_OK) return MJX_GZ_CODES;
                const int total = hlit + hdist;
                int prev = -1;
                for (int i = 0; i < total;) {
                    gz_refill(B);
                    if (gz_overrun(B)) return MJX_GZ_TRUNCATED;
                    const int sym = gz_decode(B, W.dist, 7, W.dist_cnt, W.dist_sorted);
                    if (sym < 0) return MJX_GZ_CODES;
                    int rep = 1, val = sym;
                    if (sym == 16) {
                        if (prev < 0) return MJX_GZ_CODES;
                        rep = 3 + gz_take(B, 2); val = prev;
                    } else if (sym == 17) {
                        rep = 3 + gz_take(B, 3); val = 0;
                    } else if (sym == 18) {
                        rep = 11 + gz_take(B, 7); val = 0;
                    }
                    if (i + rep > total) return MJX_GZ_CODES;
                    GZ_LEAD for (int k = 0; k < rep; k++) W.lens[i + k] = (u8)val;
                    i += rep;
                    prev = val;
                }
                MJX_SYNCWARP();
                if (W.lens[256] == 0) return MJX_GZ_CODES;
                if ((gz_build(W, W.lens, hlit, W.lit, GZ_LIT_BITS, W.lit_cnt, W.lit_sorted, lane) & 15) != GZ_CODE_OK)
                    return MJX_GZ_CODES;
                const int d = gz_build(W, W.lens + hlit, hdist, W.dist, GZ_DIST_BITS, W.dist_cnt, W.dist_sorted, lane);
                const int dcodes = (d >> 4) & 0xFFF, dlongest = d >> 16;
                if ((d & 15) == GZ_CODE_OVER || ((d & 15) == GZ_CODE_INCOMPLETE && dcodes > 1) ||
                    ((d & 15) == GZ_CODE_INCOMPLETE && dcodes == 1 && dlongest != 1))
                    return MJX_GZ_CODES;
            }
            for (;;) {  // the symbols of the block
                gz_refill(B);
                if (gz_overrun(B)) return MJX_GZ_TRUNCATED;
                const int sym = gz_decode(B, W.lit, GZ_LIT_BITS, W.lit_cnt, W.lit_sorted);
                if (sym < 0) return MJX_GZ_SYMBOL;
                if (sym < 256) {
                    if (o >= cap) return MJX_GZ_SIZE;
                    GZ_LEAD out[o] = (u8)sym;
                    o++;
                    continue;
                }
                if (sym == 256) break;
                if (sym >= 286) return MJX_GZ_SYMBOL;
                const int len = GZ_LEN_BASE[sym - 257] + (int)gz_take(B, GZ_LEN_EXTRA[sym - 257]);
                gz_refill(B);
                const int ds = gz_decode(B, W.dist, GZ_DIST_BITS, W.dist_cnt, W.dist_sorted);
                if (ds < 0 || ds >= 30) return MJX_GZ_SYMBOL;
                const int dist = GZ_DIST_BASE[ds] + (int)gz_take(B, GZ_DIST_EXTRA[ds]);
                if (gz_overrun(B)) return MJX_GZ_TRUNCATED;
                if (dist > o) return MJX_GZ_DISTANCE;
                if (o + len > cap) return MJX_GZ_SIZE;
                MJX_SYNCWARP();  // the bytes before o, written by any lane, are visible to every lane
                GZ_LANES(l) for (int k = l; k < len; k += 32) out[o + k] = out[o - dist + (dist >= len ? k : k % dist)];
                o += len;
            }
        }
        if (final_) break;
    }
    *olen = o;
    return MJX_GZ_OK;
}

// File [gb, ge) of g (n_gz bytes in all) into out[0, cap): the header as Python 3.12's gzip._read_gzip_header reads it (magic,
// CM = 8, FEXTRA / FNAME / FCOMMENT / FHCRC skipped, the rest ignored), the deflate stream, the trailer's CRC-32 and ISIZE, and
// nothing after the trailer. Every lane returns the same status.
MJX_D int gz_member(GzWarp& W, const u8* g, long long n_gz, long long gb, long long ge, u8* out, long long cap, const u32* crc_table,
                    const u32* x8, int lane) {
    long long q = gb;
    if (ge - q < 2 || g[q] != 0x1F || g[q + 1] != 0x8B) return MJX_GZ_NOT_GZIP;
    if (ge - q < 10) return MJX_GZ_HEADER;
    if (g[q + 2] != 8) return MJX_GZ_NOT_GZIP;
    const int flg = g[q + 3];
    q += 10;
    if (flg & 4) {  // FEXTRA
        if (ge - q < 2) return MJX_GZ_HEADER;
        const long long xlen = g[q] | g[q + 1] << 8;
        q += 2;
        if (ge - q < xlen) return MJX_GZ_HEADER;
        q += xlen;
    }
    for (int f = 8; f <= 16; f += 8)  // FNAME, FCOMMENT: zero-terminated
        if (flg & f) {
            while (q < ge && g[q] != 0) q++;
            if (q >= ge) return MJX_GZ_HEADER;
            q++;
        }
    if (flg & 2) {  // FHCRC (not verified, as Python does not)
        if (ge - q < 2) return MJX_GZ_HEADER;
        q += 2;
    }
    GzBits B{g, n_gz, q, ge, 0, 0};
    long long olen = 0;
    const int st = gz_inflate(W, B, out, cap, &olen, lane);
    if (st != MJX_GZ_OK) return st;
    const long long t = (B.p * 8 - B.n + 7) >> 3;  // the trailer starts at the byte after the last block
    if (t + 8 > ge) return MJX_GZ_TRUNCATED;
    const u32 crc = (u32)g[t] | (u32)g[t + 1] << 8 | (u32)g[t + 2] << 16 | (u32)g[t + 3] << 24;
    const u32 isize = (u32)g[t + 4] | (u32)g[t + 5] << 8 | (u32)g[t + 6] << 16 | (u32)g[t + 7] << 24;
    if (olen != cap || (u32)olen != isize) return MJX_GZ_SIZE;
    if (t + 8 != ge) return MJX_GZ_TRAILING;
    MJX_SYNCWARP();
    if (gz_crc32(out, olen, crc_table, x8, lane) != crc) return MJX_GZ_CRC;
    return MJX_GZ_OK;
}

// ---- key counts ---------------------------------------------------------------------------------------------------------------
struct GzKeys {
    u8 b[MJX_COUNT_KEYS_MAX][MJX_COUNT_KEY_BYTES];
    int len[MJX_COUNT_KEYS_MAX];
    int n;
};

MJX_D bool gz_key_at(const u8* p, long long left, const GzKeys& K, int k) {
    if (left < K.len[k]) return false;
    for (int j = 0; j < K.len[k]; j++)
        if (p[j] != K.b[k][j]) return false;
    return true;
}

// bytes.count of every key over p[0, len): the lanes test 32 positions at a time, and every lane walks the window's matches left
// to right, taking a match that starts at or after the end of the last one taken
MJX_D void gz_count_keys(const u8* p, long long len, const GzKeys& K, long long* cnt, int lane) {
    long long next[MJX_COUNT_KEYS_MAX];
#pragma unroll
    for (int k = 0; k < MJX_COUNT_KEYS_MAX; k++) cnt[k] = next[k] = 0;
    for (long long base = 0; base < len; base += 32) {
#pragma unroll
        for (int k = 0; k < MJX_COUNT_KEYS_MAX; k++) {
            if (k >= K.n) break;
            unsigned m = 0;
            GZ_LANES(l) {
                const long long pos = base + l;
                const bool hit = pos < len && p[pos] == K.b[k][0] && gz_key_at(p + pos, len - pos, K, k);
#ifdef MJX_HOST_EMUL
                m |= (unsigned)hit << l;
#else
                m = __ballot_sync(~0u, hit);
#endif
            }
            while (m) {
                const long long q = base + mjx_ffsll(m) - 1;
                m &= m - 1;
                if (q >= next[k]) { cnt[k]++; next[k] = q + K.len[k]; }
            }
        }
    }
}

#ifndef MJX_HOST_EMUL
__global__ void __launch_bounds__(GZ_WARPS * 32) k_gunzip(int n, const u8* gz, long long n_gz, const i64* gz_off, u8* out,
                                                          long long n_out, const i64* out_off, i32* status) {
    __shared__ GzWarp s_w[GZ_WARPS];
    __shared__ u32 s_crc[256], s_x8[GZ_X8];
    for (int k = threadIdx.x; k < 256; k += blockDim.x) s_crc[k] = gz_crc_entry(k);
    if (threadIdx.x == 0) gz_x8_table(s_x8);
    __syncthreads();
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int i = blockIdx.x * GZ_WARPS + wid;
    if (i >= n) return;
    const long long gb = gz_off[i], ge = gz_off[i + 1], ob = out_off[i], oe = out_off[i + 1];
    int st;
    if (ob < 0 || oe < ob || oe > n_out) st = MJX_GZ_SIZE;
    else if (gb < 0 || ge < gb || ge > n_gz) st = MJX_GZ_NOT_GZIP;
    else st = gz_member(s_w[wid], gz, n_gz, gb, ge, out + ob, oe - ob, s_crc, s_x8, lane);
    if (lane == 0) status[i] = st;
}

__global__ void __launch_bounds__(GZ_WARPS * 32) k_count_keys(int n_logs, const u8* text, long long n_bytes, const i64* log_off,
                                                              GzKeys K, i64* counts) {
    const int lane = threadIdx.x & 31;
    const int i = blockIdx.x * GZ_WARPS + (threadIdx.x >> 5);
    if (i >= n_logs) return;
    long long lb = log_off[i], le = log_off[i + 1];
    if (lb < 0 || le < lb || le > n_bytes) lb = le = 0;
    long long cnt[MJX_COUNT_KEYS_MAX];
    gz_count_keys(text + lb, le - lb, K, cnt, lane);
#pragma unroll
    for (int k = 0; k < MJX_COUNT_KEYS_MAX; k++)
        if (k == lane && k < K.n) counts[(long long)i * K.n + k] = cnt[k];
}
#endif

}  // namespace mjx
