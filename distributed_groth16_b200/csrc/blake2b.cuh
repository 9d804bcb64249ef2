// blake2b.cuh -- Blake2b (RFC 7693) with a state that can be exported and resumed: host code, no CUDA.
//
// A phase-1 contribution record of snarkjs stores the response hasher's state ("partialHash") and `powersoftau verify`
// resumes hashing from it, so the state itself is part of the file format.  This follows the RFC's reference
// implementation (Appendix C) step for step, including its lazy rule: a full 128-byte buffer is only compressed when
// more input arrives, so after exactly 128 k bytes the last block is still in the buffer, uncompressed, and the counter
// does not include it yet.  That rule is visible in the exported state.  Whole runs of input are copied with memcpy
// instead of byte by byte; the states it passes through are the reference's.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <string.h>

namespace b200zk {

struct blake2b_ctx {
    uint8_t b[128];      // input buffer
    uint64_t h[8];       // chained state
    uint64_t t[2];       // total number of bytes compressed
    size_t c;            // bytes in b
    size_t outlen;       // digest size
};

static const uint64_t blake2b_iv[8] = {
    0x6A09E667F3BCC908ull, 0xBB67AE8584CAA73Bull, 0x3C6EF372FE94F82Bull, 0xA54FF53A5F1D36F1ull,
    0x510E527FADE682D1ull, 0x9B05688C2B3E6C1Full, 0x1F83D9ABFB41BD6Bull, 0x5BE0CD19137E2179ull};

static inline uint64_t blake2b_rotr(uint64_t x, int n) { return (x >> n) | (x << (64 - n)); }

static inline void blake2b_compress(blake2b_ctx* ctx, int last) {
    static const uint8_t sigma[12][16] = {
        {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15}, {14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3},
        {11, 8, 12, 0, 5, 2, 15, 13, 10, 14, 3, 6, 7, 1, 9, 4}, {7, 9, 3, 1, 13, 12, 11, 14, 2, 6, 5, 10, 4, 0, 15, 8},
        {9, 0, 5, 7, 2, 4, 10, 15, 14, 1, 11, 12, 6, 8, 3, 13}, {2, 12, 6, 10, 0, 11, 8, 3, 4, 13, 7, 5, 15, 14, 1, 9},
        {12, 5, 1, 15, 14, 13, 4, 10, 0, 7, 6, 3, 9, 2, 8, 11}, {13, 11, 7, 14, 12, 1, 3, 9, 5, 0, 15, 4, 8, 6, 2, 10},
        {6, 15, 14, 9, 11, 3, 0, 8, 12, 2, 13, 7, 1, 4, 10, 5}, {10, 2, 8, 4, 7, 6, 1, 5, 15, 11, 9, 14, 3, 12, 13, 0},
        {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15}, {14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3}};
    uint64_t v[16], m[16];
    for (int i = 0; i < 8; ++i) {
        v[i] = ctx->h[i];
        v[i + 8] = blake2b_iv[i];
    }
    v[12] ^= ctx->t[0];
    v[13] ^= ctx->t[1];
    if (last) v[14] = ~v[14];
    for (int i = 0; i < 16; ++i) {
        uint64_t w = 0;
        for (int k = 7; k >= 0; --k) w = (w << 8) | ctx->b[8 * i + k];
        m[i] = w;
    }
#define B2B_G(a, b, c, d, x, y)                  \
    {                                            \
        v[a] = v[a] + v[b] + (x);                \
        v[d] = blake2b_rotr(v[d] ^ v[a], 32);    \
        v[c] = v[c] + v[d];                      \
        v[b] = blake2b_rotr(v[b] ^ v[c], 24);    \
        v[a] = v[a] + v[b] + (y);                \
        v[d] = blake2b_rotr(v[d] ^ v[a], 16);    \
        v[c] = v[c] + v[d];                      \
        v[b] = blake2b_rotr(v[b] ^ v[c], 63);    \
    }
    for (int i = 0; i < 12; ++i) {
        const uint8_t* s = sigma[i];
        B2B_G(0, 4, 8, 12, m[s[0]], m[s[1]]);
        B2B_G(1, 5, 9, 13, m[s[2]], m[s[3]]);
        B2B_G(2, 6, 10, 14, m[s[4]], m[s[5]]);
        B2B_G(3, 7, 11, 15, m[s[6]], m[s[7]]);
        B2B_G(0, 5, 10, 15, m[s[8]], m[s[9]]);
        B2B_G(1, 6, 11, 12, m[s[10]], m[s[11]]);
        B2B_G(2, 7, 8, 13, m[s[12]], m[s[13]]);
        B2B_G(3, 4, 9, 14, m[s[14]], m[s[15]]);
    }
#undef B2B_G
    for (int i = 0; i < 8; ++i) ctx->h[i] ^= v[i] ^ v[i + 8];
}

// unkeyed, outlen in 1..64
static inline void blake2b_init(blake2b_ctx* ctx, size_t outlen) {
    for (int i = 0; i < 8; ++i) ctx->h[i] = blake2b_iv[i];
    ctx->h[0] ^= 0x01010000ull ^ (uint64_t)outlen;
    ctx->t[0] = ctx->t[1] = 0;
    ctx->c = 0;
    ctx->outlen = outlen;
    memset(ctx->b, 0, sizeof(ctx->b));
}

static inline void blake2b_update(blake2b_ctx* ctx, const void* in, size_t inlen) {
    const uint8_t* p = (const uint8_t*)in;
    while (inlen > 0) {
        if (ctx->c == 128) {                         // buffer full and more input: compress it now (the lazy rule)
            ctx->t[0] += ctx->c;
            if (ctx->t[0] < ctx->c) ctx->t[1]++;
            blake2b_compress(ctx, 0);
            ctx->c = 0;
        }
        const size_t take = 128 - ctx->c < inlen ? 128 - ctx->c : inlen;
        memcpy(ctx->b + ctx->c, p, take);
        ctx->c += take;
        p += take;
        inlen -= take;
    }
}

static inline void blake2b_final(blake2b_ctx* ctx, uint8_t* out) {
    ctx->t[0] += ctx->c;
    if (ctx->t[0] < ctx->c) ctx->t[1]++;
    while (ctx->c < 128) ctx->b[ctx->c++] = 0;
    blake2b_compress(ctx, 1);
    for (size_t i = 0; i < ctx->outlen; ++i) out[i] = (uint8_t)(ctx->h[i >> 3] >> (8 * (i & 7)));
}

// The 216-byte exported state: b[128] || h[8] (u64 LE) || t[2] (u64 LE) || c (u32 LE) || outlen (u32 LE).  This is the
// context of blake2b-wasm (what snarkjs stores as a contribution's partialHash) as remembered, NOT pinned against a
// file written by snarkjs; this pair of functions is the one place that knows the layout.
static const size_t BLAKE2B_STATE_BYTES = 216;

static inline void blake2b_export(const blake2b_ctx* ctx, uint8_t* s) {
    memcpy(s, ctx->b, 128);
    for (int i = 0; i < 8; ++i)
        for (int k = 0; k < 8; ++k) s[128 + 8 * i + k] = (uint8_t)(ctx->h[i] >> (8 * k));
    for (int i = 0; i < 2; ++i)
        for (int k = 0; k < 8; ++k) s[192 + 8 * i + k] = (uint8_t)(ctx->t[i] >> (8 * k));
    for (int k = 0; k < 4; ++k) {
        s[208 + k] = (uint8_t)((uint32_t)ctx->c >> (8 * k));
        s[212 + k] = (uint8_t)((uint32_t)ctx->outlen >> (8 * k));
    }
}

// false when the state is not one blake2b_export can produce (c > 128, outlen outside 1..64)
static inline bool blake2b_import(blake2b_ctx* ctx, const uint8_t* s) {
    memcpy(ctx->b, s, 128);
    for (int i = 0; i < 8; ++i) {
        uint64_t w = 0;
        for (int k = 7; k >= 0; --k) w = (w << 8) | s[128 + 8 * i + k];
        ctx->h[i] = w;
    }
    for (int i = 0; i < 2; ++i) {
        uint64_t w = 0;
        for (int k = 7; k >= 0; --k) w = (w << 8) | s[192 + 8 * i + k];
        ctx->t[i] = w;
    }
    uint32_t c = 0, outlen = 0;
    for (int k = 3; k >= 0; --k) {
        c = (c << 8) | s[208 + k];
        outlen = (outlen << 8) | s[212 + k];
    }
    ctx->c = c;
    ctx->outlen = outlen;
    return c <= 128 && outlen >= 1 && outlen <= 64;
}

}  // namespace b200zk
