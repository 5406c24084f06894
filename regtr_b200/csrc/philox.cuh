// Counter-based randomness shared by the training-data kernels: Philox4x32-10 normals and uniforms, and the keyed
// Feistel bijection behind every permutation and subset.  A draw depends only on (seed, step, pair, side, index).
#pragma once
#include <cuda_runtime.h>

#include "../../include/regtr_b200.h"

namespace {

// ------------------------------------------------------------------------------------------- counter-based randomness
// Philox4x32-10 (Salmon et al., SC'11).
struct U4 { unsigned x, y, z, w; };

__device__ __forceinline__ U4 philox(U4 c, unsigned k0, unsigned k1) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const unsigned long long p0 = (unsigned long long)0xD2511F53u * c.x;
        const unsigned long long p1 = (unsigned long long)0xCD9E8D57u * c.z;
        c = U4{(unsigned)(p1 >> 32) ^ c.y ^ k0, (unsigned)p1, (unsigned)(p0 >> 32) ^ c.w ^ k1, (unsigned)p0};
        k0 += 0x9E3779B9u;
        k1 += 0xBB67AE85u;
    }
    return c;
}

struct Keys { unsigned k0, k1, s0, s1; };   // Philox key = seed, counter words 2..3 = step

__device__ __forceinline__ Keys make_keys(unsigned long long seed, unsigned long long step) {
    return Keys{(unsigned)seed, (unsigned)(seed >> 32), (unsigned)step, (unsigned)(step >> 32)};
}

// Keyed bijection of [0, n): an 8-round balanced Feistel network over the smallest even bit width whose range holds
// n, with cycle walking (Black & Rogaway, CT-RSA'02).  The inverse walks the inverse network, so the inverse map
// needs no scatter and no sort.  Round keys: two Philox blocks at counter (2^31 + {0,1}, 2 pair + side, step).
struct Perm {
    unsigned n, half, mask, k[8];
    bool on;
};

__device__ __forceinline__ unsigned feistel_f(unsigned r, unsigned key) {
    unsigned h = (r ^ key) * 0x9E3779B1u;
    h ^= h >> 15; h *= 0x85EBCA77u;
    h ^= h >> 13; h *= 0xC2B2AE3Du;
    return h ^ (h >> 16);
}

__device__ __forceinline__ Perm make_perm(int n, bool on, const Keys& ks, int pair, int side) {
    Perm p;
    p.n = (unsigned)n;
    p.on = on && n > 1;
    int bits = 2;
    while ((1u << bits) < (unsigned)n) ++bits;
    bits += bits & 1;
    p.half = bits / 2;
    p.mask = (1u << p.half) - 1u;
    const unsigned pc = 2u * (unsigned)pair + (unsigned)side;
    const U4 a = philox(U4{0x80000000u, pc, ks.s0, ks.s1}, ks.k0, ks.k1);
    const U4 b = philox(U4{0x80000001u, pc, ks.s0, ks.s1}, ks.k0, ks.k1);
    p.k[0] = a.x; p.k[1] = a.y; p.k[2] = a.z; p.k[3] = a.w; p.k[4] = b.x; p.k[5] = b.y; p.k[6] = b.z; p.k[7] = b.w;
    return p;
}

// output position -> input index (ShufflePoints' `src_idx[k]`)
__device__ __forceinline__ unsigned perm_fwd(const Perm& p, unsigned x) {
    if (!p.on) return x;
    do {
        unsigned L = x >> p.half, R = x & p.mask;
#pragma unroll
        for (int r = 0; r < 8; ++r) { const unsigned t = L ^ (feistel_f(R, p.k[r]) & p.mask); L = R; R = t; }
        x = (L << p.half) | R;
    } while (x >= p.n);
    return x;
}

// input index -> output position
__device__ __forceinline__ unsigned perm_inv(const Perm& p, unsigned y) {
    if (!p.on) return y;
    do {
        unsigned L = y >> p.half, R = y & p.mask;
#pragma unroll
        for (int r = 7; r >= 0; --r) { const unsigned t = R ^ (feistel_f(L, p.k[r]) & p.mask); R = L; L = t; }
        y = (L << p.half) | R;
    } while (y >= p.n);
    return y;
}

__device__ __forceinline__ double u01(unsigned v) { return ((double)v + 0.5) * 2.3283064365386963e-10; }   // (0, 1)

// ------------------------------------------------------------------------------------------ transformer dropout
// Keep decisions of the cross-encoder's six dropouts (regtr_dropout_args in include/regtr_b200.h).  Same Philox key
// and counter words 2..3 as the augmentation draws of (seed, step); the streams are told apart by counter word 1:
//   augmentation   c = (index,                 2 pair + side                        , step lo, step hi)   c1 < 2^31
//   dropout        c = (row group << 16 | col,  2^31 | cloud << 11 | layer << 7 | site << 4 | head, step lo, step hi)
// with cloud = 2 (pair_base + b) + side the GLOBAL cloud index, row / col the row within the (query) cloud and the
// column (key index within the key cloud, or feature index), row group = row / 8.  One Philox block holds the
// decisions of 8 consecutive rows of one column, 16 bits each: row 8 rg + r reads half (r & 1) of word r >> 1 and is
// kept when that 16-bit value is >= threshold = round(p 65536).  The attention passes use a whole block at a time:
// the key-major dK / dV pass owns a column and walks the rows; the query-major passes have 8 lanes draw 8 columns
// and swap them with shuffles.  The elementwise sites (the LayerNorm prologue and its backward, one warp per row)
// draw one block per element and use 1/8 of it: 256 blocks per 256-wide row, which costs a few microseconds per
// launch at the model's token counts; the feed-forward dropout has a thread own 8 rows and uses whole blocks.
// Fields: cloud < 2^20, layer < 16, site 1..6, head < 16, row < 2^19, col < 2^16.
struct DropKey {
    Keys ks;
    unsigned thr;           // round(p * 65536)
    float scale;            // fp32(1 / (1 - p))
    int pair_base, n_pairs, layer, site;
};

// counter word 1 of local cloud c (plan order: src clouds 0..B-1, then tgt clouds)
__device__ __forceinline__ unsigned drop_word1(const DropKey& d, int c, int head) {
    const unsigned cloud = 2u * (unsigned)(d.pair_base + c % d.n_pairs) + (unsigned)(c / d.n_pairs);
    return 0x80000000u | (cloud << 11) | ((unsigned)d.layer << 7) | ((unsigned)d.site << 4) | (unsigned)head;
}

// bit r set: row 8 rg + r of column col is kept
__device__ __forceinline__ unsigned drop_keep8(const DropKey& d, unsigned w1, unsigned rg, unsigned col) {
    const U4 v = philox(U4{(rg << 16) | col, w1, d.ks.s0, d.ks.s1}, d.ks.k0, d.ks.k1);
    const unsigned w[4] = {v.x, v.y, v.z, v.w};
    unsigned m = 0;
#pragma unroll
    for (int e = 0; e < 4; ++e)
        m |= ((unsigned)((w[e] & 0xffffu) >= d.thr) << (2 * e)) | ((unsigned)((w[e] >> 16) >= d.thr) << (2 * e + 1));
    return m;
}

__device__ __forceinline__ bool drop_keep(const DropKey& d, unsigned w1, unsigned row, unsigned col) {
    return (drop_keep8(d, w1, row >> 3, col) >> (row & 7u)) & 1u;
}

// host: REGTR_OK and the kernel-side key, or REGTR_ERR_ARG for fields outside the counter layout
static inline int drop_key_of(const regtr_dropout_args* a, DropKey& d) {
    if (!a || a->pair_base < 0 || a->n_pairs <= 0 || 2ll * (a->pair_base + a->n_pairs) > (1ll << 20)) return REGTR_ERR_ARG;
    if (a->layer < 0 || a->layer > 15 || a->site < 1 || a->site > 6 || a->threshold > 65536u) return REGTR_ERR_ARG;
    d.ks = Keys{(unsigned)a->seed, (unsigned)(a->seed >> 32), (unsigned)a->step, (unsigned)(a->step >> 32)};
    d.thr = a->threshold;
    d.scale = a->scale;
    d.pair_base = a->pair_base; d.n_pairs = a->n_pairs; d.layer = a->layer; d.site = a->site;
    return REGTR_OK;
}

}  // namespace
