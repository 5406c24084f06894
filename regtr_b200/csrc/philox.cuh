// Counter-based randomness shared by the training-data kernels: Philox4x32-10 normals and uniforms, and the keyed
// Feistel bijection behind every permutation and subset.  A draw depends only on (seed, step, pair, side, index).
#pragma once
#include <cuda_runtime.h>

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

}  // namespace
