// Internal to the library: the cell list's memory layout and hash, and the single-pass prefix sum, shared by the
// pyramid pre-processing (preprocess.cu) and the training-data preparation (traindata.cu).
#pragma once

#include "common.cuh"

namespace {

constexpr unsigned long long KEY_PAD = ~0ull;

// ---------------------------------------------------------------- single-pass prefix sum (own kernel)
// Exclusive prefix sum with decoupled look-back (one launch, one pass over the data): every tile publishes
// its aggregate, then its inclusive prefix; a tile adds up the published values of its predecessors until it
// meets an inclusive prefix.  Tile numbers come from an atomic ticket, so a tile only ever waits for tiles that
// already started.  The state (ticket, completion counter, per-tile flags) is zero on entry and restored to zero
// by the last tile to finish: the buffer needs to be cleared once, when it is allocated.
//   MODE 0: in int32 counts -> out int32 exclusive sums
//   MODE 1: in uint32 counts -> out uint64 { hi = number of NON-ZERO entries before, lo = sum before }
constexpr int SCAN_THREADS = 256, SCAN_ITEMS = 16, SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;

struct ScanState {                 // zero-initialised, self-cleaning
    int ticket, done, pad[62];
    // followed by: flags[num_tiles] (int), aggregate[num_tiles] (u64), inclusive[num_tiles] (u64)
};
static_assert(sizeof(ScanState) == 256, "ScanState header must stay 256 B");

__host__ __device__ inline size_t scan_state_bytes(long long n) {
    const long long tiles = (n + SCAN_TILE - 1) / SCAN_TILE + 1;
    return 256 + (size_t)tiles * (sizeof(int) + 2 * sizeof(unsigned long long)) + 64;
}

// n_dev (optional): the number of leading elements that matter is *n_dev + 1 (device-side, <= n): CTAs beyond it
// only take their ticket and leave -- the voxel grid scans its occupied part of a capacity-sized counter array.
template <int MODE>
__global__ void __launch_bounds__(SCAN_THREADS)
k_scan_lookback(const void* __restrict__ in_, void* __restrict__ out_, int n, const int* __restrict__ n_dev, ScanState* st,
                int num_tiles) {
    typedef unsigned long long u64;
    __shared__ u64 s_warp[SCAN_THREADS / 32];
    __shared__ u64 s_excl;
    __shared__ int s_tile;
    int* flags = reinterpret_cast<int*>(reinterpret_cast<char*>(st) + 256);
    u64* aggregate = reinterpret_cast<u64*>(reinterpret_cast<char*>(st) + 256 + (((size_t)num_tiles * sizeof(int) + 15) & ~(size_t)15));
    u64* inclusive = aggregate + num_tiles;
    if (n_dev) n = min(n, *n_dev + 1);
    const int live_tiles = (n + SCAN_TILE - 1) / SCAN_TILE;
    if (threadIdx.x == 0) s_tile = atomicAdd(&st->ticket, 1);
    __syncthreads();
    const int tile = s_tile;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (tile < live_tiles) {
        const int base = tile * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
        unsigned x[SCAN_ITEMS];
        if (base + SCAN_ITEMS <= n) {
#pragma unroll
            for (int j = 0; j < SCAN_ITEMS / 4; ++j) {
                const uint4 q = reinterpret_cast<const uint4*>(reinterpret_cast<const unsigned*>(in_) + base)[j];
                x[4 * j] = q.x; x[4 * j + 1] = q.y; x[4 * j + 2] = q.z; x[4 * j + 3] = q.w;
            }
        } else {
#pragma unroll
            for (int j = 0; j < SCAN_ITEMS; ++j) x[j] = base + j < n ? reinterpret_cast<const unsigned*>(in_)[base + j] : 0u;
        }
        u64 v[SCAN_ITEMS];
        u64 tsum = 0;
#pragma unroll
        for (int j = 0; j < SCAN_ITEMS; ++j) {
            v[j] = tsum;                                  // exclusive prefix inside the thread
            tsum += MODE == 0 ? (u64)x[j] : (((u64)(x[j] != 0) << 32) | x[j]);
        }
        // block-level exclusive scan of the per-thread sums
        u64 incl = tsum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const u64 t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        if (lane == 31) s_warp[warp] = incl;
        __syncthreads();
        u64 warp_off = 0, block_total = 0;
#pragma unroll
        for (int w = 0; w < SCAN_THREADS / 32; ++w) {
            if (w < warp) warp_off += s_warp[w];
            block_total += s_warp[w];
        }
        const u64 thread_excl = warp_off + incl - tsum;
        if (warp == 0) {
            // publish the aggregate, then look back a WARP of predecessors at a time: lane l reads tile - 1 - l
            // (aggregate or inclusive prefix, whichever is published); the nearest inclusive prefix ends the walk
            if (lane == 0) {
                if (tile == 0) { inclusive[0] = block_total; __threadfence(); atomicExch(&flags[0], 2); }
                else { aggregate[tile] = block_total; __threadfence(); atomicExch(&flags[tile], 1); }
            }
            u64 excl = 0;
            if (tile > 0) {
                for (int first = tile - 1;; first -= 32) {
                    const int pred = first - lane;
                    int f = 2;
                    u64 val = 0;                          // before tile 0: an inclusive prefix of zero
                    if (pred >= 0) {
                        unsigned spin = 0;
                        do {                              // bounded: a corrupted state must trap, not hang the device
                            f = atomicAdd(&flags[pred], 0);
                            if (++spin > (1u << 26)) __trap();
                        } while (f == 0);
                        __threadfence();
                        val = *reinterpret_cast<volatile u64*>(f == 2 ? &inclusive[pred] : &aggregate[pred]);
                    }
                    const unsigned done_mask = __ballot_sync(0xffffffffu, f == 2);
                    const int stop = done_mask ? __ffs(done_mask) - 1 : 31;
                    u64 part = lane <= stop ? val : 0;
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
                    excl += part;
                    if (done_mask) break;
                }
                if (lane == 0) { inclusive[tile] = excl + block_total; __threadfence(); atomicExch(&flags[tile], 2); }
            }
            if (lane == 0) s_excl = excl;
        }
        __syncthreads();
        const u64 off = s_excl + thread_excl;
        if (base + SCAN_ITEMS <= n) {
            if (MODE == 0) {
#pragma unroll
                for (int j = 0; j < SCAN_ITEMS / 4; ++j)
                    reinterpret_cast<int4*>(reinterpret_cast<int*>(out_) + base)[j] =
                        make_int4((int)(unsigned)(off + v[4 * j]), (int)(unsigned)(off + v[4 * j + 1]),
                                  (int)(unsigned)(off + v[4 * j + 2]), (int)(unsigned)(off + v[4 * j + 3]));
            } else {
#pragma unroll
                for (int j = 0; j < SCAN_ITEMS / 2; ++j)
                    reinterpret_cast<ulonglong2*>(reinterpret_cast<u64*>(out_) + base)[j] = make_ulonglong2(off + v[2 * j], off + v[2 * j + 1]);
            }
        } else {
#pragma unroll
            for (int j = 0; j < SCAN_ITEMS; ++j) {
                if (base + j < n) {
                    if (MODE == 0) reinterpret_cast<int*>(out_)[base + j] = (int)(unsigned)(off + v[j]);
                    else reinterpret_cast<u64*>(out_)[base + j] = off + v[j];
                }
            }
        }
    }
    // the last CTA to FINISH restores the zero state (nobody reads flags any more: every tile has its prefix, and
    // every launched CTA has taken its ticket)
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        s_tile = atomicAdd(&st->done, 1) == (int)gridDim.x - 1;
    }
    __syncthreads();
    if (s_tile) {
        // aggregates and prefixes too: the next call may lay the state out for another tile count, where these
        // words are somebody's flags (or, in the voxel counting sort, cell counters)
        for (int t = threadIdx.x; t < live_tiles; t += SCAN_THREADS) { flags[t] = 0; aggregate[t] = 0; inclusive[t] = 0; }
        if (threadIdx.x == 0) { st->ticket = 0; st->done = 0; }
    }
}

template <int MODE>
inline int launch_scan(const void* in, void* out, int n, const int* n_dev, void* state, cudaStream_t st) {
    const int tiles = (n + SCAN_TILE - 1) / SCAN_TILE;
    if (tiles <= 0) return REGTR_OK;
    k_scan_lookback<MODE><<<tiles, SCAN_THREADS, 0, st>>>(in, out, n, n_dev, reinterpret_cast<ScanState*>(state), tiles);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

// ------------------------------------------------------------------------- cell list

struct GridHeader {
    float cell;
    int n_cap;
    int pad[62];
};
static_assert(sizeof(GridHeader) == 256, "header must stay 256 B");

// Hash table over the occupied cells of a grid: key -> (first position in the cell-ordered arrays, point
// count).  Open addressing, linear probing, load factor <= 0.5 (>= 2 * n_cap slots).
struct CellSlot {
    unsigned long long key;
    int start;
    int count;
};
static_assert(sizeof(CellSlot) == 16, "CellSlot must be 16 B");

__host__ __device__ inline int cell_table_log2(int n_cap) {
    int b = 10;
    while ((1ll << b) < 2ll * (n_cap > 0 ? n_cap : 1)) ++b;
    return b;
}
__device__ __forceinline__ unsigned cell_hash(unsigned long long key, int log2t) {
    return (unsigned)((key * 0x9E3779B97F4A7C15ull) >> (64 - log2t));
}

// (start, count) of cell `key` in the table, (0, 0) when the cell is empty
__device__ __forceinline__ void cell_lookup(const CellSlot* __restrict__ table, int log2t, unsigned long long key,
                                            int& start, int& count) {
    const unsigned mask = (1u << log2t) - 1u;
    unsigned h = cell_hash(key, log2t);
    start = 0; count = 0;
    for (;;) {
        const CellSlot sl = table[h];
        if (sl.key == key) { start = sl.start; count = sl.count; return; }
        if (sl.key == KEY_PAD) return;
        h = (h + 1) & mask;
    }
}

// grid buffer: [GridHeader | sxyzi (n float4) | CellSlot table (2^log2t)]
inline float4* grid_sxyzi(void* grid) { return (float4*)((char*)grid + sizeof(GridHeader)); }
inline CellSlot* grid_table(void* grid, size_t n) {
    return (CellSlot*)((char*)grid + sizeof(GridHeader) + regtr_align(sizeof(float4) * n));
}

}  // namespace
