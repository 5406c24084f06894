// Pyramid pre-processing kernels: voxel-grid barycentre sub-sampling, cell-list
// construction and fixed-radius "first K in index order" neighbour search.
//
// Reference behaviour replaced (paths relative to /root/reference/src):
//   models/backbone_kpconv/kpconv.py:213-240  batch_grid_subsampling_kpconv_gpu (MinkowskiEngine)
//   models/backbone_kpconv/kpconv.py:261-288  batch_neighbors_kpconv_gpu (pytorch3d ball_query)
// Determinism rules: DESIGN.md "H1" (shared with oracle/c/preprocess_oracle.c).
//
// All data-dependent sizes stay on the device: kernels are launched over host-known
// capacities and read the real point counts from the int32 offset arrays.
#include "voxsort.cuh"

namespace {

__device__ __forceinline__ int clamp_coord(int v, uint32_t* status) {
    if (v < -32766 || v > 32766) {
        atomicOr(status, REGTR_STATUS_KEY_RANGE);
        v = v < 0 ? -32766 : 32766;
    }
    return v;
}

// key[i] = (cloud, floor(p/cell)) for i < n, KEY_PAD beyond; val[i] = i.
__global__ void k_make_keys(const float* __restrict__ xyz, const int32_t* __restrict__ offs, int n_clouds,
                            int n_cap, float cell, unsigned long long* __restrict__ keys,
                            int32_t* __restrict__ vals, uint32_t* status) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_cap) return;
    const int n = offs[n_clouds];
    unsigned long long key = KEY_PAD;
    if (i < n) {
        const int c = regtr_cloud_of(offs, n_clouds, i);
        const int vx = clamp_coord(regtr_cell_of(xyz[3 * i + 0], cell), status);
        const int vy = clamp_coord(regtr_cell_of(xyz[3 * i + 1], cell), status);
        const int vz = clamp_coord(regtr_cell_of(xyz[3 * i + 2], cell), status);
        key = regtr_pack_key(c, vx, vy, vz);
    }
    keys[i] = key;
    vals[i] = i;
}

// One thread per voxel head: fp32 running sum over the members in ascending input index
// (the radix sort is stable, so members appear in that order), then one IEEE division.
__global__ void k_voxel_mean(const float* __restrict__ xyz, const unsigned long long* __restrict__ skeys,
                             const int32_t* __restrict__ sidx, const int32_t* __restrict__ rank, int n_cap,
                             int out_cap, float* __restrict__ out_xyz, uint32_t* status) {
    int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n_cap) return;
    const unsigned long long k = skeys[j];
    if (k == KEY_PAD || (j > 0 && skeys[j - 1] == k)) return;
    if (rank[j] >= out_cap) { atomicOr(status, REGTR_STATUS_CAPACITY); return; }
    float sx = 0.f, sy = 0.f, sz = 0.f;
    int cnt = 0;
    for (int t = j; t < n_cap && skeys[t] == k; ++t) {
        const int i = sidx[t];
        sx = __fadd_rn(sx, xyz[3 * i + 0]);
        sy = __fadd_rn(sy, xyz[3 * i + 1]);
        sz = __fadd_rn(sz, xyz[3 * i + 2]);
        ++cnt;
    }
    const float c = (float)cnt;
    const int m = rank[j];
    out_xyz[3 * m + 0] = __fdiv_rn(sx, c);
    out_xyz[3 * m + 1] = __fdiv_rn(sy, c);
    out_xyz[3 * m + 2] = __fdiv_rn(sz, c);
}

// --------------------------------------------- voxel-grid sub-sampling by dense-grid counting sort (no library sort)
// The stable radix sort of (voxel key, point index) pairs is replaced by a counting sort over a DENSE grid: the
// voxel bounding box of every cloud is found first, a voxel's sort position is its linear cell number
// base[cloud] + ((x - min_x) * ny + (y - min_y)) * nz + (z - min_z) -- ascending (cloud, x, y, z), the pinned
// output order -- and one prefix sum over the cells gives, per cell, the first member slot (sum of the counts
// before) and the output row (number of occupied cells before).  Members land in their cell's slots in arrival
// order (atomics) and are put in ascending index order by the thread that averages them, so the barycentre is
// the same index-ordered fp32 running sum as before: bit-identical results, 8 kernels instead of 15, no CUB.
// The cell budget is 16 cells per point of capacity (at least 2^20): indoor fragments use ~8 cells per point
// at the first level and fewer later; a bounding box beyond the budget raises REGTR_STATUS_GRID (the caller
// then takes the sort-based path).
struct VoxCloud { int minx, miny, minz, ny, nz, base; };

__global__ void k_vox_bbox(const float* __restrict__ xyz, const int32_t* __restrict__ offs, int n_clouds, int n_cap, float dl,
                           unsigned* __restrict__ bb, uint32_t* status) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int n = offs[n_clouds];
    const bool live = i < n_cap && i < n;
    int c = -1;
    unsigned u[6] = {0, 0, 0, 0, 0, 0};              // max of (65535 - x) (the minimum), max of x, per axis; 0 = neutral
    if (live) {
        c = regtr_cloud_of(offs, n_clouds, i);
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const unsigned b = (unsigned)(clamp_coord(regtr_cell_of(xyz[3 * i + a], dl), status) + 32768);
            u[a] = 65535u - b;
            u[3 + a] = b;
        }
    }
    const unsigned m = __ballot_sync(0xffffffffu, live);
    if (!m) return;
    const int c0 = __shfl_sync(0xffffffffu, c, __ffs(m) - 1);
    if (__all_sync(0xffffffffu, !live || c == c0)) {      // the usual case: the warp's points belong to one cloud
#pragma unroll
        for (int a = 0; a < 6; ++a) u[a] = __reduce_max_sync(0xffffffffu, u[a]);
        if ((threadIdx.x & 31) == 0)
#pragma unroll
            for (int a = 0; a < 6; ++a) atomicMax(&bb[c0 * 6 + a], u[a]);
    } else if (live) {
#pragma unroll
        for (int a = 0; a < 6; ++a) atomicMax(&bb[c * 6 + a], u[a]);
    }
}

// per-cloud box -> (origin, extents, first cell); total number of cells; one thread (n_clouds is small)
__global__ void k_vox_layout(const unsigned* __restrict__ bb, int n_clouds, long long cells_cap, VoxCloud* __restrict__ lay,
                             int* __restrict__ total_cells, uint32_t* status) {
    if (blockIdx.x || threadIdx.x) return;
    long long base = 0;
    for (int c = 0; c < n_clouds; ++c) {
        VoxCloud v{0, 0, 0, 0, 0, (int)(base < cells_cap ? base : cells_cap)};
        if (bb[c * 6 + 3] != 0) {                                  // the cloud has points
            const int mn[3] = {(int)(65535u - bb[c * 6 + 0]) - 32768, (int)(65535u - bb[c * 6 + 1]) - 32768,
                               (int)(65535u - bb[c * 6 + 2]) - 32768};
            const int mx[3] = {(int)bb[c * 6 + 3] - 32768, (int)bb[c * 6 + 4] - 32768, (int)bb[c * 6 + 5] - 32768};
            v.minx = mn[0]; v.miny = mn[1]; v.minz = mn[2];
            v.ny = mx[1] - mn[1] + 1; v.nz = mx[2] - mn[2] + 1;
            base += (long long)(mx[0] - mn[0] + 1) * v.ny * v.nz;
        }
        lay[c] = v;
    }
    if (base > cells_cap) { atomicOr(status, REGTR_STATUS_GRID); base = cells_cap; }
    *total_cells = (int)base;
}

__global__ void k_vox_count(const float* __restrict__ xyz, const int32_t* __restrict__ offs, int n_clouds, int n_cap, float dl,
                            const VoxCloud* __restrict__ lay, long long cells_cap, unsigned* __restrict__ cnt,
                            int32_t* __restrict__ cell_of, uint32_t* status) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_cap) return;
    int cell = -1;
    if (i < offs[n_clouds]) {
        const int c = regtr_cloud_of(offs, n_clouds, i);
        const VoxCloud v = lay[c];
        const int vx = clamp_coord(regtr_cell_of(xyz[3 * i + 0], dl), status) - v.minx;
        const int vy = clamp_coord(regtr_cell_of(xyz[3 * i + 1], dl), status) - v.miny;
        const int vz = clamp_coord(regtr_cell_of(xyz[3 * i + 2], dl), status) - v.minz;
        const long long id = (long long)v.base + ((long long)vx * v.ny + vy) * v.nz + vz;
        if (id < cells_cap) { cell = (int)id; atomicAdd(&cnt[cell], 1u); }
    }
    cell_of[i] = cell;
}

// members[first slot of the cell + arrival rank] = point; the counters return to zero (self-cleaning state)
__global__ void k_vox_scatter(int n_cap, const int32_t* __restrict__ cell_of, const unsigned long long* __restrict__ pre,
                              unsigned* __restrict__ cnt, int32_t* __restrict__ members) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_cap) return;
    const int cell = cell_of[i];
    if (cell < 0) return;
    const unsigned k = atomicSub(&cnt[cell], 1u) - 1u;
    members[(unsigned)pre[cell] + k] = i;
}

// one thread per cell: members in ascending point index, fp32 running sum, one IEEE division (DESIGN.md H1-iii)
__global__ void k_vox_mean(const float* __restrict__ xyz, const unsigned long long* __restrict__ pre,
                           const int* __restrict__ total_cells, int32_t* __restrict__ members, int out_cap,
                           float* __restrict__ out_xyz, uint32_t* status) {
    const int cell = blockIdx.x * blockDim.x + threadIdx.x;
    if (cell >= *total_cells) return;
    const unsigned long long p0 = pre[cell], p1 = pre[cell + 1];
    const int first = (int)(unsigned)p0, cntc = (int)((unsigned)p1 - (unsigned)p0);
    if (cntc == 0) return;
    const int row = (int)(p0 >> 32);
    if (row >= out_cap) { atomicOr(status, REGTR_STATUS_CAPACITY); return; }
    int32_t* mem = members + first;
    for (int a = 1; a < cntc; ++a) {                 // insertion sort (a voxel holds a handful of points)
        const int key = mem[a];
        int b = a - 1;
        while (b >= 0 && mem[b] > key) { mem[b + 1] = mem[b]; --b; }
        mem[b + 1] = key;
    }
    float sx = 0.f, sy = 0.f, sz = 0.f;
    for (int a = 0; a < cntc; ++a) {
        const int i = mem[a];
        sx = __fadd_rn(sx, xyz[3 * i + 0]);
        sy = __fadd_rn(sy, xyz[3 * i + 1]);
        sz = __fadd_rn(sz, xyz[3 * i + 2]);
    }
    const float c = (float)cntc;
    out_xyz[3 * row + 0] = __fdiv_rn(sx, c);
    out_xyz[3 * row + 1] = __fdiv_rn(sy, c);
    out_xyz[3 * row + 2] = __fdiv_rn(sz, c);
}

// out_offs[c] = number of occupied cells before cloud c's first cell
__global__ void k_vox_offsets(const unsigned long long* __restrict__ pre, const VoxCloud* __restrict__ lay,
                              const int* __restrict__ total_cells, int n_clouds, int out_cap, int32_t* __restrict__ out_offs) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c > n_clouds) return;
    const int cell = c == n_clouds ? *total_cells : min(lay[c].base, *total_cells);
    out_offs[c] = min((int)(pre[cell] >> 32), out_cap);
}

// ------------------------------------------------------------------------- cell list


// ---- sort-free cell list: count points per cell in a hash table, prefix-sum the counts, scatter.
// The order of the points inside a cell (and of the cells in memory) is arbitrary and may differ from
// run to run; the neighbour search ranks its hits by index afterwards, so its OUTPUT is deterministic.

// slot_of[i] = table slot of point i's cell (inserted on first sight); cnt[slot] += 1.
__global__ void k_cell_count(const float* __restrict__ xyz, const int32_t* __restrict__ offs, int n_clouds, int n_cap,
                             float cell, unsigned long long* __restrict__ tkeys, int32_t* __restrict__ cnt, int log2t,
                             int32_t* __restrict__ slot_of, uint32_t* status, GridHeader* __restrict__ hdr) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) { hdr->cell = cell; hdr->n_cap = n_cap; }
    if (i >= n_cap) return;
    if (i >= offs[n_clouds]) { slot_of[i] = -1; return; }
    const int c = regtr_cloud_of(offs, n_clouds, i);
    const int vx = clamp_coord(regtr_cell_of(xyz[3 * i + 0], cell), status);
    const int vy = clamp_coord(regtr_cell_of(xyz[3 * i + 1], cell), status);
    const int vz = clamp_coord(regtr_cell_of(xyz[3 * i + 2], cell), status);
    const unsigned long long key = regtr_pack_key(c, vx, vy, vz);
    const unsigned mask = (1u << log2t) - 1u;
    unsigned h = cell_hash(key, log2t);
    for (;;) {
        const unsigned long long prev = atomicCAS(&tkeys[h], KEY_PAD, key);
        if (prev == KEY_PAD || prev == key) break;
        h = (h + 1) & mask;
    }
    atomicAdd(&cnt[h], 1);
    slot_of[i] = (int)h;
}

// position of point i = start[slot] + (arrival rank inside the cell); pads keep the tail positions.
__global__ void k_cell_scatter(const float* __restrict__ xyz, const int32_t* __restrict__ offs, int n_clouds, int n_cap,
                               const int32_t* __restrict__ slot_of, const int32_t* __restrict__ start,
                               int32_t* __restrict__ cursor, float4* __restrict__ sxyzi, int32_t* __restrict__ order) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_cap) return;
    const int h = slot_of[i];
    if (h < 0) {                                   // capacity padding: identity tail of the permutation
        sxyzi[i] = make_float4(0.f, 0.f, 0.f, __int_as_float(-1));
        if (order) order[i] = i;
        return;
    }
    const int pos = start[h] + atomicAdd(&cursor[h], 1);
    sxyzi[pos] = make_float4(xyz[3 * i + 0], xyz[3 * i + 1], xyz[3 * i + 2], __int_as_float(i));
    if (order) order[pos] = i;
}

__global__ void k_cell_pack(const unsigned long long* __restrict__ tkeys, const int32_t* __restrict__ start,
                            const int32_t* __restrict__ cnt, int t_size, CellSlot* __restrict__ table) {
    const int h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= t_size) return;
    CellSlot s;
    s.key = tkeys[h]; s.start = start[h]; s.count = cnt[h];
    table[h] = s;
}

// ------------------------------------------------------------------------ ball query

constexpr int BQ_WARPS = 8;
constexpr int BQ_HCAP = 384;   // hit staging per warp
constexpr int BQ_KMAX = 128;

// Keep the `K` smallest of hits[0..n) in ascending order in sel[0..min(n,K)).
__device__ __forceinline__ int select_smallest(const int* __restrict__ hits, int n, int K, int* __restrict__ sel,
                                               int lane) {
    for (int p = lane; p < n; p += 32) {
        const int v = hits[p];
        int r = 0;
        for (int t = 0; t < n; ++t) r += (hits[t] < v);
        if (r < K) sel[r] = v;
    }
    __syncwarp();
    return n < K ? n : K;
}

__global__ void __launch_bounds__(BQ_WARPS * 32)
k_ball_query(const float* __restrict__ q, const int32_t* __restrict__ q_offs, const int32_t* __restrict__ q_order,
             const int32_t* __restrict__ s_offs, const GridHeader* __restrict__ hdr,
             const CellSlot* __restrict__ table, int log2t, const float4* __restrict__ sxyzi, int n_clouds,
             int nq_cap, int K, float radius, int32_t* __restrict__ out32, long long* __restrict__ out64) {
    __shared__ int s_hits[BQ_WARPS][BQ_HCAP];
    __shared__ int s_sel[BQ_WARPS][BQ_KMAX];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nq = q_offs[n_clouds];
    const int ns = s_offs[n_clouds];
    const float cell = hdr->cell;
    const float r2 = __fmul_rn(radius, radius);
    int* hits = s_hits[warp];
    int* sel = s_sel[warp];
    // persistent warps: a grid of a few CTAs per SM walks the query slots (the per-launch reads -- counts, cell size --
    // and the CTA start-up are paid once per warp, not once per query)
    for (int slot = blockIdx.x * BQ_WARPS + warp; slot < nq_cap; slot += gridDim.x * BQ_WARPS) {
    const int qi = q_order ? q_order[slot] : slot;
    if (qi < 0 || qi >= nq_cap) continue;
    if (qi >= nq) {                            // capacity padding: a fully-shadow row, so that the
        for (int t = lane; t < K; t += 32) {   // whole (nq_cap, K) buffer is always initialised
            if (out32) out32[(long long)qi * K + t] = ns;
            if (out64) out64[(long long)qi * K + t] = ns;
        }
        continue;
    }
    const int c = regtr_cloud_of(q_offs, n_clouds, qi);
    const float qx = q[3 * qi + 0], qy = q[3 * qi + 1], qz = q[3 * qi + 2];
    const int cx = regtr_cell_of(qx, cell), cy = regtr_cell_of(qy, cell), cz = regtr_cell_of(qz, cell);
    // lanes 0..26: one cell of the 3x3x3 stencil each -> hash lookup of (start, count)
    int c_start = 0, c_cnt = 0;
    if (lane < 27) {
        const int x = cx + lane / 9 - 1, y = cy + (lane / 3) % 3 - 1, z = cz + lane % 3 - 1;
        if (x >= -32767 && x <= 32767 && y >= -32767 && y <= 32767 && z >= -32767 && z <= 32767) {
            const unsigned long long key = regtr_pack_key(c, x, y, z);
            const unsigned mask = (1u << log2t) - 1u;
            unsigned h = cell_hash(key, log2t);
            for (;;) {
                const CellSlot sl = table[h];
                if (sl.key == key) { c_start = sl.start; c_cnt = sl.count; break; }
                if (sl.key == KEY_PAD) break;
                h = (h + 1) & mask;
            }
        }
    }
    // inclusive prefix sum of the 27 counts: candidate i lives in the first cell whose prefix exceeds i
    int pre = c_cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, pre, o);
        if (lane >= o) pre += v;
    }
    const int total = __shfl_sync(0xffffffffu, pre, 31);
    int count = 0;
    for (int base = 0; base < total; base += 32) {
        const int i = base + lane;
        // binary search over the 32 prefix values held one per lane (5 shuffles)
        int cellid = 0;
#pragma unroll
        for (int step = 16; step > 0; step >>= 1) {
            const int probe = cellid + step - 1;
            const int pv = __shfl_sync(0xffffffffu, pre, probe);
            if (pv <= i) cellid += step;
        }
        const int cell_pre = __shfl_sync(0xffffffffu, pre, cellid);
        const int cell_cnt = __shfl_sync(0xffffffffu, c_cnt, cellid);
        const int cell_start = __shfl_sync(0xffffffffu, c_start, cellid);
        bool hit = false;
        int sidx = 0;
        if (i < total) {
            const int j = cell_start + (i - (cell_pre - cell_cnt));
            const float4 sp = sxyzi[j];
            const float dx = __fsub_rn(qx, sp.x), dy = __fsub_rn(qy, sp.y), dz = __fsub_rn(qz, sp.z);
            const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
            hit = d2 < r2;
            sidx = __float_as_int(sp.w);
        }
        const unsigned m = __ballot_sync(0xffffffffu, hit);
        if (count + 32 > BQ_HCAP) {           // staging full: keep only the K smallest so far
            __syncwarp();
            const int kept = select_smallest(hits, count, K, sel, lane);
            for (int t = lane; t < kept; t += 32) hits[t] = sel[t];
            __syncwarp();
            count = kept;
        }
        if (hit) hits[count + __popc(m & ((1u << lane) - 1u))] = sidx;
        count += __popc(m);
    }
    __syncwarp();
    const int kept = select_smallest(hits, count, K, sel, lane);
    const long long row = (long long)qi * K;
    for (int t = lane; t < K; t += 32) {
        const int v = t < kept ? sel[t] : ns;
        if (out32) out32[row + t] = v;
        if (out64) out64[row + t] = v;
    }
    __syncwarp();                              // hits / sel are reused by the next query of this warp
    }
}

}  // namespace

extern "C" {

static inline long long vox_cells_cap(int n_cap) {
    const long long c = 16ll * (n_cap > 0 ? n_cap : 1);
    return c < (1ll << 18) ? (1ll << 18) : c;
}

struct VoxWs {
    unsigned* bb;
    VoxCloud* lay;
    int* total;
    int32_t *cell_of, *members;
    unsigned long long* pre;
    size_t bb_bytes, total_bytes;
};

static VoxWs carve_vox(void* ws, int n_cap, int n_clouds) {
    VoxWs w;
    char* p = (char*)ws;
    size_t off = 0;
    auto take = [&](size_t bytes) { char* r = p ? p + off : nullptr; off += regtr_align(bytes); return (void*)r; };
    const size_t n = (size_t)(n_cap > 0 ? n_cap : 1), nc = (size_t)(n_clouds > 0 ? n_clouds : 1);
    w.bb_bytes = sizeof(unsigned) * 6 * nc;
    w.bb = (unsigned*)take(w.bb_bytes);
    w.lay = (VoxCloud*)take(sizeof(VoxCloud) * nc);
    w.total = (int*)take(sizeof(int));
    w.cell_of = (int32_t*)take(sizeof(int32_t) * n);
    w.members = (int32_t*)take(sizeof(int32_t) * n);
    w.pre = (unsigned long long*)take(sizeof(unsigned long long) * ((size_t)vox_cells_cap(n_cap) + 2));
    w.total_bytes = off;
    return w;
}

size_t regtr_grid_subsample_ws_bytes(int n_cap, int n_clouds) { return carve_vox(nullptr, n_cap, n_clouds).total_bytes; }

// state: counters (one uint32 per cell) | prefix-sum state; ZERO before the first call, every call leaves it zero
size_t regtr_grid_subsample_state_bytes(int n_cap) {
    const long long cells = vox_cells_cap(n_cap);
    return regtr_align(sizeof(unsigned) * (size_t)(cells + SCAN_TILE)) + scan_state_bytes(cells + 1);
}

int regtr_grid_subsample(const float* xyz, const int32_t* offs, int n_clouds, int n_cap, float dl,
                         float* out_xyz, int out_cap, int32_t* out_offs, uint32_t* status, void* ws,
                         size_t ws_bytes, void* state, size_t state_bytes, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (!offs || !out_offs || !status || n_clouds <= 0 || n_clouds > 32767 || n_cap < 0 || out_cap < 0 || !(dl > 0.f))
        return REGTR_ERR_ARG;
    if (n_cap == 0) {
        cudaMemsetAsync(out_offs, 0, sizeof(int32_t) * (n_clouds + 1), st);
        return REGTR_OK;
    }
    if (!xyz || !out_xyz || !ws || !state) return REGTR_ERR_ARG;
    VoxWs w = carve_vox(ws, n_cap, n_clouds);
    if (ws_bytes < w.total_bytes || state_bytes < regtr_grid_subsample_state_bytes(n_cap)) return REGTR_ERR_WORKSPACE;
    const long long cells_cap = vox_cells_cap(n_cap);
    unsigned* cnt = (unsigned*)state;
    void* scan_state = (char*)state + regtr_align(sizeof(unsigned) * (size_t)(cells_cap + SCAN_TILE));
    const int T = 256;
    if (cudaMemsetAsync(w.bb, 0, w.bb_bytes, st) != cudaSuccess) return REGTR_ERR_ARG;
    k_vox_bbox<<<regtr_cdiv(n_cap, T), T, 0, st>>>(xyz, offs, n_clouds, n_cap, dl, w.bb, status);
    REGTR_CHECK_LAUNCH();
    k_vox_layout<<<1, 32, 0, st>>>(w.bb, n_clouds, cells_cap, w.lay, w.total, status);
    REGTR_CHECK_LAUNCH();
    k_vox_count<<<regtr_cdiv(n_cap, T), T, 0, st>>>(xyz, offs, n_clouds, n_cap, dl, w.lay, cells_cap, cnt, w.cell_of, status);
    REGTR_CHECK_LAUNCH();
    const int rc = launch_scan<1>(cnt, w.pre, (int)cells_cap + 1, w.total, scan_state, st);
    if (rc != REGTR_OK) return rc;
    k_vox_scatter<<<regtr_cdiv(n_cap, T), T, 0, st>>>(n_cap, w.cell_of, w.pre, cnt, w.members);
    REGTR_CHECK_LAUNCH();
    k_vox_mean<<<regtr_cdiv(cells_cap, T), T, 0, st>>>(xyz, w.pre, w.total, w.members, out_cap, out_xyz, status);
    REGTR_CHECK_LAUNCH();
    k_vox_offsets<<<regtr_cdiv(n_clouds + 1, 128), 128, 0, st>>>(w.pre, w.lay, w.total, n_clouds, out_cap, out_offs);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

// The sort-based variant (stable CUB radix sort of (voxel key, index) pairs): any extent inside the +-32766-cell key
// range; the fallback when a bounding box exceeds the dense-grid budget (REGTR_STATUS_GRID).
size_t regtr_grid_subsample_sorted_ws_bytes(int n_cap) { return n_cap > 0 ? carve(nullptr, n_cap).total : 256; }

int regtr_grid_subsample_sorted(const float* xyz, const int32_t* offs, int n_clouds, int n_cap, float dl,
                                float* out_xyz, int out_cap, int32_t* out_offs, uint32_t* status, void* ws,
                                size_t ws_bytes, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (!offs || !out_offs || !status || n_clouds <= 0 || n_clouds > 32767 || n_cap < 0 || out_cap < 0 || !(dl > 0.f))
        return REGTR_ERR_ARG;
    if (n_cap == 0) {
        cudaMemsetAsync(out_offs, 0, sizeof(int32_t) * (n_clouds + 1), st);
        return REGTR_OK;
    }
    if (!xyz || !out_xyz || !ws) return REGTR_ERR_ARG;
    SubWs w = carve(ws, n_cap);
    if (ws_bytes < w.total) return REGTR_ERR_WORKSPACE;
    const int T = 256;
    k_make_keys<<<regtr_cdiv(n_cap, T), T, 0, st>>>(xyz, offs, n_clouds, n_cap, dl, w.keys_in, w.vals_in, status);
    REGTR_CHECK_LAUNCH();
    const int rc = sort_and_rank(w, n_cap, n_clouds, st);
    if (rc != REGTR_OK) return rc;
    k_voxel_mean<<<regtr_cdiv(n_cap, T), T, 0, st>>>(xyz, w.keys_out, w.vals_out, w.rank, n_cap, out_cap, out_xyz,
                                                     status);
    REGTR_CHECK_LAUNCH();
    k_cloud_offsets<<<regtr_cdiv(n_clouds + 1, 128), 128, 0, st>>>(w.keys_out, w.rank, n_cap, n_clouds, out_cap,
                                                                   out_offs);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

size_t regtr_cellgrid_bytes(int n_cap) {
    const size_t n = n_cap > 0 ? (size_t)n_cap : 1;
    return sizeof(GridHeader) + regtr_align(sizeof(float4) * n) + regtr_align(sizeof(CellSlot) << cell_table_log2(n_cap));
}

// workspace: slot_of (n) | zero-initialised block [tkeys (T u64) | cnt (T) | cursor (T)] | start (T + 1) | cub scan temp
struct GridWs {
    int32_t* slot_of;
    unsigned long long* tkeys;
    int32_t *cnt, *cursor, *start;
    void* cub_tmp;
    size_t cub_bytes, zero_bytes, total;
};

static GridWs carve_grid(void* ws, int n_cap) {
    GridWs w;
    char* p = (char*)ws;
    size_t off = 0;
    auto take = [&](size_t bytes) { char* r = p ? p + off : nullptr; off += regtr_align(bytes); return (void*)r; };
    const size_t t = (size_t)1 << cell_table_log2(n_cap);
    w.slot_of = (int32_t*)take(sizeof(int32_t) * (size_t)(n_cap > 0 ? n_cap : 1));
    w.tkeys = (unsigned long long*)take(sizeof(unsigned long long) * t);
    w.cnt = (int32_t*)take(sizeof(int32_t) * t);
    w.cursor = (int32_t*)take(sizeof(int32_t) * t);
    w.zero_bytes = (size_t)((char*)w.cursor - (char*)w.cnt) + regtr_align(sizeof(int32_t) * t);   // cnt + cursor
    w.start = (int32_t*)take(sizeof(int32_t) * t);
    w.cub_bytes = 0;
    w.cub_tmp = nullptr;
    w.total = off;
    return w;
}

size_t regtr_cellgrid_ws_bytes(int n_cap) { return carve_grid(nullptr, n_cap).total; }

// prefix-sum state of the build: ZERO before the first call, every call leaves it zero
size_t regtr_cellgrid_state_bytes(int n_cap) { return scan_state_bytes((long long)1 << cell_table_log2(n_cap)); }

int regtr_cellgrid_build(const float* xyz, const int32_t* offs, int n_clouds, int n_cap, float cell, void* grid,
                         int32_t* order, uint32_t* status, void* ws, size_t ws_bytes, void* state, size_t state_bytes,
                         void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (!offs || !grid || !status || n_clouds <= 0 || n_clouds > 32767 || n_cap < 0 || !(cell > 0.f))
        return REGTR_ERR_ARG;
    GridHeader* hdr = (GridHeader*)grid;
    if (n_cap == 0) {                              // header only (thread 0 writes it and leaves)
        k_cell_count<<<1, 1, 0, st>>>(nullptr, offs, n_clouds, 0, cell, nullptr, nullptr, 0, nullptr, status, hdr);
        REGTR_CHECK_LAUNCH();
        return REGTR_OK;
    }
    if (!xyz || !ws || !state) return REGTR_ERR_ARG;
    GridWs w = carve_grid(ws, n_cap);
    if (ws_bytes < w.total || state_bytes < regtr_cellgrid_state_bytes(n_cap)) return REGTR_ERR_WORKSPACE;
    const int log2t = cell_table_log2(n_cap);
    const int t_size = 1 << log2t;
    float4* sxyzi = grid_sxyzi(grid);
    CellSlot* table = grid_table(grid, (size_t)n_cap);
    const int T = 256;
    if (cudaMemsetAsync(w.tkeys, 0xFF, sizeof(unsigned long long) * (size_t)t_size, st) != cudaSuccess ||
        cudaMemsetAsync(w.cnt, 0, w.zero_bytes, st) != cudaSuccess)
        return REGTR_ERR_ARG;
    k_cell_count<<<regtr_cdiv(n_cap, T), T, 0, st>>>(xyz, offs, n_clouds, n_cap, cell, w.tkeys, w.cnt, log2t, w.slot_of,
                                                     status, hdr);
    REGTR_CHECK_LAUNCH();
    const int rc = launch_scan<0>(w.cnt, w.start, t_size, nullptr, state, st);
    if (rc != REGTR_OK) return rc;
    k_cell_scatter<<<regtr_cdiv(n_cap, T), T, 0, st>>>(xyz, offs, n_clouds, n_cap, w.slot_of, w.start, w.cursor, sxyzi,
                                                       order);
    REGTR_CHECK_LAUNCH();
    k_cell_pack<<<regtr_cdiv(t_size, T), T, 0, st>>>(w.tkeys, w.start, w.cnt, t_size, table);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

int regtr_ball_query(const float* q, const int32_t* q_offs, const int32_t* q_order, const float* s,
                     const int32_t* s_offs, const void* s_grid, int n_clouds, int nq_cap, int s_cap, int K,
                     float radius, int32_t* out_idx32, int64_t* out_idx64, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    (void)s;  // positions are read from the cell-sorted copy inside the grid
    if (!q_offs || !s_offs || !s_grid || n_clouds <= 0 || nq_cap < 0 || s_cap < 0 || K <= 0 || K > BQ_KMAX ||
        !(radius > 0.f))
        return REGTR_ERR_ARG;
    if (nq_cap == 0) return REGTR_OK;
    if (!q || (!out_idx32 && !out_idx64)) return REGTR_ERR_ARG;
    const GridHeader* hdr = (const GridHeader*)s_grid;
    const size_t n = s_cap > 0 ? (size_t)s_cap : 1;
    const float4* sxyzi = grid_sxyzi(const_cast<void*>(s_grid));
    const CellSlot* table = grid_table(const_cast<void*>(s_grid), n);
    const int bq_blocks = regtr_cdiv(nq_cap, BQ_WARPS);
    k_ball_query<<<bq_blocks < 8 * REGTR_NUM_SMS ? bq_blocks : 8 * REGTR_NUM_SMS, BQ_WARPS * 32, 0, st>>>(
        q, q_offs, q_order, s_offs, hdr, table, cell_table_log2(s_cap), sxyzi, n_clouds, nq_cap, K, radius, out_idx32,
        (long long*)out_idx64);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

}  // extern "C"
