// Training pairs for ModelNet40: the reference's crop chain on shapes that live on the device.
//
// Reference behaviour replaced (paths relative to the reference's src/):
//   data_loaders/modelnet_transforms.py   SplitSourceRef -> RandomCrop -> RandomTransformSE3_euler -> Resampler(717)
//                                         -> RandomJitter -> ShufflePoints, with the overlap masks and the
//                                         correspondences each transform maintains
// Parity rules: DESIGN.md section 8, "ModelNet training data".
//
// One CTA per pair does everything in shared memory: gather the shape, centroid and float64 distances to both crop
// planes, a bitonic sort of each side's distances for numpy's percentile threshold, the crop masks, a CTA-wide scan
// that lists the kept points in ascending raw index, the ordered subset (first n_out positions of a keyed Feistel
// bijection over the kept points), the rigid transform and the jitter, and a second scan for the correspondences.
// The per-pair scalars (crop directions, transform) come from the host; nothing else does.
#include <math.h>
#include <math_constants.h>

#include "common.cuh"
#include "philox.cuh"

static_assert(sizeof(regtr_modelnet_args) == 128, "regtr_modelnet_args layout");

namespace {

constexpr int MN_T = 512;                                  // threads per pair
constexpr int MN_N = REGTR_MODELNET_MAX_PTS;               // raw points per shape, at most
constexpr int MN_PPT = MN_N / MN_T;                        // raw points per thread: 4 t .. 4 t + 3
constexpr int MN_WARPS = MN_T / 32;

struct MnSmem {
    float x[MN_N * 3];        // the raw shape
    double d[2][MN_N];        // centroid partial sums, then each side's distances (sorted), then the kept lists
    int16_t pos[2][MN_N];     // output position of each raw point per side, or -1
    uint8_t keep[2][MN_N];    // crop masks
    int warp[MN_WARPS];
    float c[3];
    double thr[2];
};

// Exclusive scan of v over the CTA (threads in order); `total` gets the sum.  Two __syncthreads.
__device__ __forceinline__ int cta_excl_scan(int v, int* s_warp, int& total) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int u = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += u;
    }
    if (lane == 31) s_warp[w] = inc;
    __syncthreads();
    int base = 0;
    total = 0;
#pragma unroll
    for (int i = 0; i < MN_WARPS; ++i) {
        const int s = s_warp[i];
        base += i < w ? s : 0;
        total += s;
    }
    __syncthreads();
    return base + inc - v;
}

__global__ void __launch_bounds__(MN_T, 1) k_modelnet_augment(const regtr_modelnet_args a, int pair_base) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    MnSmem& s = *reinterpret_cast<MnSmem*>(smem_raw);
    const int b = blockIdx.x, t = threadIdx.x, n = a.n_pts, n_out = a.n_out;

    // 1. the shape, by its item index
    const int item = a.items[b];
    bool bad = item < 0 || item >= a.n_shapes;
    if (!bad) {
        const float* src = a.shapes + (size_t)item * n * 3;
        for (int i = t; i < 3 * n; i += MN_T) {
            const float v = src[i];
            bad |= !isfinite(v);
            s.x[i] = v;
        }
    }
    if (__syncthreads_or(bad)) {
        if (t == 0) { atomicOr(a.status, REGTR_STATUS_INPUT); a.corr_n[b] = 0; }
        return;
    }

    // 2. centroid: thread t sums points t, t + 512, t + 1024, t + 1536 left to right in float64, then a tree
    //    s[t] += s[t + h] for h = 256 .. 1; c = fp32(sum / n)
    double* red = &s.d[0][0];                              // 3 x MN_T doubles
    for (int ax = 0; ax < 3; ++ax) {
        double acc = 0.0;
        for (int r = 0; r < MN_PPT; ++r) {
            const int i = t + r * MN_T;
            if (i < n) acc = __dadd_rn(acc, (double)s.x[3 * i + ax]);
        }
        red[ax * MN_T + t] = acc;
    }
    __syncthreads();
    for (int h = MN_T / 2; h > 0; h >>= 1) {
        if (t < h)
            for (int ax = 0; ax < 3; ++ax) red[ax * MN_T + t] = __dadd_rn(red[ax * MN_T + t], red[ax * MN_T + t + h]);
        __syncthreads();
    }
    if (t < 3) s.c[t] = (float)__ddiv_rn(red[t * MN_T], (double)n);
    __syncthreads();

    // distances of this thread's points to both planes: kept in registers and copied for the sort (+inf padding)
    const double* prm = a.params + (size_t)b * REGTR_MODELNET_PARAMS;
    double dist[2][MN_PPT];
    for (int r = 0; r < MN_PPT; ++r) {
        const int i = MN_PPT * t + r;
        for (int side = 0; side < 2; ++side) {
            double v = CUDART_INF;
            if (i < n) {
                const double* u = prm + 3 * side;
                const double cx = (double)__fsub_rn(s.x[3 * i], s.c[0]), cy = (double)__fsub_rn(s.x[3 * i + 1], s.c[1]),
                             cz = (double)__fsub_rn(s.x[3 * i + 2], s.c[2]);
                v = __dadd_rn(__dadd_rn(__dmul_rn(cx, u[0]), __dmul_rn(cy, u[1])), __dmul_rn(cz, u[2]));
            }
            dist[side][r] = v;
        }
    }
    __syncthreads();                                       // the centroid sums are read by now
    for (int r = 0; r < MN_PPT; ++r) { s.d[0][MN_PPT * t + r] = dist[0][r]; s.d[1][MN_PPT * t + r] = dist[1][r]; }
    __syncthreads();

    // 3. the order statistics: bitonic sort of both sides' MN_N distances (ascending)
    if (a.k >= 0) {
        for (int kk = 2; kk <= MN_N; kk <<= 1) {
            for (int j = kk >> 1; j > 0; j >>= 1) {
                for (int q = t; q < MN_N; q += MN_T) {       // MN_N / 2 compare-exchanges per side
                    const int side = q / (MN_N / 2), i = q % (MN_N / 2);
                    const int lo = ((i & ~(j - 1)) << 1) | (i & (j - 1)), hi = lo + j;
                    const bool up = (lo & kk) == 0;
                    const double x = s.d[side][lo], y = s.d[side][hi];
                    if ((x > y) == up) { s.d[side][lo] = y; s.d[side][hi] = x; }
                }
                __syncthreads();
            }
        }
        // numpy's _lerp: a + (b - a) gamma, or b - (b - a)(1 - gamma) when gamma >= 0.5
        if (t < 2) {
            const double lo = s.d[t][a.k], hi = s.d[t][a.k + 1], diff = __dsub_rn(hi, lo);
            s.thr[t] = a.gamma >= 0.5 ? __dsub_rn(hi, __dmul_rn(diff, __dsub_rn(1.0, a.gamma)))
                                      : __dadd_rn(lo, __dmul_rn(diff, a.gamma));
        }
    } else if (t < 2) {
        s.thr[t] = 0.0;
    }
    __syncthreads();

    // 4. crop masks, and the kept points of each side in ascending raw index (one scan of both counts, packed)
    int packed = 0;
    for (int r = 0; r < MN_PPT; ++r) {
        const int i = MN_PPT * t + r;
        const bool k0 = i < n && dist[0][r] > s.thr[0], k1 = i < n && dist[1][r] > s.thr[1];
        s.keep[0][i] = k0; s.keep[1][i] = k1;
        s.pos[0][i] = -1; s.pos[1][i] = -1;
        packed += (int)k0 + ((int)k1 << 16);
    }
    int total;
    int base = cta_excl_scan(packed, s.warp, total);
    const int n_kept[2] = {total & 0xFFFF, total >> 16};
    int* kept = reinterpret_cast<int*>(&s.d[0][0]);        // kept[side * MN_N + rank]
    {
        int r0 = base & 0xFFFF, r1 = base >> 16;
        for (int r = 0; r < MN_PPT; ++r) {
            const int i = MN_PPT * t + r;
            if (s.keep[0][i]) kept[r0++] = i;
            if (s.keep[1][i]) kept[MN_N + r1++] = i;
        }
    }
    if (n_kept[0] < n_out || n_kept[1] < n_out) {
        if (t == 0) { atomicOr(a.status, REGTR_STATUS_CROP); a.corr_n[b] = 0; }
        return;
    }
    __syncthreads();

    // 5-7. the ordered subset, the transform of the source, the jitter
    const Keys ks = make_keys(a.seed, a.step);
    for (int side = 0; side < 2; ++side) {
        const Perm pm = make_perm(n_kept[side], true, ks, pair_base + b, side);
        const size_t slot = (size_t)(side * a.B + b) * n_out;
        for (int j = t; j < n_out; j += MN_T) {
            const int i = kept[side * MN_N + (int)perm_fwd(pm, (unsigned)j)];
            s.pos[side][i] = (int16_t)j;
            double v[3] = {(double)s.x[3 * i], (double)s.x[3 * i + 1], (double)s.x[3 * i + 2]};
            if (side == 0) {
                const double* m = prm + 6;
                float w[3];
                for (int ax = 0; ax < 3; ++ax) {
                    const double* row = m + 4 * ax;
                    w[ax] = (float)__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(row[0], v[0]), __dmul_rn(row[1], v[1])),
                                                       __dmul_rn(row[2], v[2])), row[3]);
                }
                for (int ax = 0; ax < 3; ++ax) v[ax] = (double)w[ax];
            }
            if (a.noise != 0.0) {
                const U4 r = philox(U4{(unsigned)i, 2u * (unsigned)(pair_base + b) + (unsigned)side, ks.s0, ks.s1},
                                    ks.k0, ks.k1);
                const double m0 = sqrt(-2.0 * log(u01(r.x))), m1 = sqrt(-2.0 * log(u01(r.z)));
                double s0, c0, s1, c1;
                sincospi(2.0 * u01(r.y), &s0, &c0);
                sincospi(2.0 * u01(r.w), &s1, &c1);
                const double g[3] = {m0 * c0, m0 * s0, m1 * c1};
                for (int ax = 0; ax < 3; ++ax)
                    v[ax] = __dadd_rn(v[ax], fmin(fmax(__dmul_rn(a.noise, g[ax]), -a.clip), a.clip));
            }
            float* o = a.out_xyz + 3 * (slot + j);
            o[0] = (float)v[0]; o[1] = (float)v[1]; o[2] = (float)v[2];
            a.out_mask[slot + j] = s.keep[1 - side][i];
        }
    }
    __syncthreads();

    // 8. correspondences: raw points present in both outputs, in ascending raw index
    int flags = 0;
    for (int r = 0; r < MN_PPT; ++r) {
        const int i = MN_PPT * t + r;
        flags += (s.pos[0][i] >= 0 && s.pos[1][i] >= 0);
    }
    base = cta_excl_scan(flags, s.warp, total);
    int32_t* c0 = a.corr + (size_t)b * 2 * n_out;
    for (int r = 0; r < MN_PPT; ++r) {
        const int i = MN_PPT * t + r;
        if (s.pos[0][i] >= 0 && s.pos[1][i] >= 0) {
            c0[base] = s.pos[0][i];
            c0[n_out + base] = s.pos[1][i];
            ++base;
        }
    }
    if (t == 0) a.corr_n[b] = total;
}

}  // namespace

extern "C" int regtr_modelnet_augment(const regtr_modelnet_args* args, int pair_base, void* stream_) {
    if (!args || pair_base < 0 || pair_base > (1 << 30)) return REGTR_ERR_ARG;
    const regtr_modelnet_args& a = *args;
    if (a.B <= 0 || a.B > 65535 || a.n_pts <= 0 || a.n_pts > REGTR_MODELNET_MAX_PTS || a.n_shapes <= 0 ||
        a.n_out <= 0 || a.n_out > a.n_pts || a.k < -1 || a.k > a.n_pts - 2 || !(a.gamma >= 0.0 && a.gamma < 1.0) ||
        !(a.noise >= 0.0) || !(a.clip >= 0.0) || !a.shapes || !a.params || !a.items || !a.out_xyz || !a.out_mask ||
        !a.corr || !a.corr_n || !a.status)
        return REGTR_ERR_ARG;
    const size_t smem = sizeof(MnSmem);
    if (cudaFuncSetAttribute(k_modelnet_augment, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
        return REGTR_ERR_UNSUPPORTED;
    k_modelnet_augment<<<a.B, MN_T, smem, (cudaStream_t)stream_>>>(a, pair_base);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}
