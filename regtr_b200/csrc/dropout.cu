// Transformer dropout, the elementwise parts: the feed-forward dropout applied in place to relu(linear1) (site 5)
// and the keep-mask export for tests and analysis.  The attention-probability dropout lives in the attention kernels
// (attention.cu, backward.cu) and the residual dropouts in the LayerNorm that follows them (norm.cu, backward.cu).
// Keep rule and counter layout: philox.cuh.
#include "common.cuh"
#include "philox.cuh"

namespace {

// thread = (8-row group, column) of one cloud (blockIdx.y): one Philox block serves its 8 rows
__global__ void k_dropout_rows(float* __restrict__ h, int F, const int32_t* __restrict__ offs, DropKey drop) {
    const int c = blockIdx.y;
    const int r0 = offs[c], len = offs[c + 1] - r0;
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int rg = (int)(t / F), col = (int)(t - (long long)rg * F);
    if (8 * rg >= len) return;
    const unsigned m = drop_keep8(drop, drop_word1(drop, c, 0), (unsigned)rg, (unsigned)col);
    const int nr = min(8, len - 8 * rg);
    float* p = h + ((size_t)r0 + 8 * rg) * F + col;
    for (int r = 0; r < nr; ++r) p[(size_t)r * F] = ((m >> r) & 1u) ? __fmul_rn(p[(size_t)r * F], drop.scale) : 0.f;
}

__global__ void k_dropout_keep_mask(DropKey drop, int cloud, int head, int rows, int cols, uint8_t* __restrict__ out) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)rows * cols) return;
    const int r = (int)(t / cols), j = (int)(t - (long long)r * cols);
    out[t] = drop_keep(drop, drop_word1(drop, cloud, head), (unsigned)r, (unsigned)j) ? 1 : 0;
}

}  // namespace

extern "C" {

int regtr_dropout_rows(float* h, int n, int F, const int32_t* offs, int max_len, const regtr_dropout_args* drop,
                       void* stream_) {
    DropKey dk;
    if (drop_key_of(drop, dk) != REGTR_OK || n < 0 || F <= 0 || max_len < 0) return REGTR_ERR_ARG;
    if (F > 65536 || max_len >= (1 << 16)) return REGTR_ERR_UNSUPPORTED;
    if (n == 0 || max_len == 0) return REGTR_OK;
    if (!h || !offs || 2 * drop->n_pairs > 65535) return REGTR_ERR_ARG;
    const long long items = (long long)regtr_cdiv(max_len, 8) * F;
    k_dropout_rows<<<dim3(regtr_cdiv(items, 256), 2 * drop->n_pairs), 256, 0, (cudaStream_t)stream_>>>(h, F, offs, dk);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

int regtr_dropout_keep_mask(const regtr_dropout_args* args, int cloud, int head, int rows, int cols, uint8_t* out,
                            void* stream_) {
    DropKey dk;
    if (drop_key_of(args, dk) != REGTR_OK || cloud < 0 || cloud >= 2 * args->n_pairs || head < 0 || head > 15)
        return REGTR_ERR_ARG;
    if (rows < 0 || cols < 0 || rows >= (1 << 19) || cols > (1 << 16)) return REGTR_ERR_ARG;
    if ((long long)rows * cols == 0) return REGTR_OK;
    if (!out) return REGTR_ERR_ARG;
    k_dropout_keep_mask<<<regtr_cdiv((long long)rows * cols, 256), 256, 0, (cudaStream_t)stream_>>>(dk, cloud, head, rows,
                                                                                                  cols, out);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

}  // extern "C"
