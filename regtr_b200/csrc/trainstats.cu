// Training-loop bookkeeping on the device: the loss meters (utils/misc.py AverageMeter, StatsMeter) with the
// loss_smooth EMA of trainer.py:127-134, and the validation pose errors (se3_compare + _aggregate_metrics).
//
// Both kernels are tiny and run on one thread per independent accumulator, in a fixed order, so that every sum is
// the same sequence of IEEE double operations the reference performs with Python floats: __dadd_rn / __dmul_rn keep
// the compiler from contracting a product and a sum into an FMA.
#include <math.h>

#include "common.cuh"

static_assert(sizeof(regtr_meter_args) == 200, "regtr_meter_args layout");
static_assert(sizeof(regtr_pose_err_args) == 72, "regtr_pose_err_args layout");

namespace {

// One thread per (bank, key) meter; thread 0 also owns the EMA and the non-finite log.
__global__ void k_meter_update(const regtr_meter_args a) {
    const int t = threadIdx.x;
    if (t < a.n_banks * a.n_keys) {
        const int b = t / a.n_keys, k = t - b * a.n_keys;
        const double v = (double)*a.vals[k];
        if (!isnan(v)) {                                  // math.isnan: +-inf is accumulated
            double* s = a.banks[b] + 4 * k;
            s[0] = v;
            s[1] = __dadd_rn(s[1], v);                    // sum += val * 1
            s[2] = __dadd_rn(s[2], __dmul_rn(v, v));      // sq_sum += val ** 2 * 1 (exact: v is an fp32 value)
            s[3] = __dadd_rn(s[3], 1.0);
        }
    }
    if (t == 0 && a.smooth != nullptr && a.total_key >= 0) {
        const double v = (double)*a.vals[a.total_key];
        if (a.smooth[1] == 0.0) {                         // loss_smooth is None: taken as-is, finite or not
            a.smooth[0] = v;
            a.smooth[1] = 1.0;
        } else if (!isfinite(v)) {                        // skipped; the host warns for this step
            if (a.log != nullptr) {
                const long long n = a.log[0];
                if (n < a.log_cap) a.log[1 + n] = a.step;
                a.log[0] = n + 1;
            }
        } else {
            a.smooth[0] = __dadd_rn(__dmul_rn(0.99, a.smooth[0]), __dmul_rn(0.01, v));
        }
    }
}

// One thread per decoder layer walks the batch's pairs in order: the accumulations do not depend on the launch.
__global__ void k_pose_errors(const regtr_pose_err_args a) {
    const int l = threadIdx.x;
    if (l >= a.L) return;
    double* acc = a.acc + 4 * l;
    for (int b = 0; b < a.B; ++b) {
        const float* P = a.pred + ((long long)l * a.B + b) * 12;
        const float* G = a.gt + (long long)b * 12;
        double R[3][3];                                   // Ra Rb^T
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) {
                double s = __dmul_rn((double)P[4 * i + 0], (double)G[4 * j + 0]);
                s = __dadd_rn(s, __dmul_rn((double)P[4 * i + 1], (double)G[4 * j + 1]));
                s = __dadd_rn(s, __dmul_rn((double)P[4 * i + 2], (double)G[4 * j + 2]));
                R[i][j] = s;
            }
        const double tr = __dadd_rn(__dadd_rn(R[0][0], R[1][1]), R[2][2]);
        double c = __dmul_rn(0.5, __dadd_rn(tr, -1.0));
        c = fmin(fmax(c, -1.0), 1.0);
        const double rot = __dmul_rn(acos(c), 180.0 / 3.14159265358979323846);
        double n2 = 0.0;
        for (int i = 0; i < 3; ++i) {                     // ta - R tb
            double rt = __dmul_rn(R[i][0], (double)G[3]);
            rt = __dadd_rn(rt, __dmul_rn(R[i][1], (double)G[7]));
            rt = __dadd_rn(rt, __dmul_rn(R[i][2], (double)G[11]));
            const double d = __dadd_rn((double)P[4 * i + 3], -rt);
            n2 = __dadd_rn(n2, __dmul_rn(d, d));
        }
        const double trans = sqrt(n2);
        const long long h = (long long)l * a.hist_cap + a.offset + b;
        a.rot_hist[h] = rot;
        a.trans_hist[h] = trans;
        acc[0] = __dadd_rn(acc[0], rot);
        acc[1] = __dadd_rn(acc[1], trans);
        if (rot < a.thresh_rot && trans < a.thresh_trans) acc[2] = __dadd_rn(acc[2], 1.0);
        acc[3] = __dadd_rn(acc[3], 1.0);
    }
}

}  // namespace

extern "C" {

int regtr_meter_update(const regtr_meter_args* args, void* stream_) {
    if (!args) return REGTR_ERR_ARG;
    const regtr_meter_args& a = *args;
    if (a.n_keys < 1 || a.n_keys > REGTR_METER_MAX_KEYS || a.n_banks < 0 || a.n_banks > REGTR_METER_MAX_BANKS ||
        a.total_key >= a.n_keys || a.log_cap < 0)
        return REGTR_ERR_ARG;
    for (int k = 0; k < a.n_keys; ++k)
        if (!a.vals[k]) return REGTR_ERR_ARG;
    for (int b = 0; b < a.n_banks; ++b)
        if (!a.banks[b]) return REGTR_ERR_ARG;
    if (a.n_banks == 0 && (a.smooth == nullptr || a.total_key < 0)) return REGTR_OK;
    const int threads = ((a.n_banks * a.n_keys + 31) / 32) * 32;
    k_meter_update<<<1, threads > 0 ? threads : 32, 0, (cudaStream_t)stream_>>>(a);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

int regtr_pose_errors(const regtr_pose_err_args* args, void* stream_) {
    if (!args) return REGTR_ERR_ARG;
    const regtr_pose_err_args& a = *args;
    if (a.L < 1 || a.L > 1024 || a.B < 0 || a.offset < 0 || (long long)a.offset + a.B > a.hist_cap ||
        !a.pred || !a.gt || !a.rot_hist || !a.trans_hist || !a.acc)
        return REGTR_ERR_ARG;
    if (a.B == 0) return REGTR_OK;
    k_pose_errors<<<1, ((a.L + 31) / 32) * 32, 0, (cudaStream_t)stream_>>>(a);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

}  // extern "C"
