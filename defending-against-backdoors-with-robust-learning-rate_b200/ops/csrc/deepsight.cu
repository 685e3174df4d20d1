// DeepSight's statistics pass (Rieger, Nguyen, Miettinen, Sadeghi, NDSS 2022; DESIGN.md section 3): for each candidate model k of
// this rank's slots, from its eval-mode logits z_k and the global model's z_g on S seeds of N random inputs (fp32 [S N][P]) and from
// the head slices of its flat parameters,
//   DDif[k][s][c] = (1/N) sum_m exp((z_k[m,c] - lse z_k[m]) - (z_g[m,c] - lse z_g[m])),   m over seed s's rows, ascending,
//   eps[k][c]     = |fp32(db_c)| + sum_j |fp32(dW_cj)|,                                   added left to right, j ascending,
//   db[k][c]      = fp32(b_k[c] - b_g[c]),
// everything after the fp32 differences in fp64.  lse z[m] = max_c z[m,c] + log(sum_c exp(z[m,c] - max)), the sum over c ascending; it
// is NaN when any logit of the row is not finite, so such a candidate's DDif is NaN and the host never accepts it.
//
// Two launches, both one thread per output and each thread adding its own terms in the stated order, so no atomics and no cross-thread
// reduction: run-to-run bitwise equal.  deepsight_lse_kernel writes lse of every row (the candidates', then the global model's) to a
// scratch vector; deepsight_stats_kernel gives its first K S P threads the DDif entries and the next K P threads eps and db.  The
// head weight W is [P][d] row-major at w_off of each flat vector, the bias [P] at b_off.  P <= kDeepSightMaxClasses (the zoo's heads
// have 10 or 62 classes); a larger P is refused, not computed.
#include "common.cuh"
#include "kernels.h"

namespace rlr {

namespace {

constexpr int kDeepSightThreads = 128;

struct DeepSightParams {
    const float* z;                              // [K][S N][P] candidates' logits
    const float* zg;                             // [S N][P] global logits
    const float* const* slots;                   // [K] flat fp32 parameters of the candidates
    const float* wg;                             // flat fp32 global parameters
    long long w_off, b_off;                      // head weight [P][d] and bias [P] offsets in the flat vectors
    int K, S, N, P, d;
    double* lse;                                 // [(K + 1) S N]: the candidates' rows, then the global model's
    double* out;                                 // [K][(S + 2) P]: DDif [S][P], eps [P], db [P]
};

__global__ void __launch_bounds__(kDeepSightThreads) deepsight_lse_kernel(DeepSightParams kp) {
    const long long SN = (long long)kp.S * kp.N;
    const long long r = (long long)blockIdx.x * kDeepSightThreads + threadIdx.x;
    if (r >= (kp.K + 1) * SN) return;
    const float* const row = r < kp.K * SN ? kp.z + r * kp.P : kp.zg + (r - kp.K * SN) * kp.P;
    double mx = -INFINITY;
    bool finite = true;
    for (int c = 0; c < kp.P; ++c) {
        const float v = row[c];
        finite = finite && isfinite(v);
        mx = fmax(mx, (double)v);
    }
    double s = 0.0;
    for (int c = 0; c < kp.P; ++c) s += exp((double)row[c] - mx);
    kp.lse[r] = finite ? mx + log(s) : (double)NAN;
}

__global__ void __launch_bounds__(kDeepSightThreads) deepsight_stats_kernel(DeepSightParams kp) {
    const int P = kp.P, S = kp.S, N = kp.N;
    const long long SN = (long long)S * N;
    const long long t = (long long)blockIdx.x * kDeepSightThreads + threadIdx.x;
    const long long n_ddif = (long long)kp.K * S * P;
    const int W = (S + 2) * P;
    if (t < n_ddif) {
        const int k = (int)(t / (S * P));
        const int s = (int)(t / P % S), c = (int)(t % P);
        const long long i0 = (long long)s * N;
        const float* const zk = kp.z + ((long long)k * SN + i0) * P + c;
        const float* const zg = kp.zg + i0 * P + c;
        const double* const lk = kp.lse + (long long)k * SN + i0;
        const double* const lg = kp.lse + (long long)kp.K * SN + i0;
        double sum = 0.0;
        for (int m = 0; m < N; ++m)                                              // seed s's samples, ascending
            sum += exp(((double)zk[(long long)m * P] - lk[m]) - ((double)zg[(long long)m * P] - lg[m]));
        kp.out[(long long)k * W + s * P + c] = sum / (double)N;
        return;
    }
    const long long u = t - n_ddif;
    if (u >= (long long)kp.K * P) return;
    const int k = (int)(u / P), c = (int)(u % P);
    const float* const w = kp.slots[k];
    const float db = __fsub_rn(w[kp.b_off + c], kp.wg[kp.b_off + c]);
    const float* const wr = w + kp.w_off + (long long)c * kp.d;
    const float* const gr = kp.wg + kp.w_off + (long long)c * kp.d;
    double eps = fabs((double)db);
    for (int j = 0; j < kp.d; ++j) eps += fabs((double)__fsub_rn(wr[j], gr[j]));   // ascending j
    kp.out[(long long)k * W + S * P + c] = eps;
    kp.out[(long long)k * W + (S + 1) * P + c] = (double)db;
}

}  // namespace

cudaError_t launch_deepsight_stats(const float* z, const float* zg, const float* const* slots, const float* wg, long long w_off,
                                   long long b_off, int K, int S, int N, int P, int d, double* out, cudaStream_t st) {
    if (K < 1 || S < 1 || N < 1 || d < 1 || !z || !zg || !slots || !wg || !out || w_off < 0 || b_off < 0) return cudaErrorInvalidValue;
    if (P < 1 || P > kDeepSightMaxClasses) return cudaErrorInvalidValue;
    DeepSightParams kp{};
    kp.z = z;
    kp.zg = zg;
    kp.slots = slots;
    kp.wg = wg;
    kp.w_off = w_off;
    kp.b_off = b_off;
    kp.K = K;
    kp.S = S;
    kp.N = N;
    kp.P = P;
    kp.d = d;
    kp.out = out;
    const long long rows = (long long)(K + 1) * S * N;
    const long long threads = (long long)K * S * P + (long long)K * P;
    const long long g1 = (rows + kDeepSightThreads - 1) / kDeepSightThreads, g2 = (threads + kDeepSightThreads - 1) / kDeepSightThreads;
    if (g1 > 0x7fffffffLL || g2 > 0x7fffffffLL) return cudaErrorInvalidValue;
    Scratch ws((size_t)rows * sizeof(double), st);
    kp.lse = ws.as<double>();
    deepsight_lse_kernel<<<dim3((unsigned)g1), kDeepSightThreads, 0, st>>>(kp);
    RLR_CUDA_CHECK(cudaGetLastError());
    deepsight_stats_kernel<<<dim3((unsigned)g2), kDeepSightThreads, 0, st>>>(kp);
    return cudaGetLastError();
}

}  // namespace rlr
