// CRFL (Xie, Chen, Chen, Li, ICML 2021; DESIGN.md section 3): the server clips the global model's parameter norm to rho and adds
// Gaussian noise N(0, sigma^2 I) to the parameters after every round's complete server step, and the final model is certified by
// smoothing it in parameter space.  Three passes:
//
//   clip / perturb   norm    q = sum_c w'[c]^2 over the real parameters (bit c of the real-coordinate mask), each square exact in fp64
//                            and added in fp64: per-thread sums in grid-stride order, block sums, per-CTA slots added in CTA order by
//                            launch_ordered_sum -- no atomics, the same q on every run;
//                    apply   s = 1 if q <= rho^2 or q is not finite, else fp32(rho / sqrt(q)), read from the device (no host sync);
//                            w[c] = fp32(fp32(w'[c] * s) + fp32(sigma * z_c)) on real coordinates (the noise term only when
//                            sigma > 0), w[c] = w'[c] everywhere else (alignment padding, BatchNorm running statistics); the bf16
//                            shadow of every coordinate is written in the same sweep.  stats = {sqrt(q), s}.
//   smoothing        the apply pass with s = 1 into a certification executor's fp32 buffer and bf16 shadow: w + sigma z_m.
//   vote count       one thread per logit row: counts[row0 + r][argmax] += 1 (lowest class on ties; a row with a non-finite logit
//                    votes for no class).  Each row belongs to one thread and the draws run in stream order: no atomics.
//
// z_c is philox_normal4(Philox(seed), c / 4, stream) (common.cuh), lane c % 4; the stream word is ops.crfl_stream of the round
// (training) or of the draw index (certification).  Bytes per coordinate: 4 + 1/8 norm, 4 + 1/8 read + 4 + 2 written apply = 14.25 B.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"
#include "kernels.h"

namespace rlr {

namespace {

constexpr int kThreads = 256;

__device__ __forceinline__ uint32_t real_nibble(const uint32_t* __restrict__ mask, long long q) {
    return (__ldg(mask + (q >> 3)) >> ((q & 7) * 4)) & 0xFu;
}

__global__ void __launch_bounds__(kThreads) crfl_norm_kernel(const float* __restrict__ w, const uint32_t* __restrict__ mask, long long n4v,
                                                            double* __restrict__ part) {
    __shared__ double sd[32];
    double acc = 0.0;
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n4v; q += (long long)gridDim.x * blockDim.x) {
        const uint32_t nib = real_nibble(mask, q);
        if (!nib) continue;
        const float4 v = ld_f4(w + 4 * q);
        if (nib & 1u) acc += (double)v.x * (double)v.x;
        if (nib & 2u) acc += (double)v.y * (double)v.y;
        if (nib & 4u) acc += (double)v.z * (double)v.z;
        if (nib & 8u) acc += (double)v.w * (double)v.w;
    }
    const double tot = block_sum<double>(acc, sd);
    if (threadIdx.x == 0) part[blockIdx.x] = tot;
}

__device__ __forceinline__ float perturb(float v, bool real, float s, float sigma, float z) {
    if (!real) return v;
    const float o = __fmul_rn(v, s);
    return sigma != 0.0f ? __fadd_rn(o, __fmul_rn(sigma, z)) : o;
}

// qsum: the norm pass's q (clip / perturb), or nullptr for s = 1 (smoothing).  stats (optional): {sqrt(q), s}.  src may be dst (the pass
// after SparseFed runs in place); rho = +inf turns the clip off.
__global__ void __launch_bounds__(kThreads) crfl_apply_kernel(const float* src, float* dst,
                                                             __nv_bfloat16* __restrict__ wb, const uint32_t* __restrict__ mask,
                                                             long long n4v, long long n4, const double* __restrict__ qsum, double rho,
                                                             float sigma, unsigned long long seed, unsigned long long stream,
                                                             double* __restrict__ stats) {
    float s = 1.0f;
    if (qsum) {
        const double q = *qsum;
        if (isfinite(q) && q > rho * rho) s = (float)(rho / sqrt(q));
        if (stats && blockIdx.x == 0 && threadIdx.x == 0) {
            stats[0] = sqrt(q);
            stats[1] = (double)s;
        }
    }
    const Philox ph(seed);
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n4; q += (long long)gridDim.x * blockDim.x) {
        float4 v = ld_f4(src + 4 * q);
        if (q < n4v) {
            const uint32_t nib = real_nibble(mask, q);
            if (nib) {
                const float4 z = sigma != 0.0f ? philox_normal4(ph, (uint64_t)q, stream) : make_float4(0.f, 0.f, 0.f, 0.f);
                v = make_float4(perturb(v.x, nib & 1u, s, sigma, z.x), perturb(v.y, nib & 2u, s, sigma, z.y),
                                perturb(v.z, nib & 4u, s, sigma, z.z), perturb(v.w, nib & 8u, s, sigma, z.w));
            }
        }
        st_f4(dst + 4 * q, v);
        if (wb) *reinterpret_cast<uint2*>(wb + 4 * q) = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
    }
}

__global__ void __launch_bounds__(kThreads) vote_count_kernel(const float* __restrict__ logits, long long rows, int classes,
                                                             int* __restrict__ counts, long long row0) {
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= rows) return;
    const float* x = logits + r * classes;
    int best = 0;
    float bv = x[0];
    bool finite = isfinite(bv);
    for (int c = 1; c < classes; ++c) {
        const float v = x[c];
        finite = finite && isfinite(v);
        if (v > bv) { bv = v; best = c; }
    }
    if (finite) counts[(row0 + r) * classes + best] += 1;
}

// grid-stride sweeps: enough CTAs for the vector, at most per_sm per SM
inline int sweep_ctas(long long n4, int num_sms, int per_sm) {
    const long long want = (n4 + kThreads - 1) / kThreads, cap = (long long)num_sms * per_sm;
    return (int)(want < 1 ? 1 : (want > cap ? cap : want));
}

}  // namespace

cudaError_t launch_crfl_clip_noise(const float* w_new, float* w, void* w_bf16, const uint32_t* mask, long long n_vote, long long n,
                                   double rho, float sigma, unsigned long long seed, unsigned long long stream, double* stats,
                                   int num_sms, cudaStream_t st) {
    if ((n_vote & 3) || (n & 3) || n_vote > n || n_vote < 0 || !(rho > 0.0)) return cudaErrorInvalidValue;
    const long long n4v = n_vote / 4, n4 = n / 4;
    const int ngrid = sweep_ctas(n4v, num_sms, 4);
    Scratch scr((size_t)(ngrid + 1) * sizeof(double), st);
    double* q = scr.as<double>();
    double* part = q + 1;
    RLR_CUDA_CHECK(cudaMemsetAsync(q, 0, sizeof(double), st));
    crfl_norm_kernel<<<ngrid, kThreads, 0, st>>>(w_new, mask, n4v, part);
    RLR_CUDA_CHECK(cudaGetLastError());
    RLR_CUDA_CHECK(launch_ordered_sum(q, part, ngrid, 1LL, st));
    crfl_apply_kernel<<<sweep_ctas(n4, num_sms, 8), kThreads, 0, st>>>(w_new, w, static_cast<__nv_bfloat16*>(w_bf16), mask, n4v, n4, q, rho,
                                                                     sigma, seed, stream, stats);
    return cudaGetLastError();
}

cudaError_t launch_crfl_smooth(const float* w, float* out, void* out_bf16, const uint32_t* mask, long long n_vote, long long n, float sigma,
                               unsigned long long seed, unsigned long long stream, int num_sms, cudaStream_t st) {
    if ((n_vote & 3) || (n & 3) || n_vote > n || n_vote < 0) return cudaErrorInvalidValue;
    crfl_apply_kernel<<<sweep_ctas(n / 4, num_sms, 8), kThreads, 0, st>>>(w, out, static_cast<__nv_bfloat16*>(out_bf16), mask, n_vote / 4,
                                                                        n / 4, nullptr, 0.0, sigma, seed, stream, nullptr);
    return cudaGetLastError();
}

cudaError_t launch_vote_count(const float* logits, long long rows, int classes, int* counts, long long row0, cudaStream_t st) {
    if (rows < 0 || classes < 1 || row0 < 0) return cudaErrorInvalidValue;
    if (rows == 0) return cudaSuccess;
    vote_count_kernel<<<(unsigned)((rows + kThreads - 1) / kThreads), kThreads, 0, st>>>(logits, rows, classes, counts, row0);
    return cudaGetLastError();
}

}  // namespace rlr
