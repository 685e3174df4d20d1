// FLDetector (Zhang, Cao, Jia and Gong, KDD 2022): find malicious agents by how far each update lies from its prediction.  Three
// memory-bound passes over a coordinate range [begin, end) of the voted coordinates, every buffer but the participant slots addressed
// through pointers offset so that absolute coordinates index them (a rank's column slice on the fused multi-GPU path):
//
//   fld_ring_kernel      s[c] = fp32(w_g[c] - w_prev[c]) into a ring row (skipped when s is null), then w_prev[c] <- w_g[c].
//   fld_hvp_kernel       Hv[c] = fp32(sum_i c_i * s_i[c]), the sum in fp64 over the ring rows in chronological order, every product and
//                        every addition rounded on its own (no contraction), rounded to fp32 once: the bits ops.fld_hvp_statement gives.
//   fld_predict_kernel   per candidate k: u = fp32(w_k[c] - w_g[c]); PREDICT: e = fp32(fp32(h_k[c] + Hv[c]) - u), d_k^2 += e^2 in fp64
//                        (e^2 is exact in fp64); then h_k[c] <- u.  The <false> instantiation only records h_k.
//
// The predict pass uses history_accumulate_kernel's decomposition (foolsgold.cu): grid.x = coordinate splits (about two waves; one
// wave on the fused multi-GPU path, where every CTA has to be resident while it waits for the cross-GPU barrier-in), grid.y = groups
// of kFldGroup candidates, w_g and Hv read once per float4 and reused for the group.  Each CTA adds its threads' d^2 partials with
// fixed-shape warp and block sums into its [K] workspace slot, and launch_ordered_sum adds the slots in split order: no atomics, so
// d^2 is bitwise identical from launch to launch.  Hv is materialised once per round (one small launch) rather than recomputed by
// every group: at K = 200 recomputing it would read the N + 1 ring rows 25 times.
#include <algorithm>

#include "common.cuh"
#include "kernels.h"

namespace rlr {

constexpr int kFldThreads = 256;
constexpr int kFldGroup = 8;                            // candidates per CTA
constexpr int kFldMaxGroups = 65535;                    // grid.y

__global__ void __launch_bounds__(256) fld_ring_kernel(const float* __restrict__ w_g, float* __restrict__ w_prev, float* __restrict__ s,
                                                       long long begin, long long end) {
    pdl_wait();
    pdl_trigger();
    for (long long i = begin + 4 * ((long long)blockIdx.x * blockDim.x + threadIdx.x); i < end; i += 4LL * gridDim.x * blockDim.x) {
        const float4 g = ld_f4(w_g + i), p = ld_f4(w_prev + i);
        if (s) st_f4(s + i, make_float4(g.x - p.x, g.y - p.y, g.z - p.z, g.w - p.w));
        st_f4(w_prev + i, g);
    }
}

__global__ void __launch_bounds__(256) fld_hvp_kernel(const float* const* __restrict__ ring, const double* __restrict__ coef, int rows,
                                                      float* __restrict__ hv, long long begin, long long end) {
    pdl_wait();
    pdl_trigger();
    for (long long i = begin + 4 * ((long long)blockIdx.x * blockDim.x + threadIdx.x); i < end; i += 4LL * gridDim.x * blockDim.x) {
        double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;
        for (int r = 0; r < rows; ++r) {
            const double c = coef[r];
            const float4 v = ld_f4(ring[r] + i);
            a0 = __dadd_rn(a0, __dmul_rn(c, (double)v.x));
            a1 = __dadd_rn(a1, __dmul_rn(c, (double)v.y));
            a2 = __dadd_rn(a2, __dmul_rn(c, (double)v.z));
            a3 = __dadd_rn(a3, __dmul_rn(c, (double)v.w));
        }
        st_f4(hv + i, make_float4(__double2float_rn(a0), __double2float_rn(a1), __double2float_rn(a2), __double2float_rn(a3)));
    }
}

struct FldKernelParams {
    FldParams p;
    long long span;                                     // coordinates per split (multiple of 4)
    double* ws;                                         // [splits][K] (PREDICT)
};

template <bool PREDICT>
__global__ void __launch_bounds__(kFldThreads, 2) fld_predict_kernel(FldKernelParams kp) {
    __shared__ double scratch[32];
    pdl_wait();
    pdl_trigger();
    const FldParams& p = kp.p;
    const int k0 = blockIdx.y * kFldGroup;
    const int nk = min(kFldGroup, p.K - k0);
    // the group's pointers live in shared memory: in registers they would cost 32 of the 128 that two CTAs per SM leave
    __shared__ const float* wp[kFldGroup];
    __shared__ float* hp[kFldGroup];
    if (threadIdx.x < kFldGroup) {
        wp[threadIdx.x] = (int)threadIdx.x < nk ? p.w_agents[k0 + threadIdx.x] : nullptr;
        hp[threadIdx.x] = (int)threadIdx.x < nk ? p.rows[k0 + threadIdx.x] : nullptr;
    }

    barrier_in(p.gate, blockIdx.x == 0 && blockIdx.y == 0);

    double acc[kFldGroup];
#pragma unroll
    for (int j = 0; j < kFldGroup; ++j) acc[j] = 0.0;
    const long long lo = p.begin + (long long)blockIdx.x * kp.span;
    const long long hi = min(p.end, lo + kp.span);
    for (long long i = lo + 4LL * threadIdx.x; i < hi; i += 4LL * kFldThreads) {
        const float4 g = ld_f4(p.w_global + i);
        float4 hv = make_float4(0.f, 0.f, 0.f, 0.f);
        if (PREDICT) hv = ld_f4(p.hv + i);
        float4 w[kFldGroup], h[kFldGroup];
#pragma unroll
        for (int j = 0; j < kFldGroup; ++j) {
            if (j < nk) {
                w[j] = ld_f4(wp[j] + i);
                if (PREDICT) h[j] = ld_f4(hp[j] + i);
            }
        }
#pragma unroll
        for (int j = 0; j < kFldGroup; ++j) {
            if (j < nk) {
                const float4 u = make_float4(w[j].x - g.x, w[j].y - g.y, w[j].z - g.z, w[j].w - g.w);
                if (PREDICT) {
                    const float ex = __fsub_rn(__fadd_rn(h[j].x, hv.x), u.x), ey = __fsub_rn(__fadd_rn(h[j].y, hv.y), u.y);
                    const float ez = __fsub_rn(__fadd_rn(h[j].z, hv.z), u.z), ew = __fsub_rn(__fadd_rn(h[j].w, hv.w), u.w);
                    acc[j] += (double)ex * ex + (double)ey * ey + (double)ez * ez + (double)ew * ew;
                }
                st_f4(hp[j] + i, u);
            }
        }
    }
    if (PREDICT) {
#pragma unroll
        for (int j = 0; j < kFldGroup; ++j) {
            const double s = block_sum<double>(acc[j], scratch);
            if (threadIdx.x == 0 && j < nk) kp.ws[(size_t)blockIdx.x * p.K + k0 + j] = s;
        }
    }
}

cudaError_t launch_fld_ring(const float* w_g, float* w_prev, float* s, long long begin, long long end, int num_sms, cudaStream_t st) {
    if ((begin & 3) || (end & 3) || end < begin || !w_g || !w_prev) return cudaErrorInvalidValue;
    if (end == begin) return cudaSuccess;
    const long long n4 = (end - begin) / 4, cap = 8LL * num_sms;
    const int grid = (int)std::max(1LL, std::min(cap, (n4 + 255) / 256));
    return launch_kernel(fld_ring_kernel, dim3(grid), dim3(256), (size_t)0, st, w_g, w_prev, s, begin, end);
}

cudaError_t launch_fld_hvp(const float* const* ring, const double* coef, int rows, float* hv, long long begin, long long end, int num_sms,
                           cudaStream_t st) {
    if ((begin & 3) || (end & 3) || end < begin || rows < 1 || !ring || !coef || !hv) return cudaErrorInvalidValue;
    if (end == begin) return cudaSuccess;
    const long long n4 = (end - begin) / 4, cap = 8LL * num_sms;
    const int grid = (int)std::max(1LL, std::min(cap, (n4 + 255) / 256));
    return launch_kernel(fld_hvp_kernel, dim3(grid), dim3(256), (size_t)0, st, ring, coef, rows, hv, begin, end);
}

cudaError_t launch_fld_predict(const FldParams& p, double* out, int num_sms, cudaStream_t st) {
    if (p.K < 1 || (p.K + kFldGroup - 1) / kFldGroup > kFldMaxGroups || !p.w_global || !p.w_agents || !p.rows)
        return cudaErrorInvalidValue;
    if ((p.begin & 3) || (p.end & 3) || p.end < p.begin || !gate_ok(p.gate) || (p.hv && !out)) return cudaErrorInvalidValue;
    const bool predict = p.hv != nullptr;
    static int occ[2] = {0, 0};
    int& o = occ[predict];
    if (!o) {
        RLR_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(
            &o, predict ? fld_predict_kernel<true> : fld_predict_kernel<false>, kFldThreads, 0));
        o = o < 1 ? 1 : o;
    }
    FldKernelParams kp{};
    kp.p = p;
    const int groups = (p.K + kFldGroup - 1) / kFldGroup;
    const long long len = p.end - p.begin;
    const long long splits = coord_splits(len, groups, (long long)o * num_sms, p.gate.world);
    kp.span = ((len + splits - 1) / splits + 3) & ~3LL;
    const dim3 grid((unsigned)splits, (unsigned)groups);
    if (!predict) return launch_kernel(fld_predict_kernel<false>, grid, dim3(kFldThreads), (size_t)0, st, kp);
    Scratch ws((size_t)(splits * p.K) * sizeof(double), st);
    kp.ws = ws.as<double>();
    RLR_CUDA_CHECK(cudaMemsetAsync(out, 0, (size_t)p.K * sizeof(double), st));
    RLR_CUDA_CHECK(launch_kernel(fld_predict_kernel<true>, grid, dim3(kFldThreads), (size_t)0, st, kp));
    return launch_ordered_sum(out, kp.ws, (int)splits, (long long)p.K, st);
}

}  // namespace rlr
