// SparseFed (Panda et al., AISTATS 2022; DESIGN.md section 3): the server applies only the top-k coordinates of its accumulated step and
// carries the rest over as error feedback.  It runs after the unchanged server step, which wrote its fp32 result w' to a scratch vector:
//
//   accumulate   for c < n_vote: e'[c] = fp32(e[c] + fp32(w'[c] - w[c])), written over e, and the first radix-histogram pass of the
//                keys bits(|e'[c]|) in the same sweep (topk_select.cuh's topk_hist_kernel with the AccumulateKeys loader);
//   select       the remaining two histogram passes over |e'| and the three bin searches: tau = the k-th largest key, on the device;
//   apply        M = {c < n_vote : key[c] >= max(tau, 1)}; w[c] <- fp32(w[c] + e'[c]) and e[c] <- 0 on M, w and e' kept elsewhere;
//                w[c] <- w'[c] for c >= n_vote (the BatchNorm running statistics keep the plain step); the bf16 shadow of every
//                coordinate is rewritten from the new w.  |M| is counted with integer atomics and ||e''||^2 goes to per-CTA fp64 partials;
//   finish       one thread adds the partials in CTA order: stats = {|M|, float(tau), ||e''||_2}.
//
// Every add is a single fp32 operation (no product to contract into an FMA), so numpy float32 arithmetic states it bit for bit
// (ops.sparsefed_statement).  Bytes per voted coordinate: 16 accumulate (w', w, e read, e written), 4 + 4 for the two later histogram
// passes, 10 apply (e and w read, the bf16 shadow written) plus 8 per applied coordinate (w and e written): 34 B + 8 B |M| / n_vote.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"
#include "kernels.h"
#include "topk_select.cuh"

namespace rlr {

namespace {

constexpr int kApplyThreads = 256;

// Pass 0 fused with the accumulation: e <- fp32(e + fp32(w' - w)), keys of the new e
struct AccumulateKeys {
    const float* __restrict__ wn;
    const float* __restrict__ w;
    float* __restrict__ e;
    __device__ __forceinline__ uint4 keys(long long q) const {
        const float4 a = ld_f4(wn + 4 * q), b = ld_f4(w + 4 * q), c = ld_f4(e + 4 * q);
        const float4 r = make_float4(__fadd_rn(c.x, __fsub_rn(a.x, b.x)), __fadd_rn(c.y, __fsub_rn(a.y, b.y)),
                                     __fadd_rn(c.z, __fsub_rn(a.z, b.z)), __fadd_rn(c.w, __fsub_rn(a.w, b.w)));
        st_f4(e + 4 * q, r);
        return make_uint4(magnitude_key(r.x), magnitude_key(r.y), magnitude_key(r.z), magnitude_key(r.w));
    }
};

// Passes 1 and 2: the keys of the accumulated error
struct ErrorKeys {
    const float* __restrict__ e;
    __device__ __forceinline__ uint4 keys(long long q) const {
        const float4 r = ld_f4(e + 4 * q);
        return make_uint4(magnitude_key(r.x), magnitude_key(r.y), magnitude_key(r.z), magnitude_key(r.w));
    }
};

__device__ __forceinline__ float take(bool in, float x) { return in ? x : 0.0f; }

__global__ void __launch_bounds__(kApplyThreads) sparsefed_apply_kernel(const float* __restrict__ wn, float* __restrict__ w,
                                                                        __nv_bfloat16* __restrict__ wb, float* __restrict__ e,
                                                                        long long n4v, long long n4, const SelectState* __restrict__ st,
                                                                        unsigned long long* __restrict__ count, double* __restrict__ part) {
    __shared__ unsigned long long su[32];
    __shared__ double sd[32];
    const uint32_t tau = max(st->prefix, 1u);
    unsigned long long pop = 0;
    double e2 = 0.0;
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n4; q += (long long)gridDim.x * blockDim.x) {
        float4 o;
        if (q < n4v) {
            const float4 r = ld_f4(e + 4 * q);
            o = ld_f4(w + 4 * q);
            const bool mx = magnitude_key(r.x) >= tau, my = magnitude_key(r.y) >= tau, mz = magnitude_key(r.z) >= tau,
                       mw = magnitude_key(r.w) >= tau;
            if (mx | my | mz | mw) {
                o = make_float4(mx ? __fadd_rn(o.x, r.x) : o.x, my ? __fadd_rn(o.y, r.y) : o.y, mz ? __fadd_rn(o.z, r.z) : o.z,
                                mw ? __fadd_rn(o.w, r.w) : o.w);
                st_f4(w + 4 * q, o);
                st_f4(e + 4 * q, make_float4(take(!mx, r.x), take(!my, r.y), take(!mz, r.z), take(!mw, r.w)));
                pop += (unsigned)mx + (unsigned)my + (unsigned)mz + (unsigned)mw;
            }
            const double x = mx ? 0.0 : (double)r.x, y = my ? 0.0 : (double)r.y, z = mz ? 0.0 : (double)r.z, v = mw ? 0.0 : (double)r.w;
            e2 += x * x;
            e2 += y * y;
            e2 += z * z;
            e2 += v * v;
        } else {
            o = ld_f4(wn + 4 * q);
            st_f4(w + 4 * q, o);
        }
        if (wb) *reinterpret_cast<uint2*>(wb + 4 * q) = make_uint2(pack_bf16x2(o.x, o.y), pack_bf16x2(o.z, o.w));
    }
    const unsigned long long tot = block_sum<unsigned long long>(pop, su);
    const double sq = block_sum<double>(e2, sd);
    if (threadIdx.x == 0) {
        if (tot) atomicAdd(count, tot);
        part[blockIdx.x] = sq;
    }
}

// stats = {|M|, float(tau), ||e''||_2}: the per-CTA partials added in CTA order
__global__ void __launch_bounds__(32) sparsefed_finish_kernel(const unsigned long long* __restrict__ count, const double* __restrict__ part,
                                                              int nparts, const SelectState* __restrict__ st, double* __restrict__ stats) {
    if (threadIdx.x != 0) return;
    double s = 0.0;
    for (int i = 0; i < nparts; ++i) s += part[i];
    stats[0] = (double)*count;
    stats[1] = (double)__uint_as_float(st->prefix);
    stats[2] = sqrt(s);
}

}  // namespace

cudaError_t launch_sparsefed(const float* w_new, float* w, void* w_bf16, float* e, long long n_vote, long long n, long long k,
                             double* stats, int num_sms, cudaStream_t st) {
    if ((n_vote & 3) || (n & 3) || n_vote > n || k < 1 || k > n_vote || n_vote >= (1LL << 32)) return cudaErrorInvalidValue;
    const long long n4v = n_vote / 4, n4 = n / 4;
    const int grid = sweep_grid(n4, kApplyThreads, num_sms, 8);
    // the select's histograms and state, then |M| and the apply pass's per-CTA partials
    const size_t bytes = kSelectScratchBytes + 8 /*align*/ + sizeof(unsigned long long) + (size_t)grid * sizeof(double);
    Scratch scr(bytes, st);
    uint32_t* hist = scr.as<uint32_t>();
    SelectState* sel = reinterpret_cast<SelectState*>(hist + 3 * kBins);
    auto* count = reinterpret_cast<unsigned long long*>(scr.as<char>() + (kSelectScratchBytes + 7) / 8 * 8);
    double* part = reinterpret_cast<double*>(count + 1);
    RLR_CUDA_CHECK(cudaMemsetAsync(scr.p, 0, bytes, st));
    const int hgrid = sweep_grid(n4v, kHistThreads, num_sms, 4);
    topk_hist_kernel<AccumulateKeys><<<hgrid, kHistThreads, 0, st>>>(AccumulateKeys{w_new, w, e}, n4v, 0, sel, hist);
    RLR_CUDA_CHECK(cudaGetLastError());
    RLR_CUDA_CHECK(topk_select(ErrorKeys{e}, n4v, k, hist, sel, hgrid, 1, st));
    sparsefed_apply_kernel<<<grid, kApplyThreads, 0, st>>>(w_new, w, static_cast<__nv_bfloat16*>(w_bf16), e, n4v, n4, sel, count, part);
    RLR_CUDA_CHECK(cudaGetLastError());
    sparsefed_finish_kernel<<<1, 32, 0, st>>>(count, part, grid, sel, stats);
    return cudaGetLastError();
}

}  // namespace rlr
