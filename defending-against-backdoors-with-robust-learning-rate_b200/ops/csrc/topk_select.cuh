// Device-side top-k radix select over 31-bit magnitude keys, shared by Neurotoxin's mask (attack.cu) and SparseFed's server step
// (sparsefed.cu).  A key is the fp32 pattern of a value with the sign bit cleared: unsigned keys that order like the magnitudes, NaN
// above +inf.  tau, the k-th largest key counted with multiplicity, is found in three histogram passes over 11 + 11 + 9 key bits, each
// restricted to the prefix the passes before it fixed.  After each histogram one small CTA finds the bin where the count from the top
// reaches the rank still wanted (topk_find_kernel), so tau never leaves the GPU and the select queues without a host sync.  Histogram
// counts are integer atomics: exact and independent of their order.  After the last find, SelectState::prefix holds tau.
//
// The histogram pass is templated on how it loads four keys: a loader is a struct with
//     __device__ uint4 keys(long long q) const      // the keys of coordinates 4q .. 4q + 3
// which may also write (SparseFed's accumulate pass produces the error vector and histograms it in one sweep).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"

namespace rlr {

namespace {

constexpr int kBins = 2048;          // 11-bit digits; the last pass uses 512 of them (9 bits)
constexpr int kHistThreads = 512;

// pass p: digit bits and the shift of the prefix fixed by the earlier passes
__device__ __forceinline__ int digit_shift(int pass) { return pass == 0 ? 20 : (pass == 1 ? 9 : 0); }
__device__ __forceinline__ uint32_t digit_mask(int pass) { return pass == 2 ? 0x1FFu : 0x7FFu; }
__device__ __forceinline__ int prefix_shift(int pass) { return pass == 1 ? 20 : 9; }

__device__ __forceinline__ uint32_t magnitude_key(float x) { return __float_as_uint(x) & 0x7FFFFFFFu; }

struct SelectState {
    uint32_t prefix;                 // key bits fixed so far (right-aligned)
    uint32_t krem;                   // rank still to find inside the selected prefix, 1-based from the top
};

template <class Keys>
__global__ void __launch_bounds__(kHistThreads) topk_hist_kernel(Keys ld, long long n4, int pass, const SelectState* __restrict__ st,
                                                                  uint32_t* __restrict__ hist /*[kBins]*/) {
    __shared__ uint32_t h[kBins];
    for (int i = threadIdx.x; i < kBins; i += blockDim.x) h[i] = 0;
    __syncthreads();
    const int sh = digit_shift(pass);
    const uint32_t dm = digit_mask(pass);
    const int psh = prefix_shift(pass);
    const uint32_t want = pass == 0 ? 0u : st->prefix;
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n4; q += (long long)gridDim.x * blockDim.x) {
        const uint4 k4 = ld.keys(q);
        const uint32_t a[4] = {k4.x, k4.y, k4.z, k4.w};
#pragma unroll
        for (int j = 0; j < 4; ++j)
            if (pass == 0 || (a[j] >> psh) == want) atomicAdd(&h[(a[j] >> sh) & dm], 1u);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < kBins; i += blockDim.x)
        if (h[i]) atomicAdd(&hist[i], h[i]);
}

// One CTA of kBins/2 threads: the bin where the count from the top reaches krem.  Thread t holds the bins 2047-2t and 2046-2t; an
// inclusive scan of the pair sums gives every thread the count above its pair, so exactly one thread sees the crossing.
__global__ void __launch_bounds__(kBins / 2) topk_find_kernel(const uint32_t* __restrict__ hist, int pass, SelectState* st,
                                                              long long k) {
    __shared__ uint32_t warp_tot[kBins / 2 / 32];
    const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
    const uint32_t krem = pass == 0 ? (uint32_t)k : st->krem;
    const uint32_t prefix = pass == 0 ? 0u : st->prefix;
    const uint32_t hi = hist[kBins - 1 - 2 * t], lo = hist[kBins - 2 - 2 * t];
    uint32_t s = hi + lo;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t v = __shfl_up_sync(0xFFFFFFFFu, s, o);
        if (lane >= o) s += v;
    }
    if (lane == 31) warp_tot[wid] = s;
    __syncthreads();
    uint32_t base = 0;
    for (int w = 0; w < wid; ++w) base += warp_tot[w];
    const uint32_t incl = base + s, above = incl - (hi + lo);
    __syncthreads();                 // every thread has read krem / prefix before the winner rewrites them
    const int bits = pass == 2 ? 9 : 11;
    if (above < krem && above + hi >= krem) {
        st->prefix = (prefix << bits) | (uint32_t)(kBins - 1 - 2 * t);
        st->krem = krem - above;
    } else if (above + hi < krem && incl >= krem) {
        st->prefix = (prefix << bits) | (uint32_t)(kBins - 2 - 2 * t);
        st->krem = krem - above - hi;
    }
}

// Bytes of the select's device scratch: three histograms and the select state, zeroed together before the first pass.
constexpr size_t kSelectScratchBytes = 3 * kBins * sizeof(uint32_t) + sizeof(SelectState);

// The three histogram + find pairs over the keys `ld` loads (n4 groups of four), into `hist` (three zeroed histograms) and `sel`.
// `first_pass`: 1 when the caller has already run pass 0's histogram (fused into a pass of its own) into hist[0 .. kBins).
template <class Keys>
inline cudaError_t topk_select(const Keys& ld, long long n4, long long k, uint32_t* hist, SelectState* sel, int grid, int first_pass,
                               cudaStream_t st) {
    for (int pass = 0; pass < 3; ++pass) {
        if (pass >= first_pass) {
            topk_hist_kernel<Keys><<<grid, kHistThreads, 0, st>>>(ld, n4, pass, sel, hist + pass * kBins);
            RLR_CUDA_CHECK(cudaGetLastError());
        }
        topk_find_kernel<<<1, kBins / 2, 0, st>>>(hist + pass * kBins, pass, sel, k);
        RLR_CUDA_CHECK(cudaGetLastError());
    }
    return cudaSuccess;
}

inline int sweep_grid(long long n4, int threads, int num_sms, int per_sm) {
    const long long want = (n4 + threads - 1) / threads, cap = (long long)num_sms * per_sm;
    return (int)(want < 1 ? 1 : (want > cap ? cap : want));
}

}  // namespace

}  // namespace rlr
