// Model-poisoning attackers (DESIGN.md section 3): Neurotoxin's top-k mask of the last global update and the boosted update.
//
// Neurotoxin (Zhang et al. 2022): a[c] = bits(|fp32(w_g[c] - w_prev[c])|) for c < n_vote (the fp32 pattern with the sign bit cleared:
// 31-bit unsigned keys that order like the magnitudes, NaN above +inf).  tau is the k-th largest key, counted with multiplicity, found
// by a radix select over the 31 key bits in three histogram passes (11 + 11 + 9 bits), each restricted to the prefix the previous one
// fixed.  The bin that crosses k is found on the device by one small CTA between the passes, so tau never leaves the GPU and the whole
// pass queues on the round's stream without a host sync.  Histogram counts are integer atomics (exact, order-free).  The last pass
// writes M = {c : a[c] >= tau, a[c] > 0} as ceil(n_vote/32) bit words, its popcount, and w_prev <- w_g.
//
// Every pass recomputes a[c] from w_g and w_prev (8 B per coordinate) instead of staging the keys in a 4 B scratch copy: 36 B per
// coordinate in all (3 x 8 read, 8 read + 4 written by the mask pass) against 32 B with a 45 MB scratch at the ResNet-18 size.
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"
#include "kernels.h"
#include "topk_select.cuh"

namespace rlr {

namespace {

__device__ __forceinline__ uint32_t key_of(float g, float p) { return magnitude_key(g - p); }

// Neurotoxin's keys: a[c] = bits(|fp32(w_g[c] - w_prev[c])|)
struct DiffKeys {
    const float* __restrict__ wg;
    const float* __restrict__ wp;
    __device__ __forceinline__ uint4 keys(long long q) const {
        const float4 g = ld_f4(wg + 4 * q), p = ld_f4(wp + 4 * q);
        return make_uint4(key_of(g.x, p.x), key_of(g.y, p.y), key_of(g.z, p.z), key_of(g.w, p.w));
    }
};

// M = {c < n_vote : a[c] >= max(tau, 1)} as bit words (bit c % 32 of word c / 32), |M| into *count, and w_prev <- w_g.  Each thread
// takes one float4 (4 mask bits); the 8 lanes that share a word OR their nibbles together.
__global__ void __launch_bounds__(256) neurotoxin_mask_kernel(const float* __restrict__ wg, float* __restrict__ wp, long long n4,
                                                              const SelectState* __restrict__ st, uint32_t* __restrict__ mask,
                                                              unsigned long long* __restrict__ count) {
    __shared__ unsigned long long scratch[32];
    const uint32_t tau = max(st->prefix, 1u);
    unsigned long long pop = 0;
    // the loop bound keeps whole warps together, so the shuffles below always see all 32 lanes
    const long long step = (long long)gridDim.x * blockDim.x;
    const long long n4w = (n4 + 31) / 32 * 32;
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n4w; q += step) {
        uint32_t nib = 0;
        if (q < n4) {
            const float4 g = ld_f4(wg + 4 * q), p = ld_f4(wp + 4 * q);
            nib = (key_of(g.x, p.x) >= tau ? 1u : 0u) | (key_of(g.y, p.y) >= tau ? 2u : 0u) | (key_of(g.z, p.z) >= tau ? 4u : 0u) |
                  (key_of(g.w, p.w) >= tau ? 8u : 0u);
            st_f4(wp + 4 * q, g);
        }
        uint32_t word = nib << ((q & 7) * 4);
        word |= __shfl_xor_sync(0xFFFFFFFFu, word, 1);
        word |= __shfl_xor_sync(0xFFFFFFFFu, word, 2);
        word |= __shfl_xor_sync(0xFFFFFFFFu, word, 4);
        if ((q & 7) == 0 && q < n4) mask[q >> 3] = word;
        pop += __popc(nib);
    }
    const unsigned long long tot = block_sum<unsigned long long>(pop, scratch);
    if (threadIdx.x == 0 && tot) atomicAdd(count, tot);
}

// slot[c] = fp32(w_g[c] + gamma * fp32(slot[c] - w_g[c])) in fp64, rounded once per operation (no contraction into an FMA), so the
// numpy statement matches bit for bit
__global__ void __launch_bounds__(256) boost_update_kernel(float* __restrict__ slot, const float* __restrict__ wg, long long n4,
                                                           double gamma) {
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n4; q += (long long)gridDim.x * blockDim.x) {
        const float4 s = ld_f4(slot + 4 * q), g = ld_f4(wg + 4 * q);
        float4 o;
        o.x = __double2float_rn(__dadd_rn((double)g.x, __dmul_rn(gamma, (double)(s.x - g.x))));
        o.y = __double2float_rn(__dadd_rn((double)g.y, __dmul_rn(gamma, (double)(s.y - g.y))));
        o.z = __double2float_rn(__dadd_rn((double)g.z, __dmul_rn(gamma, (double)(s.z - g.z))));
        o.w = __double2float_rn(__dadd_rn((double)g.w, __dmul_rn(gamma, (double)(s.w - g.w))));
        st_f4(slot + 4 * q, o);
    }
}

// Attack schedules: data[idx[i]] <-> side[i] (row_bytes each) and targets[idx[i]] <-> side_targets[i] for i < n.  One warp per row in
// a grid-stride loop over the rows, the lanes striding over the row's W-sized words; lane 0 swaps the label.  The idx are distinct, so
// no two threads touch the same byte: no atomics, and the swap is its own inverse.
template <typename W>
__global__ void __launch_bounds__(256) swap_samples_kernel(unsigned char* __restrict__ data, long long* __restrict__ targets,
                                                           const long long* __restrict__ idx, unsigned char* __restrict__ side,
                                                           long long* __restrict__ side_targets, long long n, int row_words) {
    pdl_wait();
    pdl_trigger();
    const int lane = threadIdx.x & 31;
    const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long i = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); i < n; i += warps) {
        const long long j = idx[i];
        W* a = reinterpret_cast<W*>(data) + j * row_words;
        W* b = reinterpret_cast<W*>(side) + i * row_words;
#pragma unroll 2                     // the default 4-way unroll of the 16-byte words spills
        for (int w = lane; w < row_words; w += 32) {
            const W x = a[w], y = b[w];
            a[w] = y;
            b[w] = x;
        }
        if (lane == 0) {
            const long long x = targets[j];
            targets[j] = side_targets[i];
            side_targets[i] = x;
        }
    }
}

}  // namespace

cudaError_t launch_swap_samples(void* data, long long* targets, const long long* idx, void* side, long long* side_targets, long long n,
                                long long row_bytes, int num_sms, cudaStream_t st) {
    if (n < 0 || row_bytes <= 0) return cudaErrorInvalidValue;
    if (n == 0) return cudaSuccess;
    const dim3 grid(sweep_grid(n * 32, 256, num_sms, 8)), block(256);
    auto* d = static_cast<unsigned char*>(data);
    auto* s = static_cast<unsigned char*>(side);
    // the widest word that divides the row and both base addresses
    const uintptr_t align = reinterpret_cast<uintptr_t>(data) | reinterpret_cast<uintptr_t>(side) | (uintptr_t)row_bytes;
    if (align % 16 == 0)
        return launch_kernel(swap_samples_kernel<uint4>, grid, block, (size_t)0, st, d, targets, idx, s, side_targets, n,
                             (int)(row_bytes / 16));
    if (align % 4 == 0)
        return launch_kernel(swap_samples_kernel<uint32_t>, grid, block, (size_t)0, st, d, targets, idx, s, side_targets, n,
                             (int)(row_bytes / 4));
    return launch_kernel(swap_samples_kernel<unsigned char>, grid, block, (size_t)0, st, d, targets, idx, s, side_targets, n,
                         (int)row_bytes);
}

cudaError_t launch_neurotoxin_mask(const float* w_g, float* w_prev, long long n_vote, long long k, uint32_t* mask, long long* count,
                                   int num_sms, cudaStream_t st) {
    if ((n_vote & 3) || k < 0 || k > n_vote || n_vote >= (1LL << 32)) return cudaErrorInvalidValue;
    const long long n4 = n_vote / 4, words = (n_vote + 31) / 32;
    RLR_CUDA_CHECK(cudaMemsetAsync(count, 0, sizeof(long long), st));
    if (n_vote == 0) return cudaSuccess;
    if (k == 0) {                    // empty mask: clear it and refresh w_prev
        RLR_CUDA_CHECK(cudaMemsetAsync(mask, 0, (size_t)words * sizeof(uint32_t), st));
        return cudaMemcpyAsync(w_prev, w_g, (size_t)n_vote * sizeof(float), cudaMemcpyDeviceToDevice, st);
    }
    Scratch scr(kSelectScratchBytes, st);
    uint32_t* hist = scr.as<uint32_t>();
    SelectState* sel = reinterpret_cast<SelectState*>(hist + 3 * kBins);
    RLR_CUDA_CHECK(cudaMemsetAsync(hist, 0, kSelectScratchBytes, st));
    RLR_CUDA_CHECK(topk_select(DiffKeys{w_g, w_prev}, n4, k, hist, sel, sweep_grid(n4, kHistThreads, num_sms, 4), 0, st));
    neurotoxin_mask_kernel<<<sweep_grid(n4, 256, num_sms, 8), 256, 0, st>>>(w_g, w_prev, n4, sel, mask,
                                                                              reinterpret_cast<unsigned long long*>(count));
    return cudaGetLastError();
}

cudaError_t launch_boost_update(float* slot, const float* w_g, long long n_vote, double gamma, int num_sms, cudaStream_t st) {
    if (n_vote & 3) return cudaErrorInvalidValue;
    if (n_vote == 0) return cudaSuccess;
    boost_update_kernel<<<sweep_grid(n_vote / 4, 256, num_sms, 8), 256, 0, st>>>(slot, w_g, n_vote / 4, gamma);
    return cudaGetLastError();
}

}  // namespace rlr
