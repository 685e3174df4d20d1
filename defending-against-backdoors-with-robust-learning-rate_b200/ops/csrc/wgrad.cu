// wgmma weight-gradient kernels for sm_90a:   dW[co][tap][ci] = sum_pix dY[pix][co] * X[pix (+) tap][ci]
//
// The reduction runs over PIXELS, which is the slow dimension of both NHWC operands, so both MMA operands are
// MN-major: a k-block is 64 pixels, the A tile is dY[64 pix][128 co] (two 64-channel TMA boxes, one per consumer warpgroup) and
// the B tile of tap t is X[64 shifted pix][64 ci] (one 4-D TMA box, zero-filled at the borders = padding).  One CTA keeps the
// accumulators of up to THREE taps (one filter row: one m64n192 wgmma per warpgroup and k-step) in registers so each dY tile is
// loaded once per filter row, runs a contiguous slice of the pixel range (split-K over CTAs) and reduces its 128 x 64 x taps
// partial result into a slot of a scratch buffer; the slots are then added into the fp32 flat gradient in split order, so the
// result does not depend on CTA scheduling (one split: the CTA adds its tile straight into the gradient).
// Plain mode (mode 0) is the same kernel on 2-D operands: dW[n][k] = sum_b dY[b][n] X[b][k] for linear layers.
// Replaces cuDNN wgrad / cuBLAS GEMM^T behind loss.backward() (reference src/agent.py:48).
#include <cuda.h>
#include <stdlib.h>

#include "common.cuh"
#include "gemm.h"
#include "wgmma.cuh"

namespace rlr {

using namespace wg;

cudaError_t make_tmap_bf16(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                           const uint32_t* box, const uint32_t* elem_strides = nullptr);  // gemm.cu

constexpr int WG_BM = 128, WG_BK = 64;                        // co tile, pixels per k-block
constexpr int WG_STAGES = 3;
constexpr int WG_A_BYTES = 2 * 64 * WG_BK * 2;                // two 64-channel groups x 64 pixel rows x 128 B
constexpr int WG_THREADS = 256 + 32;                          // two consumer warpgroups + the TMA producer warp
template <int BNW>                                            // ci tile width: 64 or 128 channels
struct WgCfg {
    static constexpr int kGroups = BNW / 64;
    static constexpr int kBBytes = kGroups * 64 * WG_BK * 2;  // per tap
    static constexpr int kStageBytes = WG_A_BYTES + 3 * kBBytes;   // 40 KB / 64 KB
    static constexpr int kSmem = WG_STAGES * kStageBytes + 2048;
};

struct WgradParams {
    int mode;                 // 0 plain 2-D, 1 conv
    int num_kb;               // total 64-pixel k-blocks
    int kb_per_cta;
    int a_groups;             // 1 (Cout tile of 64 valid channels) or 2
    int ntaps_cta;            // taps handled by one CTA (1 or 3)
    int T;                    // total taps of the filter
    int TW, TH, TN, tiles_w, tiles_h;
    int8_t dh[9], dw[9];
    int dn[9];
    int in_stride;            // 2: x is read through a strided TMA box (every other pixel), no parity-split copy
    int ci_tiles;
    int Cout, Cin_valid;      // rows / columns of dW that exist (Cin_valid < 64 for the channel-padded stem)
    float* dW;                // [Cout][T][Cin_valid] fp32 (accumulated)
    float* part;              // split-K > 1: [splits][Cout][T][Cin_valid] partial gradients (one slot per blockIdx.z)
};

struct __align__(8) WgShared {
    uint64_t full[WG_STAGES];
    uint64_t empty[WG_STAGES];
};

// Host-side count of the weight-gradient launches of each kernel: [0] umma_wgrad_kernel, [1] umma_wgrad_halo_kernel,
// [2] umma_wgrad_rows_kernel.  Tests read it (wgrad_launch_counts) to check which kernel a shape is dispatched to.
static long long g_wgrad_launches[3] = {0, 0, 0};
void wgrad_launch_counts(long long* out) { for (int i = 0; i < 3; ++i) out[i] = g_wgrad_launches[i]; }

// acc column c of warpgroup row `co` (fragment layout) -> dW[co][tap0 + c / BNW][ci0 + c % BNW], pairs of adjacent columns per thread;
// with `part` the values are stored into this split's slot of the partial buffer instead of being added into dW
template <int NACC, int BNW>
__device__ __forceinline__ void wgrad_flush(const float (&acc)[NACC / 2], float* dW, float* part, int co, int Cout, int T, int tap0, int ci0,
                                            int Cin_valid, int t) {
    if (part) dW = part + (size_t)blockIdx.z * Cout * T * Cin_valid;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int row = co + 8 * h;
        if (row >= Cout) continue;
#pragma unroll
        for (int j = 0; j < NACC / 8; ++j) {
            const int c = frag_col(t, 4 * j), tap = c / BNW, ci = ci0 + c % BNW;
            float* dst = dW + ((size_t)row * T + tap0 + tap) * Cin_valid + ci;
            const float a = acc[4 * j + 2 * h], b = acc[4 * j + 2 * h + 1];
            if (part) {
                if (ci < Cin_valid) dst[0] = a;
                if (ci + 1 < Cin_valid) dst[1] = b;
            } else if ((Cin_valid & 1) == 0) {
                if (ci < Cin_valid) asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(dst), "f"(a), "f"(b) : "memory");
            } else {
                if (ci < Cin_valid) atomicAdd(dst, a);
                if (ci + 1 < Cin_valid) atomicAdd(dst + 1, b);
            }
        }
    }
}

template <int BNW, int kTaps>
__global__ void __launch_bounds__(WG_THREADS, 1)
umma_wgrad_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const WgradParams p) {
    using Cfg = WgCfg<BNW>;
    constexpr int WG_BN = BNW, WG_B_BYTES = Cfg::kBBytes, WG_STAGE_BYTES = Cfg::kStageBytes;
    constexpr int NACC = kTaps * BNW;                         // 64, 128 or 192 accumulator columns
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    WgShared* sh = reinterpret_cast<WgShared*>(smem + WG_STAGES * WG_STAGE_BYTES);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int co_tile = blockIdx.x / p.ci_tiles, ci_tile = blockIdx.x - co_tile * p.ci_tiles;
    const int tap0 = blockIdx.y * kTaps;
    const int kb_begin = blockIdx.z * p.kb_per_cta;
    const int kb_end = min(p.num_kb, kb_begin + p.kb_per_cta);
    const int nkb = kb_end - kb_begin;

    if (warp == 8 && lane == 0) {
        prefetch_tmap(&tmA); prefetch_tmap(&tmB);
        for (int s = 0; s < WG_STAGES; ++s) { mbar_init(&sh->full[s], 1); mbar_init(&sh->empty[s], 4 * p.a_groups); }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();        // prologue above: parameters and shared memory only
    pdl_trigger();

    if (warp == 8) {
        if (lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            const uint32_t bytes = p.a_groups * 8192 + kTaps * WG_B_BYTES;
            for (int i = 0; i < nkb; ++i) {
                const int kb = kb_begin + i;
                mbar_wait(&sh->empty[stage], phase ^ 1);
                uint8_t* sa = smem + stage * WG_STAGE_BYTES;
                uint8_t* sb = sa + WG_A_BYTES;
                mbar_expect_tx(&sh->full[stage], bytes);
                if (p.mode == 1) {
                    const int tw_i = kb % p.tiles_w, th_i = (kb / p.tiles_w) % p.tiles_h, tn_i = kb / (p.tiles_w * p.tiles_h);
                    const int w0 = tw_i * p.TW, h0 = th_i * p.TH, n0 = tn_i * p.TN;
                    for (int g = 0; g < p.a_groups; ++g)
                        tma_load_4d(&tmA, &sh->full[stage], sa + g * 8192, co_tile * WG_BM + g * 64, w0, h0, n0);
                    for (int t = 0; t < kTaps; ++t)
                        for (int g = 0; g < Cfg::kGroups; ++g)
                            tma_load_4d(&tmB, &sh->full[stage], sb + t * WG_B_BYTES + g * 8192, ci_tile * WG_BN + g * 64,
                                        w0 * p.in_stride + p.dw[tap0 + t], h0 * p.in_stride + p.dh[tap0 + t], n0 + p.dn[tap0 + t]);
                } else {
                    for (int g = 0; g < p.a_groups; ++g)
                        tma_load_2d(&tmA, &sh->full[stage], sa + g * 8192, co_tile * WG_BM + g * 64, kb * WG_BK);
                    for (int g = 0; g < Cfg::kGroups; ++g)
                        tma_load_2d(&tmB, &sh->full[stage], sb + g * 8192, ci_tile * WG_BN + g * 64, kb * WG_BK);
                }
                if (++stage == WG_STAGES) { stage = 0; phase ^= 1; }
            }
        }
    } else if (nkb > 0 && (threadIdx.x >> 7) < p.a_groups) {
        // warpgroup wgi: output channels co_tile * 128 + 64 wgi + [0, 64) = A group wgi.  When that group does not exist (a_groups == 1)
        // the warpgroup has no work and leaves at once: the stage-release barriers count only the warps of the active warpgroups, and
        // no MMA sits under a per-warpgroup branch (which makes ptxas serialize every wgmma of the kernel)
        const int wgi = threadIdx.x >> 7, t = threadIdx.x & 127;
        float acc[NACC / 2];
#pragma unroll
        for (int i = 0; i < NACC / 2; ++i) acc[i] = 0.f;
        int stage = 0, prev = -1;
        uint32_t phase = 0;
        for (int i = 0; i < nkb; ++i) {
            mbar_wait(&sh->full[stage], phase);
            const uint32_t sa = smem_u32(smem + stage * WG_STAGE_BYTES) + wgi * 8192;
            const uint32_t sb = smem_u32(smem + stage * WG_STAGE_BYTES) + WG_A_BYTES;
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < WG_BK / 16; ++k) {   // 16 pixel rows (2 swizzle atoms) per MMA
                // B: the tap tiles (and 64-wide ci groups inside them) are N groups 8 KB apart -> one MMA covers all kTaps taps
                wgmma_bf16<NACC, 1, 1>(acc, smem_desc_sw128(sa + k * 2048, 8192, 1024), smem_desc_sw128(sb + k * 2048, 8192, 1024),
                                       (i > 0 || k > 0) ? 1u : 0u);
            }
            wgmma_commit();
            wgmma_wait<1>();
            if (prev >= 0 && lane == 0) mbar_arrive(&sh->empty[prev]);
            prev = stage;
            if (++stage == WG_STAGES) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        fence_acc(acc);
        wgrad_flush<NACC, BNW>(acc, p.dW, p.part, co_tile * WG_BM + wgi * 64 + frag_row(t, 0), p.Cout, p.T, tap0, ci_tile * WG_BN, p.Cin_valid, t);
    }
}

// split-K so that the grid of `base` CTAs per split is (at most) a whole number of waves of one CTA per SM: no ragged tail wave.
// Below one wave, `low_waves` (0 = 1) waves.  Returns the split count and the k-blocks per split; the split count fixes the
// order of every dW element's sum, so the filter-row kernel computes it from the CTA count of the kernel it replaces.
static int wg_splits(int base, int num_kb, int num_sms, int low_waves, int* kb_per_cta) {
    const int waves = base >= num_sms ? (base + num_sms - 1) / num_sms : (low_waves > 0 ? low_waves : 1);
    int splits = (waves * num_sms) / base;
    if (splits > num_kb) splits = num_kb;
    if (splits < 1) splits = 1;
    *kb_per_cta = (num_kb + splits - 1) / splits;
    return (num_kb + *kb_per_cta - 1) / *kb_per_cta;
}
// one wave measured faster (fewer split-K atomics), RLR_WG_WAVES overrides
static int wg_tune_waves() {
    static const int w = [] { const char* e = getenv("RLR_WG_WAVES"); return e ? atoi(e) : 0; }();
    return w;
}

template <int BNW, int kTaps>
static cudaError_t launch_wg(const CUtensorMap& tmA, const CUtensorMap& tmB, WgradParams& p, int co_tiles, int tap_groups,
                             int num_sms, cudaStream_t st) {
    static bool configured = false;
    if (!configured) {
        RLR_CUDA_CHECK(cudaFuncSetAttribute(umma_wgrad_kernel<BNW, kTaps>, cudaFuncAttributeMaxDynamicSharedMemorySize, WgCfg<BNW>::kSmem));
        configured = true;
    }
    const int splits = wg_splits(co_tiles * p.ci_tiles * tap_groups, p.num_kb, num_sms, wg_tune_waves(), &p.kb_per_cta);
    const dim3 grid(co_tiles * p.ci_tiles, tap_groups, splits);
    ++g_wgrad_launches[0];
    if (splits == 1) return launch_kernel(umma_wgrad_kernel<BNW, kTaps>, grid, dim3(WG_THREADS), (size_t)WgCfg<BNW>::kSmem, st, tmA, tmB, p);
    const long long plane = (long long)p.Cout * p.T * p.Cin_valid;
    Scratch part((size_t)splits * plane * sizeof(float), st);
    p.part = part.as<float>();
    RLR_CUDA_CHECK(launch_kernel(umma_wgrad_kernel<BNW, kTaps>, grid, dim3(WG_THREADS), (size_t)WgCfg<BNW>::kSmem, st, tmA, tmB, p));
    return launch_ordered_sum(p.dW, p.part, splits, plane, st);
}

// ---------------------------------------------------------------------------------------------------------------------
// Halo-reuse variant for 3x3 / stride-1 / pad-1 filters over 64 input channels (stem, layer1, first VGG block).
// A k-block is one 16x8 output tile (128 pixels); its dY tile (128 px x 64/128 co) and ONE 18x16-pixel halo of X (36 KB)
// are loaded once and serve every filter tap: the B operand of tap (dy,dx) and MMA k-step j (16 pixels = image rows 2j,2j+1)
// is the MN-major view starting at halo + ((2j+dy)*16 + dx)*128 B with an 8-row group stride (SBO) of 2048 B -- the tensor
// core applies the 128-byte swizzle on absolute smem address bits, so unaligned starts need no special handling
// (see conv_halo.cu).  The three dx taps of a filter row are the SAME view shifted by one pixel (128 B), i.e. three
// 64-channel "N groups" with a leading-dimension byte offset of 128: one N = 192 MMA per k-step computes all three, which
// moves the instruction out of the smem-bandwidth-bound N = 64 regime.  grid.y = 3 filter rows (3 x 192 columns do not fit
// registers).  L2 traffic per 128 pixels: 3 x (36 + 16..32) KB instead of 3 x 2 x (24 + 8..16) KB.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int WH_STAGES = 3;
constexpr int WH_A_BYTES = 2 * 128 * 128;                      // up to two 64-channel groups x 128 pixel rows x 128 B
constexpr int WH_HALO_BYTES = 18 * 16 * 128;                   // 36864
constexpr int WH_STAGE_BYTES = WH_A_BYTES + WH_HALO_BYTES;     // 69632
constexpr int WH_SMEM = WH_STAGES * WH_STAGE_BYTES + 2048;

struct WgHaloParams {
    int NB, H, W, tiles_h, tiles_w;
    int num_kb, kb_per_cta;
    int a_groups;
    int Cout, Cin_valid;
    float* dW;                // [Cout][9][Cin_valid]
    float* part;              // split-K > 1: [splits][Cout][9][Cin_valid] partial gradients
};

__global__ void __launch_bounds__(WG_THREADS, 1)
umma_wgrad_halo_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const WgHaloParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    WgShared* sh = reinterpret_cast<WgShared*>(smem + WH_STAGES * WH_STAGE_BYTES);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int co_tile = blockIdx.x;
    const int dy = blockIdx.y, tap0 = dy * 3;
    const int kb_begin = blockIdx.z * p.kb_per_cta;
    const int kb_end = min(p.num_kb, kb_begin + p.kb_per_cta);
    const int nkb = kb_end - kb_begin;
    const int tiles_per_img = p.tiles_h * p.tiles_w;

    if (warp == 8 && lane == 0) {
        prefetch_tmap(&tmA); prefetch_tmap(&tmB);
        for (int s = 0; s < WH_STAGES; ++s) { mbar_init(&sh->full[s], 1); mbar_init(&sh->empty[s], 4 * p.a_groups); }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();        // prologue above: parameters and shared memory only
    pdl_trigger();

    if (warp == 8) {
        if (lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            const uint32_t bytes = p.a_groups * 16384 + WH_HALO_BYTES;
            for (int i = 0; i < nkb; ++i) {
                const int kb = kb_begin + i;
                const int n = kb / tiles_per_img, r = kb - n * tiles_per_img;
                const int h0 = (r / p.tiles_w) * 16, w0 = (r % p.tiles_w) * 8;
                mbar_wait(&sh->empty[stage], phase ^ 1);
                uint8_t* sa = smem + stage * WH_STAGE_BYTES;
                mbar_expect_tx(&sh->full[stage], bytes);
                for (int g = 0; g < p.a_groups; ++g)
                    tma_load_4d(&tmA, &sh->full[stage], sa + g * 16384, co_tile * WG_BM + g * 64, w0, h0, n);
                tma_load_4d(&tmB, &sh->full[stage], sa + WH_A_BYTES, 0, w0 - 1, h0 - 1, n);
                if (++stage == WH_STAGES) { stage = 0; phase ^= 1; }
            }
        }
    } else if (nkb > 0 && (threadIdx.x >> 7) < p.a_groups) {   // as in umma_wgrad_kernel: a warpgroup without an A group leaves
        const int wgi = threadIdx.x >> 7, t = threadIdx.x & 127;
        float acc[96];
#pragma unroll
        for (int i = 0; i < 96; ++i) acc[i] = 0.f;
        int stage = 0, prev = -1;
        uint32_t phase = 0;
        for (int i = 0; i < nkb; ++i) {
            mbar_wait(&sh->full[stage], phase);
            const uint32_t sa = smem_u32(smem + stage * WH_STAGE_BYTES) + wgi * 16384;
            const uint32_t halo = smem_u32(smem + stage * WH_STAGE_BYTES) + WH_A_BYTES;
            wgmma_fence();
#pragma unroll
            for (int j = 0; j < 8; ++j) {                     // 16 pixels = output rows 2j, 2j+1 of the tile
                // N groups 0,1,2 = taps dx = 0,1,2: same halo view shifted by one pixel -> LBO = 128 B; SBO = one image row
                wgmma_bf16<192, 1, 1>(acc, smem_desc_sw128(sa + j * 2048, 16384, 1024),
                                      smem_desc_sw128(halo + ((2 * j + dy) * 16) * 128, 128, 2048), (i > 0 || j > 0) ? 1u : 0u);
            }
            wgmma_commit();
            wgmma_wait<1>();
            if (prev >= 0 && lane == 0) mbar_arrive(&sh->empty[prev]);
            prev = stage;
            if (++stage == WH_STAGES) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        fence_acc(acc);
        wgrad_flush<192, 64>(acc, p.dW, p.part, co_tile * WG_BM + wgi * 64 + frag_row(t, 0), p.Cout, 9, tap0, 0, p.Cin_valid, t);
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// Filter-row variant for 3x3 / stride-1 / pad-1 filters: ONE CTA computes all nine taps of a 64-co x 64-ci filter tile for one
// split-K range.  A k-block loads one dY box (64 co) and one input halo, shared by three consumer warpgroups, one per filter
// row dy; warpgroup dy reads the three dx taps as the halo's MN-major view shifted by one pixel (LBO = 128 B, as in
// umma_wgrad_halo_kernel), starting at halo row dy.  Zero padding is the TMA zero fill of the halo.
// The output tile of a k-block is TH x TW = 64 pixels, whole rows of one image (umma_wgrad_kernel's box when TN == 1 and TW == Wo,
// TW % 8 == 0); its halo is (TH + 2) x (TW + 2) pixels at (h0 - 1, w0 - 1).  Output pixel 16j = (row r, column c) starts
// k-step j; r * TW + c = 16j, so the view of filter row dy starts at halo pixel (r + dy) (TW + 2) + c = 16j + 2r + dy (TW + 2), and the second 8-pixel core group of the k-step
// is 8 pixels further (TW >= 16, SBO = 1024 B) or one halo row further (TW = 8, SBO = (TW + 2) * 128 B).
// That is the pixel order of umma_wgrad_kernel<64, 3>, so every dW element gets the same products through the same k16 steps in
// the same k-block order, and the caller keeps that kernel's split count: the result is bit-identical.
// Bytes per k-block: 8 KB of dY + 13.5 KB of halo (16 x 4 tile) instead of 3 x (16 + 3 x 8) KB over the three filter-row CTAs.
// The same scheme on umma_wgrad_halo_kernel's 16 x 8 tiles (Cin = 64) ran layer 1 of ResNet-18 on 44 CTAs at 84 us, slower than the
// halo kernel on 132, and did not shorten the training step (docs/PROFILE_H100.md), so those shapes keep the halo kernel.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int WR_STAGES = 4;
constexpr int WR_KSTEPS = 4;                                 // 64 pixels per k-block
constexpr int WR_THREADS = 3 * 128 + 32;                     // one consumer warpgroup per filter row + the TMA producer warp

struct __align__(8) WgRowsShared {
    uint64_t full[WR_STAGES];
    uint64_t empty[WR_STAGES];
};

struct WgRowsParams {
    int num_kb, kb_per_cta;
    int TW, TH, log2_tw;      // output tile of one k-block (TW, TH powers of two, TW * TH = 64)
    int tiles_w, tiles_h;     // k-block kb = (n * tiles_h + th) * tiles_w + tw
    int stage_bytes;          // dY box + halo, rounded up to 1024 B
    uint32_t halo_bytes;      // (TH + 2) (TW + 2) 128 B
    uint32_t sbo;             // byte offset of the second 8-pixel core group of a k-step
    int ci_tiles;
    int Cout, Cin_valid;
    float* dW;                // [Cout][9][Cin_valid]
    float* part;              // split-K > 1: [splits][Cout][9][Cin_valid] partial gradients (one slot per blockIdx.z)
};

__global__ void __launch_bounds__(WR_THREADS, 1)
umma_wgrad_rows_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const WgRowsParams p) {
    constexpr int kSteps = WR_KSTEPS;
    constexpr uint32_t kABytes = kSteps * 2048;               // 64 pixel rows x 128 B
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    WgRowsShared* sh = reinterpret_cast<WgRowsShared*>(smem + WR_STAGES * p.stage_bytes);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int co_tile = blockIdx.x / p.ci_tiles, ci_tile = blockIdx.x - co_tile * p.ci_tiles;
    const int kb_begin = blockIdx.z * p.kb_per_cta;
    const int kb_end = min(p.num_kb, kb_begin + p.kb_per_cta);
    const int nkb = kb_end - kb_begin;

    if (warp == 12 && lane == 0) {
        prefetch_tmap(&tmA); prefetch_tmap(&tmB);
        for (int s = 0; s < WR_STAGES; ++s) { mbar_init(&sh->full[s], 1); mbar_init(&sh->empty[s], 12); }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();        // prologue above: parameters and shared memory only
    pdl_trigger();

    if (warp == 12) {
        if (lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int i = 0; i < nkb; ++i) {
                const int kb = kb_begin + i;
                const int tw = kb % p.tiles_w, th = (kb / p.tiles_w) % p.tiles_h, n = kb / (p.tiles_w * p.tiles_h);
                const int w0 = tw * p.TW, h0 = th * p.TH;
                mbar_wait(&sh->empty[stage], phase ^ 1);
                uint8_t* sa = smem + stage * p.stage_bytes;
                mbar_expect_tx(&sh->full[stage], kABytes + p.halo_bytes);
                tma_load_4d(&tmA, &sh->full[stage], sa, co_tile * 64, w0, h0, n);
                tma_load_4d(&tmB, &sh->full[stage], sa + kABytes, ci_tile * 64, w0 - 1, h0 - 1, n);
                if (++stage == WR_STAGES) { stage = 0; phase ^= 1; }
            }
        }
    } else if (nkb > 0) {
        const int dy = threadIdx.x >> 7, t = threadIdx.x & 127;
        const uint32_t row0 = dy * (p.TW + 2);                // first halo pixel of filter row dy
        float acc[96];
#pragma unroll
        for (int i = 0; i < 96; ++i) acc[i] = 0.f;
        int stage = 0, prev = -1;
        uint32_t phase = 0;
        for (int i = 0; i < nkb; ++i) {
            mbar_wait(&sh->full[stage], phase);
            const uint32_t sa = smem_u32(smem + stage * p.stage_bytes);
            const uint32_t halo = sa + kABytes + row0 * 128;
            wgmma_fence();
#pragma unroll
            for (int j = 0; j < kSteps; ++j) {                   // 16 output pixels 16j .. 16j + 15
                const uint32_t px = 16 * j + 2 * ((16 * j) >> p.log2_tw);
                wgmma_bf16<192, 1, 1>(acc, smem_desc_sw128(sa + j * 2048, kABytes, 1024), smem_desc_sw128(halo + px * 128, 128, p.sbo),
                                      (i > 0 || j > 0) ? 1u : 0u);
            }
            wgmma_commit();
            wgmma_wait<1>();
            if (prev >= 0 && lane == 0) mbar_arrive(&sh->empty[prev]);
            prev = stage;
            if (++stage == WR_STAGES) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        fence_acc(acc);
        wgrad_flush<192, 64>(acc, p.dW, p.part, co_tile * 64 + frag_row(t, 0), p.Cout, 9, 3 * dy, ci_tile * 64, p.Cin_valid, t);
    }
}

static int g_wgrad_rows = 1;
void set_wgrad_rows(int on) { g_wgrad_rows = on ? 1 : 0; }

// dW[Cout][9][Cin_valid] += wgrad3x3(dy[NB][H][W][Cout], x[NB][H][W][Cin]), stride 1, pad 1, over TH x TW output tiles (TW == W,
// TH | H or the last tile row zero-filled, TW >= 8, TW * TH = 64), with the split count of `splits_base` CTAs per split.
static cudaError_t launch_wgrad_rows(const void* dy, const void* x, float* dW, int NB, int H, int W, int Cin, int Cin_valid, int Cout,
                                     int TW, int TH, int splits_base, int low_waves, int num_sms, cudaStream_t st) {
    constexpr int kSteps = WR_KSTEPS;
    constexpr int kSmemMax = WR_STAGES * (kSteps * 2048 + 25600) + 2048;   // 25600: the largest halo, 66 x 3 pixels (TW = 64)
    static bool configured = false;
    if (!configured) {
        RLR_CUDA_CHECK(cudaFuncSetAttribute(umma_wgrad_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemMax));
        configured = true;
    }
    WgRowsParams p{};
    p.TW = TW; p.TH = TH;
    while ((1 << p.log2_tw) < TW) ++p.log2_tw;
    p.tiles_w = (W + TW - 1) / TW; p.tiles_h = (H + TH - 1) / TH; p.num_kb = p.tiles_w * p.tiles_h * NB;
    p.halo_bytes = (uint32_t)((TW + 2) * (TH + 2) * 128);
    p.stage_bytes = (int)((kSteps * 2048 + p.halo_bytes + 1023) / 1024 * 1024);
    p.sbo = TW >= 16 ? 1024u : (uint32_t)((TW + 2) * 128);
    p.ci_tiles = Cin / 64; p.Cout = Cout; p.Cin_valid = Cin_valid; p.dW = dW;
    const size_t smem = (size_t)WR_STAGES * p.stage_bytes + 2048;
    if (TW * TH != 16 * kSteps || TW < 8 || (TW & (TW - 1)) || smem > (size_t)kSmemMax) return cudaErrorInvalidValue;
    const int splits = wg_splits(splits_base, p.num_kb, num_sms, low_waves, &p.kb_per_cta);
    CUtensorMap tmA, tmB;
    {
        const uint64_t d[4] = {(uint64_t)Cout, (uint64_t)W, (uint64_t)H, (uint64_t)NB};
        const uint64_t s[3] = {(uint64_t)Cout * 2, (uint64_t)W * Cout * 2, (uint64_t)H * W * Cout * 2};
        const uint32_t b[4] = {64, (uint32_t)TW, (uint32_t)TH, 1};
        RLR_CUDA_CHECK(make_tmap_bf16(&tmA, dy, 4, d, s, b));
    }
    {
        const uint64_t d[4] = {(uint64_t)Cin, (uint64_t)W, (uint64_t)H, (uint64_t)NB};
        const uint64_t s[3] = {(uint64_t)Cin * 2, (uint64_t)W * Cin * 2, (uint64_t)H * W * Cin * 2};
        const uint32_t b[4] = {64, (uint32_t)TW + 2, (uint32_t)TH + 2, 1};
        RLR_CUDA_CHECK(make_tmap_bf16(&tmB, x, 4, d, s, b));
    }
    const dim3 grid((Cout + 63) / 64 * p.ci_tiles, 1, splits);
    ++g_wgrad_launches[2];
    if (splits == 1) return launch_kernel(umma_wgrad_rows_kernel, grid, dim3(WR_THREADS), smem, st, tmA, tmB, p);
    const long long plane = (long long)Cout * 9 * Cin_valid;
    Scratch part((size_t)splits * plane * sizeof(float), st);
    p.part = part.as<float>();
    RLR_CUDA_CHECK(launch_kernel(umma_wgrad_rows_kernel, grid, dim3(WR_THREADS), smem, st, tmA, tmB, p));
    return launch_ordered_sum(dW, p.part, splits, plane, st);
}

// dW[Cout][9][Cin_valid] += wgrad3x3(dy[NB][H][W][Cout], x[NB][H][W][64]); stride 1, pad 1, H % 16 == 0, W % 8 == 0
cudaError_t launch_conv_wgrad_halo_bf16(const void* dy, const void* x, float* dW, int NB, int H, int W, int Cin_valid, int Cout,
                                        int num_sms, cudaStream_t st) {
    if (H % 16 || W % 8 || Cout % 8 || !((Cout <= 64) || Cout % 128 == 0)) return cudaErrorInvalidValue;
    const int co_tiles = (Cout + WG_BM - 1) / WG_BM;
    static bool configured = false;
    if (!configured) {
        RLR_CUDA_CHECK(cudaFuncSetAttribute(umma_wgrad_halo_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, WH_SMEM));
        configured = true;
    }
    WgHaloParams p{};
    p.NB = NB; p.H = H; p.W = W; p.tiles_h = H / 16; p.tiles_w = W / 8; p.num_kb = NB * p.tiles_h * p.tiles_w;
    p.a_groups = (Cout % 128 == 0) ? 2 : 1; p.Cout = Cout; p.Cin_valid = Cin_valid; p.dW = dW;
    const int splits = wg_splits(co_tiles * 3, p.num_kb, num_sms, 1, &p.kb_per_cta);
    CUtensorMap tmA, tmB;
    {
        const uint64_t d[4] = {(uint64_t)Cout, (uint64_t)W, (uint64_t)H, (uint64_t)NB};
        const uint64_t s[3] = {(uint64_t)Cout * 2, (uint64_t)W * Cout * 2, (uint64_t)H * W * Cout * 2};
        const uint32_t b[4] = {64, 8, 16, 1};
        RLR_CUDA_CHECK(make_tmap_bf16(&tmA, dy, 4, d, s, b));
    }
    {
        const uint64_t d[4] = {64, (uint64_t)W, (uint64_t)H, (uint64_t)NB};
        const uint64_t s[3] = {128, (uint64_t)W * 128, (uint64_t)H * W * 128};
        const uint32_t b[4] = {64, 16, 18, 1};
        RLR_CUDA_CHECK(make_tmap_bf16(&tmB, x, 4, d, s, b));
    }
    ++g_wgrad_launches[1];
    if (splits == 1) return launch_kernel(umma_wgrad_halo_kernel, dim3(co_tiles, 3, splits), dim3(WG_THREADS), (size_t)WH_SMEM, st, tmA, tmB, p);
    const long long plane = (long long)Cout * 9 * Cin_valid;
    Scratch part((size_t)splits * plane * sizeof(float), st);
    p.part = part.as<float>();
    RLR_CUDA_CHECK(launch_kernel(umma_wgrad_halo_kernel, dim3(co_tiles, 3, splits), dim3(WG_THREADS), (size_t)WH_SMEM, st, tmA, tmB, p));
    return launch_ordered_sum(dW, p.part, splits, plane, st);
}

static int pow2_ceil_(int x) { int q = 1; while (q < x) q <<= 1; return q; }

// tap t = (dy, dx) reads input pixel (h + dy - 1, w + dx - 1) of the same plane
static bool standard_3x3_taps(const int* dh, const int* dw, const int* dplane) {
    for (int t = 0; t < 9; ++t)
        if (dh[t] != t / 3 - 1 || dw[t] != t % 3 - 1 || dplane[t] != 0) return false;
    return true;
}

// dW[Cout][T][Cin_valid] += wgrad(dy[NB][Ho][Wo][Cout], x[planes*NB][Hin][Win][Cin])   (Cin multiple of 64)
cudaError_t launch_conv_wgrad_bf16(const void* dy, const void* x, float* dW, int NB, int planes, int Hin, int Win, int Cin, int Cin_valid,
                                   int Ho, int Wo, int Cout, int ntaps, const int* dh, const int* dw, const int* dplane, int num_sms,
                                   cudaStream_t st, int in_stride) {
    if (Cin % 64 || Cout % 8 || (ntaps != 1 && ntaps != 9)) return cudaErrorInvalidValue;
    if (in_stride < 1 || in_stride > 2 || (in_stride > 1 && planes != 1)) return cudaErrorInvalidValue;
    WgradParams p{};
    p.in_stride = in_stride;
    int TW = pow2_ceil_(Wo); if (TW > 64) TW = 64;
    int TH = pow2_ceil_(Ho); if (TW * TH > 64) TH = 64 / TW;
    const int TN = 64 / (TW * TH);
    // the filter-row kernel takes 3x3 / stride-1 / pad-1 filters whose tile is whole rows of one image, at least one 8-pixel core
    // group wide, on unpadded channels; same split count as umma_wgrad_kernel<64, 3> (128-co tiles, three filter-row CTAs)
    if (g_wgrad_rows && ntaps == 9 && in_stride == 1 && planes == 1 && Hin == Ho && Win == Wo && TN == 1 && TW == Wo && TW % 8 == 0 &&
        Cin_valid == Cin && standard_3x3_taps(dh, dw, dplane))
        return launch_wgrad_rows(dy, x, dW, NB, Ho, Wo, Cin, Cin_valid, Cout, TW, TH, (Cout + WG_BM - 1) / WG_BM * (Cin / 64) * 3,
                                    wg_tune_waves(), num_sms, st);
    p.mode = 1; p.TW = TW; p.TH = TH; p.TN = TN;
    p.tiles_w = (Wo + TW - 1) / TW; p.tiles_h = (Ho + TH - 1) / TH;
    p.num_kb = p.tiles_w * p.tiles_h * ((NB + TN - 1) / TN);
    p.T = ntaps; p.ntaps_cta = ntaps == 9 ? 3 : 1;
    for (int t = 0; t < ntaps; ++t) { p.dh[t] = (int8_t)dh[t]; p.dw[t] = (int8_t)dw[t]; p.dn[t] = dplane[t] * NB; }
    // 128-wide ci tiles only for one-tap filters: three taps of 128 channels would need 192 accumulator registers per thread
    const bool wide = (Cin % 128 == 0) && (Cin_valid == Cin) && ntaps == 1;
    p.ci_tiles = wide ? Cin / 128 : Cin / 64; p.Cout = Cout; p.Cin_valid = Cin_valid; p.dW = dW;
    p.a_groups = Cout > 64 ? 2 : 1;        // the second 64-channel box is zero-filled beyond Cout
    const int co_tiles = (Cout + WG_BM - 1) / WG_BM;
    CUtensorMap tmA, tmB;
    {
        const uint64_t d[4] = {(uint64_t)Cout, (uint64_t)Wo, (uint64_t)Ho, (uint64_t)NB};
        const uint64_t s[3] = {(uint64_t)Cout * 2, (uint64_t)Wo * Cout * 2, (uint64_t)Ho * Wo * Cout * 2};
        const uint32_t b[4] = {64, (uint32_t)TW, (uint32_t)TH, (uint32_t)TN};
        RLR_CUDA_CHECK(make_tmap_bf16(&tmA, dy, 4, d, s, b));
    }
    {
        const uint64_t d[4] = {(uint64_t)Cin, (uint64_t)Win, (uint64_t)Hin, (uint64_t)planes * NB};
        const uint64_t s[3] = {(uint64_t)Cin * 2, (uint64_t)Win * Cin * 2, (uint64_t)Hin * Win * Cin * 2};
        const uint32_t b[4] = {64, (uint32_t)TW, (uint32_t)TH, (uint32_t)TN};
        const uint32_t es[4] = {1, (uint32_t)in_stride, (uint32_t)in_stride, 1};
        RLR_CUDA_CHECK(make_tmap_bf16(&tmB, x, 4, d, s, b, in_stride > 1 ? es : nullptr));
    }
    if (wide) return launch_wg<128, 1>(tmA, tmB, p, co_tiles, ntaps, num_sms, st);
    return ntaps == 9 ? launch_wg<64, 3>(tmA, tmB, p, co_tiles, 3, num_sms, st) : launch_wg<64, 1>(tmA, tmB, p, co_tiles, 1, num_sms, st);
}

// dW[N][K] += dy[B][N]^T x[B][K]     (N, K multiples of 64)
cudaError_t launch_linear_wgrad_bf16(const void* dy, const void* x, float* dW, int B, int N, int K, int num_sms, cudaStream_t st) {
    if (N % 8 || K % 64) return cudaErrorInvalidValue;
    WgradParams p{};
    p.mode = 0; p.num_kb = (B + WG_BK - 1) / WG_BK; p.T = 1; p.ntaps_cta = 1; p.in_stride = 1;
    const bool wide = K % 128 == 0;
    p.ci_tiles = wide ? K / 128 : K / 64; p.Cout = N; p.Cin_valid = K; p.dW = dW;
    p.a_groups = N > 64 ? 2 : 1;
    const int co_tiles = (N + WG_BM - 1) / WG_BM;
    CUtensorMap tmA, tmB;
    {
        const uint64_t d[2] = {(uint64_t)N, (uint64_t)B}, s[1] = {(uint64_t)N * 2};
        const uint32_t b[2] = {64, WG_BK};
        RLR_CUDA_CHECK(make_tmap_bf16(&tmA, dy, 2, d, s, b));
    }
    {
        const uint64_t d[2] = {(uint64_t)K, (uint64_t)B}, s[1] = {(uint64_t)K * 2};
        const uint32_t b[2] = {64, WG_BK};
        RLR_CUDA_CHECK(make_tmap_bf16(&tmB, x, 2, d, s, b));
    }
    return wide ? launch_wg<128, 1>(tmA, tmB, p, co_tiles, 1, num_sms, st) : launch_wg<64, 1>(tmA, tmB, p, co_tiles, 1, num_sms, st);
}

}  // namespace rlr
