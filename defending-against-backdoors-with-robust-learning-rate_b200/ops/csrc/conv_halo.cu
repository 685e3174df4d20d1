// Persistent wgmma 3x3 / stride-1 convolution for 64-channel inputs with SHARED-MEMORY HALO REUSE (sm_90a).
//
// The generic implicit-GEMM kernel (gemm.cu) fetches one 128x64 input tile per filter tap, i.e. it re-reads every input
// pixel 9 times from L2 (TMA bypasses L1), which makes the 64-channel 32x32 layers L2-bandwidth bound.
// Here an output tile is 16 rows x 8 columns of one image and its whole receptive field -- 18 x 10 pixels x 64 channels,
// stored with a 16-pixel row pitch = 36 KB -- is loaded ONCE by a single 4-D TMA box (zero fill at the borders = padding).
// The A operand of tap (dy,dx) is then just a *view* into that halo: 16 groups (image rows) of 8 pixel-rows, group stride
// SBO = 16 px * 128 B = 2048 B, start address offset by (dy*16 + dx) * 128 B.  That start is not aligned to the 1024-byte
// swizzle atom; the descriptor's base-offset field is 0 by default (bo_mode 0, the swizzle follows the absolute shared-memory
// address bits like the TMA unit that wrote the tile) or (addr >> 7) & 7 (bo_mode 1); tests/test_gpu_native.py checks both.
// All 9 x 64 x 64 filter taps (72 KB) stay resident in shared memory for the lifetime of the persistent CTA, so per output tile
// the kernel moves 36 KB instead of 216 KB.  The two consumer warpgroups take alternate tiles, each computing the whole 128 x 64
// tile (two m64n64 wgmma per k-step) into registers and running its own epilogue (bias / ReLU / residual-accumulate / bf16 /
// coalesced stores / BatchNorm statistics) from its own staging tile, so one warpgroup's epilogue overlaps the other's MMAs.
// Used for the stem and layer1 forward convolutions and layer1 data gradients of ResNet-18 and the 64-channel VGG layers.
#include <cuda.h>

#include "common.cuh"
#include "gemm.h"
#include "wgmma.cuh"

namespace rlr {

using namespace wg;

cudaError_t make_tmap_bf16(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                           const uint32_t* box, const uint32_t* elem_strides = nullptr);  // gemm.cu

constexpr int HL_THREADS = 256 + 32;                  // two consumer warpgroups + the TMA producer warp
constexpr int HL_TH = 16, HL_TW = 8;                  // output tile: 16 rows x 8 cols = 128 pixels
constexpr int HL_PITCH = 16;                          // halo row pitch in pixels (8 + 2 halo + 6 pad) -> SBO = 2048 B
constexpr int HL_HALO_BYTES = (HL_TH + 2) * HL_PITCH * 128;   // 36864
constexpr int HL_W_BYTES = 9 * 64 * 128;              // 73728: [tap][cout 64][cin 64] bf16, K-major, one n-tile
constexpr int HL_STAGES = 3;
constexpr int HL_PITCH_OUT = 64 * 2 + 16;             // staging row pitch (bytes)
constexpr int HL_STAGING = 128 * HL_PITCH_OUT;        // per warpgroup
constexpr int HL_SMEM = HL_W_BYTES + HL_STAGES * HL_HALO_BYTES + 2 * HL_STAGING + 1024 + 1024;

struct HaloParams {
    int NB, H, W;                 // OUTPUT spatial size; input = output + 2 - 2*pad
    int pad;                      // 0 (valid conv), 1 (same), 2 (full: data gradient of a valid conv)
    int tiles_h, tiles_w, num_tiles;
    int N;                        // Cout (valid columns of this launch's n-tile range)
    void* out; int ldc;
    const float* bias;
    float* stats;
    int relu, accumulate;
    long long* dbg;               // optional per-tile clock64 timeline of CTA 0 (tuning aid): [tile][8]
    int bo_mode;                  // 0: descriptor base-offset field 0;  1: (addr >> 7) & 7
};

struct __align__(8) HaloShared {
    uint64_t w_full;
    uint64_t halo_full[HL_STAGES];
    uint64_t halo_empty[HL_STAGES];
    float red[128];               // per-CTA column sums (sum, sum of squares)
    float bias[64];
};

template <bool kStats, bool kAcc>
__global__ void __launch_bounds__(HL_THREADS, 1)
umma_conv3x3_halo_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW, const HaloParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* s_w = smem;                                   // 72 KB resident filter
    uint8_t* s_halo = smem + HL_W_BYTES;                   // 3 x 36 KB ring
    uint8_t* s_stage = s_halo + HL_STAGES * HL_HALO_BYTES; // 2 epilogue staging tiles
    HaloShared* sh = reinterpret_cast<HaloShared*>(s_stage + 2 * HL_STAGING);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tile_n = blockIdx.y;
    const int col0 = tile_n * 64;

    if (warp == 8 && lane == 0) {
        prefetch_tmap(&tmX); prefetch_tmap(&tmW);
        mbar_init(&sh->w_full, 1);
        for (int s = 0; s < HL_STAGES; ++s) { mbar_init(&sh->halo_full[s], 1); mbar_init(&sh->halo_empty[s], 4); }
        fence_barrier_init();
    }
    if (threadIdx.x < 128) sh->red[threadIdx.x] = 0.f;
    const int tiles_per_img = p.tiles_h * p.tiles_w;
    pdl_wait();
    pdl_trigger();
    if (threadIdx.x < 64) sh->bias[threadIdx.x] = (p.bias && col0 + (int)threadIdx.x < p.N) ? p.bias[col0 + threadIdx.x] : 0.f;
    __syncthreads();

    if (warp == 8) {
        // ===================== producer: filter once, then one halo box per tile =====================================
        if (lane == 0) {
            mbar_expect_tx(&sh->w_full, HL_W_BYTES);
            for (int t = 0; t < 9; ++t) tma_load_2d(&tmW, &sh->w_full, s_w + t * 8192, t * 64, tile_n * 64);
            int stage = 0;
            uint32_t phase = 0;
            for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
                const int n = tile / tiles_per_img, r = tile - n * tiles_per_img;
                const int h0 = (r / p.tiles_w) * HL_TH, w0 = (r % p.tiles_w) * HL_TW;
                mbar_wait(&sh->halo_empty[stage], phase ^ 1);
                mbar_expect_tx(&sh->halo_full[stage], HL_HALO_BYTES);
                tma_load_4d(&tmX, &sh->halo_full[stage], s_halo + stage * HL_HALO_BYTES, 0, w0 - p.pad, h0 - p.pad, n);
                if (++stage == HL_STAGES) { stage = 0; phase ^= 1; }
            }
        }
    } else {
        // ===================== consumers: warpgroup wgi takes the tiles of ordinal q = wgi, wgi + 2, ... ====================
        const int wgi = threadIdx.x >> 7, t = threadIdx.x & 127;
        uint8_t* stage_buf = s_stage + wgi * HL_STAGING;
        const int r0 = frag_row(t, 0);                         // rows r0 (+8) of each 64-row half
        __nv_bfloat16* out = reinterpret_cast<__nv_bfloat16*>(p.out);
        float st1[16], st2[16];                                // statistics of this thread's 16 columns over all its tiles
#pragma unroll
        for (int i = 0; i < 16; ++i) { st1[i] = 0.f; st2[i] = 0.f; }
        const uint32_t w_base = smem_u32(s_w);
        mbar_wait(&sh->w_full, 0);
        for (int q = wgi;; q += 2) {
            const int tile = blockIdx.x + q * gridDim.x;
            if (tile >= p.num_tiles) break;
            const int stage = q % HL_STAGES;
            const uint32_t phase = (uint32_t)(q / HL_STAGES) & 1u;
            const int n = tile / tiles_per_img, r = tile - n * tiles_per_img;
            const int h0 = (r / p.tiles_w) * HL_TH, w0 = (r % p.tiles_w) * HL_TW;
            // residual-accumulate operand: issue all loads BEFORE the MMAs so their latency overlaps them
            uint4 oldv[8];
            if (kAcc) {
#pragma unroll
                for (int it = 0; it < 8; ++it) {
                    const int idx = t + it * 128, rr = idx >> 3, ch = idx & 7;
                    const int h = h0 + (rr >> 3), w = w0 + (rr & 7);
                    oldv[it] = make_uint4(0, 0, 0, 0);
                    if (col0 + ch * 8 < p.N && h < p.H && w < p.W)
                        oldv[it] = *reinterpret_cast<const uint4*>(out + (((size_t)n * p.H + h) * p.W + w) * p.ldc + col0 + ch * 8);
                }
            }
            const bool trace = p.dbg && blockIdx.x == 0 && blockIdx.y == 0 && t == 0;
            if (trace) p.dbg[q * 8 + 0] = clock64();
            mbar_wait(&sh->halo_full[stage], phase);
            if (trace) p.dbg[q * 8 + 2] = clock64();
            const uint32_t halo = smem_u32(s_halo + stage * HL_HALO_BYTES);
            float acc[2][32];
#pragma unroll
            for (int m = 0; m < 2; ++m)
#pragma unroll
                for (int i = 0; i < 32; ++i) acc[m][i] = 0.f;
            wgmma_fence();
#pragma unroll
            for (int tp = 0; tp < 9; ++tp) {
                const int dy = tp / 3, dx = tp - dy * 3;
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const uint64_t db = smem_desc_sw128(w_base + tp * 8192 + k * 32, 16, 1024);
#pragma unroll
                    for (int m = 0; m < 2; ++m) {                  // rows 64 m .. 64 m + 63 = image rows 8 m .. 8 m + 7 of the tile
                        const uint32_t a0 = halo + (dy * HL_PITCH + dx) * 128 + m * 8 * HL_PITCH * 128 + k * 32;
                        const uint32_t bo = p.bo_mode ? ((a0 >> 7) & 7u) : 0u;
                        wgmma_bf16<64, 0, 0>(acc[m], smem_desc_sw128(a0, 16, HL_PITCH * 128, bo), db, (tp > 0 || k > 0) ? 1u : 0u);
                    }
                }
            }
            wgmma_commit();
            wgmma_wait<0>();
            fence_acc(acc[0]);
            fence_acc(acc[1]);
            if (lane == 0) mbar_arrive(&sh->halo_empty[stage]);   // 4 arrivals (this warpgroup's warps) release the halo stage
            if (trace) p.dbg[q * 8 + 3] = clock64();
#pragma unroll
            for (int m = 0; m < 2; ++m)
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int c = frag_col(t, 4 * j);
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        float a = acc[m][4 * j + 2 * h], b = acc[m][4 * j + 2 * h + 1];
                        a += sh->bias[c]; b += sh->bias[c + 1];
                        if (p.relu) { a = fmaxf(a, 0.f); b = fmaxf(b, 0.f); }
                        const uint32_t packed = pack_bf16x2(a, b);
                        if (kStats) {   // statistics of the bf16-rounded values that BatchNorm will read back (whole tiles only)
                            const float2 rq = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&packed));
                            st1[2 * j] += rq.x; st1[2 * j + 1] += rq.y;
                            st2[2 * j] += rq.x * rq.x; st2[2 * j + 1] += rq.y * rq.y;
                        }
                        *reinterpret_cast<uint32_t*>(stage_buf + (m * 64 + r0 + 8 * h) * HL_PITCH_OUT + c * 2) = packed;
                    }
                }
            named_bar(1 + wgi, 128);
            if (trace) p.dbg[q * 8 + 6] = clock64();
            // coalesced stores: tile row rr = g*8 + px  ->  image pixel (h0+g, w0+px)
#pragma unroll
            for (int it = 0; it < 8; ++it) {
                const int idx = t + it * 128;
                const int rr = idx >> 3, ch = idx & 7;
                if (col0 + ch * 8 >= p.N) continue;
                const int h = h0 + (rr >> 3), w = w0 + (rr & 7);
                if (h >= p.H || w >= p.W) continue;
                const size_t gi = ((size_t)n * p.H + h) * p.W + w;
                uint4 val = *reinterpret_cast<const uint4*>(stage_buf + rr * HL_PITCH_OUT + ch * 16);
                uint4* gp = reinterpret_cast<uint4*>(out + gi * p.ldc + col0 + ch * 8);
                if (kAcc) {
                    const __nv_bfloat162* o2 = reinterpret_cast<const __nv_bfloat162*>(&oldv[it]);
                    __nv_bfloat162* v2 = reinterpret_cast<__nv_bfloat162*>(&val);
#pragma unroll
                    for (int qq = 0; qq < 4; ++qq) {
                        const float2 a = __bfloat1622float2(v2[qq]), b = __bfloat1622float2(o2[qq]);
                        v2[qq] = __floats2bfloat162_rn(a.x + b.x, a.y + b.y);
                    }
                }
                *gp = val;
            }
            named_bar(1 + wgi, 128);                                // staging may be overwritten by this warpgroup's next tile
            if (trace) p.dbg[q * 8 + 7] = clock64();
        }
        if (kStats) {
            // column sums over the 8 lanes sharing this thread's columns, then one shared atomic per column and warp
#pragma unroll
            for (int i = 0; i < 16; ++i)
#pragma unroll
                for (int o = 4; o < 32; o <<= 1) {
                    st1[i] += __shfl_xor_sync(0xffffffffu, st1[i], o);
                    st2[i] += __shfl_xor_sync(0xffffffffu, st2[i], o);
                }
            if (lane < 4)
#pragma unroll
                for (int i = 0; i < 16; ++i) {
                    const int c = frag_col(t, 2 * (i & ~1)) + (i & 1);
                    atomicAdd(&sh->red[c], st1[i]);
                    atomicAdd(&sh->red[64 + c], st2[i]);
                }
            named_bar(3, 256);
            // one global reduction per CTA and channel (instead of per tile), spread over kStatSlots slots to cut same-address
            // contention in L2; bn_finalize sums the slots
            if (threadIdx.x < 128 && col0 + (threadIdx.x & 63) < p.N)
                atomicAdd(p.stats + (size_t)(blockIdx.x % kStatSlots) * 2 * p.N + (threadIdx.x < 64 ? 0 : p.N) + col0 + (threadIdx.x & 63),
                          sh->red[threadIdx.x]);
        }
    }
}

// y[NB][H][W][Cout] = conv3x3(x[NB][Hin][Win][64], w[Cout][9*64]), stride 1, padding pad = (H - Hin + 2) / 2 in {0, 1, 2} (valid / same /
// full).  Any H, W: the image is covered by ceil(H/16) x ceil(W/8) tiles, pixels beyond the output are masked in the epilogue and input
// pixels beyond the image are the TMA unit's zero fill.  BatchNorm statistics need whole tiles (H % 16 == 0, W % 8 == 0).
cudaError_t launch_conv3x3_halo_bf16(const void* x, const void* w, void* out, int NB, int Hin, int Win, int H, int W, int Cout, const float* bias,
                                     int relu, int accumulate, float* stats, int bo_mode, long long* dbg, int num_sms, cudaStream_t st) {
    const int pad = (H - Hin + 2) / 2;
    if (pad < 0 || pad > 2 || H != Hin + 2 * pad - 2 || W != Win + 2 * pad - 2 || H < 1 || W < 1 || Cout % 8) return cudaErrorInvalidValue;
    if (stats && (H % HL_TH || W % HL_TW)) return cudaErrorInvalidValue;
    static bool configured = false;
    if (!configured) {
        RLR_CUDA_CHECK(cudaFuncSetAttribute(umma_conv3x3_halo_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, HL_SMEM));
        RLR_CUDA_CHECK(cudaFuncSetAttribute(umma_conv3x3_halo_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, HL_SMEM));
        RLR_CUDA_CHECK(cudaFuncSetAttribute(umma_conv3x3_halo_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, HL_SMEM));
        configured = true;
    }
    if (stats && accumulate) return cudaErrorInvalidValue;
    HaloParams p{};
    p.NB = NB; p.H = H; p.W = W; p.pad = pad;
    p.tiles_h = (H + HL_TH - 1) / HL_TH; p.tiles_w = (W + HL_TW - 1) / HL_TW; p.num_tiles = NB * p.tiles_h * p.tiles_w;
    p.N = Cout; p.out = out; p.ldc = Cout; p.bias = bias; p.stats = stats; p.relu = relu; p.accumulate = accumulate; p.bo_mode = bo_mode; p.dbg = dbg;
    CUtensorMap tmX, tmW;
    {
        const uint64_t d[4] = {64, (uint64_t)Win, (uint64_t)Hin, (uint64_t)NB};
        const uint64_t s[3] = {128, (uint64_t)Win * 128, (uint64_t)Hin * Win * 128};
        const uint32_t b[4] = {64, HL_PITCH, HL_TH + 2, 1};
        RLR_CUDA_CHECK(make_tmap_bf16(&tmX, x, 4, d, s, b));
    }
    {
        const uint64_t d[2] = {9 * 64, (uint64_t)Cout}, s[1] = {9 * 64 * 2};
        const uint32_t b[2] = {64, 64};
        RLR_CUDA_CHECK(make_tmap_bf16(&tmW, w, 2, d, s, b));
    }
    const int n_tiles_n = (Cout + 63) / 64;
    int gx = num_sms / n_tiles_n;
    if (gx > p.num_tiles) gx = p.num_tiles;
    if (gx < 1) gx = 1;
    const dim3 grid(gx, n_tiles_n);
    if (stats) return launch_kernel(umma_conv3x3_halo_kernel<true, false>, grid, dim3(HL_THREADS), HL_SMEM, st, tmX, tmW, p);
    if (accumulate) return launch_kernel(umma_conv3x3_halo_kernel<false, true>, grid, dim3(HL_THREADS), HL_SMEM, st, tmX, tmW, p);
    return launch_kernel(umma_conv3x3_halo_kernel<false, false>, grid, dim3(HL_THREADS), HL_SMEM, st, tmX, tmW, p);
}

}  // namespace rlr
