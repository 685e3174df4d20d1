// Three-taps-per-MMA variant of the persistent 3x3 / stride-1 halo convolution for 64 input channels (opt-in: RLR_HALO3=1).
//
// conv_halo.cu issues nine N = 64 MMAs per 16-deep k-step (one per filter tap).  Here the three taps of a filter ROW share one A view:
//   D_j[h][w] = sum_ci x[h + dy - 1][w] * W[dy][j][ci][:]      for j = 0, 1, 2 at once  ->  one N = 192 MMA per (dy, k-step)
// (B = the three consecutive 64 x 64 tap tiles of the resident filter, 192 rows, K-major), and the column shift of the taps moves
// into the epilogue:
//   out[h][c] = D_0[h][c - 1] + D_1[h][c] + D_2[h][c + 1]
// Tile rows are (h, w) = 16 x 8 with w the fast index; in the wgmma accumulator fragment w = lane / 4, so "c -+ 1" is the value held
// four lanes away: two warp shuffles per value.  Only the six interior columns of a tile have both neighbours, so tiles advance by 6
// columns (8-column A views overlapping by 2): 75 % of the MMA rows are useful.
// The halo box shrinks to 8 x 18 pixels (18 KB, row-group pitch 1024 B = the swizzle atom, so the three A views start atom-aligned).
// Two consumer warpgroups (image rows 0-7 / 8-15 of the tile, 96 accumulator registers each), filter resident (72 KB), 4-stage halo ring.
#include <cuda.h>

#include "common.cuh"
#include "gemm.h"
#include "wgmma.cuh"

namespace rlr {

using namespace wg;

cudaError_t make_tmap_bf16(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                           const uint32_t* box, const uint32_t* elem_strides = nullptr);  // gemm.cu

namespace {

constexpr int H3_THREADS = 256 + 32;
constexpr int H3_TH = 16, H3_TWD = 8, H3_VALID = 6;      // 16 x 8 accumulator rows per tile, 6 output columns of them valid
constexpr int H3_HALO_BYTES = (H3_TH + 2) * H3_TWD * 128; // 18432
constexpr int H3_W_BYTES = 9 * 64 * 128;                  // 73728
constexpr int H3_STAGES = 4;
constexpr int H3_PITCH_OUT = 64 * 2 + 16;
constexpr int H3_STAGING = 128 * H3_PITCH_OUT;
constexpr int H3_SMEM = H3_W_BYTES + H3_STAGES * H3_HALO_BYTES + H3_STAGING + 1024 + 1024;

struct Halo3Params {
    int NB, H, W;
    int tiles_h, tiles_w, num_tiles;
    int N;
    void* out; int ldc;
    const float* bias;
    int relu;
};

struct __align__(8) Halo3Shared {
    uint64_t w_full;
    uint64_t halo_full[H3_STAGES];
    uint64_t halo_empty[H3_STAGES];
};

template <bool kAcc>
__global__ void __launch_bounds__(H3_THREADS, 1)
umma_conv3x3_halo3_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW, const Halo3Params p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* s_w = smem;
    uint8_t* s_halo = smem + H3_W_BYTES;
    uint8_t* s_stage = s_halo + H3_STAGES * H3_HALO_BYTES;
    Halo3Shared* sh = reinterpret_cast<Halo3Shared*>(s_stage + H3_STAGING);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tile_n = blockIdx.y;

    if (warp == 8 && lane == 0) {
        prefetch_tmap(&tmX); prefetch_tmap(&tmW);
        mbar_init(&sh->w_full, 1);
        for (int s = 0; s < H3_STAGES; ++s) { mbar_init(&sh->halo_full[s], 1); mbar_init(&sh->halo_empty[s], 8); }
        fence_barrier_init();
    }
    __syncthreads();
    const int tiles_per_img = p.tiles_h * p.tiles_w;
    pdl_wait();
    pdl_trigger();

    if (warp == 8) {
        // ===================== producer: filter once, then one 8 x 18 pixel box per tile ==================================
        if (lane == 0) {
            mbar_expect_tx(&sh->w_full, H3_W_BYTES);
            for (int t = 0; t < 9; ++t) tma_load_2d(&tmW, &sh->w_full, s_w + t * 8192, t * 64, tile_n * 64);
            int stage = 0;
            uint32_t phase = 0;
            for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
                const int n = tile / tiles_per_img, r = tile - n * tiles_per_img;
                const int h0 = (r / p.tiles_w) * H3_TH, c0 = (r % p.tiles_w) * H3_VALID - 1;     // first accumulator column (may be -1)
                mbar_wait(&sh->halo_empty[stage], phase ^ 1);
                mbar_expect_tx(&sh->halo_full[stage], H3_HALO_BYTES);
                tma_load_4d(&tmX, &sh->halo_full[stage], s_halo + stage * H3_HALO_BYTES, 0, c0, h0 - 1, n);
                if (++stage == H3_STAGES) { stage = 0; phase ^= 1; }
            }
        }
    } else {
        // ===================== consumers: 3 filter rows x 4 k-steps of N = 192, shift-add, bias / ReLU / accumulate, stores =====
        const int et = threadIdx.x;
        const int wgi = et >> 7, t = et & 127;
        const int r0 = wgi * 64 + frag_row(t, 0);               // accumulator rows r0, r0 + 8 (row = h * 8 + w, w = lane / 4)
        const int col0 = tile_n * 64;
        const uint32_t w_base = smem_u32(s_w);
        __nv_bfloat16* out = reinterpret_cast<__nv_bfloat16*>(p.out);
        int stage = 0;
        uint32_t phase = 0;
        mbar_wait(&sh->w_full, 0);
        for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
            const int n = tile / tiles_per_img, r = tile - n * tiles_per_img;
            const int h0 = (r / p.tiles_w) * H3_TH, oc0 = (r % p.tiles_w) * H3_VALID;    // first OUTPUT column of the tile
            uint4 oldv[4];
            if (kAcc) {
#pragma unroll
                for (int it = 0; it < 4; ++it) {
                    const int idx = et + it * 256, rr = idx >> 3, ch = idx & 7;
                    const int wl = rr & 7, h = h0 + (rr >> 3), c = oc0 + wl - 1;
                    oldv[it] = make_uint4(0, 0, 0, 0);
                    if (wl >= 1 && wl <= H3_VALID && col0 + ch * 8 < p.N && h < p.H && c < p.W)
                        oldv[it] = *reinterpret_cast<const uint4*>(out + (((size_t)n * p.H + h) * p.W + c) * p.ldc + col0 + ch * 8);
                }
            }
            mbar_wait(&sh->halo_full[stage], phase);
            const uint32_t halo = smem_u32(s_halo + stage * H3_HALO_BYTES) + wgi * 8 * 1024;   // image rows 8 wgi .. 8 wgi + 7
            float acc[96];
#pragma unroll
            for (int i = 0; i < 96; ++i) acc[i] = 0.f;
            wgmma_fence();
#pragma unroll
            for (int dy = 0; dy < 3; ++dy) {
                const uint32_t a0 = halo + dy * H3_TWD * 128;            // box row dy: 1024-byte (atom) aligned
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    wgmma_bf16<192, 0, 0>(acc, smem_desc_sw128(a0 + k * 32, 16, 1024),
                                          smem_desc_sw128(w_base + dy * 3 * 8192 + k * 32, 16, 1024),   // taps (dy,0..2): 192 rows
                                          (dy > 0 || k > 0) ? 1u : 0u);
            }
            wgmma_commit();
            wgmma_wait<0>();
            fence_acc(acc);
            if (lane == 0) mbar_arrive(&sh->halo_empty[stage]);
            if (++stage == H3_STAGES) { stage = 0; phase ^= 1; }
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int c = frag_col(t, 4 * j);
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    float v[2];
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int i = 4 * j + 2 * h + e;
                        // tap column j = 0 contributes to the output one pixel (4 lanes) to the right, j = 2 one pixel to the left
                        v[e] = acc[32 + i] + __shfl_up_sync(0xffffffffu, acc[i], 4) + __shfl_down_sync(0xffffffffu, acc[64 + i], 4);
                        if (p.bias && col0 + c + e < p.N) v[e] += p.bias[col0 + c + e];
                        if (p.relu) v[e] = fmaxf(v[e], 0.f);
                    }
                    *reinterpret_cast<uint32_t*>(s_stage + (r0 + 8 * h) * H3_PITCH_OUT + c * 2) = pack_bf16x2(v[0], v[1]);
                }
            }
            named_bar(1, 256);
            // stores: accumulator row rr = (h, wl); wl = 1..6 are the valid output columns oc0 + wl - 1 (w = 0 and 7 lack a neighbour
            // and are dropped)
#pragma unroll
            for (int it = 0; it < 4; ++it) {
                const int idx = et + it * 256, rr = idx >> 3, ch = idx & 7;
                const int wl = rr & 7, h = h0 + (rr >> 3), c = oc0 + wl - 1;
                if (wl < 1 || wl > H3_VALID || col0 + ch * 8 >= p.N || h >= p.H || c >= p.W) continue;
                uint4 val = *reinterpret_cast<const uint4*>(s_stage + rr * H3_PITCH_OUT + ch * 16);
                uint4* gp = reinterpret_cast<uint4*>(out + (((size_t)n * p.H + h) * p.W + c) * p.ldc + col0 + ch * 8);
                if (kAcc) {
                    const __nv_bfloat162* o2 = reinterpret_cast<const __nv_bfloat162*>(&oldv[it]);
                    __nv_bfloat162* v2 = reinterpret_cast<__nv_bfloat162*>(&val);
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const float2 a = __bfloat1622float2(v2[q]), b = __bfloat1622float2(o2[q]);
                        v2[q] = __floats2bfloat162_rn(a.x + b.x, a.y + b.y);
                    }
                }
                *gp = val;
            }
            named_bar(1, 256);
        }
    }
}

}  // namespace

// y[NB][H][W][Cout] (+)= conv3x3(x[NB][H][W][64], w[Cout][9*64]), stride 1, pad 1; H % 16 == 0.
cudaError_t launch_conv3x3_halo3_bf16(const void* x, const void* w, void* out, int NB, int H, int W, int Cout, const float* bias, int relu,
                                      int accumulate, int num_sms, cudaStream_t st) {
    if (H % H3_TH || Cout % 8) return cudaErrorInvalidValue;
    static bool configured = false;
    if (!configured) {
        RLR_CUDA_CHECK(cudaFuncSetAttribute(umma_conv3x3_halo3_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, H3_SMEM));
        RLR_CUDA_CHECK(cudaFuncSetAttribute(umma_conv3x3_halo3_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, H3_SMEM));
        configured = true;
    }
    Halo3Params p{};
    p.NB = NB; p.H = H; p.W = W; p.tiles_h = H / H3_TH; p.tiles_w = (W + H3_VALID - 1) / H3_VALID; p.num_tiles = NB * p.tiles_h * p.tiles_w;
    p.N = Cout; p.out = out; p.ldc = Cout; p.bias = bias; p.relu = relu;
    CUtensorMap tmX, tmW;
    {
        const uint64_t d[4] = {64, (uint64_t)W, (uint64_t)H, (uint64_t)NB};
        const uint64_t s[3] = {128, (uint64_t)W * 128, (uint64_t)H * W * 128};
        const uint32_t b[4] = {64, H3_TWD, H3_TH + 2, 1};
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
    if (accumulate) return launch_kernel(umma_conv3x3_halo3_kernel<true>, grid, dim3(H3_THREADS), (size_t)H3_SMEM, st, tmX, tmW, p);
    return launch_kernel(umma_conv3x3_halo3_kernel<false>, grid, dim3(H3_THREADS), (size_t)H3_SMEM, st, tmX, tmW, p);
}

}  // namespace rlr
