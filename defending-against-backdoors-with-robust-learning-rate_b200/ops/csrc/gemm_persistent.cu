// Persistent variant of the implicit-GEMM conv / GEMM kernel of gemm.cu (opt-in: RLR_PERSISTENT_CONV=1; default for the stem GEMM).
//
// Same operands, tap tables and epilogue semantics as umma_conv_gemm_kernel, but the CTA loops over output tiles (tile = blockIdx.x,
// += gridDim.x; consecutive tiles share the filter n-tile) with a deeper operand ring (7 x 24 KB for BN = 64, 5 x 32 KB for BN = 128)
// and a dedicated staging tile: the producer warp runs straight through tile boundaries, so the operands of tile i+1 are in flight
// while the two consumer warpgroups (64 rows each) run the epilogue of tile i.  No statistics path (BatchNorm statistics are taken
// by the streaming pass, see models/native.py).
#include <cuda.h>

#include "common.cuh"
#include "gemm.h"
#include "stem_gather.cuh"
#include "wgmma.cuh"

namespace rlr {

using namespace wg;

constexpr int PBM = 128, PBK = 64, PConsumers = 256, PThreads = PConsumers + 32;

// kOcc = 1: one CTA per SM with a deep ring (7 x 24 KB / 5 x 32 KB).  kOcc = 2: two CTAs per SM with a 3-stage ring -- for the stem GEMM,
// whose one-k-block tiles are EPILOGUE bound: two CTAs give the SM two sets of epilogue warpgroups (and two TMA streams) to drain them.
template <int BN, int kOcc = 1>
struct PCfg {
    static constexpr int kStages = kOcc == 2 ? 3 : (BN == 64 ? 7 : 5);
    static constexpr int kABytes = PBM * PBK * 2;
    static constexpr int kBBytes = BN * PBK * 2;
    static constexpr int kStageBytes = kABytes + kBBytes;
    static constexpr int kPitch = BN * 2 + 16;
    static constexpr int kStagingBytes = PBM * kPitch;
    static constexpr int kRingBytes = kStages * kStageBytes;
    static constexpr int kTailBytes = BN == 128 ? 2048 : 1024;    // PShared (704 B) + the n-tile's bias values (BN floats)
    static constexpr int kSmemBytes = kRingBytes + kStagingBytes + 1024 + kTailBytes;
};

struct __align__(8) PShared {
    uint64_t full[8];
    uint64_t empty[8];
    int row_index[PBM];
};
static_assert(sizeof(PShared) <= 704, "the bias slice starts 704 bytes into the tail");

template <int BN, bool kBMN, int kOcc = 1>
__global__ void __launch_bounds__(PThreads, kOcc)
umma_conv_gemm_persistent_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const ConvGemmParams p,
                                  const int m_tiles, const int total_tiles) {
    using Cfg = PCfg<BN, kOcc>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* staging = smem + Cfg::kRingBytes;
    PShared* sh = reinterpret_cast<PShared*>(staging + Cfg::kStagingBytes);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (warp == 8 && lane == 0) {
        prefetch_tmap(&tmA); prefetch_tmap(&tmB);
        for (int s = 0; s < Cfg::kStages; ++s) { mbar_init(&sh->full[s], 1); mbar_init(&sh->empty[s], 8); }
        fence_barrier_init();
    }
    __syncthreads();

    // tile -> (tile_m, tile_n) and image-space origin
    auto origin = [&](int tile, int& tile_m, int& tile_n, int& n0, int& h0, int& w0) {
        tile_m = tile % m_tiles; tile_n = tile / m_tiles;
        n0 = h0 = w0 = 0;
        if (p.mode == 1) {
            const int tw_i = tile_m % p.tiles_w, th_i = (tile_m / p.tiles_w) % p.tiles_h, tn_i = tile_m / (p.tiles_w * p.tiles_h);
            w0 = tw_i * p.TW; h0 = th_i * p.TH; n0 = tn_i * p.TN;
        }
    };

    if (warp == 8) {
        // stem GEMM (b_src: one k-block, one n-tile): the B tile is built ONCE per CTA by this warp in the B slot of stage 0 (no stage ever
        // loads a B tile in this mode, so the slot is never overwritten) and every tile's MMAs read it there; per tile only A is fetched.
        // The first full[0] arrival orders the gather before every consumer read of the slot.
        if (p.b_src) stem_gather_b(p, smem + Cfg::kABytes, BN, 0, lane);
        if (lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
                int tile_m, tile_n, n0, h0, w0;
                origin(tile, tile_m, tile_n, n0, h0, w0);
                for (int kb = 0; kb < p.num_kb; ++kb) {
                    mbar_wait(&sh->empty[stage], phase ^ 1);
                    uint8_t* sa = smem + stage * Cfg::kStageBytes;
                    uint8_t* sb = sa + Cfg::kABytes;
                    mbar_expect_tx(&sh->full[stage], p.b_src ? Cfg::kABytes : Cfg::kStageBytes);
                    const int tap = p.mode == 1 ? kb / p.cblocks : 0, cb = p.mode == 1 ? kb - tap * p.cblocks : 0;
                    if (p.mode == 1) tma_load_4d(&tmA, &sh->full[stage], sa, cb * PBK, w0 * p.in_stride + p.dw[tap], h0 * p.in_stride + p.dh[tap],
                                                n0 + p.dn[tap]);
                    else tma_load_2d(&tmA, &sh->full[stage], sa, kb * PBK, tile_m * PBM);
                    if (p.b_src) {
                        // resident B tile (above)
                    } else if (kBMN) {
                        for (int g = 0; g < BN / 64; ++g)
                            tma_load_2d(&tmB, &sh->full[stage], sb + g * 8192, p.wtap[tap] * p.wcols + tile_n * BN + g * 64, cb * PBK);
                    } else {
                        tma_load_2d(&tmB, &sh->full[stage], sb, kb * PBK, tile_n * BN);
                    }
                    if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else {
        const int et = threadIdx.x;                 // 0..255
        const int wgi = et >> 7, t = et & 127;
        const int r0 = wgi * 64 + frag_row(t, 0);   // this thread's two tile rows: r0, r0 + 8
        __nv_bfloat16* out = reinterpret_cast<__nv_bfloat16*>(p.out);
        constexpr int kChunks = BN * 2 / 16;
        constexpr int kIters = PBM * kChunks / PConsumers;
        constexpr int kBatch = kIters < 8 ? kIters : 8;
        float* bias_s = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(sh) + 704);
        int bias_tile_n = -1;
        int stage = 0;
        uint32_t phase = 0;
        const uint32_t b_fixed = p.b_src ? smem_u32(smem + Cfg::kABytes) : 0u;
        for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
            int tile_m, tile_n, n0, h0, w0;
            origin(tile, tile_m, tile_n, n0, h0, w0);
            const int col0 = tile_n * BN;
            if (p.bias && tile_n != bias_tile_n) {   // (re)load this n-tile's bias values; consecutive tiles share the n-tile
                for (int i = et; i < BN; i += PConsumers) bias_s[i] = (col0 + i < p.N) ? p.bias[col0 + i] : 0.f;
                bias_tile_n = tile_n;
            }
            if (et < PBM) {   // global output row of every tile row (-1 = masked); the previous tile's readers are past the end-of-tile barrier
                const int row = et;
                int gi;
                if (p.mode == 1) {
                    const int tw = row % p.TW, th = (row / p.TW) % p.TH, tn = row / (p.TW * p.TH);
                    const int w = w0 + tw, h = h0 + th, n = n0 + tn;
                    gi = (w < p.Wo && h < p.Ho && n < p.NB)
                             ? ((n * p.OutH + h * p.out_stride + p.out_ph) * p.OutW + w * p.out_stride + p.out_pw) : -1;
                } else {
                    gi = tile_m * PBM + row;
                    if (gi >= p.M) gi = -1;
                }
                sh->row_index[row] = gi;
            }
            float acc[BN / 2];
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
            consumer_mainloop<BN, Cfg::kStages, Cfg::kStageBytes, Cfg::kABytes, kBMN>(acc, smem, sh->full, sh->empty, p.num_kb,
                                                                                       (uint32_t)wgi * 64 * 128, b_fixed, stage, phase, lane);
            named_bar(1, PConsumers);                // bias slice and row_index of this tile are written
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
                const int c = frag_col(t, 4 * j);
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    float a = acc[4 * j + 2 * h], b = acc[4 * j + 2 * h + 1];
                    if (p.bias) { a += bias_s[c]; b += bias_s[c + 1]; }
                    if (p.relu) { a = fmaxf(a, 0.f); b = fmaxf(b, 0.f); }
                    *reinterpret_cast<uint32_t*>(staging + (r0 + 8 * h) * Cfg::kPitch + c * 2) = pack_bf16x2(a, b);
                }
            }
            named_bar(1, PConsumers);                // staging tile complete
#pragma unroll
            for (int it0 = 0; it0 < kIters; it0 += kBatch) {
                uint4 oldv[kBatch];
                if (p.accumulate) {
#pragma unroll
                    for (int j = 0; j < kBatch; ++j) {
                        const int idx = et + (it0 + j) * PConsumers, r = idx / kChunks, ch = idx - r * kChunks;
                        const int gi = sh->row_index[r];
                        oldv[j] = make_uint4(0, 0, 0, 0);
                        if (gi >= 0 && col0 + ch * 8 < p.N) oldv[j] = *reinterpret_cast<const uint4*>(out + (size_t)gi * p.ldc + col0 + ch * 8);
                    }
                }
#pragma unroll
                for (int j = 0; j < kBatch; ++j) {
                    const int idx = et + (it0 + j) * PConsumers, r = idx / kChunks, ch = idx - r * kChunks;
                    const int gi = sh->row_index[r];
                    if (gi < 0 || col0 + ch * 8 >= p.N) continue;
                    uint4 val = *reinterpret_cast<const uint4*>(staging + r * Cfg::kPitch + ch * 16);
                    if (p.accumulate) {
                        const __nv_bfloat162* o2 = reinterpret_cast<const __nv_bfloat162*>(&oldv[j]);
                        __nv_bfloat162* v2 = reinterpret_cast<__nv_bfloat162*>(&val);
#pragma unroll
                        for (int q = 0; q < 4; ++q) {
                            const float2 a = __bfloat1622float2(v2[q]), b = __bfloat1622float2(o2[q]);
                            v2[q] = __floats2bfloat162_rn(a.x + b.x, a.y + b.y);
                        }
                    }
                    *reinterpret_cast<uint4*>(out + (size_t)gi * p.ldc + col0 + ch * 8) = val;
                }
            }
            named_bar(1, PConsumers);                // staging / row_index / bias slice may be overwritten by the next tile
        }
    }
}

template <int BN>
cudaError_t launch_persistent_bn(const CUtensorMap& tmA, const CUtensorMap& tmB, const ConvGemmParams& p, int m_tiles, int num_sms,
                                 cudaStream_t st, int occ) {
    const int n_tiles = (p.N + BN - 1) / BN;
    const int total = m_tiles * n_tiles;
    if (occ == 2 && !p.b_mn) {
        using Cfg = PCfg<BN, 2>;
        static bool configured2 = false;
        if (!configured2) {
            RLR_CUDA_CHECK(cudaFuncSetAttribute(umma_conv_gemm_persistent_kernel<BN, false, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
            configured2 = true;
        }
        const int grid = total < 2 * num_sms ? total : 2 * num_sms;
        umma_conv_gemm_persistent_kernel<BN, false, 2><<<grid, PThreads, Cfg::kSmemBytes, st>>>(tmA, tmB, p, m_tiles, total);
        return cudaGetLastError();
    }
    using Cfg = PCfg<BN>;
    static bool configured = false;
    if (!configured) {
        RLR_CUDA_CHECK(cudaFuncSetAttribute(umma_conv_gemm_persistent_kernel<BN, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
        RLR_CUDA_CHECK(cudaFuncSetAttribute(umma_conv_gemm_persistent_kernel<BN, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
        configured = true;
    }
    const int grid = total < num_sms ? total : num_sms;
    if (p.b_mn) umma_conv_gemm_persistent_kernel<BN, true><<<grid, PThreads, Cfg::kSmemBytes, st>>>(tmA, tmB, p, m_tiles, total);
    else umma_conv_gemm_persistent_kernel<BN, false><<<grid, PThreads, Cfg::kSmemBytes, st>>>(tmA, tmB, p, m_tiles, total);
    return cudaGetLastError();
}
template cudaError_t launch_persistent_bn<64>(const CUtensorMap&, const CUtensorMap&, const ConvGemmParams&, int, int, cudaStream_t, int);
template cudaError_t launch_persistent_bn<128>(const CUtensorMap&, const CUtensorMap&, const ConvGemmParams&, int, int, cudaStream_t, int);

}  // namespace rlr
