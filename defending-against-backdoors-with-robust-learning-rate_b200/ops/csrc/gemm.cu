// wgmma / TMA GEMM and implicit-GEMM convolution for sm_90a (forward and data-gradient of every conv / linear layer of the
// model zoo; replaces the cuDNN / cuBLAS calls behind src/models.py:22-31,47-58 and autograd).
//
//   C[M, N] = A[M, K] * B[N, K]^T      bf16 operands (K-major, 128-byte swizzled tiles), fp32 accumulation in registers
//
// * plain mode: A is a row-major [M][K] matrix (linear layers).
// * conv mode : A is never materialised.  The activation tensor is NHWC; for filter tap (dy,dx) the 128 x 64 A tile of
//   k-block (tap, channel-block) is ONE 4-D TMA box {64 ch, TW, TH, TN} of the input at spatial offset (dy-pad, dx-pad);
//   out-of-bounds coordinates are zero-filled by the TMA unit, which implements the padding.  Strided (2x) convolutions
//   read a parity-split copy of the input ([4][N][H/2][W/2][C], see space_to_depth in norm.cu) through per-tap plane
//   offsets, so they use the same kernel.  The data-gradient of a 3x3/s1 conv is the same kernel on dY with the
//   tap-flipped, transposed filter.
// * warp-specialised CTA (320 threads): warps 0-7 = two consumer warpgroups, each issuing the m64 wgmma of its half of the
//   128-row tile and then running the epilogue on its accumulator registers (bias / ReLU / dropout, bf16 pack, staging through
//   shared memory for TMA tensor stores or fully coalesced 16-byte global stores, and per-channel sum / sum-of-squares
//   reductions that feed BatchNorm -- fused here so the conv output is not re-read for statistics); warp 8 = TMA producer,
//   warp 9 = second TMA producer for the B tiles.
// * 4-stage (BN=64) / 3-stage (BN=128) smem ring with full/empty mbarriers; a stage is released once the wgmma group that read
//   it has retired; two CTAs are resident per SM (<= 113 KB smem each) so one CTA's epilogue overlaps the other's mainloop.
#include <cuda.h>
#include <stdlib.h>

#include "common.cuh"
#include "gemm.h"
#include "stem_gather.cuh"
#include "wgmma.cuh"

namespace rlr {

using namespace wg;

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int kConsumers = 256;                 // two warpgroups
constexpr int kThreads = kConsumers + 64;       // + producer warps 8, 9
constexpr int kEpiThreads = kConsumers;

template <int BN, int kOcc = 2>
struct TileCfg {
    // two CTAs per SM: 4 x 24 KB / 3 x 32 KB ring; three CTAs per SM (kOcc = 3): 3 x 24 KB / 2 x 32 KB ring
    static constexpr int kStages = kOcc == 3 ? (BN == 64 ? 3 : 2) : (BN == 64 ? 4 : 3);
    static constexpr int kABytes = BM * BK * 2;
    static constexpr int kBBytes = BN * BK * 2;
    static constexpr int kStageBytes = kABytes + kBBytes;
    static constexpr int kPitch = BN * 2 + 16;                    // staging row pitch (bytes), conflict-free 16 B stores
    static constexpr int kStagingBytes = BM * kPitch;
    static constexpr int kRingBytes = kStages * kStageBytes;
    static_assert(kStagingBytes + 2 * BN * 4 <= kRingBytes, "staging aliases the operand ring");
    static constexpr int kTailBytes = BN == 128 ? 2048 : 1024;   // barriers, row index (640 B) + the tile's bias values (BN floats)
    static constexpr int kSmemBytes = kRingBytes + 1024 /*align slack*/ + kTailBytes;
};

struct __align__(8) SharedTail {
    uint64_t full[4];
    uint64_t empty[4];
    uint64_t pad0;
    uint32_t pad1;
    uint32_t pad2;
    int row_index[BM];   // global output row of each tile row, -1 = masked
};
static_assert(sizeof(SharedTail) <= 640, "the bias slice starts 640 bytes into the tail");

template <int BN, bool kStats, bool kBMN, int kOcc = 2>
__global__ void __launch_bounds__(kThreads, kOcc)
umma_conv_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmC,
                       const ConvGemmParams p) {
    using Cfg = TileCfg<BN, kOcc>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    SharedTail* tail = reinterpret_cast<SharedTail*>(smem + Cfg::kRingBytes);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tile_m = blockIdx.x, tile_n = blockIdx.y;
    long long* dbg = p.dbg ? p.dbg + ((size_t)blockIdx.y * gridDim.x + blockIdx.x) * 8 : nullptr;
    if (dbg && threadIdx.x == 0) { dbg[0] = (long long)gtimer(); uint32_t sm; asm volatile("mov.u32 %0, %%smid;" : "=r"(sm)); dbg[7] = sm; }

    // ---- tile origin -------------------------------------------------------------------------------------------------
    int n0 = 0, h0 = 0, w0 = 0;
    if (p.mode == 1) {
        const int tw_i = tile_m % p.tiles_w;
        const int th_i = (tile_m / p.tiles_w) % p.tiles_h;
        const int tn_i = tile_m / (p.tiles_w * p.tiles_h);
        w0 = tw_i * p.TW; h0 = th_i * p.TH; n0 = tn_i * p.TN;
    }

    if (warp == 8 && lane == 0) {
        prefetch_tmap(&tmA);
        prefetch_tmap(&tmB);
        if (p.tma_store) prefetch_tmap(&tmC);
        for (int s = 0; s < Cfg::kStages; ++s) { mbar_init(&tail->full[s], (p.split_prod || p.b_src) ? 2 : 1); mbar_init(&tail->empty[s], 8); }
        fence_barrier_init();
    }
    if (threadIdx.x < BM) {   // resolve the global output row of every tile row once
        const int r = threadIdx.x;
        int gi;
        if (p.mode == 1) {
            const int tw = r % p.TW, th = (r / p.TW) % p.TH, tn = r / (p.TW * p.TH);
            const int w = w0 + tw, h = h0 + th, n = n0 + tn;
            gi = (w < p.Wo && h < p.Ho && n < p.NB) ? ((n * p.OutH + h * p.out_stride + p.out_ph) * p.OutW + w * p.out_stride + p.out_pw) : -1;
        } else {
            gi = tile_m * BM + r;
            if (gi >= p.M) gi = -1;
        }
        tail->row_index[r] = gi;
    }
    __syncthreads();
    pdl_wait();        // everything above touched only parameters and shared memory
    pdl_trigger();
    if (dbg && threadIdx.x == 0) dbg[1] = (long long)gtimer();

    if (warp == 8) {
        // ================================ TMA producer =====================================================================
        if (p.b_src) {
            // stem GEMM (ONE k-block, mode 0): the A tile is requested first, then -- while it is in flight -- the whole warp builds the
            // B tile from the un-padded filter; full[0] takes two arrivals (the TMA transaction and this warp).
            if (lane == 0) {
                mbar_expect_tx(&tail->full[0], Cfg::kABytes);
                tma_load_2d(&tmA, &tail->full[0], smem, 0, tile_m * BM);
            }
            stem_gather_b(p, smem + Cfg::kABytes, BN, tile_n, lane);               // stage 0's B slot
            if (lane == 0) mbar_arrive(&tail->full[0]);
        } else if (lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int kb = 0; kb < p.num_kb; ++kb) {
                mbar_wait(&tail->empty[stage], phase ^ 1);
                uint8_t* sa = smem + stage * Cfg::kStageBytes;
                uint8_t* sb = sa + Cfg::kABytes;
                mbar_expect_tx(&tail->full[stage], p.split_prod ? Cfg::kABytes : Cfg::kStageBytes);
                if (dbg && kb == 0) dbg[2] = (long long)gtimer();
                if (p.mode == 1) {
                    const int tap = kb / p.cblocks, cb = kb - tap * p.cblocks;
                    tma_load_4d(&tmA, &tail->full[stage], sa, cb * BK, w0 * p.in_stride + p.dw[tap], h0 * p.in_stride + p.dh[tap],
                                n0 + p.dn[tap]);
                } else {
                    tma_load_2d(&tmA, &tail->full[stage], sa, kb * BK, tile_m * BM);
                }
                if (p.split_prod) {
                    // B tile loaded by the second producer (warp 9)
                } else if (kBMN) {
                    // data gradient: B[k = co][n = ci] is a 64 x 64 box of the ORIGINAL filter W[co][tap][ci] (ci contiguous ->
                    // MN-major operand); one box per 64-wide ci group.  No transposed filter copy is ever materialised.
                    const int tap = kb / p.cblocks, cb = kb - tap * p.cblocks;
                    for (int g = 0; g < BN / 64; ++g)
                        tma_load_2d(&tmB, &tail->full[stage], sb + g * 8192, p.wtap[tap] * p.wcols + tile_n * BN + g * 64, cb * BK);
                } else {
                    tma_load_2d(&tmB, &tail->full[stage], sb, kb * BK, tile_n * BN);
                }
                if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
            }
        }
    } else if (warp == 9) {
        if (p.split_prod && lane == 0) {
            // second TMA producer: the B (filter) tiles of every k-block -- an independent request stream next to warp 8's A stream
            int stage = 0;
            uint32_t phase = 0;
            for (int kb = 0; kb < p.num_kb; ++kb) {
                mbar_wait(&tail->empty[stage], phase ^ 1);
                uint8_t* sb = smem + stage * Cfg::kStageBytes + Cfg::kABytes;
                mbar_expect_tx(&tail->full[stage], Cfg::kBBytes);
                if (kBMN) {
                    const int tap = kb / p.cblocks, cb = kb - tap * p.cblocks;
                    for (int g = 0; g < BN / 64; ++g)
                        tma_load_2d(&tmB, &tail->full[stage], sb + g * 8192, p.wtap[tap] * p.wcols + tile_n * BN + g * 64, cb * BK);
                } else {
                    tma_load_2d(&tmB, &tail->full[stage], sb, kb * BK, tile_n * BN);
                }
                if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
            }
        }
    } else {
        // ================================ consumers: 2 warpgroups x 64 rows ==================================================
        const int et = threadIdx.x;                      // 0..255
        const int wgi = et >> 7, t = et & 127;
        const int col0 = tile_n * BN;
        const bool has_bias = !kBMN && p.bias != nullptr;   // data gradients (MN-major B) never carry a bias
        // the tile's bias values go to shared memory while the main loop runs
        float* bias_w = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(tail) + 640);
        if (has_bias)
            for (int i = et; i < BN; i += kEpiThreads) bias_w[i] = (col0 + i < p.N) ? p.bias[col0 + i] : 0.f;
        float acc[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
        {
            int stage = 0;
            uint32_t phase = 0;
            consumer_mainloop<BN, Cfg::kStages, Cfg::kStageBytes, Cfg::kABytes, kBMN>(
                acc, smem, tail->full, tail->empty, p.num_kb, (uint32_t)wgi * 64 * 128, p.b_src ? smem_u32(smem + Cfg::kABytes) : 0u,
                stage, phase, lane);
        }
        if (dbg && et == 0) dbg[4] = (long long)gtimer();
        named_bar(1, kEpiThreads);                       // both warpgroups are done with the ring (and the bias slice is written)
        if (dbg && et == 0) dbg[5] = (long long)gtimer();
        const float* bias_s = bias_w;
        uint8_t* staging = smem;                         // operand ring is idle now: reuse it
        float* red = reinterpret_cast<float*>(staging + Cfg::kStagingBytes);   // [2][BN] per-tile column sums
        const int r0 = wgi * 64 + frag_row(t, 0);        // this thread's two tile rows: r0, r0 + 8
        int gi_r[2];
        gi_r[0] = tail->row_index[r0];
        gi_r[1] = tail->row_index[r0 + 8];
        if (kStats) {
            for (int i = et; i < 2 * BN; i += kEpiThreads) red[i] = 0.f;
            named_bar(1, kEpiThreads);
        }
        const bool tma_out = !kStats && p.tma_store;
        // registers -> bias / ReLU / dropout / bf16 pack -> staging tile.
        // Staging layout: TMA-store path = 128-byte-swizzled [64-channel group][128 rows][128 B] tiles (what cp.async.bulk.tensor reads);
        //                 accumulate / statistics path = padded row pitch for the coalesced read-modify-write stores below.
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
            const int c = frag_col(t, 4 * j);            // even column of this thread inside the 8-column group j
            float s1[2] = {0.f, 0.f}, s2[2] = {0.f, 0.f};
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = r0 + 8 * h, gi_row = gi_r[h];
                float a = acc[4 * j + 2 * h], b = acc[4 * j + 2 * h + 1];
                if (has_bias) { a += bias_s[c]; b += bias_s[c + 1]; }
                if (p.relu) { a = fmaxf(a, 0.f); b = fmaxf(b, 0.f); }
                if (p.drop.thr) {   // fused dropout (linear layers): keep-mask of the 8-column group of this row
                    const uint32_t keep8 = dropout_keep8(p.drop, ((long long)(gi_row < 0 ? 0 : gi_row) * p.ldc + col0 + 8 * j) >> 3);
                    a = (keep8 >> (c & 7) & 1) ? a * p.drop.scale : 0.f;
                    b = (keep8 >> ((c & 7) + 1) & 1) ? b * p.drop.scale : 0.f;
                }
                const uint32_t packed = pack_bf16x2(a, b);
                if (kStats && gi_row >= 0) {   // statistics of the bf16-rounded values BatchNorm will read back; masked rows count as zero
                    const float2 rq = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&packed));
                    s1[0] += rq.x; s1[1] += rq.y; s2[0] += rq.x * rq.x; s2[1] += rq.y * rq.y;
                }
                if (tma_out)
                    *reinterpret_cast<uint32_t*>(staging + (c >> 6) * (BM * 128) + row * 128 + ((((c & 63) >> 3) ^ (row & 7)) << 4) + (c & 7) * 2) = packed;
                else
                    *reinterpret_cast<uint32_t*>(staging + row * Cfg::kPitch + c * 2) = packed;
            }
            if (kStats) {   // column sums over the 8 lanes that share this thread's columns, then the warps meet in shared memory
#pragma unroll
                for (int o = 4; o < 32; o <<= 1)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        s1[e] += __shfl_xor_sync(0xffffffffu, s1[e], o);
                        s2[e] += __shfl_xor_sync(0xffffffffu, s2[e], o);
                    }
                if (lane < 4) {
                    atomicAdd(&red[c], s1[0]); atomicAdd(&red[c + 1], s1[1]);
                    atomicAdd(&red[BN + c], s2[0]); atomicAdd(&red[BN + c + 1], s2[1]);
                }
            }
        }
        if (tma_out) {
            fence_proxy_async_smem();                        // generic-proxy staging writes -> TMA (async proxy) reads
            named_bar(1, kEpiThreads);
            if (dbg && et == 0) dbg[6] = (long long)gtimer();
            if (et == 0) {
                // one TMA tensor store per 64-channel group: the box is the tile's pixel box of the NHWC output (rows / columns outside
                // the tensor are clipped by the TMA unit) -- no per-thread address arithmetic, fully coalesced, asynchronous
#pragma unroll
                for (int g = 0; g < BN / 64; ++g) {
                    if (col0 + g * 64 >= p.N) break;
                    if (p.mode == 1) tma_store_4d(&tmC, staging + g * (BM * 128), col0 + g * 64, w0, h0, n0);
                    else tma_store_2d(&tmC, staging + g * (BM * 128), col0 + g * 64, tile_m * BM);
                }
                tma_store_commit();
            }
            if (p.stats) {
                // BatchNorm statistics of this tile while the TMA unit drains it: kEpiThreads / BN threads per output column, each walking
                // the staged bf16 tile -- exactly the values BatchNorm will read back -- down its share of the rows (masked rows skipped);
                // ONE pair of global reductions per thread, spread over the stat_slots partial buffers
                constexpr int kPerCol = kEpiThreads / BN, kRows = BM / kPerCol;
                const int c = et % BN;
                const int r_lo = (et / BN) * kRows, r_hi = r_lo + kRows;
                const uint8_t* colp = staging + (c >> 6) * (BM * 128) + (c & 7) * 2;
                const int chunk = (c & 63) >> 3;
                float s1 = 0.f, s2 = 0.f;
#pragma unroll 8
                for (int r = r_lo; r < r_hi; ++r) {
                    if (tail->row_index[r] < 0) continue;
                    const float v = __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(colp + r * 128 + ((chunk ^ (r & 7)) << 4)));
                    s1 += v; s2 += v * v;
                }
                if (col0 + c < p.N) {
                    float* dst = p.stats + (size_t)(blockIdx.x % p.stat_slots) * 2 * p.N + col0 + c;
                    atomicAdd(dst, s1);
                    atomicAdd(dst + p.N, s2);
                }
            }
            if (et == 0) tma_store_wait_read();
        } else {
        named_bar(1, kEpiThreads);                       // staging tile complete
        if (dbg && et == 0) dbg[6] = (long long)gtimer();
        // ---- coalesced 16-byte stores (optionally accumulating into the existing output) ----
        constexpr int kChunks = BN * 2 / 16;             // 16 B chunks per row
        __nv_bfloat16* out = reinterpret_cast<__nv_bfloat16*>(p.out);
        constexpr int kIters = BM * kChunks / kEpiThreads;   // 4 (BN=64) / 8 (BN=128) chunks per thread
        constexpr int kBatch = kIters < 8 ? kIters : 8;
#pragma unroll
        for (int it0 = 0; it0 < kIters; it0 += kBatch) {
            uint4 oldv[kBatch];
            if (p.accumulate) {                             // batch the read-modify-write loads: one latency per batch
#pragma unroll
                for (int j = 0; j < kBatch; ++j) {
                    const int idx = et + (it0 + j) * kEpiThreads, r = idx / kChunks, ch = idx - r * kChunks;
                    const int gi = tail->row_index[r];
                    oldv[j] = make_uint4(0, 0, 0, 0);
                    if (gi >= 0 && col0 + ch * 8 < p.N) oldv[j] = *reinterpret_cast<const uint4*>(out + (size_t)gi * p.ldc + col0 + ch * 8);
                }
            }
#pragma unroll
            for (int j = 0; j < kBatch; ++j) {
                const int idx = et + (it0 + j) * kEpiThreads, r = idx / kChunks, ch = idx - r * kChunks;
                const int gi = tail->row_index[r];
                if (gi < 0 || col0 + ch * 8 >= p.N) continue;     // masked row / column chunk beyond Cout
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
        // ---- per-channel statistics: one global reduction per column and tile, spread over kStatSlots partial buffers ----
        if (kStats) {
            named_bar(1, kEpiThreads);                   // (also orders the smem atomics above; the bar before the stores did too)
            for (int i = et; i < 2 * BN; i += kEpiThreads)
                if (col0 + (i % BN) < p.N)
                    atomicAdd(p.stats + (size_t)(blockIdx.x % kStatSlots) * 2 * p.N + (i < BN ? 0 : p.N) + col0 + (i % BN), red[i]);
        }
        }   // !tma_out
    }
}

// =====================================================================================================================
// host side: tensor maps + launch
// =====================================================================================================================
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess || !f) return nullptr;
        fn = reinterpret_cast<EncodeTiledFn>(f);
    }
    return fn;
}

// bf16 tensor of `rank` dims (innermost first), 128-byte swizzle, zero fill out of bounds.
// `elem_strides` (optional, per dimension, 1..8): traversal stride -- the box then covers box[i] * stride elements of dimension i
// and TMA loads every stride-th one (box[i] elements land in shared memory).  Used for stride-2 convolutions without a
// parity-split copy of the input.
cudaError_t make_tmap_bf16(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                           const uint32_t* box, const uint32_t* elem_strides = nullptr) {
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) return cudaErrorNotSupported;
    cuuint64_t gd[5], gs[4];
    cuuint32_t bx[5], es[5];
    for (int i = 0; i < rank; ++i) {
        gd[i] = dims[i];
        es[i] = elem_strides ? elem_strides[i] : 1;
        bx[i] = box[i] * es[i];       // "to load N elements along dimension i, boxDim[i] must be N * elementStrides[i]"
        if (bx[i] > 256 || es[i] < 1 || es[i] > 8) return cudaErrorInvalidValue;
    }
    for (int i = 0; i + 1 < rank; ++i) gs[i] = strides_bytes[i];
    const CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base), gd, gs, bx, es,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? cudaSuccess : cudaErrorInvalidValue;
}

// gemm_persistent.cu (opt-in, RLR_PERSISTENT_CONV=1): one CTA per SM looping over tiles, operand ring running ahead of the epilogue
template <int BN>
cudaError_t launch_persistent_bn(const CUtensorMap& tmA, const CUtensorMap& tmB, const ConvGemmParams& p, int m_tiles, int num_sms,
                                 cudaStream_t st, int occ = 1);

// 0: two CTAs per SM for every tile | 1 (default): three for the 64-wide tile.  Levels above 1 select 1: three 320-thread CTAs of the
// 128-wide tile would need 64 accumulator registers of a 64-register budget per thread.  -1: take RLR_CONV_OCC3 from the environment on first use.
static int g_occ3 = -1;
void set_conv_occ3(int level) { g_occ3 = level < 0 ? 0 : (level > 1 ? 1 : level); }
static int conv_occ3() {
    if (g_occ3 < 0) { const char* e = getenv("RLR_CONV_OCC3"); set_conv_occ3(e ? atoi(e) : 1); }
    return g_occ3;
}

// default (RLR_CONV_OCC3=0 disables): 64-wide tiles with a 3-stage ring at three CTAs per SM (three TMA producers / MMA issue threads per SM)
template <int BN>
static cudaError_t launch_bn_occ3(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmC, const ConvGemmParams& p, int m_tiles,
                                  cudaStream_t st) {
    using Cfg = TileCfg<BN, 3>;
    static bool configured = false;
    if (!configured) {
        RLR_CUDA_CHECK(cudaFuncSetAttribute(umma_conv_gemm_kernel<BN, false, false, 3>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
        RLR_CUDA_CHECK(cudaFuncSetAttribute(umma_conv_gemm_kernel<BN, false, true, 3>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
        configured = true;
    }
    dim3 grid(m_tiles, (p.N + BN - 1) / BN);
    if (p.b_mn) return launch_kernel(umma_conv_gemm_kernel<BN, false, true, 3>, grid, dim3(kThreads), Cfg::kSmemBytes, st, tmA, tmB, tmC, p);
    return launch_kernel(umma_conv_gemm_kernel<BN, false, false, 3>, grid, dim3(kThreads), Cfg::kSmemBytes, st, tmA, tmB, tmC, p);
}

static int sm_count() {
    static const int sms = [] {
        int dev = 0, n = 0;
        if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 132;
        return n;
    }();
    return sms;
}

static int g_persistent = -1;   // -1: take RLR_PERSISTENT_CONV from the environment on first use
void set_persistent_conv(int on) { g_persistent = on ? 1 : 0; }

static int persistent_sms() {
    if (g_persistent < 0) { const char* e = getenv("RLR_PERSISTENT_CONV"); g_persistent = (e && atoi(e) > 0) ? 1 : 0; }
    if (!g_persistent) return 0;
    static const int sms = [] {
        int dev = 0, n = 0;
        if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 0;
        return n;
    }();
    return sms;
}

static int g_split_prod = -1;
void set_conv_split_producer(int on) { g_split_prod = on ? 1 : 0; }
static long long* g_trace = nullptr;
void set_conv_trace(long long* buf) { g_trace = buf; }
long long* conv_trace_buf() { return g_trace; }

static int g_tma_store = -1;    // epilogue through TMA tensor stores (default on; RLR_TMA_STORE=0 restores the per-thread coalesced stores)
void set_conv_tma_store(int on) { g_tma_store = on ? 1 : 0; }
static bool tma_store_enabled() {
    if (g_tma_store < 0) { const char* e = getenv("RLR_TMA_STORE"); g_tma_store = (e && atoi(e) == 0) ? 0 : 1; }
    return g_tma_store != 0;
}
// Output tensor map for the TMA-store epilogue: the [M][N] matrix (plain) or the NHWC image grid the tile's pixel box addresses
// (conv; a strided data-gradient plane is expressed through doubled global strides and an offset base).  64-channel (128-byte) boxes.
static cudaError_t make_out_tmap(CUtensorMap* tmC, const ConvGemmParams& p) {
    if (p.ldc % 8) return cudaErrorInvalidValue;
    if (p.mode == 1) {
        const uint64_t d[4] = {(uint64_t)p.N, (uint64_t)p.Wo, (uint64_t)p.Ho, (uint64_t)p.NB};
        const uint64_t s[3] = {(uint64_t)p.out_stride * p.ldc * 2, (uint64_t)p.out_stride * p.OutW * p.ldc * 2, (uint64_t)p.OutH * p.OutW * p.ldc * 2};
        const uint32_t b[4] = {64, (uint32_t)p.TW, (uint32_t)p.TH, (uint32_t)p.TN};
        const char* base = reinterpret_cast<const char*>(p.out) + ((size_t)p.out_ph * p.OutW + p.out_pw) * p.ldc * 2;
        return make_tmap_bf16(tmC, base, 4, d, s, b);
    }
    const uint64_t d[2] = {(uint64_t)p.N, (uint64_t)p.M}, s[1] = {(uint64_t)p.ldc * 2};
    const uint32_t b[2] = {64, BM};
    return make_tmap_bf16(tmC, p.out, 2, d, s, b);
}

template <int BN>
static cudaError_t launch_bn(const CUtensorMap& tmA, const CUtensorMap& tmB, const ConvGemmParams& p_in, int m_tiles, cudaStream_t st) {
    using Cfg = TileCfg<BN>;
    ConvGemmParams p = p_in;
    p.dbg = g_trace;
    CUtensorMap tmC = tmA;                                       // dummy unless the TMA-store epilogue applies
    {   // slots used by the TMA-store epilogue's statistics (RLR_EPI_STAT_SLOTS; python reads the same variable for the prefix it reduces)
        static const int epi_slots = [] { const char* e = getenv("RLR_EPI_STAT_SLOTS"); int v = e ? atoi(e) : 2; return v < 1 ? 1 : (v > kStatSlots ? kStatSlots : v); }();
        p.stat_slots = epi_slots;
    }
    p.tma_store = 0;
    if (tma_store_enabled() && !p.accumulate && ((reinterpret_cast<uintptr_t>(p.out) & 15) == 0) && make_out_tmap(&tmC, p) == cudaSuccess)
        p.tma_store = 1;
    if (g_split_prod < 0) { const char* e = getenv("RLR_SPLIT_PRODUCER"); g_split_prod = (e && atoi(e) == 0) ? 0 : 1; }   // default on
    p.split_prod = (g_split_prod && !p.b_src) ? 1 : 0;
    if (p.b_src && !p.stats && p.N <= BN) {
        // stem GEMM: ONE k-block per output tile, so a one-tile CTA is all fixed cost (set-up, the filter gather, a lone TMA round trip).
        // The persistent kernel builds the B tile once per SM, streams the A tiles through its ring and overlaps every tile's epilogue
        // with the next tile's operand loads.  RLR_STEM_PERSISTENT=0 restores the one-tile-per-CTA launch.
        // (RLR_STEM_PERSISTENT=1: one CTA per SM with the deep ring; default 2: two CTAs per SM, 3-stage rings -- the tiles are epilogue bound)
        static const int stem_persistent = [] { const char* e = getenv("RLR_STEM_PERSISTENT"); return e ? atoi(e) : 2; }();
        if (stem_persistent && m_tiles >= 2 * sm_count())
            return launch_persistent_bn<BN>(tmA, tmB, p, m_tiles, sm_count(), st, stem_persistent == 2 ? 2 : 1);
    }
    if (!p.stats && !p.b_src && persistent_sms() > 0 && m_tiles * ((p.N + BN - 1) / BN) > persistent_sms())
        return launch_persistent_bn<BN>(tmA, tmB, p, m_tiles, persistent_sms(), st);
    // statistics ride on the TMA-store epilogue of the plain instantiation (runtime p.stats); without TMA stores: the kStats variant below
    if constexpr (BN == 64)
        if ((!p.stats || p.tma_store) && conv_occ3() >= 1) return launch_bn_occ3<BN>(tmA, tmB, tmC, p, m_tiles, st);
    static bool configured = false;
    if (!configured) {
        RLR_CUDA_CHECK(cudaFuncSetAttribute(umma_conv_gemm_kernel<BN, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
        RLR_CUDA_CHECK(cudaFuncSetAttribute(umma_conv_gemm_kernel<BN, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
        RLR_CUDA_CHECK(cudaFuncSetAttribute(umma_conv_gemm_kernel<BN, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
        configured = true;
    }
    dim3 grid(m_tiles, (p.N + BN - 1) / BN);
    if (p.b_mn) return launch_kernel(umma_conv_gemm_kernel<BN, false, true>, grid, dim3(kThreads), Cfg::kSmemBytes, st, tmA, tmB, tmC, p);
    if (p.stats && !p.tma_store) return launch_kernel(umma_conv_gemm_kernel<BN, true, false>, grid, dim3(kThreads), Cfg::kSmemBytes, st, tmA, tmB, tmC, p);
    return launch_kernel(umma_conv_gemm_kernel<BN, false, false>, grid, dim3(kThreads), Cfg::kSmemBytes, st, tmA, tmB, tmC, p);
}

static int pick_bn(int N) { return (N % 128 == 0) ? 128 : 64; }

// Plain GEMM: out[M][ldc] (bf16) = A[M][K] * B[N][K]^T (+bias)(relu).  K % 64 == 0, N % 64 == 0.
cudaError_t launch_gemm_bf16(const void* A, const void* B, void* out, int M, int N, int K, int lda, int ldb, int ldc,
                             const float* bias, int relu, int accumulate, float* stats, cudaStream_t st, const DropSpec* drop) {
    if (K % BK || N % 8 || M <= 0) return cudaErrorInvalidValue;
    if (drop && drop->thr && (accumulate || stats || ldc % 8)) return cudaErrorInvalidValue;
    const int m_tiles = (M + BM - 1) / BM;
    int bn = pick_bn(N);
    {   // opt-in (RLR_GEMM_SMALL_BN64=1): small-batch linear layers (M = 256: two M tiles) get twice the CTAs
        static const int small64 = [] { const char* e = getenv("RLR_GEMM_SMALL_BN64"); return e ? atoi(e) : 0; }();
        if (small64 && bn == 128 && m_tiles * (N / 128) < sm_count()) bn = 64;
    }
    CUtensorMap tmA, tmB;
    {
        const uint64_t d[2] = {(uint64_t)K, (uint64_t)M}, s[1] = {(uint64_t)lda * 2};
        const uint32_t b[2] = {BK, BM};
        RLR_CUDA_CHECK(make_tmap_bf16(&tmA, A, 2, d, s, b));
    }
    {
        const uint64_t d[2] = {(uint64_t)K, (uint64_t)N}, s[1] = {(uint64_t)ldb * 2};
        const uint32_t b[2] = {BK, (uint32_t)bn};
        RLR_CUDA_CHECK(make_tmap_bf16(&tmB, B, 2, d, s, b));
    }
    ConvGemmParams p{};
    p.M = M; p.N = N; p.num_kb = K / BK; p.mode = 0; p.in_stride = 1; p.out_stride = 1;
    p.out = out; p.ldc = ldc; p.bias = bias; p.stats = stats; p.relu = relu; p.accumulate = accumulate;
    if (drop && drop->thr) p.drop = *drop;      // fused dropout lives in the epilogue
    return bn == 128 ? launch_bn<128>(tmA, tmB, p, m_tiles, st) : launch_bn<64>(tmA, tmB, p, m_tiles, st);
}

// Stem GEMM (tiny-K first layer): A is the im2col matrix [M][64] (gather_im2col), W the un-padded bf16 filter [N][ldw] with kvalid <= 64
// valid columns, read by the producer warp (ConvGemmParams::b_src) -- from the trainer's own shadow, or straight from the multicast
// broadcast buffer behind the ready flags.
cudaError_t launch_stem_gemm_bf16(const void* A, const void* W, void* out, int M, int N, int kvalid, int ldw, const float* bias, int relu,
                                  float* stats, const uint32_t* wait_flags, int wait_lo, int wait_hi, const uint32_t* wait_epoch,
                                  cudaStream_t st) {
    if (N % 8 || M <= 0 || kvalid < 1 || kvalid > BK || ldw < kvalid) return cudaErrorInvalidValue;
    if (wait_flags && (!wait_epoch || wait_lo > wait_hi || wait_lo < 0)) return cudaErrorInvalidValue;
    const int m_tiles = (M + BM - 1) / BM;
    const int bn = pick_bn(N);
    CUtensorMap tmA;
    {
        const uint64_t d[2] = {(uint64_t)BK, (uint64_t)M}, s[1] = {(uint64_t)BK * 2};
        const uint32_t b[2] = {BK, BM};
        RLR_CUDA_CHECK(make_tmap_bf16(&tmA, A, 2, d, s, b));
    }
    ConvGemmParams p{};
    p.M = M; p.N = N; p.num_kb = 1; p.mode = 0; p.in_stride = 1; p.out_stride = 1;
    p.out = out; p.ldc = N; p.bias = bias; p.stats = stats; p.relu = relu; p.accumulate = 0;
    p.b_src = reinterpret_cast<const __nv_bfloat16*>(W); p.b_ld = ldw; p.b_kvalid = kvalid;
    p.wait_flags = wait_flags; p.wait_lo = wait_lo; p.wait_hi = wait_hi; p.wait_epoch = wait_epoch;
    return bn == 128 ? launch_bn<128>(tmA, tmA, p, m_tiles, st) : launch_bn<64>(tmA, tmA, p, m_tiles, st);   // tmB unused: B is gathered by the warp
}

static int pow2_ceil(int x) { int p = 1; while (p < x) p <<= 1; return p; }

// Implicit-GEMM convolution.  `x` is [planes*NB][Hin][Win][Cin] bf16 NHWC (planes = 1, or 4 parity planes for stride 2),
// `w` is [Cout][ntaps*Cin] bf16 (tap-major K), out is [NB*Ho*Wo][ldc] bf16.  Taps are given as input offsets.
cudaError_t launch_conv_bf16(const void* x, const void* w, void* out, int NB, int planes, int Hin, int Win, int Cin, int Ho, int Wo,
                             int Cout, int ldc, int ntaps, const int* dh, const int* dw, const int* dplane, const float* bias,
                             int relu, int accumulate, float* stats, cudaStream_t st, const int* wtap, int w_taps_total,
                             int in_stride, int out_stride, int out_ph, int out_pw) {
    if (Cin % BK || Cout % 8 || ntaps < 1 || ntaps > 9) return cudaErrorInvalidValue;
    if (in_stride < 1 || in_stride > 2 || out_stride < 1 || out_stride > 2 || (in_stride > 1 && planes != 1)) return cudaErrorInvalidValue;
    if (wtap && (stats || Cout % 64)) return cudaErrorInvalidValue;   // MN-major filter path: whole 64-wide ci groups, no statistics
    int bn = pick_bn(Cout);
    ConvGemmParams p{};
    {   // few M tiles (deep layers at small batch / 4x4 maps): prefer the 64-wide tile so the grid covers all SMs
        static const int small_bn64 = [] { const char* e = getenv("RLR_SMALL_BN64"); return e ? atoi(e) : 1; }();
        const long long px = (long long)NB * Ho * Wo;
        if (small_bn64 && bn == 128 && ((px + BM - 1) / BM) * (Cout / 128) < sm_count()) bn = 64;
    }
    // output tile: TW x TH x TN = 128 output pixels, TW/TH powers of two covering the image
    int TW = pow2_ceil(Wo); if (TW > BM) TW = BM;
    int TH = pow2_ceil(Ho); if (TW * TH > BM) TH = BM / TW;
    int TN = BM / (TW * TH);
    p.TW = TW; p.TH = TH; p.TN = TN;
    p.tiles_w = (Wo + TW - 1) / TW; p.tiles_h = (Ho + TH - 1) / TH;
    const int tiles_n = (NB + TN - 1) / TN;
    const int m_tiles = p.tiles_w * p.tiles_h * tiles_n;
    p.M = NB * Ho * Wo; p.N = Cout; p.mode = 1; p.cblocks = Cin / BK; p.num_kb = ntaps * p.cblocks; p.ntaps = ntaps;
    p.Ho = Ho; p.Wo = Wo; p.NB = NB;
    // Ho x Wo is the logical output grid; it is stored into an image of (out_stride * Ho) x (out_stride * Wo) pixels at parity
    // (out_ph, out_pw) -- stride-2 data gradients write their four parity planes straight into dX
    p.in_stride = in_stride; p.out_stride = out_stride; p.out_ph = out_ph; p.out_pw = out_pw; p.OutH = Ho * out_stride; p.OutW = Wo * out_stride;
    for (int t = 0; t < ntaps; ++t) { p.dh[t] = (int8_t)dh[t]; p.dw[t] = (int8_t)dw[t]; p.dn[t] = dplane[t] * NB; }
    p.out = out; p.ldc = ldc; p.bias = bias; p.stats = stats; p.relu = relu; p.accumulate = accumulate;
    CUtensorMap tmA, tmB;
    {
        const uint64_t d[4] = {(uint64_t)Cin, (uint64_t)Win, (uint64_t)Hin, (uint64_t)planes * NB};
        const uint64_t s[3] = {(uint64_t)Cin * 2, (uint64_t)Win * Cin * 2, (uint64_t)Hin * Win * Cin * 2};
        const uint32_t b[4] = {BK, (uint32_t)TW, (uint32_t)TH, (uint32_t)TN};
        const uint32_t es[4] = {1, (uint32_t)in_stride, (uint32_t)in_stride, 1};
        RLR_CUDA_CHECK(make_tmap_bf16(&tmA, x, 4, d, s, b, in_stride > 1 ? es : nullptr));
    }
    if (wtap) {
        // data gradient on the un-transposed filter: w is the forward filter [K = Cin of this call][w_taps_total * Cout of this call]
        if (bias) return cudaErrorInvalidValue;                 // the MN-major (data-gradient) kernels are compiled without the bias path
        p.b_mn = 1; p.wcols = Cout;
        for (int t = 0; t < ntaps; ++t) p.wtap[t] = wtap[t];
        const uint64_t cols = (uint64_t)w_taps_total * Cout;
        const uint64_t d[2] = {cols, (uint64_t)Cin}, s[1] = {cols * 2};
        const uint32_t b[2] = {64, BK};
        RLR_CUDA_CHECK(make_tmap_bf16(&tmB, w, 2, d, s, b));
    } else {
        const uint64_t K = (uint64_t)ntaps * Cin;
        const uint64_t d[2] = {K, (uint64_t)Cout}, s[1] = {K * 2};
        const uint32_t b[2] = {BK, (uint32_t)bn};
        RLR_CUDA_CHECK(make_tmap_bf16(&tmB, w, 2, d, s, b));
    }
    return bn == 128 ? launch_bn<128>(tmA, tmB, p, m_tiles, st) : launch_bn<64>(tmA, tmB, p, m_tiles, st);
}

}  // namespace rlr
