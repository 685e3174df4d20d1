// Split-K variant of the plain wgmma GEMM for small-M / deep-K problems (default for K >= 1024 with at most 16 output
// tiles, e.g. fc1 of the reference CNNs; RLR_SPLITK=0 turns it off).
//
// The first dense layer of the reference's FMNIST CNN is out[256][128] = x[256][9216] W[128][9216]^T: two 128 x 128 output tiles
// that each walk 144 k-blocks in sequence (pure pipeline latency on two of the GPU's SMs); at the runner's batch size 64 it is a
// single tile.  Here grid.z CTAs share a tile's k range, each accumulates its slice in registers and stores it into its slot of an
// fp32 partial buffer [splits][M][N]; `splitk_finish_kernel` then adds the slots in split order (the result does not depend on CTA
// scheduling), applies bias / ReLU and packs bf16.
// Same roles and operand layouts as gemm.cu (two consumer warpgroups of 64 rows each, one TMA producer warp; K-major SW128 operands).
#include <cuda.h>

#include "common.cuh"
#include "gemm.h"
#include "wgmma.cuh"

namespace rlr {

using namespace wg;

cudaError_t make_tmap_bf16(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                           const uint32_t* box, const uint32_t* elem_strides = nullptr);  // gemm.cu

namespace {

constexpr int SBM = 128, SBN = 128, SBK = 64, SThreads = 256 + 32, SStages = 4;
constexpr int SABytes = SBM * SBK * 2;
constexpr int SStageBytes = (SBM + SBN) * SBK * 2;          // 32 KB
constexpr int SSmem = SStages * SStageBytes + 1024 + 1024;

struct SplitKParams {
    int M, N, num_kb, kb_per_split;
    float* part;               // [splits][M][N] fp32 partial products, one slot per blockIdx.z
};

struct __align__(8) SKShared {
    uint64_t full[SStages];
    uint64_t empty[SStages];
};

__global__ void __launch_bounds__(SThreads, 1)
umma_gemm_splitk_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const SplitKParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    SKShared* sh = reinterpret_cast<SKShared*>(smem + SStages * SStageBytes);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tile_m = blockIdx.x, tile_n = blockIdx.y;
    const int kb0 = blockIdx.z * p.kb_per_split;
    const int kb1 = min(p.num_kb, kb0 + p.kb_per_split);
    const int nkb = kb1 - kb0;                               // >= 1 by construction of the grid

    if (warp == 8 && lane == 0) {
        prefetch_tmap(&tmA); prefetch_tmap(&tmB);
        for (int s = 0; s < SStages; ++s) { mbar_init(&sh->full[s], 1); mbar_init(&sh->empty[s], 8); }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();
    pdl_trigger();

    if (warp == 8) {
        if (lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int i = 0; i < nkb; ++i) {
                mbar_wait(&sh->empty[stage], phase ^ 1);
                uint8_t* sa = smem + stage * SStageBytes;
                mbar_expect_tx(&sh->full[stage], SStageBytes);
                tma_load_2d(&tmA, &sh->full[stage], sa, (kb0 + i) * SBK, tile_m * SBM);
                tma_load_2d(&tmB, &sh->full[stage], sa + SABytes, (kb0 + i) * SBK, tile_n * SBN);
                if (++stage == SStages) { stage = 0; phase ^= 1; }
            }
        }
    } else {
        const int wgi = threadIdx.x >> 7, t = threadIdx.x & 127;
        float acc[SBN / 2];
#pragma unroll
        for (int i = 0; i < SBN / 2; ++i) acc[i] = 0.f;
        int stage = 0;
        uint32_t phase = 0;
        consumer_mainloop<SBN, SStages, SStageBytes, SABytes, false>(acc, smem, sh->full, sh->empty, nkb, (uint32_t)wgi * 64 * 128, 0u,
                                                                     stage, phase, lane);
        const int row0 = tile_m * SBM + wgi * 64 + frag_row(t, 0);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = row0 + 8 * h;
            if (row >= p.M) continue;
#pragma unroll
            for (int j = 0; j < SBN / 8; ++j) {
                const int col = tile_n * SBN + frag_col(t, 4 * j);
                if (col < p.N)          // N % 8 == 0: whole pairs are valid or not
                    *reinterpret_cast<float2*>(p.part + ((size_t)blockIdx.z * p.M + row) * p.N + col) =
                        make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
            }
        }
    }
}

// out = bf16(act(sum of the split slots + bias))
// drop.thr != 0: dropout fused into this finishing pass (keep-mask of output element 4 q + i, common.cuh: dropout_keep8)
__global__ void __launch_bounds__(256) splitk_finish_kernel(const float* __restrict__ part, int splits, const float* __restrict__ bias,
                                                              __nv_bfloat16* __restrict__ out, long long n4, int N, int relu, DropSpec drop) {
    pdl_wait();
    pdl_trigger();
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n4; q += (long long)gridDim.x * blockDim.x) {
        float4 v = *reinterpret_cast<const float4*>(part + 4 * q);
        for (int z = 1; z < splits; ++z) {
            const float4 u = *reinterpret_cast<const float4*>(part + (size_t)z * 4 * n4 + 4 * q);
            v.x += u.x; v.y += u.y; v.z += u.z; v.w += u.w;
        }
        if (bias) {
            const int c = (int)((4 * q) % N);
            v.x += bias[c]; v.y += bias[c + 1]; v.z += bias[c + 2]; v.w += bias[c + 3];
        }
        if (relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
        if (drop.thr) {
            const uint32_t keep = dropout_keep8(drop, q >> 1) >> ((q & 1) * 4);       // elements 4 q .. 4 q + 3 of their group of eight
            v.x = (keep & 1) ? v.x * drop.scale : 0.f; v.y = (keep & 2) ? v.y * drop.scale : 0.f;
            v.z = (keep & 4) ? v.z * drop.scale : 0.f; v.w = (keep & 8) ? v.w * drop.scale : 0.f;
        }
        *reinterpret_cast<uint2*>(out + 4 * q) = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
    }
}

}  // namespace

// out[M][N] (bf16) = act(A[M][K] B[N][K]^T + bias).  K % 64 == 0, N % 8 == 0.  `ws` ([M][N] fp32, zero) is left untouched: the
// partial products live in scratch memory of the launch stream.
cudaError_t launch_gemm_splitk_bf16(const void* A, const void* B, void* out, float* ws, int M, int N, int K, const float* bias, int relu,
                                    int num_sms, cudaStream_t st, const DropSpec* drop) {
    if (K % SBK || N % 8 || M <= 0) return cudaErrorInvalidValue;
    static bool configured = false;
    if (!configured) {
        RLR_CUDA_CHECK(cudaFuncSetAttribute(umma_gemm_splitk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SSmem));
        configured = true;
    }
    CUtensorMap tmA, tmB;
    {
        const uint64_t d[2] = {(uint64_t)K, (uint64_t)M}, s[1] = {(uint64_t)K * 2};
        const uint32_t b[2] = {SBK, SBM};
        RLR_CUDA_CHECK(make_tmap_bf16(&tmA, A, 2, d, s, b));
    }
    {
        const uint64_t d[2] = {(uint64_t)K, (uint64_t)N}, s[1] = {(uint64_t)K * 2};
        const uint32_t b[2] = {SBK, SBN};
        RLR_CUDA_CHECK(make_tmap_bf16(&tmB, B, 2, d, s, b));
    }
    SplitKParams p{};
    p.M = M; p.N = N; p.num_kb = K / SBK;
    const int m_tiles = (M + SBM - 1) / SBM, n_tiles = (N + SBN - 1) / SBN;
    int splits = num_sms / (m_tiles * n_tiles);                 // one wave
    if (splits > p.num_kb / 2) splits = p.num_kb / 2;            // at least two k-blocks per CTA
    if (splits < 1) splits = 1;
    p.kb_per_split = (p.num_kb + splits - 1) / splits;
    splits = (p.num_kb + p.kb_per_split - 1) / p.kb_per_split;   // no empty CTA
    Scratch part((size_t)splits * M * N * sizeof(float), st);
    p.part = part.as<float>();
    RLR_CUDA_CHECK(launch_kernel(umma_gemm_splitk_kernel, dim3(m_tiles, n_tiles, splits), dim3(SThreads), (size_t)SSmem, st, tmA, tmB, p));
    const long long n4 = (long long)M * N / 4;
    long long blocks = (n4 + 255) / 256;
    if (blocks > num_sms * 4) blocks = num_sms * 4;
    return launch_kernel(splitk_finish_kernel, dim3((int)blocks), dim3(256), (size_t)0, st, (const float*)p.part, splits, bias,
                         reinterpret_cast<__nv_bfloat16*>(out), n4, N, relu, drop ? *drop : DropSpec{});
}

}  // namespace rlr
