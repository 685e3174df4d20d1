// Pairwise squared distances of the participants' updates for Krum / Multi-Krum selection (Blanchard et al. 2017):
//   D[i][j] = sum_c (x_i[c] - x_j[c])^2,  x_k = w_k (no clipping: w_global cancels, so w_i - w_j is formed directly -- one fp32
//   rounding per coordinate, and bitwise-identical participants are exactly 0 apart) or x_k = (w_k - w_global) * s_k (server clipping).
// The differences are formed per coordinate; a Gram formulation (|a|^2 + |b|^2 - 2 a.b) would cancel catastrophically exactly where
// Krum matters, between near-duplicate updates.
//
// Work decomposition:
//   grid.x  the upper triangle of 64 x 64 participant tiles (a tile pairs 64 "row" with 64 "column" participants; a diagonal tile
//           pairs a set with itself, so with K <= 64 every vector is read once),
//   grid.y  coordinate splits, sized so the grid covers about two waves (one wave on the fused multi-GPU path, where every CTA has to
//           be resident while it waits for the cross-GPU barrier-in) and the workspace stays <= kMaxWorkspace bytes.
// A CTA streams its coordinate range in chunks: the tile's participants are staged in shared memory with 16-byte loads, and each thread
// accumulates a 4 x 4 register block of pairs in fp32 over (its share of) one chunk -- at most 256 coordinates -- and folds it into
// fp64.  Small tiles give each pair block several coordinate lanes; the lanes are added in lane order at the end.  Every (tile, split)
// CTA writes its tile, mirrored, to its split's [K][K] workspace slot and launch_ordered_sum adds the slots in split order.  No atomics:
// the matrix is bitwise identical from run to run.
//
// The same kernel with GRAM = true is FLAME's Gram pass: G[i][j] = sum_c Δi[c] Δj[c] with Δk = w_k - w_global formed per coordinate in
// fp32 while staging, one FMA per pair and coordinate, and the diagonal (the squared update norms) kept.  Cosines are taken from G
// directly: deriving them from D through (|a|^2 + |b|^2 - D) / 2 cancels near cos = 0, where honest high-dimensional updates sit.
// With ROWS = true as well it is FoolsGold's Gram pass over the candidates' history rows, staged as they are (no w_global).
#include "common.cuh"
#include "kernels.h"

namespace rlr {

constexpr int kDistThreads = 256;
constexpr int kDistTile = 64;                           // participants per tile side
constexpr int kDistStage = 16384;                       // fp32 values per chunk (staged participants x chunk coordinates)
constexpr int kDistStageFloats = kDistStage + 4 * 2 * kDistTile;   // + 4 padding floats per staged row (bank spread)
constexpr size_t kDistSmem = (size_t)kDistStageFloats * sizeof(float);
constexpr int kDistMaxAgents = 1024;
constexpr long long kMaxWorkspace = 64LL << 20;         // bytes of per-split partial matrices
constexpr int kStageBatch = 8;                          // 16-byte loads in flight per thread while staging (16 would spill)

struct DistKernelParams {
    DistParams p;
    int tiles_side;
    long long span;                                     // coordinates per split (multiple of 4)
    double* ws;                                         // [splits][K][K]
};

template <bool GRAM, bool ROWS = false>
__global__ void __launch_bounds__(kDistThreads, 2) pairwise_sqdist_kernel(DistKernelParams kp) {
    extern __shared__ float4 stage4[];
    float* const stage = reinterpret_cast<float*>(stage4);
    __shared__ const float* wp[2 * kDistTile];
    __shared__ float scs[2 * kDistTile];
    const DistParams& p = kp.p;
    const int tid = threadIdx.x, K = p.K;

    // tile (ti, tj), ti <= tj, row-major over the upper triangle
    int ti = 0, rem = blockIdx.x;
    while (rem >= kp.tiles_side - ti) { rem -= kp.tiles_side - ti; ++ti; }
    const int tj = ti + rem;
    const bool diag = ti == tj;
    const int r0 = ti * kDistTile, c0 = tj * kDistTile;
    const int nr = min(kDistTile, K - r0), nc = min(kDistTile, K - c0);
    const int nbr = (nr + 3) >> 2, nbc = (nc + 3) >> 2;
    const int col_base = diag ? 0 : 4 * nbr;            // staged row of the first column participant
    const int P = diag ? 4 * nbr : 4 * nbr + 4 * nbc;   // staged rows (padding participants are staged as zeros)
    const int CH = (kDistStage / P) & ~63;              // chunk coordinates: >= 128, multiple of 64
    const int RS = CH + 4;                              // staged row stride in floats (16-byte aligned)
    const int G = CH >> 2;                              // float4 groups per staged row

    for (int q = tid; q < P; q += kDistThreads) {
        const int k = q < col_base ? r0 + q : (diag ? r0 + q : c0 + (q - col_base));
        const bool valid = diag ? q < nr : (q < col_base ? q < nr : q - col_base < nc);
        wp[q] = valid ? p.w_agents[k] : nullptr;
        scs[q] = valid && p.scales ? p.scales[k] : 1.0f;
    }
    barrier_in(p.gate, blockIdx.x == 0 && blockIdx.y == 0);

    // this thread's pair block (bi, bj) and coordinate lane l
    const int NB = diag ? nbr * (nbr + 1) / 2 : nbr * nbc;
    const int L = NB >= kDistThreads ? 1 : kDistThreads / NB;
    const bool active = tid < NB * L;
    const int b = tid % NB, l = tid / NB;
    int bi = 0, bj = 0;
    if (diag) {
        int r = b;
        while (r >= nbr - bi) { r -= nbr - bi; ++bi; }
        bj = bi + r;
    } else {
        bi = b / nbc; bj = b % nbc;
    }
    const float4* const ra = stage4 + (size_t)(4 * bi) * (RS >> 2);
    const float4* const cb = stage4 + (size_t)(col_base + 4 * bj) * (RS >> 2);

    double accd[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) accd[r][c] = 0.0;

    const long long lo = p.begin + (long long)blockIdx.y * kp.span;
    const long long hi = min(p.end, lo + kp.span);
    for (long long cc = lo; cc < hi; cc += CH) {
        const int ng = (int)(min((long long)CH, hi - cc) >> 2);     // valid float4 groups of this chunk
        __syncthreads();                                             // the previous chunk has been consumed
        // stage: consecutive threads read consecutive 16-byte groups of one participant; kStageBatch loads in flight per thread
        for (int base = tid; base < P * G; base += kStageBatch * kDistThreads) {
            float4 v[kStageBatch];
#pragma unroll
            for (int u = 0; u < kStageBatch; ++u) {
                const int idx = base + u * kDistThreads;
                const int q = idx / G, g = idx - q * G;
                v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
                if (idx < P * G && g < ng && wp[q]) {
                    const long long i = cc + 4 * g;
                    v[u] = ld_f4(wp[q] + i);
                    if (GRAM && !ROWS) {
                        const float4 gg = ld_f4(p.w_global + i);
                        v[u] = make_float4(v[u].x - gg.x, v[u].y - gg.y, v[u].z - gg.z, v[u].w - gg.w);
                    } else if (p.scales) {
                        const float4 gg = ld_f4(p.w_global + i);
                        const float s = scs[q];
                        v[u] = make_float4((v[u].x - gg.x) * s, (v[u].y - gg.y) * s, (v[u].z - gg.z) * s, (v[u].w - gg.w) * s);
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < kStageBatch; ++u) {
                const int idx = base + u * kDistThreads;
                if (idx < P * G) {
                    const int q = idx / G, g = idx - q * G;
                    stage4[(size_t)q * (RS >> 2) + g] = v[u];
                }
            }
        }
        __syncthreads();
        if (active) {
            float acc[4][4];
#pragma unroll
            for (int r = 0; r < 4; ++r)
#pragma unroll
                for (int c = 0; c < 4; ++c) acc[r][c] = 0.f;
            for (int g = l; g < ng; g += L) {
                float4 a[4];
#pragma unroll
                for (int r = 0; r < 4; ++r) a[r] = ra[r * (RS >> 2) + g];
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const float4 x = cb[c * (RS >> 2) + g];
#pragma unroll
                    for (int r = 0; r < 4; ++r) {
                        if (GRAM) {
                            acc[r][c] = __fmaf_rn(a[r].x, x.x, acc[r][c]);
                            acc[r][c] = __fmaf_rn(a[r].y, x.y, acc[r][c]);
                            acc[r][c] = __fmaf_rn(a[r].z, x.z, acc[r][c]);
                            acc[r][c] = __fmaf_rn(a[r].w, x.w, acc[r][c]);
                        } else {
                            float d;
                            d = a[r].x - x.x; acc[r][c] = __fmaf_rn(d, d, acc[r][c]);
                            d = a[r].y - x.y; acc[r][c] = __fmaf_rn(d, d, acc[r][c]);
                            d = a[r].z - x.z; acc[r][c] = __fmaf_rn(d, d, acc[r][c]);
                            d = a[r].w - x.w; acc[r][c] = __fmaf_rn(d, d, acc[r][c]);
                        }
                    }
                }
            }
#pragma unroll
            for (int r = 0; r < 4; ++r)
#pragma unroll
                for (int c = 0; c < 4; ++c) accd[r][c] += (double)acc[r][c];
        }
    }

    // coordinate lanes of a pair block: added in lane order through shared memory (the stage is free now)
    __syncthreads();
    double* const red = reinterpret_cast<double*>(stage);            // [kDistThreads][16] doubles = 32 KiB <= stage
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) red[tid * 16 + r * 4 + c] = accd[r][c];
    __syncthreads();
    if (tid < NB) {
        double* const out = kp.ws + (size_t)blockIdx.y * K * K;
#pragma unroll
        for (int r = 0; r < 4; ++r) {
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                double v = red[tid * 16 + r * 4 + c];
                for (int ll = 1; ll < L; ++ll) v += red[(ll * NB + tid) * 16 + r * 4 + c];
                const int i = r0 + 4 * bi + r, j = c0 + 4 * bj + c;
                if (4 * bi + r < nr && 4 * bj + c < nc) {
                    if (!GRAM && i == j) v = 0.0;
                    out[(size_t)i * K + j] = v;
                    out[(size_t)j * K + i] = v;
                }
            }
        }
    }
}

template <bool GRAM, bool ROWS = false>
static cudaError_t launch_pairwise(const DistParams& p, double* out, int num_sms, cudaStream_t st) {
    if (p.K < 1 || p.K > kDistMaxAgents) return cudaErrorInvalidValue;
    if ((p.begin & 3) || (p.end & 3) || p.end < p.begin) return cudaErrorInvalidValue;
    if ((((GRAM && !ROWS) || p.scales) && !p.w_global) || (GRAM && p.scales) || !gate_ok(p.gate)) return cudaErrorInvalidValue;
    static int occ = 0;
    if (!occ) {
        RLR_CUDA_CHECK(cudaFuncSetAttribute(pairwise_sqdist_kernel<GRAM, ROWS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kDistSmem));
        RLR_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, pairwise_sqdist_kernel<GRAM, ROWS>, kDistThreads, kDistSmem));
        occ = occ < 1 ? 1 : occ;
    }
    DistKernelParams kp{};
    kp.p = p;
    kp.tiles_side = (p.K + kDistTile - 1) / kDistTile;
    const int tiles = kp.tiles_side * (kp.tiles_side + 1) / 2;
    const long long len = p.end - p.begin;
    const long long kk = (long long)p.K * p.K;
    const long long splits = coord_splits(len, tiles, (long long)occ * num_sms, p.gate.world, kMaxWorkspace / (kk * (long long)sizeof(double)));
    kp.span = ((len + splits - 1) / splits + 3) & ~3LL;
    Scratch ws((size_t)(splits * kk) * sizeof(double), st);
    kp.ws = ws.as<double>();
    RLR_CUDA_CHECK(cudaMemsetAsync(out, 0, (size_t)kk * sizeof(double), st));
    pairwise_sqdist_kernel<GRAM, ROWS><<<dim3((unsigned)tiles, (unsigned)splits), kDistThreads, kDistSmem, st>>>(kp);
    RLR_CUDA_CHECK(cudaGetLastError());
    return launch_ordered_sum(out, kp.ws, (int)splits, kk, st);
}

cudaError_t launch_pairwise_sqdist(const DistParams& p, double* out, int num_sms, cudaStream_t st) {
    return launch_pairwise<false>(p, out, num_sms, st);
}

cudaError_t launch_pairwise_gram(const DistParams& p, double* out, int num_sms, cudaStream_t st) {
    return launch_pairwise<true>(p, out, num_sms, st);
}

cudaError_t launch_history_gram(const DistParams& p, double* out, int num_sms, cudaStream_t st) {
    return launch_pairwise<true, true>(p, out, num_sms, st);
}

// DnC's sampled, centred updates (Shejwalkar and Houmansadr, NDSS 2021).  One thread per (iteration t, row position q): with c the
// sample's coordinate at position lo_t + q, x_k = (w_k[c] - w_global[c]) (* s_k) in fp64, mu = (sum of the finite x_k, k ascending) /
// (their count), and Y[t][k][q] = fp32(x_k - mu), every fp64 operation rounded on its own (the bits ops.dnc_gather_statement gives).
// A non-finite x_k stays out of the mean and leaves its own entry non-finite, so it spoils only its own row of the Gram matrix.
// Positions q >= hi_t - lo_t are written as zeros, the rows' padding to a multiple of 4.  Grid-stride loop over T * len_pad positions
// on at most one wave of CTAs (every CTA has to be resident while the leader waits in barrier_in); nothing is reduced across threads.
constexpr int kDncThreads = 256;

__global__ void __launch_bounds__(kDncThreads) dnc_gather_kernel(DncParams p) {
    barrier_in(p.gate, blockIdx.x == 0);
    const long long total = (long long)p.T * p.len_pad;
    for (long long e = (long long)blockIdx.x * kDncThreads + threadIdx.x; e < total; e += (long long)gridDim.x * kDncThreads) {
        const int t = (int)(e / p.len_pad), q = (int)(e - (long long)t * p.len_pad);
        float* const y = p.y + (size_t)t * p.K * p.len_pad + q;
        const int lo = p.ranges[2 * t], hi = p.ranges[2 * t + 1];
        if (q >= hi - lo) {
            for (int k = 0; k < p.K; ++k) y[(size_t)k * p.len_pad] = 0.f;
            continue;
        }
        const long long c = p.sample[(size_t)t * p.stride + lo + q];
        const double g = (double)ld_f1(p.w_global + c);
        auto x = [&](int k) {
            const double d = __dsub_rn((double)ld_f1(p.w_agents[k] + c), g);
            return p.scales ? __dmul_rn(d, (double)p.scales[k]) : d;
        };
        double mu = 0.0;
        int n = 0;
        for (int k = 0; k < p.K; ++k) {
            const double v = x(k);
            if (isfinite(v)) { mu = __dadd_rn(mu, v); ++n; }
        }
        mu = n ? __ddiv_rn(mu, (double)n) : 0.0;
        for (int k = 0; k < p.K; ++k) y[(size_t)k * p.len_pad] = __double2float_rn(__dsub_rn(x(k), mu));
    }
}

cudaError_t launch_dnc_gather(const DncParams& p, int num_sms, cudaStream_t st) {
    if (p.K < 1 || p.T < 1 || p.len_pad < 4 || (p.len_pad & 3) || p.stride < 0 || !p.w_agents || !p.w_global || !p.sample || !p.ranges || !p.y)
        return cudaErrorInvalidValue;
    if (!gate_ok(p.gate)) return cudaErrorInvalidValue;
    static int occ = 0;
    if (!occ) {
        RLR_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, dnc_gather_kernel, kDncThreads, 0));
        occ = occ < 1 ? 1 : occ;
    }
    // every rank launches at least one CTA, whatever its share of the sample: the barrier-in waits for all of them
    const long long need = ((long long)p.T * p.len_pad + kDncThreads - 1) / kDncThreads;
    const long long cap = (long long)occ * num_sms;
    const int grid = (int)(need < 1 ? 1 : (need < cap ? need : cap));
    dnc_gather_kernel<<<grid, kDncThreads, 0, st>>>(p);
    return cudaGetLastError();
}

}  // namespace rlr
