// Squared distances of the participants' updates to their weighted mean: the pass of RFA's smoothed Weiszfeld iteration (robust
// federated aggregation by the geometric median, Pillutla, Kakade and Harchaoui, IEEE TSP 2022):
//   out[k] = sum_{begin <= c < end} (x_k[c] - z[c])^2,   z[c] = sum_j b_j x_j[c],   sum_j b_j = 1,
// x_k = w_k (no clipping: w_global cancels because the b_j sum to 1) or x_k = (w_k - w_global) * s_k (server clipping).
// z is formed coordinate by coordinate from the staged values and never stored.  Deriving out[k] from the Krum matrix through
// sum_j b_j D_kj - 1/2 sum_ij b_i b_j D_ij would cost O(K^2) and cancels catastrophically exactly where RFA matters: one boosted update
// far from a tight honest cluster, whose large distances swamp the honest participants' small ones.  select.cu and trust.cu form their
// values per coordinate for the same reason.
//
// Work decomposition: grid.x = coordinate splits, sized so the grid covers about two waves (one wave on the fused multi-GPU path, where
// every CTA has to be resident while it waits for the cross-GPU barrier-in).  A CTA streams its range in chunks of CH coordinates:
//   1. stage CH coordinates of every participant in shared memory with 16-byte loads, so each value crosses HBM / NVLink once per pass;
//   2. z[c] in fp64 from shared memory, in position order.  When the chunk has fewer coordinates than half the CTA's threads (large K),
//      L = 256 / CH threads share a coordinate: each sums a contiguous block of positions in position order and the blocks are added in
//      block order.  z is kept as the fp32 pair hi = fp32(z), lo = fp32(z - hi);
//   3. each thread owns fixed participants (k = t, t + 256, ... for K >= 256; for K < 256 participant t % K on coordinate lane t / K of
//      256 / K lanes) and accumulates d = (x - hi) - lo, d^2 in fp32 over its <= 128 coordinates of the chunk, then folds the chunk into
//      fp64.
// The coordinate lanes of a participant are added in lane order at the end, every split writes its [K] workspace slot and
// launch_ordered_sum adds the slots in split order.  No atomics: the distances are bitwise identical from run to run.
#include "common.cuh"
#include "kernels.h"

namespace rlr {

constexpr int kRfaThreads = 256;
constexpr int kRfaStage = 16384;                        // fp32 values per chunk (staged participants x padded chunk coordinates)
constexpr int kRfaMaxChunk = 1024;                      // chunk coordinates at most (small K)
constexpr int kRfaMaxAgents = 1024;
constexpr int kRfaSlots = 4;                            // participants a thread owns at most (kRfaMaxAgents / kRfaThreads)
constexpr int kRfaStageBatch = 8;                       // 16-byte loads in flight per thread while staging
// dynamic shared memory: the stage, the chunk of w_global (clipping), z as hi / lo, and the position-block partials of z
constexpr size_t kRfaSmem = (size_t)(kRfaStage + 3 * kRfaMaxChunk) * sizeof(float) + (size_t)kRfaThreads * sizeof(double);

struct RfaKernelParams {
    RfaParams p;
    int chunk;                                          // CH: coordinates per chunk (multiple of 4)
    int row;                                            // staged row stride in floats (multiple of 4, an odd number of float4)
    long long span;                                     // coordinates per split (multiple of 4)
    double* ws;                                         // [splits][K]
};

__global__ void __launch_bounds__(kRfaThreads, 2) rfa_sqdist_kernel(RfaKernelParams kp) {
    extern __shared__ float4 smem4[];
    float* const stage = reinterpret_cast<float*>(smem4);
    float4* const gst4 = smem4 + kRfaStage / 4;                          // [CH / 4] w_global chunk
    float4* const zhi4 = gst4 + kRfaMaxChunk / 4;                        // [CH / 4]
    float4* const zlo4 = zhi4 + kRfaMaxChunk / 4;                        // [CH / 4]
    double* const zpart = reinterpret_cast<double*>(zlo4 + kRfaMaxChunk / 4);   // [L][CH], L * CH <= kRfaThreads
    __shared__ const float* wp[kRfaMaxAgents];
    __shared__ double bs[kRfaMaxAgents];
    __shared__ float scs[kRfaMaxAgents];
    const RfaParams& p = kp.p;
    const int tid = threadIdx.x, K = p.K, CH = kp.chunk, RS = kp.row, G = CH >> 2;

    for (int q = tid; q < K; q += kRfaThreads) {
        wp[q] = p.w_agents[q];
        bs[q] = p.b[q];
        scs[q] = p.scales ? p.scales[q] : 1.0f;
    }
    barrier_in(p.gate, blockIdx.x == 0);

    // z: LZ threads per coordinate, each over a contiguous block of positions
    const int LZ = CH >= kRfaThreads ? 1 : kRfaThreads / CH;
    const int zc = tid % CH, zl = tid / CH;
    const int jb = (int)((long long)zl * K / LZ), je = (int)((long long)(zl + 1) * K / LZ);
    // distances: participants t0, t0 + 256, ... on coordinate lane l of LD
    const int M = K < kRfaThreads ? K : kRfaThreads;
    const int LD = kRfaThreads / M;
    const int t0 = tid % M, l = tid / M;
    const bool active = l < LD;

    double accd[kRfaSlots];
#pragma unroll
    for (int i = 0; i < kRfaSlots; ++i) accd[i] = 0.0;

    const long long lo = p.begin + (long long)blockIdx.x * kp.span;
    const long long hi = min(p.end, lo + kp.span);
    for (long long cc = lo; cc < hi; cc += CH) {
        const int ng = (int)(min((long long)CH, hi - cc) >> 2);     // valid float4 groups of this chunk
        const int nc = 4 * ng;
        __syncthreads();                                             // the previous chunk has been consumed
        if (p.scales) {
            for (int g = tid; g < ng; g += kRfaThreads) gst4[g] = ld_f4(p.w_global + cc + 4 * g);
            __syncthreads();
        }
        // 1. stage: consecutive threads read consecutive 16-byte groups of one participant
        for (int base = tid; base < K * G; base += kRfaStageBatch * kRfaThreads) {
            float4 v[kRfaStageBatch];
#pragma unroll
            for (int u = 0; u < kRfaStageBatch; ++u) {
                const int idx = base + u * kRfaThreads;
                const int q = idx / G, g = idx - q * G;
                v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
                if (idx < K * G && g < ng) {
                    v[u] = ld_f4(wp[q] + cc + 4 * g);
                    if (p.scales) {
                        const float4 gg = gst4[g];
                        const float s = scs[q];
                        v[u] = make_float4((v[u].x - gg.x) * s, (v[u].y - gg.y) * s, (v[u].z - gg.z) * s, (v[u].w - gg.w) * s);
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < kRfaStageBatch; ++u) {
                const int idx = base + u * kRfaThreads;
                if (idx < K * G) {
                    const int q = idx / G, g = idx - q * G;
                    smem4[(size_t)q * (RS >> 2) + g] = v[u];
                }
            }
        }
        __syncthreads();
        // 2. z in fp64, positions in order
        float* const zhi = reinterpret_cast<float*>(zhi4);
        float* const zlo = reinterpret_cast<float*>(zlo4);
        if (LZ == 1) {
            for (int c = tid; c < nc; c += kRfaThreads) {
                double z = 0.0;
                for (int j = 0; j < K; ++j) z = fma(bs[j], (double)stage[(size_t)j * RS + c], z);
                const float h = __double2float_rn(z);
                zhi[c] = h;
                zlo[c] = __double2float_rn(z - (double)h);
            }
        } else {
            if (zl < LZ && zc < nc) {
                double z = 0.0;
                for (int j = jb; j < je; ++j) z = fma(bs[j], (double)stage[(size_t)j * RS + zc], z);
                zpart[zl * CH + zc] = z;
            }
            __syncthreads();
            if (tid < nc) {
                double z = zpart[tid];
                for (int b = 1; b < LZ; ++b) z += zpart[b * CH + tid];
                const float h = __double2float_rn(z);
                zhi[tid] = h;
                zlo[tid] = __double2float_rn(z - (double)h);
            }
        }
        __syncthreads();
        // 3. squared distances of the owned participants over this lane's groups, folded into fp64 once per chunk
        if (active) {
            float acc[kRfaSlots];
#pragma unroll
            for (int i = 0; i < kRfaSlots; ++i) acc[i] = 0.f;
            for (int g = l; g < ng; g += LD) {
                const float4 h = zhi4[g], o = zlo4[g];
#pragma unroll
                for (int i = 0; i < kRfaSlots; ++i) {
                    const int k = t0 + i * kRfaThreads;
                    if (k < K) {
                        const float4 x = smem4[(size_t)k * (RS >> 2) + g];
                        float d;
                        d = (x.x - h.x) - o.x; acc[i] = __fmaf_rn(d, d, acc[i]);
                        d = (x.y - h.y) - o.y; acc[i] = __fmaf_rn(d, d, acc[i]);
                        d = (x.z - h.z) - o.z; acc[i] = __fmaf_rn(d, d, acc[i]);
                        d = (x.w - h.w) - o.w; acc[i] = __fmaf_rn(d, d, acc[i]);
                    }
                }
            }
#pragma unroll
            for (int i = 0; i < kRfaSlots; ++i) accd[i] += (double)acc[i];
        }
    }

    // coordinate lanes of a participant: added in lane order through shared memory (the stage is free now)
    __syncthreads();
    double* const red = reinterpret_cast<double*>(stage);               // [kRfaThreads][kRfaSlots] doubles = 8 KiB <= stage
#pragma unroll
    for (int i = 0; i < kRfaSlots; ++i) red[tid * kRfaSlots + i] = accd[i];
    __syncthreads();
    if (tid < M) {
        double* const out = kp.ws + (size_t)blockIdx.x * K;
#pragma unroll
        for (int i = 0; i < kRfaSlots; ++i) {
            const int k = tid + i * kRfaThreads;
            if (k < K) {
                double v = red[tid * kRfaSlots + i];
                for (int ll = 1; ll < LD; ++ll) v += red[(ll * M + tid) * kRfaSlots + i];
                out[k] = v;
            }
        }
    }
}

cudaError_t launch_rfa_sqdist(const RfaParams& p, double* out, int num_sms, cudaStream_t st) {
    if (p.K < 1 || p.K > kRfaMaxAgents || !p.b) return cudaErrorInvalidValue;
    if ((p.begin & 3) || (p.end & 3) || p.end < p.begin) return cudaErrorInvalidValue;
    if ((p.scales && !p.w_global) || !gate_ok(p.gate)) return cudaErrorInvalidValue;
    static int occ = 0;
    if (!occ) {
        RLR_CUDA_CHECK(cudaFuncSetAttribute(rfa_sqdist_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kRfaSmem));
        RLR_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, rfa_sqdist_kernel, kRfaThreads, kRfaSmem));
        occ = occ < 1 ? 1 : occ;
    }
    RfaKernelParams kp{};
    kp.p = p;
    const int per = kRfaStage / p.K;                                     // staged floats per participant (>= 16)
    kp.chunk = min(kRfaMaxChunk, (per - 4) & ~3);
    kp.row = ((kp.chunk >> 2) | 1) << 2;                                 // <= chunk + 4; odd float4 stride: conflict-free row reads
    const long long len = p.end - p.begin;
    const long long splits = coord_splits(len, 1, (long long)occ * num_sms, p.gate.world);
    kp.span = ((len + splits - 1) / splits + 3) & ~3LL;
    Scratch ws((size_t)(splits * p.K) * sizeof(double), st);
    kp.ws = ws.as<double>();
    RLR_CUDA_CHECK(cudaMemsetAsync(out, 0, (size_t)p.K * sizeof(double), st));
    rfa_sqdist_kernel<<<dim3((unsigned)splits), kRfaThreads, kRfaSmem, st>>>(kp);
    RLR_CUDA_CHECK(cudaGetLastError());
    return launch_ordered_sum(out, kp.ws, (int)splits, (long long)p.K, st);
}

}  // namespace rlr
