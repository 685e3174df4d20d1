// Colluding attackers with full knowledge: ALIE (A Little Is Enough, Baruch, Baruch and Goldberg, NeurIPS 2019) and the Min-Max /
// Min-Sum attacks (Shejwalkar and Houmansadr, NDSS 2021).  The corrupt participants read the round's honest updates and all submit one
// crafted update m.  Per voted coordinate c, with x_k = (double)w_k[c] - (double)w_g[c] and every fp64 operation rounded on its own
// (__dadd_rn & co.: no FMA contraction, so ops.collude_statement matches the crafted slots bit for bit):
//   mu  = the mean of the honest x_k, added in position order (a non-finite x_k is left out; mu = 0 when none is finite);
//   sig = sqrt(sum_k (x_k - mu)^2 / (n - 1)) over the same x_k, two-pass (0 when n < 2);
//   xc  = the mean of the corrupt x_k, likewise (mu when none is finite);
//   u   = sig (std), sign(mu) (sign), mu (unit) or mu - xc (backdoor);
//   m   = mu - z sig (alie, std), clamp(xc, mu - z sig, mu + z sig) (alie, backdoor) or mu - gamma u (minmax / minsum);
//   every output slot gets fp32((double)w_g[c] + m).
// Two kernels share one body:
//   STATS (minmax / minsum): out[2H + 1] = a_k = sum_c (mu - x_k)^2, e_k = sum_c (mu - x_k) u for every honest k, then q = sum_c u^2;
//   WRITE (alie, and minmax / minsum once the host has gamma): writes m into the output slots, out[1] = sum_c (m - mu)^2.
// The write pass recomputes mu and u from the re-staged slots instead of keeping them in an fp64 scratch vector: that reads 4 (K + 1)
// bytes per coordinate against the scratch's 16 written and 16 read back, and holds no 16 bytes per voted coordinate of device memory.
//
// Work decomposition as in rfa.cu: grid.x = coordinate splits (about two waves; one wave on the fused multi-GPU path, where every CTA
// has to be resident while it waits for the cross-GPU barrier-in).  A CTA streams its range in chunks of CH coordinates:
//   1. stage CH coordinates of every participant (honest first, then corrupt) and of w_global in shared memory with 16-byte loads, so
//      each value crosses HBM / NVLink once per pass;
//   2. one thread per coordinate forms mu, sig, xc and u (and m) from the stage;
//   3. STATS: each thread owns fixed honest participants (k = t, t + 256, ... for H >= 256; for H < 256 participant t % H on coordinate
//      lane t / H of 256 / H lanes) and accumulates a_k and e_k over its float4 groups of the chunk in fp64.
// At the end the lanes of a participant and the coordinate threads' q (or deviation) are added in a fixed order, every split writes its
// workspace slot and launch_ordered_sum adds the slots in split order.  No atomics: the sums are bitwise identical from run to run.
#include "common.cuh"
#include "kernels.h"

namespace rlr {

constexpr int kColThreads = 256;
constexpr int kColStage = 16384;                        // fp32 values per chunk (staged participants x padded chunk coordinates)
constexpr int kColMaxChunk = 1024;                      // chunk coordinates at most (small K)
constexpr int kColMaxAgents = 1024;
constexpr int kColSlots = 4;                            // honest participants a thread owns at most (kColMaxAgents / kColThreads)
constexpr int kColStageBatch = 8;                       // 16-byte loads in flight per thread while staging
// dynamic shared memory: the stage, the chunk of w_global, and mu / u of the chunk in fp64
constexpr size_t kColSmem = (size_t)(kColStage + kColMaxChunk) * sizeof(float) + 2 * (size_t)kColMaxChunk * sizeof(double);

struct ColKernelParams {
    ColludeParams p;
    int chunk;                                          // CH: coordinates per chunk (multiple of 4)
    int row;                                            // staged row stride in floats (multiple of 4, an odd number of float4)
    long long span;                                     // coordinates per split (multiple of 4)
    double* ws;                                         // [splits][2H + 1] (STATS) or [splits][1]
};

template <bool STATS>
__global__ void __launch_bounds__(kColThreads, 2) collude_kernel(ColKernelParams kp) {
    extern __shared__ float4 smem4[];
    float* const stage = reinterpret_cast<float*>(smem4);
    float4* const gst4 = smem4 + kColStage / 4;                          // [CH / 4] w_global chunk
    const float* const gst = reinterpret_cast<const float*>(gst4);
    double* const mus = reinterpret_cast<double*>(gst4 + kColMaxChunk / 4);   // [CH]
    double* const us = mus + kColMaxChunk;                               // [CH]
    __shared__ const float* wp[kColMaxAgents];
    __shared__ float* op[kColMaxAgents];
    const ColludeParams& p = kp.p;
    const int tid = threadIdx.x, H = p.H, K = p.H + p.C, CH = kp.chunk, RS = kp.row, G = CH >> 2;
    const bool need_sig = p.dir == 1 || (!STATS && p.mode == 0);

    for (int q = tid; q < K; q += kColThreads) wp[q] = p.w_agents[q];
    if (!STATS)
        for (int q = tid; q < p.n_out; q += kColThreads) op[q] = p.w_out[q];
    barrier_in(p.gate, blockIdx.x == 0);

    // a_k / e_k: honest participants t0, t0 + 256, ... on coordinate lane l of LD
    const int M = H < kColThreads ? H : kColThreads;
    const int LD = kColThreads / M;
    const int t0 = tid % M, l = tid / M;
    double acca[kColSlots], acce[kColSlots];
#pragma unroll
    for (int i = 0; i < kColSlots; ++i) acca[i] = acce[i] = 0.0;
    double accq = 0.0;                                                   // q (STATS) or the deviation, over this thread's coordinates

    const long long lo = p.begin + (long long)blockIdx.x * kp.span;
    const long long hi = min(p.end, lo + kp.span);
    for (long long cc = lo; cc < hi; cc += CH) {
        const int ng = (int)(min((long long)CH, hi - cc) >> 2);     // valid float4 groups of this chunk
        const int nc = 4 * ng;
        __syncthreads();                                             // the previous chunk has been consumed
        for (int g = tid; g < ng; g += kColThreads) gst4[g] = ld_f4(p.w_global + cc + 4 * g);
        // 1. stage: consecutive threads read consecutive 16-byte groups of one participant
        for (int base = tid; base < K * G; base += kColStageBatch * kColThreads) {
            float4 v[kColStageBatch];
#pragma unroll
            for (int u = 0; u < kColStageBatch; ++u) {
                const int idx = base + u * kColThreads;
                const int q = idx / G, g = idx - q * G;
                v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
                if (idx < K * G && g < ng) v[u] = ld_f4(wp[q] + cc + 4 * g);
            }
#pragma unroll
            for (int u = 0; u < kColStageBatch; ++u) {
                const int idx = base + u * kColThreads;
                if (idx < K * G) {
                    const int q = idx / G, g = idx - q * G;
                    smem4[(size_t)q * (RS >> 2) + g] = v[u];
                }
            }
        }
        __syncthreads();
        // 2. the per-coordinate statistics, one thread per coordinate, positions in order
        for (int c = tid; c < nc; c += kColThreads) {
            const double g = (double)gst[c];
            double s = 0.0;
            int n = 0;
            for (int j = 0; j < H; ++j) {
                const double x = __dsub_rn((double)stage[(size_t)j * RS + c], g);
                if (isfinite(x)) { s = __dadd_rn(s, x); ++n; }
            }
            const double mu = n ? __ddiv_rn(s, (double)n) : 0.0;
            double sig = 0.0;
            if (need_sig && n >= 2) {
                double v = 0.0;
                for (int j = 0; j < H; ++j) {
                    const double x = __dsub_rn((double)stage[(size_t)j * RS + c], g);
                    if (isfinite(x)) {
                        const double d = __dsub_rn(x, mu);
                        v = __dadd_rn(v, __dmul_rn(d, d));
                    }
                }
                sig = __dsqrt_rn(__ddiv_rn(v, (double)(n - 1)));
            }
            double xc = mu;
            if (p.dir == 0) {
                double sc = 0.0;
                int ncor = 0;
                for (int j = H; j < K; ++j) {
                    const double x = __dsub_rn((double)stage[(size_t)j * RS + c], g);
                    if (isfinite(x)) { sc = __dadd_rn(sc, x); ++ncor; }
                }
                if (ncor) xc = __ddiv_rn(sc, (double)ncor);
            }
            const double u = p.dir == 1 ? sig : p.dir == 2 ? (double)((mu > 0.0) - (mu < 0.0)) : p.dir == 3 ? mu : __dsub_rn(mu, xc);
            if (STATS) {
                mus[c] = mu;
                us[c] = u;
                accq = fma(u, u, accq);
            } else {
                double m;
                if (p.mode == 0) {
                    const double t = __dmul_rn(p.z, sig);
                    m = p.dir == 1 ? __dsub_rn(mu, t) : fmin(fmax(xc, __dsub_rn(mu, t)), __dadd_rn(mu, t));
                } else {
                    m = __dsub_rn(mu, __dmul_rn(p.gamma, u));
                }
                const float o = __double2float_rn(__dadd_rn(g, m));
                for (int q = 0; q < p.n_out; ++q) op[q][cc + c] = o;
                const double dv = m - mu;
                accq = fma(dv, dv, accq);
            }
        }
        // 3. a_k and e_k of the owned honest participants over this lane's groups
        if (STATS) {
            __syncthreads();
            if (l < LD) {
                for (int g4 = l; g4 < ng; g4 += LD) {
                    const float4 gg = gst4[g4];
                    const float gv[4] = {gg.x, gg.y, gg.z, gg.w};
#pragma unroll
                    for (int i = 0; i < kColSlots; ++i) {
                        const int k = t0 + i * kColThreads;
                        if (k < H) {
                            const float4 xv = smem4[(size_t)k * (RS >> 2) + g4];
                            const float xs[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
                            for (int e = 0; e < 4; ++e) {
                                const double x = (double)xs[e] - (double)gv[e];
                                if (isfinite(x)) {
                                    const double d = mus[4 * g4 + e] - x;
                                    acca[i] = fma(d, d, acca[i]);
                                    acce[i] = fma(d, us[4 * g4 + e], acce[i]);
                                }
                            }
                        }
                    }
                }
            }
        }
    }

    // lanes of a participant and the coordinate threads: added in a fixed order through shared memory (the stage is free now)
    __syncthreads();
    double* const red = reinterpret_cast<double*>(stage);               // [kColThreads][2 kColSlots] + [kColThreads] doubles <= stage
    double* const redq = red + kColThreads * 2 * kColSlots;
    if (STATS) {
#pragma unroll
        for (int i = 0; i < kColSlots; ++i) {
            red[tid * 2 * kColSlots + i] = acca[i];
            red[tid * 2 * kColSlots + kColSlots + i] = acce[i];
        }
    }
    redq[tid] = accq;
    __syncthreads();
    const int nout = STATS ? 2 * H + 1 : 1;
    double* const out = kp.ws + (size_t)blockIdx.x * nout;
    if (STATS && tid < M) {
#pragma unroll
        for (int i = 0; i < kColSlots; ++i) {
            const int k = tid + i * kColThreads;
            if (k < H) {
                double a = red[tid * 2 * kColSlots + i], e = red[tid * 2 * kColSlots + kColSlots + i];
                for (int ll = 1; ll < LD; ++ll) {
                    a += red[(ll * M + tid) * 2 * kColSlots + i];
                    e += red[(ll * M + tid) * 2 * kColSlots + kColSlots + i];
                }
                out[k] = a;
                out[H + k] = e;
            }
        }
    }
    if (tid == 0) {
        double s = redq[0];
        for (int t = 1; t < kColThreads; ++t) s += redq[t];
        out[nout - 1] = s;
    }
}

template <bool STATS>
static cudaError_t launch_collude(const ColludeParams& p, double* out, int num_sms, cudaStream_t st) {
    const int K = p.H + p.C;
    if (p.H < 1 || p.C < 0 || K > kColMaxAgents || !p.w_agents || !p.w_global) return cudaErrorInvalidValue;
    if (!STATS && (p.n_out < 0 || p.n_out > kColMaxAgents || (p.n_out && !p.w_out))) return cudaErrorInvalidValue;
    if (p.mode < 0 || p.mode > 1 || p.dir < 0 || p.dir > 3) return cudaErrorInvalidValue;
    if ((p.begin & 3) || (p.end & 3) || p.end < p.begin || !gate_ok(p.gate)) return cudaErrorInvalidValue;
    static int occ = 0;
    if (!occ) {
        RLR_CUDA_CHECK(cudaFuncSetAttribute(collude_kernel<STATS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kColSmem));
        RLR_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, collude_kernel<STATS>, kColThreads, kColSmem));
        occ = occ < 1 ? 1 : occ;
    }
    ColKernelParams kp{};
    kp.p = p;
    const int per = kColStage / K;                                       // staged floats per participant (>= 16)
    kp.chunk = min(kColMaxChunk, (per - 4) & ~3);
    kp.row = ((kp.chunk >> 2) | 1) << 2;                                 // <= chunk + 4; odd float4 stride: conflict-free row reads
    const long long len = p.end - p.begin;
    const long long splits = coord_splits(len, 1, (long long)occ * num_sms, p.gate.world);
    kp.span = ((len + splits - 1) / splits + 3) & ~3LL;
    const long long nout = STATS ? 2LL * p.H + 1 : 1;
    Scratch ws((size_t)(splits * nout) * sizeof(double), st);
    kp.ws = ws.as<double>();
    RLR_CUDA_CHECK(cudaMemsetAsync(out, 0, (size_t)nout * sizeof(double), st));
    collude_kernel<STATS><<<dim3((unsigned)splits), kColThreads, kColSmem, st>>>(kp);
    RLR_CUDA_CHECK(cudaGetLastError());
    return launch_ordered_sum(out, kp.ws, (int)splits, nout, st);
}

cudaError_t launch_collude_stats(const ColludeParams& p, double* out, int num_sms, cudaStream_t st) {
    return launch_collude<true>(p, out, num_sms, st);
}

cudaError_t launch_collude_write(const ColludeParams& p, double* out, int num_sms, cudaStream_t st) {
    return launch_collude<false>(p, out, num_sms, st);
}

}  // namespace rlr
