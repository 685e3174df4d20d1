// Fused federated server step for sm_90a: one pass over the flat parameter vector that
//   * reads every participating agent's local parameters w_k (local HBM, or a PEER GPU's HBM through
//     NVLink/NVSwitch-mapped pointers) and forms the update d_k = w_k - w_g in registers (never materialised),
//   * takes the per-coordinate sign vote  s = |sum_k sign(d_k)|  ->  lr = +server_lr if s >= theta else -server_lr
//     (Robust Learning Rate; reference src/aggregation.py:48-54),
//   * aggregates: data-size-weighted mean (:57-64) | lower coordinate median (:66-69) | sign majority (:71-75),
//   * adds optional Gaussian noise (in-kernel Philox; :34-35) BEFORE the lr multiply, like the reference,
//   * applies the server step  w_g' = w_g + lr * agg  (:38-40) in fp64 then rounds to fp32 -- or, with --server_opt, the server
//     optimizer (FedAvgM momentum, FedAdagrad, FedAdam, FedYogi) on the pseudo-gradient ±agg, its fp32 state m, v read and
//     written in the same pass (state index i - state_base: a rank keeps only its own slice on the fused multi-GPU path),
//   * and writes w_g' (+ its bf16 GEMM-operand shadow) to every GPU: one NVLS `multimem.st` per 16 bytes when a
//     multicast mapping exists, else one P2P store per peer.  This store IS the next round's broadcast
//     (reference src/federated.py:72).
// Across GPUs rank r owns coordinates [begin,end); the kernel is reduce-scatter ∘ compute ∘ all-gather in one
// launch.  Synchronisation is by release/acquire flags on peer-mapped signal words (no NCCL, no host sync):
//   barrier-in  : every rank's slots are final (also: nobody reads the old w_global any more),
//   hand-off    : either the classic barrier-out (every slice has landed everywhere when the kernel ends), or -- p.handoff = 1 --
//                 rank r only PUBLISHES "slice r of round e has landed" into every peer's ready word and exits; the consumer of
//                 the broadcast (the next round's first-layer GEMM, gemm.cu, and acquire_slices_kernel) acquires the words of the
//                 slices it is about to read, so the first local forward overlaps the rest of the broadcast.
// Coordinates >= n_vote (BatchNorm running statistics; SURVEY.md quirk 13) get a plain weighted mean, no vote, no clip scale.
//
// Coordinate median for real participant counts (reference runs K = 10, 40 and 33-of-3383; src/runner.sh:12-38):
//   K <= 8   odd-even transposition network on four coordinates per thread (registers),
//   K <= 64  Batcher odd-even merge network generated at compile time for N in {12,16,24,32,40,48,64} (K is padded with +inf;
//            one coordinate per thread, everything in registers: 42 ... 543 compare-exchanges),
//   K > 64   storage-free selection: 32 rounds of bit-wise bisection on the order-preserving integer image of the updates,
//            the K values staged once per coordinate in shared memory (or re-read from L2 when they do not fit).
// torch.median's LOWER median for even K is kept in every path.
#include "common.cuh"
#include "kernels.h"

namespace rlr {

constexpr int kAggThreads = 256;
constexpr int kSelThreads = 128;     // bisection path: fewer threads -> more shared memory per coordinate
constexpr int kMaxAgents = 1024;     // capacity of the per-block pointer / weight tables

template <int K>
__device__ __forceinline__ float lower_median_fixed(float (&v)[K]) {
    // odd-even transposition network, fully unrolled -> registers only
#pragma unroll
    for (int pass = 0; pass < K; ++pass) {
#pragma unroll
        for (int j = pass & 1; j + 1 < K; j += 2) {
            const float lo = fminf(v[j], v[j + 1]), hi = fmaxf(v[j], v[j + 1]);
            v[j] = lo; v[j + 1] = hi;
        }
    }
    return v[(K - 1) / 2];  // torch.median returns the LOWER median for even K
}

// Batcher's odd-even merge sort for an arbitrary (compile-time) length.  The comparator list is produced by a constexpr function,
// so the device code is ONE fully unrolled loop over compile-time index pairs and v[] lives in registers.
// Comparator counts: 42 / 63 / 132 / 191 / 305 / 384 / 543 for N = 12 / 16 / 24 / 32 / 40 / 48 / 64.
template <int N>
struct BatcherNet {
    static constexpr int kMax = N * 10;
    int n = 0;
    short a[kMax] = {}, b[kMax] = {};
    constexpr BatcherNet() {
        for (int p = 1; p < N; p <<= 1)
            for (int k = p; k >= 1; k >>= 1)
                for (int j = k % p; j + k <= N - 1; j += 2 * k)
                    for (int i = 0; i < k && i + j + k <= N - 1; ++i)
                        if ((i + j) / (2 * p) == (i + j + k) / (2 * p)) { a[n] = (short)(i + j); b[n] = (short)(i + j + k); ++n; }
    }
};
template <int N>
__device__ __forceinline__ void batcher_sort(float (&v)[N]) {
    constexpr BatcherNet<N> net{};
#pragma unroll
    for (int c = 0; c < net.n; ++c) {
        const float lo = fminf(v[net.a[c]], v[net.b[c]]), hi = fmaxf(v[net.a[c]], v[net.b[c]]);
        v[net.a[c]] = lo; v[net.b[c]] = hi;
    }
}

__device__ __forceinline__ int sgn(float d) { return (d > 0.f) - (d < 0.f); }
// order-preserving map float -> uint32 (negative values reversed, sign bit flipped for positives)
__device__ __forceinline__ uint32_t ordered_bits(float f) {
    const uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float from_ordered_bits(uint32_t o) {
    return __uint_as_float((o & 0x80000000u) ? (o & 0x7FFFFFFFu) : ~o);
}

struct AggShared {
    const float* w[kMaxAgents];
    double wt[kMaxAgents];
    float sc[kMaxAgents];
    unsigned long long scratch[32];
    int last;
};

// ---- prologue shared by all variants: tables into shared memory, barrier-in ---------------------------------------------------
__device__ __forceinline__ void agg_prologue(const AggParams& p, AggShared& sh, int K) {
    for (int k = threadIdx.x; k < K; k += blockDim.x) {
        sh.w[k] = p.w_agents[k];
        sh.wt[k] = p.weights[k];
        sh.sc[k] = p.scales ? p.scales[k] : 1.0f;
    }
    // barrier-in: every peer's local training has finished and its w_k is globally visible
    if (p.world > 1) {
        if (blockIdx.x == 0) {
            xgpu_barrier(p.flag_ptrs, 0, p.rank, p.world, p.epoch);
            __syncthreads();
            if (threadIdx.x == 0) st_release_gpu(p.local_sync, p.epoch);
        } else if (threadIdx.x == 0) {
            while ((int32_t)(ld_acquire_gpu(p.local_sync) - p.epoch) < 0) { __nanosleep(32); }
        }
    }
    __syncthreads();
}

// ---- epilogue: flipped counter, then barrier-out or slice publication ------------------------------------------------------------
__device__ __forceinline__ void agg_epilogue(const AggParams& p, AggShared& sh, unsigned long long flipped) {
    if (p.flipped) {
        const unsigned long long tot = block_sum<unsigned long long>(flipped, sh.scratch);
        if (threadIdx.x == 0 && tot) atomicAdd(p.flipped, tot);
    }
    if (p.world > 1) {
        __threadfence_system();                    // this thread's (multicast / peer) stores are ordered before the flag stores below
        __syncthreads();
        if (threadIdx.x == 0) {
            const unsigned prev = atomicAdd(p.local_sync + 1, 1u);
            sh.last = (prev == gridDim.x - 1);
            if (sh.last) { p.local_sync[1] = 0; }
            __threadfence();
        }
        __syncthreads();
        if (sh.last) {                             // the last CTA of this GPU: every CTA's stores are fenced
            if (p.handoff) {
                // publish "slice `rank` of round `epoch` has landed" to every peer (slot 2*world + rank of its flag words); nobody waits
                if ((int)threadIdx.x < p.world) st_release_sys(p.flag_ptrs[threadIdx.x] + 2 * p.world + p.rank, p.epoch);
            } else {
                xgpu_barrier(p.flag_ptrs, p.world, p.rank, p.world, p.epoch);
            }
        }
    }
}

// ---- one coordinate: noise, RLR flip, server step -----------------------------------------------------------------------------
// The server optimizers (Reddi et al., Adaptive Federated Optimization, Algorithm 2, no bias correction; FedAvgM for momentum) act on
// the pseudo-gradient d = ±(agg + noise).  m and v are this coordinate's state: read and rounded back to fp32 here, while the new
// weight uses this round's unrounded fp64 values.  sgd keeps the exact expression of the plain step.
enum : int { kOptSgd = 0, kOptMomentum = 1, kOptAdagrad = 2, kOptAdam = 3, kOptYogi = 4 };

__device__ __forceinline__ float server_step(const AggParams& p, float g, double agg, int s, float nz, unsigned long long& flipped,
                                             float& m, float& v, bool stateful = true) {
    const double a = agg + (double)nz;
    const bool keep = (p.theta <= 0) || (abs(s) >= p.theta);
    flipped += keep ? 0 : 1;
    if (!stateful || p.opt == kOptSgd) {
        const double lr = keep ? (double)p.server_lr : -(double)p.server_lr;
        return (float)((double)g + lr * a);
    }
    const double d = keep ? a : -a;
    double m1, step;
    if (p.opt == kOptMomentum) {
        m1 = p.beta1 * (double)m + d;
        step = m1;
    } else {
        m1 = p.beta1 * (double)m + (1.0 - p.beta1) * d;
        const double v0 = (double)v, d2 = d * d;
        const double v1 = p.opt == kOptAdagrad ? v0 + d2
                        : p.opt == kOptAdam    ? p.beta2 * v0 + (1.0 - p.beta2) * d2
                                               : v0 - (1.0 - p.beta2) * d2 * (double)((v0 > d2) - (v0 < d2));   // yogi
        v = (float)v1;
        step = m1 / (sqrt(v1) + p.tau);
    }
    m = (float)m1;
    return (float)((double)g + (double)p.server_lr * step);
}

__device__ __forceinline__ void store4(const AggParams& p, long long i, const float (&out)[4]) {
    const float4 o4 = make_float4(out[0], out[1], out[2], out[3]);
    const uint2 b4 = make_uint2(pack_bf16x2(out[0], out[1]), pack_bf16x2(out[2], out[3]));
    if (p.use_multimem) {
        multimem_st_f4(p.out_ptrs[0] + i, o4);
        if (p.out_bf16_ptrs) multimem_st_b2(reinterpret_cast<uint2*>(p.out_bf16_ptrs[0] + i), b4);
    } else {
        for (int d = 0; d < p.n_out; ++d) {
            st_f4(p.out_ptrs[d] + i, o4);
            if (p.out_bf16_ptrs) *reinterpret_cast<uint2*>(p.out_bf16_ptrs[d] + i) = b4;
        }
    }
}

// =================================================================================================================================
// vector path: four coordinates per thread.  MODE 0 avg, 1 comed (KT = 1..8 participants, compile time), 2 sign.
// OPT: a server optimizer with state (float4 loads / stores of m, v).  A compile-time switch here: with a run-time one the sgd build of
// the K = 8 median spills at ptxas's 64-register choice.  The stateful builds are allowed 2 CTAs per SM so ptxas keeps their fp64 step
// (~80 registers) out of local memory.
// =================================================================================================================================
template <int MODE, int KT, bool OPT>
__global__ void __launch_bounds__(kAggThreads, OPT ? 2 : 0) fused_aggregate_kernel(AggParams p) {
    __shared__ AggShared sh;
    const int K = KT > 0 ? KT : p.K;
    agg_prologue(p, sh, K);

    const Philox ph(p.seed);
    const double inv_total = 1.0 / p.total_weight;
    unsigned long long flipped = 0;
    const long long n4 = (p.end - p.begin) >> 2;
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n4; q += (long long)gridDim.x * blockDim.x) {
        const long long i = p.begin + (q << 2);
        const bool tail = i >= p.n_vote;
        const float4 g4 = ld_f4(p.w_global + i);
        const float g[4] = {g4.x, g4.y, g4.z, g4.w};
        int s[4] = {0, 0, 0, 0};
        double acc[4] = {0., 0., 0., 0.};
        float agg[4] = {0.f, 0.f, 0.f, 0.f};
        if (MODE == 1 && !tail) {
            constexpr int KV = KT > 0 ? KT : 1;
            float v0[KV], v1[KV], v2[KV], v3[KV];
#pragma unroll
            for (int k = 0; k < KV; ++k) {
                const float4 w = ld_f4(sh.w[k] + i);
                const float sc = sh.sc[k];
                v0[k] = (w.x - g[0]) * sc; v1[k] = (w.y - g[1]) * sc; v2[k] = (w.z - g[2]) * sc; v3[k] = (w.w - g[3]) * sc;
                s[0] += sgn(v0[k]); s[1] += sgn(v1[k]); s[2] += sgn(v2[k]); s[3] += sgn(v3[k]);
            }
            agg[0] = lower_median_fixed<KV>(v0); agg[1] = lower_median_fixed<KV>(v1);
            agg[2] = lower_median_fixed<KV>(v2); agg[3] = lower_median_fixed<KV>(v3);
        } else {
#pragma unroll 4
            for (int k = 0; k < K; ++k) {
                const float4 w = ld_f4(sh.w[k] + i);
                const float sc = tail ? 1.0f : sh.sc[k];
                const float d[4] = {(w.x - g[0]) * sc, (w.y - g[1]) * sc, (w.z - g[2]) * sc, (w.w - g[3]) * sc};
                const double wt = sh.wt[k];
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    s[c] += sgn(d[c]);
                    if (MODE == 0 || tail) acc[c] += wt * (double)d[c];
                }
            }
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                if (!(MODE == 0 || tail)) agg[c] = (float)((s[c] > 0) - (s[c] < 0));  // sign majority
            }
        }
        float out[4];
        if (tail) {
#pragma unroll
            for (int c = 0; c < 4; ++c) out[c] = (float)((double)g[c] + acc[c] * inv_total);
        } else {
            float nz[4] = {0.f, 0.f, 0.f, 0.f};
            if (p.noise_std > 0.f) {
                const float4 z = philox_normal4(ph, (uint64_t)(i >> 2), p.noise_stream);
                nz[0] = z.x * p.noise_std; nz[1] = z.y * p.noise_std; nz[2] = z.z * p.noise_std; nz[3] = z.w * p.noise_std;
            }
            float4 m4 = make_float4(0.f, 0.f, 0.f, 0.f), v4 = m4;
            if (OPT) m4 = ld_f4(p.opt_m + (i - p.state_base));
            if (OPT && p.opt_v) v4 = ld_f4(p.opt_v + (i - p.state_base));
            float m[4] = {m4.x, m4.y, m4.z, m4.w}, v[4] = {v4.x, v4.y, v4.z, v4.w};
#pragma unroll
            for (int c = 0; c < 4; ++c)   // avg keeps its fp64 mean; comed / sign values are exact in fp32
                out[c] = server_step(p, g[c], (MODE == 0) ? acc[c] * inv_total : (double)agg[c], s[c], nz[c], flipped, m[c], v[c], OPT);
            if (OPT) st_f4(p.opt_m + (i - p.state_base), make_float4(m[0], m[1], m[2], m[3]));
            if (OPT && p.opt_v) st_f4(p.opt_v + (i - p.state_base), make_float4(v[0], v[1], v[2], v[3]));
        }
        store4(p, i, out);
    }
    agg_epilogue(p, sh, flipped);
}

// =================================================================================================================================
// scalar median path: one coordinate per thread, results re-grouped by four lanes for the 16-byte (multicast) stores.
//   NT > 0 : Batcher network of NT >= K registers (padding = +inf)
//   NT == 0: bit-wise bisection select, K values staged in shared memory (use_smem) or re-read from global / L2
// =================================================================================================================================
template <int NT>
__global__ void __launch_bounds__(NT > 0 ? kAggThreads : kSelThreads) fused_aggregate_median_kernel(AggParams p, int use_smem) {
    __shared__ AggShared sh;
    extern __shared__ float stage[];                  // NT == 0 && use_smem: [K][blockDim.x]
    const int K = p.K;
    agg_prologue(p, sh, K);

    const Philox ph(p.seed);
    const double inv_total = 1.0 / p.total_weight;
    unsigned long long flipped = 0;
    const long long n = p.end - p.begin;
    const int lane = threadIdx.x & 31;
    const int m = (K - 1) / 2;                          // rank of the lower median
    // every warp walks whole 32-coordinate groups (n % 4 == 0: a 4-lane store group is all-valid or all-invalid)
    for (long long base = ((long long)blockIdx.x * blockDim.x + (threadIdx.x & ~31)); base < n; base += (long long)gridDim.x * blockDim.x) {
        const long long i = p.begin + base + lane;
        const bool valid = base + lane < n;
        const bool tail = i >= p.n_vote;
        float out = 0.f;
        if (valid) {
            const float g = p.w_global[i];
            int s = 0;
            float med = 0.f;
            if (tail) {
                double acc = 0.;
                for (int k = 0; k < K; ++k) acc += sh.wt[k] * (double)(sh.w[k][i] - g);
                out = (float)((double)g + acc * inv_total);
            } else {
                if constexpr (NT > 0) {
                    float v[NT];
#pragma unroll
                    for (int k = 0; k < NT; ++k) {
                        v[k] = INFINITY;
                        if (k < K) {
                            v[k] = (sh.w[k][i] - g) * sh.sc[k];
                            s += sgn(v[k]);
                        }
                    }
                    batcher_sort<NT>(v);
                    // the rank is a run-time value: select it with a compile-time scan (no dynamic register indexing)
#pragma unroll
                    for (int k = 0; k < NT; ++k) med = (k == m) ? v[k] : med;
                } else {
                    // answer = the (m+1)-th smallest ordered image, built bit by bit from the MSB: keep the candidate bit whenever
                    // at most m values lie strictly below the candidate prefix
                    float* mine = stage + threadIdx.x;
                    if (use_smem) {
                        for (int k = 0; k < K; ++k) {
                            const float d = (sh.w[k][i] - g) * sh.sc[k];
                            mine[(size_t)k * blockDim.x] = d;
                            s += sgn(d);
                        }
                    } else {
                        for (int k = 0; k < K; ++k) s += sgn((sh.w[k][i] - g) * sh.sc[k]);
                    }
                    uint32_t ans = 0;
                    for (int b = 31; b >= 0; --b) {
                        const uint32_t cand = ans | (1u << b);
                        int below = 0;
                        if (use_smem) {
#pragma unroll 4
                            for (int k = 0; k < K; ++k) below += ordered_bits(mine[(size_t)k * blockDim.x]) < cand;
                        } else {
#pragma unroll 4
                            for (int k = 0; k < K; ++k) below += ordered_bits((sh.w[k][i] - g) * sh.sc[k]) < cand;
                        }
                        if (below <= m) ans = cand;
                    }
                    med = from_ordered_bits(ans);
                }
                float nz = 0.f;
                if (p.noise_std > 0.f) {
                    const float4 z = philox_normal4(ph, (uint64_t)(i >> 2), p.noise_stream);   // same stream as the vector path
                    const int c = (int)(i & 3);
                    nz = (c == 0 ? z.x : c == 1 ? z.y : c == 2 ? z.z : z.w) * p.noise_std;
                }
                float* const mp = p.opt_m ? p.opt_m + (i - p.state_base) : nullptr;
                float* const vp = p.opt_v ? p.opt_v + (i - p.state_base) : nullptr;
                float m = mp ? *mp : 0.f, v = vp ? *vp : 0.f;
                out = server_step(p, g, (double)med, s, nz, flipped, m, v);
                if (mp) *mp = m;
                if (vp) *vp = v;
            }
        }
        // regroup: lanes 4j .. 4j+3 -> one 16-byte store by lane 4j
        const float o1 = __shfl_down_sync(0xffffffffu, out, 1), o2 = __shfl_down_sync(0xffffffffu, out, 2),
                    o3 = __shfl_down_sync(0xffffffffu, out, 3);
        if (valid && (lane & 3) == 0) {
            const float o[4] = {out, o1, o2, o3};
            store4(p, i, o);
        }
    }
    agg_epilogue(p, sh, flipped);
}

template <int MODE, int KT>
static cudaError_t launch_vec(const AggParams& p, int grid, cudaStream_t st) {
    if (p.opt == kOptSgd) fused_aggregate_kernel<MODE, KT, false><<<grid, kAggThreads, 0, st>>>(p);
    else fused_aggregate_kernel<MODE, KT, true><<<grid, kAggThreads, 0, st>>>(p);
    return cudaGetLastError();
}
template <int NT>
static cudaError_t launch_net(const AggParams& p, int grid, cudaStream_t st) {
    fused_aggregate_median_kernel<NT><<<grid, kAggThreads, 0, st>>>(p, 0);
    return cudaGetLastError();
}

int aggregate_max_agents() { return kMaxAgents; }

cudaError_t launch_fused_aggregate(const AggParams& p, int num_sms, cudaStream_t st) {
    if (p.K < 1 || p.K > kMaxAgents) return cudaErrorInvalidValue;
    if (((p.end - p.begin) & 3) || (p.begin & 3) || (p.n_vote & 3)) return cudaErrorInvalidValue;
    if (p.opt < kOptSgd || p.opt > kOptYogi || (p.state_base & 3) || p.state_base > p.begin) return cudaErrorInvalidValue;
    if ((p.opt != kOptSgd && !p.opt_m) || (p.opt >= kOptAdagrad && !p.opt_v)) return cudaErrorInvalidValue;
    const long long n = p.end - p.begin;
    const bool scalar = p.mode == 1 && p.K > 8;
    const long long per_block = scalar ? (p.K > 64 ? kSelThreads : kAggThreads) : 4LL * kAggThreads;
    long long want = (n + per_block - 1) / per_block;
    // all CTAs co-resident so the intra-kernel flag barriers can never starve: <= 8 per SM for the vector path, <= 2 for the
    // register-heavy networks / shared-memory staged selection
    const long long cap = (long long)num_sms * (scalar ? 2 : 8);
    const int grid = (int)(want < 1 ? 1 : (want > cap ? cap : want));
    switch (p.mode) {
        case 0: return launch_vec<0, 0>(p, grid, st);
        case 2: return launch_vec<2, 0>(p, grid, st);
        case 1:
            switch (p.K) {
                case 1: return launch_vec<1, 1>(p, grid, st);
                case 2: return launch_vec<1, 2>(p, grid, st);
                case 3: return launch_vec<1, 3>(p, grid, st);
                case 4: return launch_vec<1, 4>(p, grid, st);
                case 5: return launch_vec<1, 5>(p, grid, st);
                case 6: return launch_vec<1, 6>(p, grid, st);
                case 7: return launch_vec<1, 7>(p, grid, st);
                case 8: return launch_vec<1, 8>(p, grid, st);
                default: break;
            }
            if (p.K <= 12) return launch_net<12>(p, grid, st);
            if (p.K <= 16) return launch_net<16>(p, grid, st);
            if (p.K <= 24) return launch_net<24>(p, grid, st);
            if (p.K <= 32) return launch_net<32>(p, grid, st);
            if (p.K <= 40) return launch_net<40>(p, grid, st);
            if (p.K <= 48) return launch_net<48>(p, grid, st);
            if (p.K <= 64) return launch_net<64>(p, grid, st);
            {
                const size_t stage_bytes = (size_t)p.K * kSelThreads * sizeof(float);
                const int use_smem = stage_bytes <= 160 * 1024;            // K <= 320: values staged once, bisection out of shared memory
                static bool configured = false;
                if (!configured) {
                    RLR_CUDA_CHECK(cudaFuncSetAttribute(fused_aggregate_median_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
                    configured = true;
                }
                const int g2 = use_smem ? (grid > num_sms ? num_sms : grid) : grid;   // one CTA per SM when the stage fills shared memory
                fused_aggregate_median_kernel<0><<<g2, kSelThreads, use_smem ? stage_bytes : 0, st>>>(p, use_smem);
                return cudaGetLastError();
            }
        default: return cudaErrorInvalidValue;
    }
}

// ---- consumer side of the hand-off: acquire broadcast slices (+ seed the trainer's BatchNorm running statistics) -------------------
// One warp.  Waits until the ready words [first, last] of this rank carry `epoch` (the owners' multicast stores of those slices
// have landed in this GPU's memory), then copies tail_n floats (the BatchNorm running statistics stored behind n_vote) from the
// broadcast buffer into the trainer's working parameters.  Kernels launched after it in the stream may read those slices freely.
__global__ void __launch_bounds__(32) acquire_slices_kernel(const uint32_t* ready, int first, int last, const uint32_t* epoch_ptr,
                                                              const float* __restrict__ tail_src, float* __restrict__ tail_dst, long long tail_n) {
    if (ready) {
        const uint32_t epoch = *epoch_ptr;       // device word written by the host before the (captured) step is replayed
        for (int r = first + (int)threadIdx.x; r <= last; r += 32)
            while ((int32_t)(ld_acquire_sys(ready + r) - epoch) < 0) { __nanosleep(64); }
        __syncwarp();
        __threadfence();      // order the acquired data before the plain loads below and before dependent kernels
    }
    for (long long i = threadIdx.x; i < tail_n; i += 32) tail_dst[i] = ld_f1(tail_src + i);
}
cudaError_t launch_acquire_slices(const uint32_t* ready, int first, int last, const uint32_t* epoch, const float* tail_src, float* tail_dst,
                                  long long tail_n, cudaStream_t st) {
    if (ready && !epoch) return cudaErrorInvalidValue;
    acquire_slices_kernel<<<1, 32, 0, st>>>(ready, first, last, epoch, tail_src, tail_dst, tail_n);
    return cudaGetLastError();
}

// ---- per-agent update L2 norms  ||w_k - w_g||_2^2  (server clipping + the Norms/* diagnostics) -------------
__global__ void __launch_bounds__(256) update_sqnorm_kernel(const float* const* w_agents, const float* w_global,
                                                              long long n, double* out /*[K]*/) {
    __shared__ double scratch[32];
    const float* w = w_agents[blockIdx.y];
    double acc = 0.0;
    for (long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4; i < n; i += (long long)gridDim.x * blockDim.x * 4) {
        const float4 a = ld_f4(w + i), g = ld_f4(w_global + i);
        const float d0 = a.x - g.x, d1 = a.y - g.y, d2 = a.z - g.z, d3 = a.w - g.w;
        acc += (double)(d0 * d0 + d1 * d1) + (double)(d2 * d2 + d3 * d3);
    }
    const double tot = block_sum<double>(acc, scratch);
    if (threadIdx.x == 0) atomicAdd(out + blockIdx.y, tot);
}

cudaError_t launch_update_sqnorm(const float* const* w_agents, const float* w_global, long long n, int K, double* out,
                                 int num_sms, cudaStream_t st) {
    if (n & 3) return cudaErrorInvalidValue;
    RLR_CUDA_CHECK(cudaMemsetAsync(out, 0, sizeof(double) * K, st));
    long long want = (n / 4 + 255) / 256;
    int gx = (int)(want > num_sms * 4 ? num_sms * 4 : (want < 1 ? 1 : want));
    update_sqnorm_kernel<<<dim3(gx, K), 256, 0, st>>>(w_agents, w_global, n, out);
    return cudaGetLastError();
}

}  // namespace rlr
