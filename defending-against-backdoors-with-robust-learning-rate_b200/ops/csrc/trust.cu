// Per-participant statistics of FLTrust (Cao et al., NDSS 2021) against the server's root update Δ0 = w_ref - w_global:
//   out[k] = d_k = sum_c Δk[c] Δ0[c],   out[K + k] = q_k = sum_c Δk[c]^2,   out[2K] = q0 = sum_c Δ0[c]^2,   Δk = w_k - w_global,
// over the coordinates [begin, end).  The dot product is formed per coordinate: the Gram identity Δk.Δ0 = (|Δk|^2 + |Δ0|^2 -
// |w_k - w_ref|^2) / 2 cancels catastrophically when the cosine is near 0, which is where the trust score's ReLU decides whether a
// participant counts (and honest cosines are small in high dimension).
// With w_ref = w_global (Δ0 = 0) the q_k are the squared update norms of server clipping and the Norms/* diagnostics (ops.update_norms).
//
// Work decomposition:
//   grid.x  coordinate splits, sized so the grid covers about two waves (one wave on the fused multi-GPU path, where every CTA has to
//           be resident while it waits for the cross-GPU barrier-in),
//   grid.y  groups of kTrustGroup participants.
// A thread forms Δ0 and loads w_global for its float4 once and reuses them for every participant of its group, so each participant's
// vector is read exactly once and w_ref / w_global are read once per group.  Products are accumulated in fp32 over at most 256
// coordinates per thread, then folded into fp64.  The CTA reduction has a fixed order (warp butterflies, then the warps in order), every
// (split, group) CTA writes its values to its split's [2K + 1] workspace slot and launch_ordered_sum adds the slots in split order.
// No atomics: the statistics are bitwise identical from run to run.
#include "common.cuh"
#include "kernels.h"

namespace rlr {

constexpr int kTrustThreads = 256;
constexpr int kTrustGroup = 8;                          // participants per CTA
constexpr int kTrustFold = 64;                          // float4 groups (256 coordinates) per thread between fp64 folds
constexpr int kTrustVals = 2 * kTrustGroup + 1;         // (d_k, q_k) of the group + q0
constexpr int kTrustMaxAgents = 1024;

struct TrustKernelParams {
    TrustParams p;
    long long span;                                     // coordinates per split (multiple of 4)
    double* ws;                                         // [splits][2K + 1]
};

__global__ void __launch_bounds__(kTrustThreads) trust_stats_kernel(TrustKernelParams kp) {
    __shared__ double red[kTrustThreads / kWarp][kTrustVals];
    const TrustParams& p = kp.p;
    const int tid = threadIdx.x, K = p.K;
    const int k0 = blockIdx.y * kTrustGroup;
    const int nk = min(kTrustGroup, K - k0);
    const float* wp[kTrustGroup];
#pragma unroll
    for (int j = 0; j < kTrustGroup; ++j) wp[j] = j < nk ? p.w_agents[k0 + j] : nullptr;

    barrier_in(p.gate, blockIdx.x == 0 && blockIdx.y == 0);

    double dd[kTrustGroup], qd[kTrustGroup], q0d = 0.0;
#pragma unroll
    for (int j = 0; j < kTrustGroup; ++j) { dd[j] = 0.0; qd[j] = 0.0; }
    float df[kTrustGroup], qf[kTrustGroup], q0f = 0.f;
#pragma unroll
    for (int j = 0; j < kTrustGroup; ++j) { df[j] = 0.f; qf[j] = 0.f; }

    const long long lo = p.begin + (long long)blockIdx.x * kp.span;
    const long long hi = min(p.end, lo + kp.span);
    int since = 0;
    for (long long i = lo + 4LL * tid; i < hi; i += 4LL * kTrustThreads) {
        const float4 g = ld_f4(p.w_global + i);
        const float4 r = ld_f4(p.w_ref + i);
        const float4 e = make_float4(r.x - g.x, r.y - g.y, r.z - g.z, r.w - g.w);
        q0f = __fmaf_rn(e.x, e.x, q0f); q0f = __fmaf_rn(e.y, e.y, q0f); q0f = __fmaf_rn(e.z, e.z, q0f); q0f = __fmaf_rn(e.w, e.w, q0f);
        float4 w[kTrustGroup];
#pragma unroll
        for (int j = 0; j < kTrustGroup; ++j) w[j] = j < nk ? ld_f4(wp[j] + i) : g;
#pragma unroll
        for (int j = 0; j < kTrustGroup; ++j) {
            const float x = w[j].x - g.x, y = w[j].y - g.y, z = w[j].z - g.z, u = w[j].w - g.w;
            df[j] = __fmaf_rn(x, e.x, df[j]); df[j] = __fmaf_rn(y, e.y, df[j]); df[j] = __fmaf_rn(z, e.z, df[j]); df[j] = __fmaf_rn(u, e.w, df[j]);
            qf[j] = __fmaf_rn(x, x, qf[j]); qf[j] = __fmaf_rn(y, y, qf[j]); qf[j] = __fmaf_rn(z, z, qf[j]); qf[j] = __fmaf_rn(u, u, qf[j]);
        }
        if (++since == kTrustFold) {
            since = 0;
            q0d += (double)q0f; q0f = 0.f;
#pragma unroll
            for (int j = 0; j < kTrustGroup; ++j) { dd[j] += (double)df[j]; qd[j] += (double)qf[j]; df[j] = 0.f; qf[j] = 0.f; }
        }
    }
    q0d += (double)q0f;
#pragma unroll
    for (int j = 0; j < kTrustGroup; ++j) { dd[j] += (double)df[j]; qd[j] += (double)qf[j]; }

    // fixed-order CTA reduction: butterfly within each warp, then the warps in order
    const int lane = tid & (kWarp - 1), warp = tid / kWarp;
#pragma unroll
    for (int j = 0; j < kTrustGroup; ++j) {
        dd[j] = warp_sum(dd[j]);
        qd[j] = warp_sum(qd[j]);
    }
    q0d = warp_sum(q0d);
    if (lane == 0) {
#pragma unroll
        for (int j = 0; j < kTrustGroup; ++j) { red[warp][j] = dd[j]; red[warp][kTrustGroup + j] = qd[j]; }
        red[warp][2 * kTrustGroup] = q0d;
    }
    __syncthreads();
    if (tid < kTrustVals) {
        double v = red[0][tid];
        for (int w = 1; w < kTrustThreads / kWarp; ++w) v += red[w][tid];
        double* const out = kp.ws + (size_t)blockIdx.x * (2 * K + 1);
        if (tid < kTrustGroup) {
            if (tid < nk) out[k0 + tid] = v;
        } else if (tid < 2 * kTrustGroup) {
            if (tid - kTrustGroup < nk) out[K + k0 + tid - kTrustGroup] = v;
        } else if (blockIdx.y == 0) {
            out[2 * K] = v;
        }
    }
}

cudaError_t launch_trust_stats(const TrustParams& p, double* out, int num_sms, cudaStream_t st) {
    if (p.K < 1 || p.K > kTrustMaxAgents || !p.w_ref || !p.w_global) return cudaErrorInvalidValue;
    if ((p.begin & 3) || (p.end & 3) || p.end < p.begin || !gate_ok(p.gate)) return cudaErrorInvalidValue;
    static int occ = 0;
    if (!occ) {
        RLR_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, trust_stats_kernel, kTrustThreads, 0));
        occ = occ < 1 ? 1 : occ;
    }
    TrustKernelParams kp{};
    kp.p = p;
    const int groups = (p.K + kTrustGroup - 1) / kTrustGroup;
    const long long len = p.end - p.begin;
    const long long nvals = 2LL * p.K + 1;
    const long long splits = coord_splits(len, groups, (long long)occ * num_sms, p.gate.world);
    kp.span = ((len + splits - 1) / splits + 3) & ~3LL;
    Scratch ws((size_t)(splits * nvals) * sizeof(double), st);
    kp.ws = ws.as<double>();
    RLR_CUDA_CHECK(cudaMemsetAsync(out, 0, (size_t)nvals * sizeof(double), st));
    trust_stats_kernel<<<dim3((unsigned)splits, (unsigned)groups), kTrustThreads, 0, st>>>(kp);
    RLR_CUDA_CHECK(cudaGetLastError());
    return launch_ordered_sum(out, kp.ws, (int)splits, nvals, st);
}

}  // namespace rlr
