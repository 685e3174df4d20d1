// FoolsGold's update history (Fung, Yoon and Beschastnikh, "The Limitations of Federated Learning in Sybil Settings", RAID 2020): every
// agent a keeps the sum of the updates it submitted in a row H[a] of fp32, and each round every candidate k folds its update in,
//   H[a_k][c] <- fp32(H[a_k][c] + fp32(w_k[c] - w_global[c])),   begin <= c < end.
// Both operations are single fp32 roundings, so any correct implementation produces the same bits.  The Gram matrix of the updated
// rows is the distance kernel of select.cu on the rows as they are (pairwise_sqdist_kernel<true, true>).  The two are separate
// launches: a participant sits in several Gram tiles, and one tile's CTA would otherwise read a row that another tile has rewritten.
//
// A history row may hold only this rank's coordinate slice (the fused multi-GPU path): its pointer is offset so that absolute
// coordinates index it, and only [begin, end) is ever touched.
//
// Work decomposition: grid.x = coordinate splits (about two waves; one wave on the fused multi-GPU path, where every CTA has to be
// resident while it waits for the cross-GPU barrier-in), grid.y = groups of kHistGroup candidates.  A thread loads w_global for its
// float4 once and reuses it for every candidate of its group.  Nothing is reduced: no workspace and no atomics.
#include "common.cuh"
#include "kernels.h"

namespace rlr {

constexpr int kHistThreads = 256;
constexpr int kHistGroup = 8;                           // candidates per CTA
constexpr int kHistMaxGroups = 65535;                   // grid.y

struct HistKernelParams {
    HistParams p;
    long long span;                                     // coordinates per split (multiple of 4)
};

__global__ void __launch_bounds__(kHistThreads) history_accumulate_kernel(HistKernelParams kp) {
    const HistParams& p = kp.p;
    const int k0 = blockIdx.y * kHistGroup;
    const int nk = min(kHistGroup, p.K - k0);
    const float* wp[kHistGroup];
    float* hp[kHistGroup];
#pragma unroll
    for (int j = 0; j < kHistGroup; ++j) {
        wp[j] = j < nk ? p.w_agents[k0 + j] : nullptr;
        hp[j] = j < nk ? p.rows[k0 + j] : nullptr;
    }

    barrier_in(p.gate, blockIdx.x == 0 && blockIdx.y == 0);

    const long long lo = p.begin + (long long)blockIdx.x * kp.span;
    const long long hi = min(p.end, lo + kp.span);
    for (long long i = lo + 4LL * threadIdx.x; i < hi; i += 4LL * kHistThreads) {
        const float4 g = ld_f4(p.w_global + i);
        float4 w[kHistGroup], h[kHistGroup];
#pragma unroll
        for (int j = 0; j < kHistGroup; ++j) {
            if (j < nk) {
                w[j] = ld_f4(wp[j] + i);
                h[j] = ld_f4(hp[j] + i);
            }
        }
#pragma unroll
        for (int j = 0; j < kHistGroup; ++j) {
            if (j < nk) {
                const float4 d = make_float4(w[j].x - g.x, w[j].y - g.y, w[j].z - g.z, w[j].w - g.w);
                st_f4(hp[j] + i, make_float4(h[j].x + d.x, h[j].y + d.y, h[j].z + d.z, h[j].w + d.w));
            }
        }
    }
}

cudaError_t launch_history_accumulate(const HistParams& p, int num_sms, cudaStream_t st) {
    if (p.K < 1 || (p.K + kHistGroup - 1) / kHistGroup > kHistMaxGroups || !p.w_global || !p.w_agents || !p.rows)
        return cudaErrorInvalidValue;
    if ((p.begin & 3) || (p.end & 3) || p.end < p.begin || !gate_ok(p.gate)) return cudaErrorInvalidValue;
    static int occ = 0;
    if (!occ) {
        RLR_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, history_accumulate_kernel, kHistThreads, 0));
        occ = occ < 1 ? 1 : occ;
    }
    HistKernelParams kp{};
    kp.p = p;
    const int groups = (p.K + kHistGroup - 1) / kHistGroup;
    const long long len = p.end - p.begin;
    const long long splits = coord_splits(len, groups, (long long)occ * num_sms, p.gate.world);
    kp.span = ((len + splits - 1) / splits + 3) & ~3LL;
    history_accumulate_kernel<<<dim3((unsigned)splits, (unsigned)groups), kHistThreads, 0, st>>>(kp);
    return cudaGetLastError();
}

}  // namespace rlr
