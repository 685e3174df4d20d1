// Host-callable launchers of the sm_90a kernels (raw pointers + stream; no torch headers so the .cu
// translation units compile in seconds).  Python bindings live in binding.cpp.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

namespace rlr {

// Cross-GPU gate of the server step's launches (world > 1: the fused multi-GPU path).  The aggregate, distance and trust kernels open
// with the barrier-in on it (barrier_in, common.cuh); the aggregate kernel also runs its barrier-out or hand-off on these words.
struct Gate {
    uint32_t* const* flag_ptrs;     // [world] peer-mapped signal words, 3*world per rank (in / out barrier, broadcast-ready words)
    uint32_t* local_sync;           // [2] intra-GPU: ready flag, finished-CTA counter
    int rank, world;
    uint32_t epoch;                 // monotonically increasing per call
};

struct AggParams {
    const float* const* w_agents;   // [K] device pointers: each participant's flat params (local or peer-mapped)
    const double* weights;          // [K] data sizes n_k
    const float* scales;            // [K] optional per-agent update scale (server clipping) or nullptr
    double total_weight;            // sum_k n_k
    const float* w_global;          // current global params (local copy)
    float* const* out_ptrs;         // [n_out] destinations of the new global params (1 = local or multicast)
    __nv_bfloat16* const* out_bf16_ptrs;  // optional bf16 shadows (same count) or nullptr
    int n_out;
    int use_multimem;               // out_ptrs[0] is an NVLS multicast address
    int K;
    long long begin, end;           // coordinate slice owned by this rank (multiples of 4)
    long long n_vote;               // coordinates >= n_vote: plain weighted mean (BN statistics)
    int mode;                       // 0 avg, 1 comed, 2 sign
    int theta;                      // RLR threshold (0 = off)
    float server_lr;
    float noise_std;
    uint64_t seed, noise_stream;
    unsigned long long* flipped;    // optional counter of coordinates with negated lr
    Gate gate;
    int handoff;                   // 1: publish this rank's slice in the peers' ready words (flag slot 2*world + rank) instead of the barrier-out
    // server optimizer applied to the voted coordinates (0 sgd, 1 momentum, 2 adagrad, 3 adam, 4 yogi); state fp32, indexed by i - state_base
    int opt;
    double beta1, beta2, tau;
    float* opt_m;                   // first moment (every optimizer but sgd) or nullptr
    float* opt_v;                   // second moment (adagrad / adam / yogi) or nullptr
    long long state_base;           // coordinate of opt_m[0] / opt_v[0] (multiple of 4; = begin when the state is sharded)
};
cudaError_t launch_fused_aggregate(const AggParams& p, int num_sms, cudaStream_t st);
int aggregate_max_agents();         // capacity of the kernel's participant tables
// consumer side of the hand-off: wait for ready words [first, last] >= epoch (ready may be null), then copy the BatchNorm-statistics tail
cudaError_t launch_acquire_slices(const uint32_t* ready, int first, int last, const uint32_t* epoch, const float* tail_src, float* tail_dst,
                                  long long tail_n, cudaStream_t st);

// ---- participant selection (Krum / Multi-Krum): pairwise squared distances of the participants' updates ----------------------------
// out[i][j] = sum_{begin <= c < end} (x_i[c] - x_j[c])^2 in fp64 ([K][K], symmetric, zero diagonal), x_k = w_k without scales and
// x_k = (w_k - w_global) * scales[k] with them.  Fixed-order sums, no atomics: bitwise reproducible.
struct DistParams {
    const float* const* w_agents;   // [K] device pointers (local or peer-mapped)
    const float* w_global;          // only read with scales
    const float* scales;            // [K] server clipping scales or nullptr
    long long begin, end;           // coordinate range (multiples of 4), already clipped to [0, n_vote)
    int K;
    Gate gate;                      // world > 1: the aggregation's barrier-in
};
cudaError_t launch_pairwise_sqdist(const DistParams& p, double* out, int num_sms, cudaStream_t st);
// FLAME's Gram matrix of the updates: out[i][j] = sum_{begin <= c < end} Δi[c] Δj[c] in fp64 ([K][K], symmetric, diagonal = squared
// update norms), Δk = w_k - w_global formed in fp32.  Same kernel, tiles and fixed-order sums as the distances; needs w_global, no scales.
cudaError_t launch_pairwise_gram(const DistParams& p, double* out, int num_sms, cudaStream_t st);

// ---- FLTrust: each participant's update against the server's root update Δ0 = w_ref - w_global -----------------------------------------
// out[k] = sum_c Δk[c] Δ0[c], out[K + k] = sum_c Δk[c]^2, out[2K] = sum_c Δ0[c]^2 over [begin, end), fp64 [2K + 1], Δk = w_k - w_global.
// Fixed-order sums, no atomics: bitwise reproducible.
struct TrustParams {
    const float* const* w_agents;   // [K] device pointers (local or peer-mapped)
    const float* w_ref;             // the root job's parameters (local or peer-mapped)
    const float* w_global;          // this rank's global parameters
    long long begin, end;           // coordinate range (multiples of 4), already clipped to [0, n_vote)
    int K;
    Gate gate;                      // world > 1: the aggregation's barrier-in
};
cudaError_t launch_trust_stats(const TrustParams& p, double* out, int num_sms, cudaStream_t st);

// ---- RFA (smoothed Weiszfeld geometric median): each participant's squared distance to the b-weighted mean of the updates -------------
// out[k] = sum_{begin <= c < end} (x_k[c] - z[c])^2 in fp64 [K], z[c] = sum_j b[j] x_j[c] (sum_j b[j] = 1), x_k = w_k without scales and
// x_k = (w_k - w_global) * scales[k] with them.  Fixed-order sums, no atomics: bitwise reproducible.
struct RfaParams {
    const float* const* w_agents;   // [K] device pointers (local or peer-mapped)
    const double* b;                // [K] normalised weights
    const float* w_global;          // only read with scales
    const float* scales;            // [K] server clipping scales or nullptr
    long long begin, end;           // coordinate range (multiples of 4), already clipped to [0, n_vote)
    int K;
    Gate gate;                      // world > 1: the aggregation's barrier-in
};
cudaError_t launch_rfa_sqdist(const RfaParams& p, double* out, int num_sms, cudaStream_t st);

// ---- data path ---------------------------------------------------------------------------------------
// out_kind: 0 fp32, 1 bf16.  nchw: output layout NCHW (Cpad ignored) else NHWC with channels padded to c_pad.
// Both gathers: crop_pad > 0 or flip turns on the training augmentation (AugSpec, common.cuh): sample b of the batch is drawn
// at position (cursor ? *cursor : start) + b from the Philox stream word *aug_stream under key seed.
cudaError_t launch_gather_normalize(const void* data, int in_is_float, const int64_t* idx, const int* cursor,
                                    const int64_t* targets, void* out, int out_kind, int64_t* out_labels, int B, int H,
                                    int W, int C, int c_pad, int nchw, const float* mean, const float* stdv,
                                    int crop_pad, int flip, long long seed, const long long* aug_stream, long long start,
                                    cudaStream_t st);
// gather + normalise + im2col for the stem conv (C*k*k <= 64): A[B*Ho*Wo][64] bf16, (tap, channel) column order, zero padded
cudaError_t launch_gather_im2col(const void* data, int in_is_float, const int64_t* idx, const int* cursor, const int64_t* targets,
                                 __nv_bfloat16* A, int64_t* out_labels, int B, int H, int W, int C, int k, int pad, const float* mean,
                                 const float* stdv, int crop_pad, int flip, long long seed, const long long* aug_stream, long long start,
                                 cudaStream_t st);
cudaError_t launch_stamp_pixels(void* data, int is_float, const int64_t* sel, int S, const int* rows, const int* cols,
                                const float* vals, int P, int H, int W, int C, int mode, cudaStream_t st);
cudaError_t launch_advance_cursor(int* cursor, int delta, long long* step /*optional: += 1*/, cudaStream_t st);
// dst[R][Kp] (bf16) = src[R][K] zero-padded along the row | dst[R][K] (fp32) += src[R][Kp][:K]
cudaError_t launch_pad_rows(const __nv_bfloat16* src, __nv_bfloat16* dst, long long R, int K, int Kp, int num_sms, cudaStream_t st);
cudaError_t launch_unpad_add(const float* src, float* dst, long long R, int K, int Kp, int num_sms, cudaStream_t st);

// ---- optimiser over flat buffers -------------------------------------------------------------------------
cudaError_t launch_round_init(const float* w_global, float* w_local, __nv_bfloat16* w_bf16, float* mom, long long n,
                              cudaStream_t st);
cudaError_t launch_sqnorm(const float* x, long long n, double* out /*accumulates*/, int num_sms, cudaStream_t st);
cudaError_t launch_sgd_step(float* w, const float* g, float* m, const float* w0, __nv_bfloat16* w_bf16, long long n,
                            float lr, float momentum, float max_grad_norm, const double* g_sqnorm, double* d_sqnorm,
                            int num_sms, cudaStream_t st, long long n_pgd = 0 /*PGD norm over [0, n_pgd); 0 = n*/,
                            const float* w_in = nullptr /*first step of a round: read params from w_in, momentum = 0, keep w[n_pgd:]*/);
cudaError_t launch_pgd_project(float* w, const float* w0, __nv_bfloat16* w_bf16, long long n, float clip,
                               const double* d_sqnorm, int num_sms, cudaStream_t st, long long n_pgd = 0);

// ---- loss / evaluation -----------------------------------------------------------------------------------
// logits [B,C] (kind 0 fp32 / 1 bf16); writes dlogits (same kind, scaled by 1/B) and accumulates loss_sum / correct.
cudaError_t launch_softmax_xent(const void* logits, int kind, const int64_t* labels, void* dlogits, float* loss_sum,
                                int* correct, int B, int C, float grad_scale, cudaStream_t st);
cudaError_t launch_eval_metrics(const void* logits, int kind, const int64_t* labels, int B, int C, double* loss_sum,
                                long long* confusion /*[C*C]*/, cudaStream_t st);

}  // namespace rlr
