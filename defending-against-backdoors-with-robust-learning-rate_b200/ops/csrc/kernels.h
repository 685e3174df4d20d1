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
// FoolsGold's Gram matrix of history rows taken as they are: out[i][j] = sum_{begin <= c < end} w_agents[i][c] w_agents[j][c] in fp64
// (the w_agents are the candidates' history rows, offset so that absolute coordinates index them).  Same kernel, tiles and fixed-order
// sums as the distances; reads neither w_global nor scales.
cudaError_t launch_history_gram(const DistParams& p, double* out, int num_sms, cudaStream_t st);
// DnC: the participants' updates at T sampled coordinate sets, centred per coordinate.  For iteration t the coordinates are
// sample[t][ranges[2t] .. ranges[2t + 1]) (sorted, < 2^31); y[t][k][q] = fp32(x_k - mu) at the q-th of them, x_k = (w_k - w_global)
// (* scales[k]) in fp64 and mu the fp64 mean of the finite x_k in ascending k; rows zero-padded to len_pad (a multiple of 4), so
// launch_history_gram takes them as its table.  No reductions across threads: bitwise reproducible.
struct DncParams {
    const float* const* w_agents;   // [K] device pointers (local or peer-mapped)
    const float* w_global;          // this rank's global parameters
    const float* scales;            // [K] server clipping scales or nullptr
    const int* sample;              // [T][stride] sorted coordinates
    const int* ranges;              // [T][2] position range [lo, hi) of row t that this launch gathers (hi - lo <= len_pad)
    float* y;                       // [T][K][len_pad]
    int T, K, stride, len_pad;
    Gate gate;                      // world > 1: the aggregation's barrier-in
};
cudaError_t launch_dnc_gather(const DncParams& p, int num_sms, cudaStream_t st);

// ---- FoolsGold: each candidate's update folded into its agent's history row ------------------------------------------------------
// rows[k][c] <- fp32(rows[k][c] + fp32(w_agents[k][c] - w_global[c])) for begin <= c < end.  Exact fp32: bitwise reproducible.
struct HistParams {
    const float* const* w_agents;   // [K] device pointers (local or peer-mapped)
    float* const* rows;             // [K] history rows, offset so that absolute coordinates index them
    const float* w_global;          // this rank's global parameters
    long long begin, end;           // coordinate range (multiples of 4), already clipped to [0, n_vote)
    int K;
    Gate gate;                      // world > 1: the aggregation's barrier-in
};
cudaError_t launch_history_accumulate(const HistParams& p, int num_sms, cudaStream_t st);

// ---- FLDetector (fldetector.cu): the global-update ring, the Hessian-vector product and the prediction pass --------------------------
// ring: s[c] = fp32(w_g[c] - w_prev[c]) (s may be null), then w_prev[c] <- w_g[c], over [begin, end); w_prev and s offset so that absolute
// coordinates index them.
cudaError_t launch_fld_ring(const float* w_g, float* w_prev, float* s, long long begin, long long end, int num_sms, cudaStream_t st);
// Hv[c] = fp32(sum_{r < rows} coef[r] * ring[r][c]), fp64 products and sums each rounded on their own, r ascending.
cudaError_t launch_fld_hvp(const float* const* ring, const double* coef, int rows, float* hv, long long begin, long long end, int num_sms,
                           cudaStream_t st);
// per candidate k over [begin, end): u = fp32(w_agents[k][c] - w_global[c]); with hv: out[k] = sum_c fp32(fp32(rows[k][c] + hv[c]) - u)^2
// in fp64 (fixed-order sums); then rows[k][c] <- u.  Without hv only the rows are written (out untouched, may be null).
struct FldParams {
    const float* const* w_agents;   // [K] device pointers (local or peer-mapped)
    float* const* rows;             // [K] last-update rows, offset so that absolute coordinates index them
    const float* w_global;          // this rank's global parameters
    const float* hv;                // Hv, offset so that absolute coordinates index it, or nullptr (record only)
    long long begin, end;           // coordinate range (multiples of 4), already clipped to [0, n_vote)
    int K;
    Gate gate;                      // world > 1: the aggregation's barrier-in
};
cudaError_t launch_fld_predict(const FldParams& p, double* out, int num_sms, cudaStream_t st);

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

// ---- colluding attackers (collude.cu): ALIE and Min-Max / Min-Sum craft one update from the round's honest ones ---------------------
// Per coordinate of [begin, end): mu, sig (ddof 1) and the corrupt mean xc of x_k = w_k - w_global in fp64, the direction u and the
// crafted m (the statement is in collude.cu).  stats: out[2H + 1] = (a_k, e_k for the H honest participants, q).  write: every w_out slot
// gets fp32(w_global + m) and out[1] = sum (m - mu)^2.  Fixed-order sums, no atomics: bitwise reproducible.
struct ColludeParams {
    const float* const* w_agents;   // [H + C] device pointers (local or peer-mapped): the honest participants, then the corrupt ones
    float* const* w_out;            // [n_out] slots the write pass fills with the crafted update (may be the corrupt inputs)
    const float* w_global;
    long long begin, end;           // coordinate range (multiples of 4), already clipped to [0, n_vote)
    int H, C, n_out;
    int mode;                       // 0 alie, 1 minmax / minsum (m = mu - gamma u)
    int dir;                        // u: 0 backdoor (mu - xc), 1 std (sig), 2 sign (sign mu), 3 unit (mu)
    double z, gamma;                // alie's z; the host's gamma* of minmax / minsum
    Gate gate;                      // world > 1: the aggregation's barrier-in
};
cudaError_t launch_collude_stats(const ColludeParams& p, double* out, int num_sms, cudaStream_t st);
cudaError_t launch_collude_write(const ColludeParams& p, double* out, int num_sms, cudaStream_t st);

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
// mask (optional): gradient mask bit words (bit c % 32 of word c / 32 set = g[c] reads as zero) over [0, n_mask) for sqnorm and over
// [0, n_pgd) for sgd_step; pgd_project leaves masked coordinates untouched
cudaError_t launch_sqnorm(const float* x, long long n, double* out /*accumulates*/, int num_sms, cudaStream_t st,
                          const uint32_t* mask = nullptr, long long n_mask = 0);
cudaError_t launch_sgd_step(float* w, const float* g, float* m, const float* w0, __nv_bfloat16* w_bf16, long long n,
                            float lr, float momentum, float max_grad_norm, const double* g_sqnorm, double* d_sqnorm,
                            int num_sms, cudaStream_t st, long long n_pgd = 0 /*PGD norm over [0, n_pgd); 0 = n*/,
                            const float* w_in = nullptr /*first step of a round: read params from w_in, momentum = 0, keep w[n_pgd:]*/,
                            const uint32_t* mask = nullptr);
cudaError_t launch_pgd_project(float* w, const float* w0, __nv_bfloat16* w_bf16, long long n, float clip,
                               const double* d_sqnorm, int num_sms, cudaStream_t st, long long n_pgd = 0, const uint32_t* mask = nullptr);

// ---- model-poisoning attackers (attack.cu) ----------------------------------------------------------------------------------------
// Neurotoxin: a[c] = bits(|fp32(w_g[c] - w_prev[c])|) over [0, n_vote); tau = the k-th largest a (with multiplicity) by an on-device
// radix select; mask = {c : a[c] >= tau, a[c] > 0} as ceil(n_vote/32) bit words; *count = |mask|; then w_prev <- w_g[:n_vote].
// k = 0: empty mask.  No host sync, no float atomics: bitwise reproducible.  n_vote % 4 == 0, 0 <= k <= n_vote < 2^32.
cudaError_t launch_neurotoxin_mask(const float* w_g, float* w_prev, long long n_vote, long long k, uint32_t* mask, long long* count,
                                   int num_sms, cudaStream_t st);
// boosted update: slot[c] = fp32((double)w_g[c] + gamma * (double)fp32(slot[c] - w_g[c])) over [0, n_vote), each fp64 operation
// rounded on its own
cudaError_t launch_boost_update(float* slot, const float* w_g, long long n_vote, double gamma, int num_sms, cudaStream_t st);
// attack schedules: data[idx[i]] <-> side[i] (row_bytes bytes each) and targets[idx[i]] <-> side_targets[i] for i < n, in one launch.
// The idx must be distinct and in range (checked by the caller once, when the side copy is built).  n = 0 launches nothing.
cudaError_t launch_swap_samples(void* data, long long* targets, const long long* idx, void* side, long long* side_targets, long long n,
                                long long row_bytes, int num_sms, cudaStream_t st);

// ---- loss / evaluation -----------------------------------------------------------------------------------
// logits [B,C] (kind 0 fp32 / 1 bf16); writes dlogits (same kind, scaled by 1/B) and accumulates loss_sum / correct.
cudaError_t launch_softmax_xent(const void* logits, int kind, const int64_t* labels, void* dlogits, float* loss_sum,
                                int* correct, int B, int C, float grad_scale, cudaStream_t st);
cudaError_t launch_eval_metrics(const void* logits, int kind, const int64_t* labels, int B, int C, double* loss_sum,
                                long long* confusion /*[C*C]*/, cudaStream_t st);

}  // namespace rlr
