// wgmma / TMA GEMM + implicit-GEMM convolution launchers (gemm.cu, wgrad.cu) and the memory-bound layer kernels
// (the tensor-core kernels keep their historical umma_* names; all of them issue Hopper wgmma, see wgmma.cuh)
// (norm.cu).  Raw pointers + stream; bindings in gemm_binding.cpp.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

#include "dropspec.h"

namespace rlr {

// conv epilogues reduce per-channel statistics into one of kStatSlots partial buffers ([slots][2][C]) chosen by CTA index, so
// same-address atomics in L2 are spread 16x; bn_finalize sums the slots.
constexpr int kStatSlots = 16;

struct ConvGemmParams {
    int M, N, num_kb;
    int mode;                  // 0 plain [M][K] A operand, 1 implicit conv (4-D NHWC A operand)
    int cblocks;               // Cin / 64
    int TW, TH, TN;            // output tile = TW x TH x TN pixels (= 128)
    int Ho, Wo, NB;
    int tiles_w, tiles_h;
    int ntaps;
    int in_stride;             // input pixel of output pixel o and tap t is in_stride * o + d[t]: 2 = strided TMA box (element strides)
    int out_stride, out_ph, out_pw, OutH, OutW;   // output pixel (h, w) of the Ho x Wo grid is stored at (out_stride*h + out_ph, ...)
    int8_t dh[9], dw[9];       // per tap: input row / col offset relative to the output pixel (in plane coordinates)
    int dn[9];                 // per tap: image offset (parity plane * NB) for strided convs
    int b_mn;                  // 1: B operand is read MN-major straight from the un-transposed filter (data gradients)
    int wtap[9];               // b_mn: filter tap that k-block tap t multiplies (flipped / parity-selected)
    int wcols;                 // b_mn: columns per filter tap in the 2-D filter view (= Cin of the forward conv)
    // stem GEMM (tiny-K first layer, mode 0, one k-block): the B tile is NOT loaded by TMA but gathered by the producer warp from the
    // un-padded bf16 filter b_src[N][b_ld] (b_kvalid <= 64 valid columns, zero beyond) and written in the 128-byte-swizzled operand layout.
    // With wait_flags the producer first acquires the broadcast-ready words [wait_lo, wait_hi] (>= *wait_epoch): b_src then points into
    // the NVLS-multicast parameter shadow that the aggregation kernels of ALL GPUs are still filling -- the first local-forward GEMM of
    // a round starts as soon as the slice holding its filter has landed (broadcast (+) first-GEMM fusion, parallel/fused_agg.py).
    DropSpec drop;             // thr != 0: dropout fused into the epilogue (after bias / ReLU): keep-mask of output element (row * ldc + col), common.cuh
    int tma_store;             // 1: epilogue writes the tile with TMA tensor stores from a swizzled staging tile (tmC valid; no accumulate / stats)
    int split_prod;            // 1: two TMA producer threads per CTA (warp 0 loads A, warp 2 loads B): two request streams into the TMA unit
    long long* dbg;            // optional [CTAs][8] timeline (globaltimer ns): entry, setup done, first TMA issued, first data landed,
                               // all MMAs issued, accumulator complete, epilogue done, SM id  (scripts/trace_conv.py)
    const __nv_bfloat16* b_src;
    int b_ld, b_kvalid;
    const uint32_t* wait_flags;
    int wait_lo, wait_hi;
    const uint32_t* wait_epoch;
    void* out;                 // bf16 [M][ldc]
    int ldc;
    const float* bias;         // [N] or null
    float* stats;              // [slots][2][N] (sum, sum of squares) partial buffers or null
    int stat_slots;            // TMA-store epilogue: CTA b adds into slot b % stat_slots (0 -> kStatSlots); the caller reduces over that prefix
    int relu, accumulate;
};

cudaError_t launch_gemm_bf16(const void* A, const void* B, void* out, int M, int N, int K, int lda, int ldb, int ldc,
                             const float* bias, int relu, int accumulate, float* stats, cudaStream_t st, const DropSpec* drop = nullptr);
// stem GEMM: out[M][N] = A[M][64] * pad64(W[N][kvalid])^T (+bias)(relu); W is read un-padded by the producer warp (optionally after
// acquiring broadcast-ready flags [wait_lo, wait_hi] >= *wait_epoch -- see ConvGemmParams::b_src)
cudaError_t launch_stem_gemm_bf16(const void* A, const void* W, void* out, int M, int N, int kvalid, int ldw, const float* bias, int relu,
                                  float* stats, const uint32_t* wait_flags, int wait_lo, int wait_hi, const uint32_t* wait_epoch,
                                  cudaStream_t st);
// programmatic dependent launch for the hot kernels (common.cuh: launch_kernel / pdl_wait); default: RLR_PDL env, off
void set_pdl(int on);
// gemm_splitk.cu: small-M / deep-K GEMM, grid.z CTAs share a tile's k range and store fp32 partials into per-split slots of stream
// scratch memory, then one finishing pass adds them in split order, applies bias / ReLU and packs bf16 (`ws` is not used)
cudaError_t launch_gemm_splitk_bf16(const void* A, const void* B, void* out, float* ws, int M, int N, int K, const float* bias, int relu,
                                    int num_sms, cudaStream_t st, const DropSpec* drop = nullptr);
// opt-in persistent tile scheduler for the generic conv / GEMM kernel (gemm_persistent.cu); default: RLR_PERSISTENT_CONV env
void set_persistent_conv(int on);
// three CTAs per SM: level 0 never, 1 (default) for the 64-wide tile (RLR_CONV_OCC3 env; higher levels select 1)
void set_conv_occ3(int level);
// per-CTA timeline buffer for the NEXT launches of the generic conv / GEMM kernel (nullptr = off); see ConvGemmParams::dbg
void set_conv_tma_store(int on);           // epilogue via TMA tensor stores (default on; RLR_TMA_STORE=0)
void set_conv_split_producer(int on);      // experiment: two TMA producer threads per CTA (RLR_SPLIT_PRODUCER env)
void set_conv_trace(long long* buf);
long long* conv_trace_buf();
cudaError_t launch_conv_bf16(const void* x, const void* w, void* out, int NB, int planes, int Hin, int Win, int Cin, int Ho, int Wo,
                             int Cout, int ldc, int ntaps, const int* dh, const int* dw, const int* dplane, const float* bias,
                             int relu, int accumulate, float* stats, cudaStream_t st, const int* wtap = nullptr, int w_taps_total = 0,
                             int in_stride = 1, int out_stride = 1, int out_ph = 0, int out_pw = 0);

// ---- conv_halo.cu: persistent 3x3/s1/p1 conv for 64 input channels with smem halo reuse + resident filter ------------------
cudaError_t launch_conv3x3_halo_bf16(const void* x, const void* w, void* out, int NB, int Hin, int Win, int H, int W, int Cout, const float* bias,
                                     int relu, int accumulate, float* stats, int bo_mode, long long* dbg, int num_sms, cudaStream_t st);

// ---- conv_halo3.cu (opt-in): the three taps of a filter row in ONE N = 192 MMA, column shift-add in the epilogue -----------------
cudaError_t launch_conv3x3_halo3_bf16(const void* x, const void* w, void* out, int NB, int H, int W, int Cout, const float* bias, int relu,
                                      int accumulate, int num_sms, cudaStream_t st);

// ---- wgrad.cu: MN-major wgmma weight gradients (fp32, added into dW; split-K partials summed in split order) ---------
cudaError_t launch_conv_wgrad_bf16(const void* dy, const void* x, float* dW, int NB, int planes, int Hin, int Win, int Cin, int Cin_valid,
                                   int Ho, int Wo, int Cout, int ntaps, const int* dh, const int* dw, const int* dplane, int num_sms,
                                   cudaStream_t st, int in_stride = 1);
cudaError_t launch_conv_wgrad_halo_bf16(const void* dy, const void* x, float* dW, int NB, int H, int W, int Cin_valid, int Cout,
                                        int num_sms, cudaStream_t st);
cudaError_t launch_linear_wgrad_bf16(const void* dy, const void* x, float* dW, int B, int N, int K, int num_sms, cudaStream_t st);

// ---- norm.cu: NHWC bf16 layer kernels -----------------------------------------------------------------------------
// per-channel sum / sum of squares of x[M][C]
// only_sum: accumulate just sum x into stats[0..C) (bias gradients written straight into the flat gradient)
cudaError_t launch_channel_stats(const __nv_bfloat16* x, long long M, int C, float* stats /*[nslots][2][C], accumulates*/, int num_sms, cudaStream_t st,
                                 int only_sum = 0, int nslots = 1);
// finalize statistics: mean/rstd (+ running stats update with momentum, unbiased variance)
cudaError_t launch_bn_finalize(const float* stats, int slots, float* mean_rstd, float* running_mean, float* running_var, int C,
                               float count, float eps, float momentum, int train, cudaStream_t st);
// y = act(gamma * (x - mean) * rstd + beta [+ res])
// fin_mode 0: mean_rstd given | 1: training, derive from raw sums `stats` [slots][2][C] (also writes mean_rstd + running stats) |
// 2: evaluation, derive from the running statistics
cudaError_t launch_bn_apply(const __nv_bfloat16* x, const __nv_bfloat16* res, __nv_bfloat16* y, const float* gamma, const float* beta,
                            float* mean_rstd, long long M, int C, int relu, int fin_mode, const float* stats, int slots, float count,
                            float eps, float momentum, float* running_mean, float* running_var, int num_sms, cudaStream_t st);
// dsum[0][c] = sum dz, dsum[1][c] = sum dz * xhat   (dz = dy * mask; relu 1: mask = (y > 0), relu 2: mask recomputed from x, gamma, beta)
cudaError_t launch_bn_bwd_reduce(const __nv_bfloat16* dy, const __nv_bfloat16* y, const __nv_bfloat16* x, const float* mean_rstd,
                                 float* dsum /*[nslots][2][C], accumulates*/, long long M, int C, int relu, int num_sms, cudaStream_t st,
                                 const float* gamma = nullptr, const float* beta = nullptr, int nslots = 1);
// dx = gamma * rstd * (dz - dsum0/M - xhat * dsum1/M); dres = dz; dgamma = dsum1, dbeta = dsum0
cudaError_t launch_bn_bwd_apply(const __nv_bfloat16* dy, const __nv_bfloat16* y, const __nv_bfloat16* x, const float* gamma,
                                const float* mean_rstd, const float* dsum, __nv_bfloat16* dx, __nv_bfloat16* dres, float* dgamma,
                                float* dbeta, long long M, int C, int relu, int num_sms, cudaStream_t st, const float* beta = nullptr, int nslots = 1);
// scale != 1: the output went through fused dropout (mask = y > 0 covers ReLU and dropout together)
cudaError_t launch_relu_bwd(__nv_bfloat16* dy, const __nv_bfloat16* y, long long n, int num_sms, cudaStream_t st, float scale = 1.0f);
// drop_p > 0: dropout fused into the pooling kernel (Philox keep-mask of the pooled element, recomputed by the backward kernel; no mask tensor)
cudaError_t launch_maxpool2_fwd(const __nv_bfloat16* x, __nv_bfloat16* y, uint8_t* idx, int B, int H, int W, int C, cudaStream_t st,
                                float drop_p = 0.f, uint64_t seed = 0, const long long* step = nullptr, uint64_t stream = 0);
cudaError_t launch_maxpool2_bwd(const __nv_bfloat16* dy, const uint8_t* idx, __nv_bfloat16* dx, int B, int H, int W, int C, cudaStream_t st,
                                float drop_p, uint64_t seed, const long long* step, uint64_t stream, const __nv_bfloat16* zmask);
cudaError_t launch_avgpool_fwd(const __nv_bfloat16* x, __nv_bfloat16* y, int B, int HW, int C, cudaStream_t st);
cudaError_t launch_avgpool_bwd(const __nv_bfloat16* dy, __nv_bfloat16* dx, int B, int HW, int C, cudaStream_t st);
cudaError_t launch_dropout_fwd(const __nv_bfloat16* x, __nv_bfloat16* y, uint8_t* mask, long long n, float p, uint64_t seed,
                               const long long* step, uint64_t stream, cudaStream_t st);
cudaError_t launch_dropout_bwd(const __nv_bfloat16* dy, const uint8_t* mask, __nv_bfloat16* dx, long long n, float p, cudaStream_t st);
// x[NB][H][W][C] -> four parity planes [4][NB][H/2][W/2][C] (plane = (h&1)*2 + (w&1)); H, W even
cudaError_t launch_space_to_depth(const __nv_bfloat16* x, __nv_bfloat16* y, int NB, int H, int W, int C, int num_sms, cudaStream_t st);
// stem convs (C*k*k <= 64, stride 1): A[NB*Ho*Wo][64] = zero-padded patches of x[NB][H][W][C] in (tap, channel) order
cudaError_t launch_im2col_small(const __nv_bfloat16* x, __nv_bfloat16* A, int NB, int H, int W, int C, int Ho, int Wo, int k, int pad,
                                int num_sms, cudaStream_t st);
cudaError_t launch_depth_to_space(const __nv_bfloat16* x4, __nv_bfloat16* y, int NB, int H, int W, int C, int accumulate, int plane_mask,
                                  int num_sms, cudaStream_t st);
cudaError_t launch_filter_gather_transpose(const __nv_bfloat16* w, __nv_bfloat16* wt, int Cout, int T, int Cin, int nsub, const int* taps,
                                           cudaStream_t st);
// tap-flipped transposed filter for the data gradient: wt[ci][8-t][co] = w[co][t][ci]   (3x3) / wt[ci][co] = w[co][ci] (1x1)
cudaError_t launch_filter_transpose(const __nv_bfloat16* w, __nv_bfloat16* wt, int Cout, int ntaps, int Cin, cudaStream_t st);
// small dense layers on CUDA cores (heads with N=10): y = x W^T + b ; dx = dy W ; dW = dy^T x ; db = sum dy
cudaError_t launch_linear_small_fwd(const __nv_bfloat16* x, const __nv_bfloat16* w, const float* bias, __nv_bfloat16* y, int B, int K,
                                    int N, int relu, cudaStream_t st);
// v2 head kernels (opt-in): more blocks / staged weights; bwd2 ACCUMULATES into dW, db (must be zero on entry)
cudaError_t launch_linear_small_fwd2(const __nv_bfloat16* x, const __nv_bfloat16* w, const float* bias, __nv_bfloat16* y, int B, int K,
                                     int N, int relu, cudaStream_t st);
cudaError_t launch_linear_small_bwd2(const __nv_bfloat16* x, const __nv_bfloat16* dy, const __nv_bfloat16* w, __nv_bfloat16* dx,
                                     float* dw, float* db, int B, int K, int N, int accumulate_dx, cudaStream_t st);
cudaError_t launch_linear_small_bwd(const __nv_bfloat16* x, const __nv_bfloat16* dy, const __nv_bfloat16* w, __nv_bfloat16* dx,
                                    float* dw, float* db, int B, int K, int N, int accumulate_dx, cudaStream_t st);

}  // namespace rlr
