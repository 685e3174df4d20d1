// Python bindings for the wgmma GEMM / implicit-GEMM conv kernels (gemm.cu) and the NHWC layer kernels (norm.cu).
#include <torch/extension.h>
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>
#include <c10/cuda/CUDACachingAllocator.h>

#include <vector>

#include "gemm.h"

namespace rlr {
// scratch memory of the deterministic reductions (common.cuh): PyTorch's caching allocator, ordered on the launch stream
void* scratch_alloc(size_t bytes, cudaStream_t st) {
    return c10::cuda::CUDACachingAllocator::raw_alloc_with_stream(bytes < 256 ? 256 : bytes, st);
}
void scratch_free(void* p) { c10::cuda::CUDACachingAllocator::raw_delete(p); }
}  // namespace rlr

namespace {
inline cudaStream_t cur_stream() { return c10::cuda::getCurrentCUDAStream().stream(); }
inline int num_sms() { return at::cuda::getCurrentDeviceProperties()->multiProcessorCount; }
inline void check(cudaError_t e, const char* what) { TORCH_CHECK(e == cudaSuccess, what, ": ", cudaGetErrorString(e)); }
template <typename T>
inline T* opt(const c10::optional<at::Tensor>& t) { return t.has_value() && t->defined() ? reinterpret_cast<T*>(t->data_ptr()) : nullptr; }
inline const __nv_bfloat16* bf(const at::Tensor& t) {
    TORCH_CHECK(t.is_cuda() && t.scalar_type() == at::kBFloat16 && t.is_contiguous(), "expected contiguous CUDA bf16 tensor");
    return reinterpret_cast<const __nv_bfloat16*>(t.data_ptr());
}
inline __nv_bfloat16* bfm(at::Tensor& t) { return const_cast<__nv_bfloat16*>(bf(t)); }
inline const __nv_bfloat16* bfo(const c10::optional<at::Tensor>& t) { return t.has_value() && t->defined() ? bf(*t) : nullptr; }
inline float* f32(const at::Tensor& t) {
    TORCH_CHECK(t.is_cuda() && t.scalar_type() == at::kFloat && t.is_contiguous(), "expected contiguous CUDA fp32 tensor");
    return reinterpret_cast<float*>(t.data_ptr());
}

// out[M][N] = A[M][K] @ B[N][K]^T (+bias)(relu)
// fused-dropout arguments of the python API: p in (0, 1) (0 = off), Philox seed, device int64 step counter, node id
static rlr::DropSpec drop_spec(double p, int64_t seed, const c10::optional<at::Tensor>& step, int64_t stream) {
    rlr::DropSpec d{};
    if (p > 0.0) {
        TORCH_CHECK(p < 1.0 && step.has_value() && step->defined() && step->scalar_type() == at::kLong, "fused dropout needs p < 1 and an int64 step counter");
        d.thr = (uint32_t)(p * 65536.0); d.scale = (float)(1.0 / (1.0 - p)); d.seed = (uint64_t)seed; d.stream = (uint64_t)stream;
        d.step = reinterpret_cast<const long long*>(step->data_ptr<int64_t>());
    }
    return d;
}

void gemm_bf16(at::Tensor A, at::Tensor B, at::Tensor out, c10::optional<at::Tensor> bias, bool relu, bool accumulate,
               c10::optional<at::Tensor> stats, double drop_p, int64_t drop_seed, c10::optional<at::Tensor> drop_step, int64_t drop_stream) {
    c10::cuda::CUDAGuard g(A.device());
    const rlr::DropSpec drop = drop_spec(drop_p, drop_seed, drop_step, drop_stream);
    const int M = A.size(0), K = A.size(1), N = B.size(0);
    TORCH_CHECK(B.size(1) == K && out.size(0) == M && out.size(1) == N);
    TORCH_CHECK(!stats.has_value() || !stats->defined() || stats->numel() == (int64_t)rlr::kStatSlots * 2 * N, "stats must be [STAT_SLOTS,2,N]");
    check(rlr::launch_gemm_bf16(bf(A), bf(B), bfm(out), M, N, K, K, K, N, opt<const float>(bias), relu, accumulate, opt<float>(stats),
                                cur_stream(), drop.thr ? &drop : nullptr), "gemm_bf16");
}

// stem convolution as one 64-deep GEMM: out[M][N] = A[M][64] @ pad64(W[N][kvalid])^T; W is the UN-padded filter, gathered by the kernel's
// producer warp.  ready_ptr != 0: device address of this rank's broadcast-ready words; the producer acquires words [lo, hi] >= *epoch first
void stem_gemm_bf16(at::Tensor A, at::Tensor W, at::Tensor out, c10::optional<at::Tensor> bias, bool relu, c10::optional<at::Tensor> stats,
                    int64_t ready_ptr, int64_t lo, int64_t hi, c10::optional<at::Tensor> epoch) {
    c10::cuda::CUDAGuard g(A.device());
    const int M = A.size(0), N = W.size(0), kvalid = W.size(1);
    TORCH_CHECK(A.dim() == 2 && A.size(1) == 64 && W.dim() == 2 && W.is_contiguous() && out.size(0) == M && out.size(1) == N, "stem_gemm shapes");
    TORCH_CHECK(ready_ptr == 0 || (epoch.has_value() && epoch->defined() && epoch->scalar_type() == at::kInt), "epoch must be an int32 device tensor");
    check(rlr::launch_stem_gemm_bf16(bf(A), bf(W), bfm(out), M, N, kvalid, kvalid, opt<const float>(bias), relu, opt<float>(stats),
                                     reinterpret_cast<const uint32_t*>(ready_ptr), (int)lo, (int)hi,
                                     ready_ptr ? reinterpret_cast<const uint32_t*>(epoch->data_ptr()) : nullptr, cur_stream()), "stem_gemm_bf16");
}

// x: [planes*NB, Hin, Win, Cin]; w: [Cout, ntaps*Cin]; out: [NB, Ho, Wo, Cout]
void conv_bf16(at::Tensor x, at::Tensor w, at::Tensor out, int64_t NB, int64_t planes, std::vector<int64_t> dh, std::vector<int64_t> dw,
               std::vector<int64_t> dplane, c10::optional<at::Tensor> bias, bool relu, bool accumulate, c10::optional<at::Tensor> stats,
               std::vector<int64_t> wtap, int64_t w_taps_total) {
    c10::cuda::CUDAGuard g(x.device());
    TORCH_CHECK(x.dim() == 4 && out.dim() == 4 && w.dim() == 2);
    const int Hin = x.size(1), Win = x.size(2), Cin = x.size(3), Ho = out.size(1), Wo = out.size(2), Cout = out.size(3);
    const int T = (int)dh.size();
    const bool bmn = !wtap.empty();   // data gradient reading the forward filter w[Cin_here][w_taps_total * Cout_here] MN-major
    TORCH_CHECK(x.size(0) == planes * NB && out.size(0) == NB);
    TORCH_CHECK(bmn ? (w.size(0) == Cin && w.size(1) == w_taps_total * Cout && (int)wtap.size() == T)
                    : (w.size(0) == Cout && w.size(1) == (int64_t)T * Cin), "filter shape");
    TORCH_CHECK(!stats.has_value() || !stats->defined() || stats->numel() == (int64_t)rlr::kStatSlots * 2 * Cout, "stats must be [STAT_SLOTS,2,Cout]");
    int a[9], b[9], c[9], wt[9];
    for (int t = 0; t < T; ++t) { a[t] = (int)dh[t]; b[t] = (int)dw[t]; c[t] = (int)dplane[t]; wt[t] = bmn ? (int)wtap[t] : 0; }
    check(rlr::launch_conv_bf16(bf(x), bf(w), bfm(out), (int)NB, (int)planes, Hin, Win, Cin, Ho, Wo, Cout, Cout, T, a, b, c,
                                opt<const float>(bias), relu, accumulate, opt<float>(stats), cur_stream(), bmn ? wt : nullptr,
                                (int)w_taps_total), "conv_bf16");
}

// out[M][N] = act(A[M][K] @ B[N][K]^T + bias) with split-K partial sums in ws ([M][N] fp32, zero on entry, left zero)
void gemm_splitk_bf16(at::Tensor A, at::Tensor B, at::Tensor out, at::Tensor ws, c10::optional<at::Tensor> bias, bool relu, double drop_p,
                      int64_t drop_seed, c10::optional<at::Tensor> drop_step, int64_t drop_stream) {
    c10::cuda::CUDAGuard g(A.device());
    const rlr::DropSpec drop = drop_spec(drop_p, drop_seed, drop_step, drop_stream);
    const int M = A.size(0), K = A.size(1), N = B.size(0);
    TORCH_CHECK(B.size(1) == K && out.size(0) == M && out.size(1) == N && ws.numel() == (int64_t)M * N);
    check(rlr::launch_gemm_splitk_bf16(bf(A), bf(B), bfm(out), f32(ws), M, N, K, opt<const float>(bias), relu, num_sms(), cur_stream(),
                                       drop.thr ? &drop : nullptr), "gemm_splitk_bf16");
}

// Strided variant without parity-split copies: x [NB,Hin,Win,Cin] is the ORIGINAL input, read through a TMA box with element
// strides (in_stride, 2 for stride-2 forward convs); `out` [NB,OutH,OutW,Cout] is the FULL output image and this launch fills the
// pixels (out_stride*h + out_ph, out_stride*w + out_pw) of it (out_stride 2 = one parity plane of a stride-2 data gradient).
// Tap offsets dh/dw are in input pixels relative to in_stride * (output grid coordinate).
void conv_bf16_strided(at::Tensor x, at::Tensor w, at::Tensor out, std::vector<int64_t> dh, std::vector<int64_t> dw,
                       c10::optional<at::Tensor> bias, bool relu, bool accumulate, std::vector<int64_t> wtap, int64_t w_taps_total,
                       int64_t in_stride, int64_t out_stride, int64_t out_ph, int64_t out_pw) {
    c10::cuda::CUDAGuard g(x.device());
    TORCH_CHECK(x.dim() == 4 && out.dim() == 4 && w.dim() == 2 && x.size(0) == out.size(0));
    TORCH_CHECK(out.size(1) % out_stride == 0 && out.size(2) % out_stride == 0, "output image must be a multiple of out_stride");
    const int NB = x.size(0), Hin = x.size(1), Win = x.size(2), Cin = x.size(3), Cout = out.size(3);
    const int Ho = out.size(1) / out_stride, Wo = out.size(2) / out_stride;
    const int T = (int)dh.size();
    const bool bmn = !wtap.empty();
    TORCH_CHECK(bmn ? (w.size(0) == Cin && w.size(1) == w_taps_total * Cout && (int)wtap.size() == T)
                    : (w.size(0) == Cout && w.size(1) == (int64_t)T * Cin), "filter shape");
    int a[9], b[9], c[9] = {0}, wt[9];
    for (int t = 0; t < T; ++t) { a[t] = (int)dh[t]; b[t] = (int)dw[t]; wt[t] = bmn ? (int)wtap[t] : 0; }
    check(rlr::launch_conv_bf16(bf(x), bf(w), bfm(out), NB, 1, Hin, Win, Cin, Ho, Wo, Cout, Cout, T, a, b, c, opt<const float>(bias), relu,
                                accumulate, nullptr, cur_stream(), bmn ? wt : nullptr, (int)w_taps_total, (int)in_stride, (int)out_stride,
                                (int)out_ph, (int)out_pw), "conv_bf16_strided");
}

// x: [NB,H,W,64]; w: [Cout, 9*64]; out: [NB,H,W,Cout]   (3x3, stride 1, pad 1)
void conv3x3_halo_bf16(at::Tensor x, at::Tensor w, at::Tensor out, c10::optional<at::Tensor> bias, bool relu, bool accumulate,
                       c10::optional<at::Tensor> stats, int64_t bo_mode, c10::optional<at::Tensor> dbg) {
    c10::cuda::CUDAGuard g(x.device());
    TORCH_CHECK(x.dim() == 4 && x.size(3) == 64 && out.dim() == 4 && w.dim() == 2 && w.size(1) == 9 * 64 && w.size(0) == out.size(3));
    TORCH_CHECK(out.size(0) == x.size(0) && out.size(1) - x.size(1) == out.size(2) - x.size(2), "halo conv: output = input + 2*pad - 2, pad in {0,1,2}");
    TORCH_CHECK(!stats.has_value() || !stats->defined() || stats->numel() == (int64_t)rlr::kStatSlots * 2 * out.size(3), "stats must be [STAT_SLOTS,2,Cout]");
    check(rlr::launch_conv3x3_halo_bf16(bf(x), bf(w), bfm(out), x.size(0), x.size(1), x.size(2), out.size(1), out.size(2), out.size(3), opt<const float>(bias), relu,
                                        accumulate, opt<float>(stats), (int)bo_mode, opt<long long>(dbg), num_sms(), cur_stream()), "conv3x3_halo_bf16");
}

// same contract as conv3x3_halo_bf16 without statistics; H % 16 == 0, any W
void conv3x3_halo3_bf16(at::Tensor x, at::Tensor w, at::Tensor out, c10::optional<at::Tensor> bias, bool relu, bool accumulate) {
    c10::cuda::CUDAGuard g(x.device());
    TORCH_CHECK(x.dim() == 4 && x.size(3) == 64 && out.dim() == 4 && w.dim() == 2 && w.size(1) == 9 * 64 && w.size(0) == out.size(3));
    TORCH_CHECK(out.size(0) == x.size(0) && out.size(1) == x.size(1) && out.size(2) == x.size(2));
    check(rlr::launch_conv3x3_halo3_bf16(bf(x), bf(w), bfm(out), x.size(0), x.size(1), x.size(2), out.size(3), opt<const float>(bias), relu,
                                         accumulate, num_sms(), cur_stream()), "conv3x3_halo3_bf16");
}

// dW[Cout][T][Cin_valid] (fp32, pre-zeroed) += wgrad(dy[NB,Ho,Wo,Cout], x[planes*NB,Hin,Win,Cin])
void conv_wgrad_bf16(at::Tensor dy, at::Tensor x, at::Tensor dW, int64_t NB, int64_t planes, int64_t cin_valid, std::vector<int64_t> dh,
                     std::vector<int64_t> dw, std::vector<int64_t> dplane) {
    c10::cuda::CUDAGuard g(x.device());
    TORCH_CHECK(x.dim() == 4 && dy.dim() == 4);
    const int Hin = x.size(1), Win = x.size(2), Cin = x.size(3), Ho = dy.size(1), Wo = dy.size(2), Cout = dy.size(3);
    const int T = (int)dh.size();
    TORCH_CHECK(x.size(0) == planes * NB && dy.size(0) == NB && dW.numel() == (int64_t)Cout * T * cin_valid);
    TORCH_CHECK((Cout <= 64 && Cout % 8 == 0) || Cout % 128 == 0, "wgrad: Cout must be <= 64 or a multiple of 128");
    int a[9], b[9], c[9];
    for (int t = 0; t < T; ++t) { a[t] = (int)dh[t]; b[t] = (int)dw[t]; c[t] = (int)dplane[t]; }
    check(rlr::launch_conv_wgrad_bf16(bf(dy), bf(x), f32(dW), (int)NB, (int)planes, Hin, Win, Cin, (int)cin_valid, Ho, Wo, Cout, T, a, b, c,
                                      num_sms(), cur_stream()), "conv_wgrad_bf16");
}
// stride-2 weight gradient on the ORIGINAL input x [NB,Hin,Win,Cin] (strided TMA box, no parity-split copy); dh/dw in input pixels
void conv_wgrad_bf16_strided(at::Tensor dy, at::Tensor x, at::Tensor dW, int64_t cin_valid, std::vector<int64_t> dh, std::vector<int64_t> dw,
                             int64_t in_stride) {
    c10::cuda::CUDAGuard g(x.device());
    TORCH_CHECK(x.dim() == 4 && dy.dim() == 4 && x.size(0) == dy.size(0));
    const int NB = x.size(0), Hin = x.size(1), Win = x.size(2), Cin = x.size(3), Ho = dy.size(1), Wo = dy.size(2), Cout = dy.size(3);
    const int T = (int)dh.size();
    TORCH_CHECK(dW.numel() == (int64_t)Cout * T * cin_valid);
    TORCH_CHECK((Cout <= 64 && Cout % 8 == 0) || Cout % 128 == 0, "wgrad: Cout must be <= 64 or a multiple of 128");
    int a[9], b[9], c[9] = {0};
    for (int t = 0; t < T; ++t) { a[t] = (int)dh[t]; b[t] = (int)dw[t]; }
    check(rlr::launch_conv_wgrad_bf16(bf(dy), bf(x), f32(dW), NB, 1, Hin, Win, Cin, (int)cin_valid, Ho, Wo, Cout, T, a, b, c, num_sms(),
                                      cur_stream(), (int)in_stride), "conv_wgrad_bf16_strided");
}
// 3x3/s1/p1 weight gradient with smem halo reuse: x [NB,H,W,64], dy [NB,H,W,Cout], dW [Cout,9,cin_valid]
void conv_wgrad_halo_bf16(at::Tensor dy, at::Tensor x, at::Tensor dW, int64_t cin_valid) {
    c10::cuda::CUDAGuard g(x.device());
    TORCH_CHECK(x.dim() == 4 && x.size(3) == 64 && dy.dim() == 4 && dy.size(0) == x.size(0) && dy.size(1) == x.size(1) && dy.size(2) == x.size(2));
    TORCH_CHECK(dW.numel() == dy.size(3) * 9 * cin_valid);
    check(rlr::launch_conv_wgrad_halo_bf16(bf(dy), bf(x), f32(dW), x.size(0), x.size(1), x.size(2), (int)cin_valid, dy.size(3), num_sms(),
                                           cur_stream()), "conv_wgrad_halo_bf16");
}
void linear_wgrad_bf16(at::Tensor dy, at::Tensor x, at::Tensor dW) {
    c10::cuda::CUDAGuard g(x.device());
    const int B = x.size(0), K = x.size(1), N = dy.size(1);
    TORCH_CHECK(dy.size(0) == B && dW.numel() == (int64_t)N * K && ((N <= 64 && N % 8 == 0) || N % 128 == 0));
    check(rlr::launch_linear_wgrad_bf16(bf(dy), bf(x), f32(dW), B, N, K, num_sms(), cur_stream()), "linear_wgrad_bf16");
}

void channel_stats(at::Tensor x, at::Tensor stats) {
    c10::cuda::CUDAGuard g(x.device());
    const int C = x.size(-1);
    const int nslots = (int)(stats.numel() / (2 * C));       // stats is [nslots][2][C]: CTAs spread their atomics over the slots
    TORCH_CHECK(nslots >= 1 && stats.numel() == (int64_t)nslots * 2 * C, "stats must be [slots, 2, C]");
    check(rlr::launch_channel_stats(bf(x), x.numel() / C, C, f32(stats), num_sms(), cur_stream(), 0, nslots), "channel_stats");
}
// bias gradient: db[C] += sum over rows of dy[M][C]  (db is a slice of the flat fp32 gradient, zero or partially accumulated on entry)
void bias_grad(at::Tensor dy, at::Tensor db) {
    c10::cuda::CUDAGuard g(dy.device());
    const int C = dy.size(-1);
    TORCH_CHECK(db.numel() == C && db.scalar_type() == at::kFloat && dy.is_contiguous(), "bias_grad: db must be fp32 [C]");
    check(rlr::launch_channel_stats(bf(dy), dy.numel() / C, C, f32(db), num_sms(), cur_stream(), 1), "bias_grad");
}
void bn_finalize(at::Tensor stats, at::Tensor mean_rstd, at::Tensor rm, at::Tensor rv, double count, double eps, double momentum, bool train) {
    c10::cuda::CUDAGuard g(stats.device());
    const int C = mean_rstd.size(-1);
    const int slots = (int)(stats.numel() / (2 * C));
    TORCH_CHECK(slots >= 1 && stats.numel() == (int64_t)slots * 2 * C, "stats must be [slots, 2, C]");
    check(rlr::launch_bn_finalize(f32(stats), slots, f32(mean_rstd), (float*)rm.data_ptr(), (float*)rv.data_ptr(), C, (float)count, (float)eps,
                                  (float)momentum, train, cur_stream()), "bn_finalize");
}
void bn_apply(at::Tensor x, c10::optional<at::Tensor> res, at::Tensor y, at::Tensor gamma, at::Tensor beta, at::Tensor mean_rstd, bool relu,
              int64_t fin_mode, c10::optional<at::Tensor> stats, double count, double eps, double momentum,
              c10::optional<at::Tensor> rm, c10::optional<at::Tensor> rv) {
    c10::cuda::CUDAGuard g(x.device());
    const int C = x.size(-1);
    int slots = 1;
    if (fin_mode == 1) {
        TORCH_CHECK(stats.has_value() && stats->defined() && rm.has_value() && rv.has_value(), "bn_apply: training finalize needs stats and running stats");
        slots = (int)(stats->numel() / (2 * C));
        TORCH_CHECK(slots >= 1 && stats->numel() == (int64_t)slots * 2 * C, "stats must be [slots,2,C]");
    }
    if (fin_mode == 2) TORCH_CHECK(rm.has_value() && rv.has_value(), "bn_apply: eval needs running stats");
    check(rlr::launch_bn_apply(bf(x), bfo(res), bfm(y), (const float*)gamma.data_ptr(), (const float*)beta.data_ptr(), f32(mean_rstd),
                               x.numel() / C, C, relu, (int)fin_mode, opt<const float>(stats), slots, (float)count, (float)eps, (float)momentum,
                               opt<float>(rm), opt<float>(rv), num_sms(), cur_stream()), "bn_apply");
}
void bn_bwd(at::Tensor dy, at::Tensor y, at::Tensor x, at::Tensor gamma, at::Tensor mean_rstd, at::Tensor dsum, at::Tensor dx,
            c10::optional<at::Tensor> dres, at::Tensor dgamma, at::Tensor dbeta, bool relu, bool zero_dsum) {
    c10::cuda::CUDAGuard g(x.device());
    const int C = x.size(-1);
    const long long M = x.numel() / C;
    const int nslots = (int)(dsum.numel() / (2 * C));         // dsum is [nslots][2][C]
    TORCH_CHECK(nslots >= 1 && dsum.numel() == (int64_t)nslots * 2 * C, "dsum must be [slots, 2, C]");
    if (zero_dsum) check(cudaMemsetAsync(dsum.data_ptr(), 0, sizeof(float) * dsum.numel(), cur_stream()), "bn_bwd/memset");
    check(rlr::launch_bn_bwd_reduce(bf(dy), bf(y), bf(x), f32(mean_rstd), f32(dsum), M, C, relu, num_sms(), cur_stream(), nullptr, nullptr, nslots),
          "bn_bwd_reduce");
    check(rlr::launch_bn_bwd_apply(bf(dy), bf(y), bf(x), (const float*)gamma.data_ptr(), f32(mean_rstd), f32(dsum), bfm(dx),
                                   const_cast<__nv_bfloat16*>(bfo(dres)), (float*)dgamma.data_ptr(), (float*)dbeta.data_ptr(), M, C, relu,
                                   num_sms(), cur_stream(), nullptr, nslots), "bn_bwd_apply");
}
// BatchNorm + ReLU without a residual: the ReLU mask is recomputed from x (same expression as the forward), y is never read
void bn_bwd_recompute(at::Tensor dy, at::Tensor x, at::Tensor gamma, at::Tensor beta, at::Tensor mean_rstd, at::Tensor dsum, at::Tensor dx,
                      at::Tensor dgamma, at::Tensor dbeta, bool zero_dsum) {
    c10::cuda::CUDAGuard g(x.device());
    const int C = x.size(-1);
    const long long M = x.numel() / C;
    const int nslots = (int)(dsum.numel() / (2 * C));
    TORCH_CHECK(nslots >= 1 && dsum.numel() == (int64_t)nslots * 2 * C, "dsum must be [slots, 2, C]");
    if (zero_dsum) check(cudaMemsetAsync(dsum.data_ptr(), 0, sizeof(float) * dsum.numel(), cur_stream()), "bn_bwd/memset");
    check(rlr::launch_bn_bwd_reduce(bf(dy), nullptr, bf(x), f32(mean_rstd), f32(dsum), M, C, 2, num_sms(), cur_stream(),
                                    (const float*)gamma.data_ptr(), (const float*)beta.data_ptr(), nslots), "bn_bwd_reduce(recompute)");
    check(rlr::launch_bn_bwd_apply(bf(dy), nullptr, bf(x), (const float*)gamma.data_ptr(), f32(mean_rstd), f32(dsum), bfm(dx), nullptr,
                                   (float*)dgamma.data_ptr(), (float*)dbeta.data_ptr(), M, C, 2, num_sms(), cur_stream(),
                                   (const float*)beta.data_ptr(), nslots), "bn_bwd_apply(recompute)");
}
void relu_bwd(at::Tensor dy, at::Tensor y, double scale) {
    c10::cuda::CUDAGuard g(dy.device());
    check(rlr::launch_relu_bwd(bfm(dy), bf(y), dy.numel(), num_sms(), cur_stream(), (float)scale), "relu_bwd");
}
void maxpool2_fwd(at::Tensor x, at::Tensor y, at::Tensor idx, double drop_p, int64_t drop_seed, c10::optional<at::Tensor> drop_step, int64_t drop_stream) {
    c10::cuda::CUDAGuard g(x.device());
    const rlr::DropSpec d = drop_spec(drop_p, drop_seed, drop_step, drop_stream);
    check(rlr::launch_maxpool2_fwd(bf(x), bfm(y), (uint8_t*)idx.data_ptr(), x.size(0), x.size(1), x.size(2), x.size(3), cur_stream(),
                                   (float)drop_p, d.seed, d.step, d.stream), "maxpool2_fwd");
}
// relu_out (optional) = the pooled forward output: back-propagates the producer's fused ReLU in the same pass (see norm.cu)
void maxpool2_bwd(at::Tensor dy, at::Tensor idx, at::Tensor dx, double drop_p, int64_t drop_seed, c10::optional<at::Tensor> drop_step, int64_t drop_stream,
                  c10::optional<at::Tensor> relu_out) {
    c10::cuda::CUDAGuard g(dx.device());
    const rlr::DropSpec d = drop_spec(drop_p, drop_seed, drop_step, drop_stream);
    const bool zm = relu_out.has_value() && relu_out->defined();
    TORCH_CHECK(!zm || (relu_out->scalar_type() == at::kBFloat16 && relu_out->is_contiguous() && relu_out->numel() == dy.numel()), "relu_out must match dy");
    TORCH_CHECK(dy.is_contiguous() && dx.is_contiguous() && idx.is_contiguous() && dy.size(1) == dx.size(1) / 2 && dy.size(2) == dx.size(2) / 2);
    check(rlr::launch_maxpool2_bwd(bf(dy), (const uint8_t*)idx.data_ptr(), bfm(dx), dx.size(0), dx.size(1), dx.size(2), dx.size(3), cur_stream(),
                                   (float)drop_p, d.seed, d.step, d.stream, zm ? bf(*relu_out) : nullptr), "maxpool2_bwd");
}
void avgpool_fwd(at::Tensor x, at::Tensor y) {
    c10::cuda::CUDAGuard g(x.device());
    check(rlr::launch_avgpool_fwd(bf(x), bfm(y), x.size(0), x.size(1) * x.size(2), x.size(3), cur_stream()), "avgpool_fwd");
}
void avgpool_bwd(at::Tensor dy, at::Tensor dx) {
    c10::cuda::CUDAGuard g(dx.device());
    check(rlr::launch_avgpool_bwd(bf(dy), bfm(dx), dx.size(0), dx.size(1) * dx.size(2), dx.size(3), cur_stream()), "avgpool_bwd");
}
void dropout_fwd(at::Tensor x, at::Tensor y, at::Tensor mask, double p, int64_t seed, at::Tensor step, int64_t stream) {
    c10::cuda::CUDAGuard g(x.device());
    check(rlr::launch_dropout_fwd(bf(x), bfm(y), (uint8_t*)mask.data_ptr(), x.numel(), (float)p, (uint64_t)seed,
                                  (const long long*)step.data_ptr(), (uint64_t)stream, cur_stream()), "dropout_fwd");
}
void dropout_bwd(at::Tensor dy, at::Tensor mask, at::Tensor dx, double p) {
    c10::cuda::CUDAGuard g(dx.device());
    check(rlr::launch_dropout_bwd(bf(dy), (const uint8_t*)mask.data_ptr(), bfm(dx), dx.numel(), (float)p, cur_stream()), "dropout_bwd");
}
void space_to_depth(at::Tensor x, at::Tensor y) {
    c10::cuda::CUDAGuard g(x.device());
    check(rlr::launch_space_to_depth(bf(x), bfm(y), x.size(0), x.size(1), x.size(2), x.size(3), num_sms(), cur_stream()), "space_to_depth");
}
void im2col_small(at::Tensor x, at::Tensor A, int64_t k, int64_t pad) {
    c10::cuda::CUDAGuard g(x.device());
    const int NB = x.size(0), H = x.size(1), W = x.size(2), C = x.size(3);
    const int Ho = H + 2 * pad - k + 1, Wo = W + 2 * pad - k + 1;
    TORCH_CHECK(x.dim() == 4 && x.is_contiguous() && A.is_contiguous() && A.numel() == (int64_t)NB * Ho * Wo * 64, "im2col_small: A must be [NB*Ho*Wo, 64]");
    check(rlr::launch_im2col_small(bf(x), bfm(A), NB, H, W, C, Ho, Wo, (int)k, (int)pad, num_sms(), cur_stream()), "im2col_small");
}
void depth_to_space(at::Tensor x4, at::Tensor y, bool accumulate, int64_t plane_mask) {
    c10::cuda::CUDAGuard g(y.device());
    check(rlr::launch_depth_to_space(bf(x4), bfm(y), y.size(0), y.size(1), y.size(2), y.size(3), accumulate, (int)plane_mask, num_sms(),
                                     cur_stream()), "depth_to_space");
}
void filter_gather_transpose(at::Tensor w, at::Tensor wt, int64_t Cout, int64_t T, int64_t Cin, std::vector<int64_t> taps) {
    c10::cuda::CUDAGuard g(w.device());
    int t[9];
    TORCH_CHECK(taps.size() >= 1 && taps.size() <= 9);
    for (size_t i = 0; i < taps.size(); ++i) t[i] = (int)taps[i];
    check(rlr::launch_filter_gather_transpose(bf(w), bfm(wt), Cout, T, Cin, (int)taps.size(), t, cur_stream()), "filter_gather_transpose");
}
void filter_transpose(at::Tensor w, at::Tensor wt, int64_t Cout, int64_t ntaps, int64_t Cin) {
    c10::cuda::CUDAGuard g(w.device());
    check(rlr::launch_filter_transpose(bf(w), bfm(wt), Cout, ntaps, Cin, cur_stream()), "filter_transpose");
}
void linear_small_fwd(at::Tensor x, at::Tensor w, c10::optional<at::Tensor> bias, at::Tensor y, bool relu) {
    c10::cuda::CUDAGuard g(x.device());
    check(rlr::launch_linear_small_fwd(bf(x), bf(w), opt<const float>(bias), bfm(y), x.size(0), x.size(1), w.size(0), relu, cur_stream()), "linear_small_fwd");
}
void linear_small_bwd(at::Tensor x, at::Tensor dy, at::Tensor w, c10::optional<at::Tensor> dx, at::Tensor dw, c10::optional<at::Tensor> db,
                      bool accumulate_dx) {
    c10::cuda::CUDAGuard g(x.device());
    check(rlr::launch_linear_small_bwd(bf(x), bf(dy), bf(w), const_cast<__nv_bfloat16*>(bfo(dx)), (float*)dw.data_ptr(), opt<float>(db),
                                       x.size(0), x.size(1), w.size(0), accumulate_dx, cur_stream()), "linear_small_bwd");
}
void linear_small_fwd2(at::Tensor x, at::Tensor w, c10::optional<at::Tensor> bias, at::Tensor y, bool relu) {
    c10::cuda::CUDAGuard g(x.device());
    check(rlr::launch_linear_small_fwd2(bf(x), bf(w), opt<const float>(bias), bfm(y), x.size(0), x.size(1), w.size(0), relu, cur_stream()), "linear_small_fwd2");
}
// dw / db are ACCUMULATED into (zero them first)
void linear_small_bwd2(at::Tensor x, at::Tensor dy, at::Tensor w, c10::optional<at::Tensor> dx, at::Tensor dw, c10::optional<at::Tensor> db,
                       bool accumulate_dx) {
    c10::cuda::CUDAGuard g(x.device());
    check(rlr::launch_linear_small_bwd2(bf(x), bf(dy), bf(w), const_cast<__nv_bfloat16*>(bfo(dx)), (float*)dw.data_ptr(), opt<float>(db),
                                        x.size(0), x.size(1), w.size(0), accumulate_dx, cur_stream()), "linear_small_bwd2");
}
}  // namespace

void register_gemm_bindings(py::module_& m) {
    m.attr("STAT_SLOTS") = rlr::kStatSlots;
    m.def("set_persistent_conv", [](bool on) { rlr::set_persistent_conv(on ? 1 : 0); });
    m.def("set_pdl", [](bool on) { rlr::set_pdl(on ? 1 : 0); });
    m.def("set_conv_occ3", [](int64_t level) { rlr::set_conv_occ3((int)level); });
    m.def("set_conv_tma_store", [](bool on) { rlr::set_conv_tma_store(on ? 1 : 0); });
    m.def("set_conv_split_producer", [](bool on) { rlr::set_conv_split_producer(on ? 1 : 0); });
    m.def("set_conv_trace", [](c10::optional<at::Tensor> buf) {   // int64 [CTAs * 8] timeline buffer for the next generic conv / GEMM launches
        rlr::set_conv_trace(buf.has_value() && buf->defined() ? reinterpret_cast<long long*>(buf->data_ptr<int64_t>()) : nullptr);
    });
    m.def("gemm_bf16", &gemm_bf16, py::arg("A"), py::arg("B"), py::arg("out"), py::arg("bias"), py::arg("relu"), py::arg("accumulate"), py::arg("stats"),
          py::arg("drop_p") = 0.0, py::arg("drop_seed") = 0, py::arg("drop_step") = py::none(), py::arg("drop_stream") = 0);
    m.def("stem_gemm_bf16", &stem_gemm_bf16, py::arg("A"), py::arg("W"), py::arg("out"), py::arg("bias"), py::arg("relu"), py::arg("stats"),
          py::arg("ready_ptr") = 0, py::arg("lo") = 0, py::arg("hi") = 0, py::arg("epoch") = py::none());
    m.def("gemm_splitk_bf16", &gemm_splitk_bf16, py::arg("A"), py::arg("B"), py::arg("out"), py::arg("ws"), py::arg("bias"), py::arg("relu"),
          py::arg("drop_p") = 0.0, py::arg("drop_seed") = 0, py::arg("drop_step") = py::none(), py::arg("drop_stream") = 0);
    m.def("conv_bf16", &conv_bf16);
    m.def("conv_bf16_strided", &conv_bf16_strided);
    m.def("conv_wgrad_bf16_strided", &conv_wgrad_bf16_strided);
    m.def("conv3x3_halo_bf16", &conv3x3_halo_bf16);
    m.def("conv3x3_halo3_bf16", &conv3x3_halo3_bf16);
    m.def("conv_wgrad_bf16", &conv_wgrad_bf16);
    m.def("linear_wgrad_bf16", &linear_wgrad_bf16);
    m.def("conv_wgrad_halo_bf16", &conv_wgrad_halo_bf16);
    m.def("channel_stats", &channel_stats);
    m.def("bias_grad", &bias_grad);
    m.def("bn_finalize", &bn_finalize);
    m.def("bn_apply", &bn_apply);
    m.def("bn_bwd", &bn_bwd);
    m.def("bn_bwd_recompute", &bn_bwd_recompute);
    m.def("relu_bwd", &relu_bwd, py::arg("dy"), py::arg("y"), py::arg("scale") = 1.0);
    m.def("maxpool2_fwd", &maxpool2_fwd, py::arg("x"), py::arg("y"), py::arg("idx"), py::arg("drop_p") = 0.0, py::arg("drop_seed") = 0,
          py::arg("drop_step") = py::none(), py::arg("drop_stream") = 0);
    m.def("maxpool2_bwd", &maxpool2_bwd, py::arg("dy"), py::arg("idx"), py::arg("dx"), py::arg("drop_p") = 0.0, py::arg("drop_seed") = 0,
          py::arg("drop_step") = py::none(), py::arg("drop_stream") = 0, py::arg("relu_out") = py::none());
    m.def("avgpool_fwd", &avgpool_fwd);
    m.def("avgpool_bwd", &avgpool_bwd);
    m.def("dropout_fwd", &dropout_fwd);
    m.def("dropout_bwd", &dropout_bwd);
    m.def("space_to_depth", &space_to_depth);
    m.def("im2col_small", &im2col_small);
    m.def("filter_transpose", &filter_transpose);
    m.def("depth_to_space", &depth_to_space);
    m.def("filter_gather_transpose", &filter_gather_transpose);
    m.def("linear_small_fwd", &linear_small_fwd);
    m.def("linear_small_bwd", &linear_small_bwd);
    m.def("linear_small_fwd2", &linear_small_fwd2);
    m.def("linear_small_bwd2", &linear_small_bwd2);
}
