// Python bindings (pybind11 through torch/extension.h) for the sm_90a kernels and the small native runtime
// pieces (CUDA-IPC symmetric buffers).  All launches go to the CURRENT torch CUDA stream so they compose with
// stream capture (CUDA graphs) and with torch ops on the same stream.
#include <torch/extension.h>
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAStream.h>
#include <c10/cuda/CUDAGuard.h>
#include <cuda_runtime.h>

#include <string>
#include <vector>

#include "kernels.h"
#include "gemm.h"

namespace {

inline cudaStream_t cur_stream() { return c10::cuda::getCurrentCUDAStream().stream(); }
inline int num_sms() { return at::cuda::getCurrentDeviceProperties()->multiProcessorCount; }
inline void check(cudaError_t e, const char* what) {
    TORCH_CHECK(e == cudaSuccess, what, ": ", cudaGetErrorString(e));
}
template <typename T>
inline T* ptr_or_null(const c10::optional<at::Tensor>& t) {
    return t.has_value() && t->defined() ? reinterpret_cast<T*>(t->data_ptr()) : nullptr;
}
#define CHECK_CUDA(x) TORCH_CHECK((x).is_cuda() && (x).is_contiguous(), #x " must be a contiguous CUDA tensor")
// the cross-GPU gate of a server-step launch: flag_ptrs / local_sync are only needed (and checked by the launchers) when world > 1
inline rlr::Gate gate_of(const c10::optional<at::Tensor>& flag_ptrs, const c10::optional<at::Tensor>& local_sync, int64_t rank,
                         int64_t world, int64_t epoch) {
    return {ptr_or_null<uint32_t* const>(flag_ptrs), ptr_or_null<uint32_t>(local_sync), (int)rank, (int)world, (uint32_t)epoch};
}

// ---------------------------------------------------------------------------------------------------------------
void fused_aggregate(at::Tensor w_agent_ptrs, at::Tensor weights, c10::optional<at::Tensor> scales, double total_weight,
                     int64_t w_global_ptr, at::Tensor out_ptrs, c10::optional<at::Tensor> out_bf16_ptrs,
                     bool use_multimem, int64_t begin, int64_t end, int64_t n_vote, int64_t mode, int64_t theta,
                     double server_lr, double noise_std, int64_t seed, int64_t noise_stream,
                     c10::optional<at::Tensor> flipped, c10::optional<at::Tensor> flag_ptrs,
                     c10::optional<at::Tensor> local_sync, int64_t rank, int64_t world, int64_t epoch, bool handoff,
                     int64_t opt, double beta1, double beta2, double tau, c10::optional<at::Tensor> opt_m, c10::optional<at::Tensor> opt_v,
                     int64_t state_base) {
    CHECK_CUDA(w_agent_ptrs); CHECK_CUDA(weights); CHECK_CUDA(out_ptrs);
    TORCH_CHECK(w_agent_ptrs.scalar_type() == at::kLong && out_ptrs.scalar_type() == at::kLong, "pointer tables must be int64");
    TORCH_CHECK(weights.scalar_type() == at::kDouble, "weights must be float64");
    c10::cuda::CUDAGuard guard(w_agent_ptrs.device());
    rlr::AggParams p{};
    p.w_agents = reinterpret_cast<const float* const*>(w_agent_ptrs.data_ptr());
    p.weights = weights.data_ptr<double>();
    p.scales = ptr_or_null<const float>(scales);
    p.total_weight = total_weight;
    p.w_global = reinterpret_cast<const float*>(w_global_ptr);
    p.out_ptrs = reinterpret_cast<float* const*>(out_ptrs.data_ptr());
    p.out_bf16_ptrs = ptr_or_null<__nv_bfloat16* const>(out_bf16_ptrs);
    p.n_out = (int)out_ptrs.numel();
    p.use_multimem = use_multimem ? 1 : 0;
    p.K = (int)w_agent_ptrs.numel();
    p.begin = begin; p.end = end; p.n_vote = n_vote;
    p.mode = (int)mode; p.theta = (int)theta;
    p.server_lr = (float)server_lr; p.noise_std = (float)noise_std;
    p.seed = (uint64_t)seed; p.noise_stream = (uint64_t)noise_stream;
    p.flipped = ptr_or_null<unsigned long long>(flipped);
    p.gate = gate_of(flag_ptrs, local_sync, rank, world, epoch);
    p.handoff = handoff ? 1 : 0;
    // server optimizer state: fp32 on the launch device, covering [state_base, end)
    for (const auto* t : {&opt_m, &opt_v}) {
        if (!t->has_value() || !(*t)->defined()) continue;
        CHECK_CUDA(**t);
        TORCH_CHECK((*t)->scalar_type() == at::kFloat && (*t)->device() == w_agent_ptrs.device(), "optimizer state must be float32 on the launch device");
        TORCH_CHECK(state_base <= begin && state_base + (*t)->numel() >= end, "optimizer state does not cover the coordinate slice");
    }
    p.opt = (int)opt; p.beta1 = beta1; p.beta2 = beta2; p.tau = tau;
    p.opt_m = ptr_or_null<float>(opt_m);
    p.opt_v = ptr_or_null<float>(opt_v);
    p.state_base = state_base;
    check(rlr::launch_fused_aggregate(p, num_sms(), cur_stream()), "fused_aggregate");
}

// wait for broadcast slices [first, last] of round `epoch` (ready_ptr = address of this rank's ready words, 0 = nothing to wait for) and
// copy the BatchNorm-statistics tail of the broadcast buffer into the trainer's parameters
void acquire_slices(int64_t ready_ptr, int64_t first, int64_t last, c10::optional<at::Tensor> epoch, c10::optional<at::Tensor> tail_src,
                    c10::optional<at::Tensor> tail_dst) {
    TORCH_CHECK(ready_ptr == 0 || (epoch.has_value() && epoch->defined() && epoch->scalar_type() == at::kInt), "epoch must be an int32 device tensor");
    const float* src = ptr_or_null<const float>(tail_src);
    float* dst = ptr_or_null<float>(tail_dst);
    const long long n = (src && dst) ? (long long)tail_dst->numel() : 0;
    TORCH_CHECK(!(src && dst) || tail_src->numel() == tail_dst->numel(), "acquire_slices: tail size mismatch");
    check(rlr::launch_acquire_slices(reinterpret_cast<const uint32_t*>(ready_ptr), (int)first, (int)last,
                                     ready_ptr ? reinterpret_cast<const uint32_t*>(epoch->data_ptr()) : nullptr, src, dst, n, cur_stream()),
          "acquire_slices");
}

// K x K fp64 squared distances of the participants' updates over coordinates [begin, end) (Krum / Multi-Krum selection).  w_global_ptr
// is read only with scales.  world > 1: the fused multi-GPU form, which first runs the aggregation's barrier-in at `epoch`.
void pairwise_sqdist(at::Tensor w_agent_ptrs, int64_t w_global_ptr, c10::optional<at::Tensor> scales, int64_t begin, int64_t end,
                     at::Tensor out, c10::optional<at::Tensor> flag_ptrs, c10::optional<at::Tensor> local_sync, int64_t rank,
                     int64_t world, int64_t epoch) {
    CHECK_CUDA(w_agent_ptrs); CHECK_CUDA(out);
    TORCH_CHECK(w_agent_ptrs.scalar_type() == at::kLong, "pointer table must be int64");
    const int64_t K = w_agent_ptrs.numel();
    TORCH_CHECK(out.scalar_type() == at::kDouble && out.numel() == K * K, "out must be a float64 [K, K] tensor");
    const float* sc = ptr_or_null<const float>(scales);
    if (sc) {
        CHECK_CUDA(*scales);
        TORCH_CHECK(scales->scalar_type() == at::kFloat && scales->numel() == K && w_global_ptr, "scales: float32 [K], with w_global");
    }
    c10::cuda::CUDAGuard guard(out.device());
    rlr::DistParams p{};
    p.w_agents = reinterpret_cast<const float* const*>(w_agent_ptrs.data_ptr());
    p.w_global = reinterpret_cast<const float*>(w_global_ptr);
    p.scales = sc;
    p.begin = begin; p.end = end;
    p.K = (int)K;
    p.gate = gate_of(flag_ptrs, local_sync, rank, world, epoch);
    check(rlr::launch_pairwise_sqdist(p, out.data_ptr<double>(), num_sms(), cur_stream()), "pairwise_sqdist");
}

// FLAME: K x K fp64 Gram matrix of the participants' updates w_k - w_global over coordinates [begin, end), diagonal included.  world > 1:
// the fused multi-GPU form, which first runs the aggregation's barrier-in at `epoch`.
void pairwise_gram(at::Tensor w_agent_ptrs, int64_t w_global_ptr, int64_t begin, int64_t end, at::Tensor out,
                   c10::optional<at::Tensor> flag_ptrs, c10::optional<at::Tensor> local_sync, int64_t rank, int64_t world, int64_t epoch) {
    CHECK_CUDA(w_agent_ptrs); CHECK_CUDA(out);
    TORCH_CHECK(w_agent_ptrs.scalar_type() == at::kLong, "pointer table must be int64");
    const int64_t K = w_agent_ptrs.numel();
    TORCH_CHECK(out.scalar_type() == at::kDouble && out.numel() == K * K, "out must be a float64 [K, K] tensor");
    TORCH_CHECK(w_global_ptr, "pairwise_gram needs w_global");
    c10::cuda::CUDAGuard guard(out.device());
    rlr::DistParams p{};
    p.w_agents = reinterpret_cast<const float* const*>(w_agent_ptrs.data_ptr());
    p.w_global = reinterpret_cast<const float*>(w_global_ptr);
    p.begin = begin; p.end = end;
    p.K = (int)K;
    p.gate = gate_of(flag_ptrs, local_sync, rank, world, epoch);
    check(rlr::launch_pairwise_gram(p, out.data_ptr<double>(), num_sms(), cur_stream()), "pairwise_gram");
}

// FoolsGold: fold each candidate's update w_k - w_global into its history row over coordinates [begin, end).  row_ptrs holds the
// rows' addresses, offset so that absolute coordinates index them.  world > 1: the fused multi-GPU form, which first runs the
// aggregation's barrier-in at `epoch`.
void history_accumulate(at::Tensor w_agent_ptrs, at::Tensor row_ptrs, int64_t w_global_ptr, int64_t begin, int64_t end,
                        c10::optional<at::Tensor> flag_ptrs, c10::optional<at::Tensor> local_sync, int64_t rank, int64_t world, int64_t epoch) {
    CHECK_CUDA(w_agent_ptrs); CHECK_CUDA(row_ptrs);
    TORCH_CHECK(w_agent_ptrs.scalar_type() == at::kLong && row_ptrs.scalar_type() == at::kLong, "pointer tables must be int64");
    TORCH_CHECK(row_ptrs.numel() == w_agent_ptrs.numel(), "one history row per participant");
    TORCH_CHECK(w_global_ptr, "history_accumulate needs w_global");
    c10::cuda::CUDAGuard guard(w_agent_ptrs.device());
    rlr::HistParams p{};
    p.w_agents = reinterpret_cast<const float* const*>(w_agent_ptrs.data_ptr());
    p.rows = reinterpret_cast<float* const*>(row_ptrs.data_ptr());
    p.w_global = reinterpret_cast<const float*>(w_global_ptr);
    p.begin = begin; p.end = end;
    p.K = (int)w_agent_ptrs.numel();
    p.gate = gate_of(flag_ptrs, local_sync, rank, world, epoch);
    check(rlr::launch_history_accumulate(p, num_sms(), cur_stream()), "history_accumulate");
}

// FoolsGold: K x K fp64 Gram matrix of the history rows (row_ptrs, offset so that absolute coordinates index them) over [begin, end).
void history_gram(at::Tensor row_ptrs, int64_t begin, int64_t end, at::Tensor out) {
    CHECK_CUDA(row_ptrs); CHECK_CUDA(out);
    TORCH_CHECK(row_ptrs.scalar_type() == at::kLong, "pointer table must be int64");
    const int64_t K = row_ptrs.numel();
    TORCH_CHECK(out.scalar_type() == at::kDouble && out.numel() == K * K, "out must be a float64 [K, K] tensor");
    c10::cuda::CUDAGuard guard(out.device());
    rlr::DistParams p{};
    p.w_agents = reinterpret_cast<const float* const*>(row_ptrs.data_ptr());
    p.begin = begin; p.end = end;
    p.K = (int)K;
    p.gate = rlr::Gate{nullptr, nullptr, 0, 1, 0};
    check(rlr::launch_history_gram(p, out.data_ptr<double>(), num_sms(), cur_stream()), "history_gram");
}

// DnC: y [T][K][len_pad] fp32 <- the participants' centred updates at sample[t][ranges[t][0] .. ranges[t][1]), zero-padded.  world > 1:
// the fused multi-GPU form, which first runs the aggregation's barrier-in at `epoch`.
void dnc_gather(at::Tensor w_agent_ptrs, int64_t w_global_ptr, c10::optional<at::Tensor> scales, at::Tensor sample, at::Tensor ranges,
                at::Tensor y, c10::optional<at::Tensor> flag_ptrs, c10::optional<at::Tensor> local_sync, int64_t rank, int64_t world,
                int64_t epoch) {
    CHECK_CUDA(w_agent_ptrs); CHECK_CUDA(sample); CHECK_CUDA(ranges); CHECK_CUDA(y);
    TORCH_CHECK(w_agent_ptrs.scalar_type() == at::kLong, "pointer table must be int64");
    TORCH_CHECK(sample.scalar_type() == at::kInt && sample.dim() == 2, "sample must be int32 [T, S]");
    const int64_t T = sample.size(0), K = w_agent_ptrs.numel();
    TORCH_CHECK(ranges.scalar_type() == at::kInt && ranges.numel() == 2 * T, "ranges must be int32 [T, 2]");
    TORCH_CHECK(y.scalar_type() == at::kFloat && y.dim() == 3 && y.size(0) == T && y.size(1) == K, "y must be float32 [T, K, len_pad]");
    TORCH_CHECK(w_global_ptr, "dnc_gather needs w_global");
    const float* sc = ptr_or_null<const float>(scales);
    if (sc) {
        CHECK_CUDA(*scales);
        TORCH_CHECK(scales->scalar_type() == at::kFloat && scales->numel() == K, "scales: float32 [K]");
    }
    c10::cuda::CUDAGuard guard(y.device());
    rlr::DncParams p{};
    p.w_agents = reinterpret_cast<const float* const*>(w_agent_ptrs.data_ptr());
    p.w_global = reinterpret_cast<const float*>(w_global_ptr);
    p.scales = sc;
    p.sample = sample.data_ptr<int>();
    p.ranges = ranges.data_ptr<int>();
    p.y = y.data_ptr<float>();
    p.T = (int)T; p.K = (int)K; p.stride = (int)sample.size(1); p.len_pad = (int)y.size(2);
    p.gate = gate_of(flag_ptrs, local_sync, rank, world, epoch);
    check(rlr::launch_dnc_gather(p, num_sms(), cur_stream()), "dnc_gather");
}

// FLDetector ring pass over [begin, end): s_ptr (0 = none) <- w_g - w_prev, then w_prev <- w_g.  Pointers offset so that absolute
// coordinates index them.
void fld_ring(int64_t w_g_ptr, int64_t w_prev_ptr, int64_t s_ptr, int64_t begin, int64_t end) {
    TORCH_CHECK(w_g_ptr && w_prev_ptr, "fld_ring needs w_g and w_prev");
    check(rlr::launch_fld_ring(reinterpret_cast<const float*>(w_g_ptr), reinterpret_cast<float*>(w_prev_ptr), reinterpret_cast<float*>(s_ptr),
                               begin, end, num_sms(), cur_stream()), "fld_ring");
}

// FLDetector Hessian-vector product over [begin, end): hv_ptr <- fp32(sum_r coef[r] ring_ptrs[r]) (offset pointers).
void fld_hvp(at::Tensor ring_ptrs, at::Tensor coef, int64_t hv_ptr, int64_t begin, int64_t end) {
    CHECK_CUDA(ring_ptrs); CHECK_CUDA(coef);
    TORCH_CHECK(ring_ptrs.scalar_type() == at::kLong, "pointer table must be int64");
    TORCH_CHECK(coef.scalar_type() == at::kDouble && coef.numel() == ring_ptrs.numel(), "coef must be float64, one per ring row");
    TORCH_CHECK(hv_ptr, "fld_hvp needs an output");
    c10::cuda::CUDAGuard guard(coef.device());
    check(rlr::launch_fld_hvp(reinterpret_cast<const float* const*>(ring_ptrs.data_ptr()), coef.data_ptr<double>(), (int)coef.numel(),
                              reinterpret_cast<float*>(hv_ptr), begin, end, num_sms(), cur_stream()), "fld_hvp");
}

// FLDetector prediction pass over [begin, end): hv_ptr != 0 predicts (out: float64 [K] squared distances) and records, hv_ptr = 0 only
// records u_k into the rows (out ignored).  world > 1: the fused multi-GPU form, which first runs the aggregation's barrier-in at `epoch`.
void fld_predict(at::Tensor w_agent_ptrs, at::Tensor row_ptrs, int64_t w_global_ptr, int64_t hv_ptr, int64_t begin, int64_t end,
                 c10::optional<at::Tensor> out, c10::optional<at::Tensor> flag_ptrs, c10::optional<at::Tensor> local_sync, int64_t rank,
                 int64_t world, int64_t epoch) {
    CHECK_CUDA(w_agent_ptrs); CHECK_CUDA(row_ptrs);
    TORCH_CHECK(w_agent_ptrs.scalar_type() == at::kLong && row_ptrs.scalar_type() == at::kLong, "pointer tables must be int64");
    TORCH_CHECK(row_ptrs.numel() == w_agent_ptrs.numel(), "one last-update row per candidate");
    TORCH_CHECK(w_global_ptr, "fld_predict needs w_global");
    double* o = nullptr;
    if (hv_ptr) {
        TORCH_CHECK(out.has_value() && out->defined(), "a prediction pass needs out");
        CHECK_CUDA(*out);
        TORCH_CHECK(out->scalar_type() == at::kDouble && out->numel() == w_agent_ptrs.numel(), "out must be a float64 [K] tensor");
        o = out->data_ptr<double>();
    }
    c10::cuda::CUDAGuard guard(w_agent_ptrs.device());
    rlr::FldParams p{};
    p.w_agents = reinterpret_cast<const float* const*>(w_agent_ptrs.data_ptr());
    p.rows = reinterpret_cast<float* const*>(row_ptrs.data_ptr());
    p.w_global = reinterpret_cast<const float*>(w_global_ptr);
    p.hv = reinterpret_cast<const float*>(hv_ptr);
    p.begin = begin; p.end = end;
    p.K = (int)w_agent_ptrs.numel();
    p.gate = gate_of(flag_ptrs, local_sync, rank, world, epoch);
    check(rlr::launch_fld_predict(p, o, num_sms(), cur_stream()), "fld_predict");
}

// FLTrust statistics over coordinates [begin, end): fp64 [2K + 1] = (Δk.Δ0 for every k, |Δk|^2 for every k, |Δ0|^2), Δk = w_k - w_global,
// Δ0 = w_ref - w_global.  world > 1: the fused multi-GPU form, which first runs the aggregation's barrier-in at `epoch`.
void trust_stats(at::Tensor w_agent_ptrs, int64_t w_ref_ptr, int64_t w_global_ptr, int64_t begin, int64_t end, at::Tensor out,
                 c10::optional<at::Tensor> flag_ptrs, c10::optional<at::Tensor> local_sync, int64_t rank, int64_t world, int64_t epoch) {
    CHECK_CUDA(w_agent_ptrs); CHECK_CUDA(out);
    TORCH_CHECK(w_agent_ptrs.scalar_type() == at::kLong, "pointer table must be int64");
    const int64_t K = w_agent_ptrs.numel();
    TORCH_CHECK(out.scalar_type() == at::kDouble && out.numel() == 2 * K + 1, "out must be a float64 [2K + 1] tensor");
    TORCH_CHECK(w_ref_ptr && w_global_ptr, "trust_stats needs w_ref and w_global");
    c10::cuda::CUDAGuard guard(out.device());
    rlr::TrustParams p{};
    p.w_agents = reinterpret_cast<const float* const*>(w_agent_ptrs.data_ptr());
    p.w_ref = reinterpret_cast<const float*>(w_ref_ptr);
    p.w_global = reinterpret_cast<const float*>(w_global_ptr);
    p.begin = begin; p.end = end;
    p.K = (int)K;
    p.gate = gate_of(flag_ptrs, local_sync, rank, world, epoch);
    check(rlr::launch_trust_stats(p, out.data_ptr<double>(), num_sms(), cur_stream()), "trust_stats");
}

// RFA: fp64 [K] squared distances of the participants' updates to their b-weighted mean over coordinates [begin, end).  w_global_ptr is
// read only with scales.  world > 1: the fused multi-GPU form, which first runs the aggregation's barrier-in at `epoch`.
void rfa_sqdist(at::Tensor w_agent_ptrs, at::Tensor b, int64_t w_global_ptr, c10::optional<at::Tensor> scales, int64_t begin, int64_t end,
                at::Tensor out, c10::optional<at::Tensor> flag_ptrs, c10::optional<at::Tensor> local_sync, int64_t rank, int64_t world,
                int64_t epoch) {
    CHECK_CUDA(w_agent_ptrs); CHECK_CUDA(b); CHECK_CUDA(out);
    TORCH_CHECK(w_agent_ptrs.scalar_type() == at::kLong, "pointer table must be int64");
    const int64_t K = w_agent_ptrs.numel();
    TORCH_CHECK(b.scalar_type() == at::kDouble && b.numel() == K, "b must be a float64 [K] tensor");
    TORCH_CHECK(out.scalar_type() == at::kDouble && out.numel() == K, "out must be a float64 [K] tensor");
    const float* sc = ptr_or_null<const float>(scales);
    if (sc) {
        CHECK_CUDA(*scales);
        TORCH_CHECK(scales->scalar_type() == at::kFloat && scales->numel() == K && w_global_ptr, "scales: float32 [K], with w_global");
    }
    c10::cuda::CUDAGuard guard(out.device());
    rlr::RfaParams p{};
    p.w_agents = reinterpret_cast<const float* const*>(w_agent_ptrs.data_ptr());
    p.b = b.data_ptr<double>();
    p.w_global = reinterpret_cast<const float*>(w_global_ptr);
    p.scales = sc;
    p.begin = begin; p.end = end;
    p.K = (int)K;
    p.gate = gate_of(flag_ptrs, local_sync, rank, world, epoch);
    check(rlr::launch_rfa_sqdist(p, out.data_ptr<double>(), num_sms(), cur_stream()), "rfa_sqdist");
}

// Colluding attackers: the statistics pass (out = float64 [2H + 1]: a_k, e_k, q) or, with out_ptrs, the write pass (out = float64 [1]:
// sum (m - mu)^2) over coordinates [begin, end) of the H honest then C corrupt participants in w_agent_ptrs.  world > 1: the fused
// multi-GPU form, which first runs the aggregation's barrier-in at `epoch`.
rlr::ColludeParams collude_params(const at::Tensor& w_agent_ptrs, int64_t H, int64_t w_global_ptr, int64_t mode, int64_t dir, int64_t begin,
                                  int64_t end, const at::Tensor& out, int64_t nout) {
    CHECK_CUDA(w_agent_ptrs); CHECK_CUDA(out);
    TORCH_CHECK(w_agent_ptrs.scalar_type() == at::kLong, "pointer table must be int64");
    TORCH_CHECK(H >= 1 && H <= w_agent_ptrs.numel(), "collude: 1 <= H <= participants");
    TORCH_CHECK(out.scalar_type() == at::kDouble && out.numel() == nout, "collude: out must be a float64 tensor of ", nout, " values");
    TORCH_CHECK(w_global_ptr, "collude: w_global is required");
    rlr::ColludeParams p{};
    p.w_agents = reinterpret_cast<const float* const*>(w_agent_ptrs.data_ptr());
    p.w_global = reinterpret_cast<const float*>(w_global_ptr);
    p.begin = begin; p.end = end;
    p.H = (int)H; p.C = (int)(w_agent_ptrs.numel() - H);
    p.mode = (int)mode; p.dir = (int)dir;
    return p;
}

void collude_stats(at::Tensor w_agent_ptrs, int64_t H, int64_t w_global_ptr, int64_t dir, int64_t begin, int64_t end, at::Tensor out,
                   c10::optional<at::Tensor> flag_ptrs, c10::optional<at::Tensor> local_sync, int64_t rank, int64_t world, int64_t epoch) {
    rlr::ColludeParams p = collude_params(w_agent_ptrs, H, w_global_ptr, 1, dir, begin, end, out, 2 * H + 1);
    c10::cuda::CUDAGuard guard(out.device());
    p.gate = gate_of(flag_ptrs, local_sync, rank, world, epoch);
    check(rlr::launch_collude_stats(p, out.data_ptr<double>(), num_sms(), cur_stream()), "collude_stats");
}

void collude_write(at::Tensor w_agent_ptrs, int64_t H, c10::optional<at::Tensor> out_ptrs, int64_t w_global_ptr, int64_t mode, int64_t dir,
                   double z, double gamma, int64_t begin, int64_t end, at::Tensor out, c10::optional<at::Tensor> flag_ptrs,
                   c10::optional<at::Tensor> local_sync, int64_t rank, int64_t world, int64_t epoch) {
    rlr::ColludeParams p = collude_params(w_agent_ptrs, H, w_global_ptr, mode, dir, begin, end, out, 1);
    if (out_ptrs.has_value() && out_ptrs->defined()) {
        CHECK_CUDA(*out_ptrs);
        TORCH_CHECK(out_ptrs->scalar_type() == at::kLong, "output pointer table must be int64");
        p.w_out = reinterpret_cast<float* const*>(out_ptrs->data_ptr());
        p.n_out = (int)out_ptrs->numel();
    }
    p.z = z; p.gamma = gamma;
    c10::cuda::CUDAGuard guard(out.device());
    p.gate = gate_of(flag_ptrs, local_sync, rank, world, epoch);
    check(rlr::launch_collude_write(p, out.data_ptr<double>(), num_sms(), cur_stream()), "collude_write");
}

// ---------------------------------------------------------------------------------------------------------------
// training augmentation of the gathers: crop pad, flip, Philox key and the device int64 stream word (needed when either is on)
inline const long long* aug_stream_ptr(const c10::optional<at::Tensor>& stream, int64_t crop_pad, bool flip) {
    if (crop_pad == 0 && !flip) return nullptr;
    TORCH_CHECK(stream.has_value() && stream->defined() && stream->is_cuda() && stream->scalar_type() == at::kLong,
                "augmentation needs a CUDA int64 stream word");
    return reinterpret_cast<const long long*>(stream->data_ptr());
}

void gather_normalize(at::Tensor data, at::Tensor idx, c10::optional<at::Tensor> cursor, c10::optional<at::Tensor> targets,
                      at::Tensor out, c10::optional<at::Tensor> out_labels, int64_t B, int64_t c_pad, bool nchw,
                      std::vector<double> mean, std::vector<double> stdv, int64_t crop_pad, bool flip, int64_t seed,
                      c10::optional<at::Tensor> aug_stream, int64_t start) {
    CHECK_CUDA(data); CHECK_CUDA(idx); CHECK_CUDA(out);
    TORCH_CHECK(data.dim() == 4 && idx.scalar_type() == at::kLong);
    const int H = data.size(1), W = data.size(2), C = data.size(3);
    TORCH_CHECK((int)mean.size() == C && (int)stdv.size() == C);
    TORCH_CHECK(crop_pad >= 0 && crop_pad < H && crop_pad < W, "crop_pad must lie in [0, image side)");
    const int in_is_float = data.scalar_type() == at::kFloat;
    TORCH_CHECK(in_is_float || data.scalar_type() == at::kByte, "dataset must be uint8 or float32");
    const int out_kind = out.scalar_type() == at::kFloat ? 0 : 1;
    TORCH_CHECK(out_kind == 0 || out.scalar_type() == at::kBFloat16, "out must be fp32 or bf16");
    TORCH_CHECK(out.numel() >= B * H * W * (nchw ? C : c_pad), "out too small");
    float mu[4], sd[4];
    for (int c = 0; c < C; ++c) { mu[c] = (float)mean[c]; sd[c] = (float)stdv[c]; }
    c10::cuda::CUDAGuard guard(data.device());
    check(rlr::launch_gather_normalize(data.data_ptr(), in_is_float, idx.data_ptr<int64_t>(), ptr_or_null<const int>(cursor),
                                       ptr_or_null<const int64_t>(targets), out.data_ptr(), out_kind,
                                       ptr_or_null<int64_t>(out_labels), (int)B, H, W, C, (int)c_pad, nchw ? 1 : 0, mu, sd,
                                       (int)crop_pad, flip ? 1 : 0, (long long)seed, aug_stream_ptr(aug_stream, crop_pad, flip),
                                       (long long)start, cur_stream()), "gather_normalize");
}

// gather + normalise + im2col: A[B*Ho*Wo][64] (bf16) for a k x k / pad stem convolution over data[N,H,W,C]  (C*k*k <= 64)
void gather_im2col(at::Tensor data, at::Tensor idx, c10::optional<at::Tensor> cursor, c10::optional<at::Tensor> targets, at::Tensor A,
                   c10::optional<at::Tensor> out_labels, int64_t B, int64_t k, int64_t pad, std::vector<double> mean, std::vector<double> stdv,
                   int64_t crop_pad, bool flip, int64_t seed, c10::optional<at::Tensor> aug_stream, int64_t start) {
    CHECK_CUDA(data); CHECK_CUDA(idx); CHECK_CUDA(A);
    TORCH_CHECK(data.dim() == 4 && idx.scalar_type() == at::kLong && A.scalar_type() == at::kBFloat16);
    const int H = data.size(1), W = data.size(2), C = data.size(3);
    TORCH_CHECK((int)mean.size() == C && (int)stdv.size() == C && C * k * k <= 64);
    TORCH_CHECK(crop_pad >= 0 && crop_pad < H && crop_pad < W, "crop_pad must lie in [0, image side)");
    const int in_is_float = data.scalar_type() == at::kFloat;
    TORCH_CHECK(in_is_float || data.scalar_type() == at::kByte, "dataset must be uint8 or float32");
    const int64_t Ho = H + 2 * pad - k + 1, Wo = W + 2 * pad - k + 1;
    TORCH_CHECK(A.numel() >= B * Ho * Wo * 64, "A too small");
    float mu[4], sd[4];
    for (int c = 0; c < C; ++c) { mu[c] = (float)mean[c]; sd[c] = (float)stdv[c]; }
    c10::cuda::CUDAGuard guard(data.device());
    check(rlr::launch_gather_im2col(data.data_ptr(), in_is_float, idx.data_ptr<int64_t>(), ptr_or_null<const int>(cursor),
                                    ptr_or_null<const int64_t>(targets), reinterpret_cast<__nv_bfloat16*>(A.data_ptr()),
                                    ptr_or_null<int64_t>(out_labels), (int)B, H, W, C, (int)k, (int)pad, mu, sd, (int)crop_pad, flip ? 1 : 0,
                                    (long long)seed, aug_stream_ptr(aug_stream, crop_pad, flip), (long long)start, cur_stream()), "gather_im2col");
}

void stamp_pixels(at::Tensor data, at::Tensor sel, at::Tensor rows, at::Tensor cols, at::Tensor vals, int64_t mode) {
    CHECK_CUDA(data); CHECK_CUDA(sel); CHECK_CUDA(rows); CHECK_CUDA(cols); CHECK_CUDA(vals);
    TORCH_CHECK(data.dim() == 4 && sel.scalar_type() == at::kLong && rows.scalar_type() == at::kInt &&
                cols.scalar_type() == at::kInt && vals.scalar_type() == at::kFloat);
    const int is_float = data.scalar_type() == at::kFloat;
    TORCH_CHECK(is_float || data.scalar_type() == at::kByte);
    c10::cuda::CUDAGuard guard(data.device());
    check(rlr::launch_stamp_pixels(data.data_ptr(), is_float, sel.data_ptr<int64_t>(), (int)sel.numel(), rows.data_ptr<int>(),
                                   cols.data_ptr<int>(), vals.data_ptr<float>(), (int)rows.numel(), data.size(1), data.size(2),
                                   data.size(3), (int)mode, cur_stream()), "stamp_pixels");
}

void advance_cursor(at::Tensor cursor, int64_t delta, c10::optional<at::Tensor> step) {
    CHECK_CUDA(cursor);
    TORCH_CHECK(cursor.scalar_type() == at::kInt);
    TORCH_CHECK(!(step.has_value() && step->defined()) || step->scalar_type() == at::kLong, "step counter must be int64");
    c10::cuda::CUDAGuard guard(cursor.device());
    check(rlr::launch_advance_cursor(cursor.data_ptr<int>(), (int)delta, reinterpret_cast<long long*>(ptr_or_null<int64_t>(step)),
                                     cur_stream()), "advance_cursor");
}

// zero a contiguous tensor with a memset node on the current stream (no fill kernel inside captured steps)
void memset_zero(at::Tensor t) {
    CHECK_CUDA(t);
    c10::cuda::CUDAGuard guard(t.device());
    check(cudaMemsetAsync(t.data_ptr(), 0, (size_t)t.numel() * t.element_size(), cur_stream()), "memset_zero");
}

void pad_rows(at::Tensor src, at::Tensor dst) {
    CHECK_CUDA(src); CHECK_CUDA(dst);
    TORCH_CHECK(src.scalar_type() == at::kBFloat16 && dst.scalar_type() == at::kBFloat16 && src.dim() == 2 && dst.dim() == 2 &&
                src.size(0) == dst.size(0), "pad_rows: bf16 [R,K] -> [R,Kp]");
    c10::cuda::CUDAGuard guard(src.device());
    check(rlr::launch_pad_rows(reinterpret_cast<const __nv_bfloat16*>(src.data_ptr()), reinterpret_cast<__nv_bfloat16*>(dst.data_ptr()),
                               src.size(0), (int)src.size(1), (int)dst.size(1), num_sms(), cur_stream()), "pad_rows");
}

void unpad_add(at::Tensor src, at::Tensor dst) {
    CHECK_CUDA(src); CHECK_CUDA(dst);
    TORCH_CHECK(src.scalar_type() == at::kFloat && dst.scalar_type() == at::kFloat && src.dim() == 2 && dst.dim() == 2 &&
                src.size(0) == dst.size(0), "unpad_add: fp32 [R,Kp] -> [R,K]");
    c10::cuda::CUDAGuard guard(src.device());
    check(rlr::launch_unpad_add(src.data_ptr<float>(), dst.data_ptr<float>(), src.size(0), (int)dst.size(1), (int)src.size(1), num_sms(),
                                cur_stream()), "unpad_add");
}

// ---------------------------------------------------------------------------------------------------------------
void round_init(at::Tensor w_global, c10::optional<at::Tensor> w_local, c10::optional<at::Tensor> w_bf16,
                c10::optional<at::Tensor> mom) {
    CHECK_CUDA(w_global);
    c10::cuda::CUDAGuard guard(w_global.device());
    check(rlr::launch_round_init(w_global.data_ptr<float>(), ptr_or_null<float>(w_local), ptr_or_null<__nv_bfloat16>(w_bf16),
                                 ptr_or_null<float>(mom), w_global.numel(), cur_stream()), "round_init");
}

// a gradient mask: int32 bit words covering at least n coordinates
inline const uint32_t* mask_ptr(const c10::optional<at::Tensor>& mask, int64_t n) {
    if (!(mask.has_value() && mask->defined())) return nullptr;
    CHECK_CUDA(*mask);
    TORCH_CHECK(mask->scalar_type() == at::kInt && mask->numel() * 32 >= n, "mask: int32 bit words covering ", n, " coordinates");
    return reinterpret_cast<const uint32_t*>(mask->data_ptr());
}

// with w0: the local objective's norm pass, out[0:3] += [sum x^2, sum x d, sum d^2], d = fp32(w - w0) over [0, n_pgd)
void sqnorm(at::Tensor x, at::Tensor out, c10::optional<at::Tensor> mask, int64_t n_mask, c10::optional<at::Tensor> w,
            c10::optional<at::Tensor> w0, int64_t n_pgd) {
    CHECK_CUDA(x); CHECK_CUDA(out);
    TORCH_CHECK(x.scalar_type() == at::kFloat && out.scalar_type() == at::kDouble);
    const bool prox = w0.has_value() && w0->defined();
    if (prox) {
        TORCH_CHECK(w.has_value() && w->defined(), "sqnorm: the objective's norm pass needs w and w0");
        CHECK_CUDA(*w); CHECK_CUDA(*w0);
        TORCH_CHECK(w->scalar_type() == at::kFloat && w0->scalar_type() == at::kFloat && w->numel() == x.numel() &&
                    w0->numel() >= n_pgd && out.numel() >= 3, "sqnorm: fp32 w [n], w0 [>= n_pgd], fp64 out [3]");
    }
    c10::cuda::CUDAGuard guard(x.device());
    check(rlr::launch_sqnorm(x.data_ptr<float>(), x.numel(), out.data_ptr<double>(), num_sms(), cur_stream(), mask_ptr(mask, n_mask),
                             n_mask, prox ? w->data_ptr<float>() : nullptr, prox ? w0->data_ptr<float>() : nullptr, n_pgd), "sqnorm");
}

void sgd_step(at::Tensor w, at::Tensor g, at::Tensor m, c10::optional<at::Tensor> w0, c10::optional<at::Tensor> w_bf16,
              double lr, double momentum, double max_grad_norm, c10::optional<at::Tensor> g_sqnorm,
              c10::optional<at::Tensor> d_sqnorm, int64_t n_pgd, c10::optional<at::Tensor> w_in, c10::optional<at::Tensor> mask,
              c10::optional<std::vector<double>> objective) {
    CHECK_CUDA(w); CHECK_CUDA(g); CHECK_CUDA(m);
    TORCH_CHECK(w.numel() == g.numel() && w.numel() == m.numel());
    TORCH_CHECK(!(d_sqnorm.has_value() && d_sqnorm->defined()) || (w0.has_value() && w0->defined()), "PGD needs w0");
    float obj[3] = {1.f, 0.f, 0.f};
    if (objective.has_value()) {
        TORCH_CHECK(objective->size() == 3, "sgd_step: objective = (a, b, mu)");
        TORCH_CHECK(w0.has_value() && w0->defined() && g_sqnorm.has_value() && g_sqnorm->defined() && g_sqnorm->numel() >= 3,
                    "sgd_step: the objective needs w0 and the norm pass's three sums");
        for (int i = 0; i < 3; ++i) obj[i] = (float)(*objective)[i];
    }
    c10::cuda::CUDAGuard guard(w.device());
    check(rlr::launch_sgd_step(w.data_ptr<float>(), g.data_ptr<float>(), m.data_ptr<float>(), ptr_or_null<const float>(w0),
                               ptr_or_null<__nv_bfloat16>(w_bf16), w.numel(), (float)lr, (float)momentum,
                               (float)max_grad_norm, ptr_or_null<const double>(g_sqnorm), ptr_or_null<double>(d_sqnorm),
                               num_sms(), cur_stream(), n_pgd, ptr_or_null<const float>(w_in),
                               mask_ptr(mask, n_pgd > 0 && n_pgd <= w.numel() ? n_pgd : w.numel()), objective.has_value() ? obj : nullptr),
          "sgd_step");
}

void pgd_project(at::Tensor w, at::Tensor w0, c10::optional<at::Tensor> w_bf16, double clip, at::Tensor d_sqnorm, int64_t n_pgd,
                 c10::optional<at::Tensor> mask) {
    CHECK_CUDA(w); CHECK_CUDA(w0); CHECK_CUDA(d_sqnorm);
    c10::cuda::CUDAGuard guard(w.device());
    check(rlr::launch_pgd_project(w.data_ptr<float>(), w0.data_ptr<float>(), ptr_or_null<__nv_bfloat16>(w_bf16), w.numel(),
                                  (float)clip, d_sqnorm.data_ptr<double>(), num_sms(), cur_stream(), n_pgd,
                                  mask_ptr(mask, n_pgd > 0 && n_pgd <= w.numel() ? n_pgd : w.numel())), "pgd_project");
}

void neurotoxin_mask(at::Tensor w_g, at::Tensor w_prev, int64_t n_vote, int64_t k, at::Tensor mask, at::Tensor count) {
    CHECK_CUDA(w_g); CHECK_CUDA(w_prev); CHECK_CUDA(mask); CHECK_CUDA(count);
    TORCH_CHECK(w_g.scalar_type() == at::kFloat && w_prev.scalar_type() == at::kFloat && count.scalar_type() == at::kLong &&
                count.numel() >= 1);
    TORCH_CHECK(w_g.numel() >= n_vote && w_prev.numel() >= n_vote, "neurotoxin_mask: w_g / w_prev shorter than n_vote");
    mask_ptr(mask, n_vote);
    c10::cuda::CUDAGuard guard(w_g.device());
    check(rlr::launch_neurotoxin_mask(w_g.data_ptr<float>(), w_prev.data_ptr<float>(), n_vote, k,
                                      reinterpret_cast<uint32_t*>(mask.data_ptr()), reinterpret_cast<long long*>(count.data_ptr()), num_sms(), cur_stream()),
          "neurotoxin_mask");
}

void sparsefed(at::Tensor w_new, at::Tensor w, c10::optional<at::Tensor> w_bf16, at::Tensor e, int64_t n_vote, int64_t k, at::Tensor stats) {
    CHECK_CUDA(w_new); CHECK_CUDA(w); CHECK_CUDA(e); CHECK_CUDA(stats);
    TORCH_CHECK(w_new.scalar_type() == at::kFloat && w.scalar_type() == at::kFloat && e.scalar_type() == at::kFloat &&
                stats.scalar_type() == at::kDouble && stats.numel() >= 3, "sparsefed: fp32 w_new / w / e and an fp64 stats[3]");
    TORCH_CHECK(w_new.numel() == w.numel() && e.numel() >= n_vote && n_vote <= w.numel(), "sparsefed: w_new / w / e sizes");
    if (w_bf16) {
        CHECK_CUDA(*w_bf16);
        TORCH_CHECK(w_bf16->scalar_type() == at::kBFloat16 && w_bf16->numel() == w.numel(), "sparsefed: bf16 shadow of w's size");
    }
    c10::cuda::CUDAGuard guard(w.device());
    check(rlr::launch_sparsefed(w_new.data_ptr<float>(), w.data_ptr<float>(), w_bf16 ? w_bf16->data_ptr() : nullptr, e.data_ptr<float>(),
                                n_vote, w.numel(), k, stats.data_ptr<double>(), num_sms(), cur_stream()), "sparsefed");
}

static void crfl_check(const char* what, const at::Tensor& src, const at::Tensor& dst, const c10::optional<at::Tensor>& dst_bf16,
                       const at::Tensor& mask, int64_t n_vote) {
    CHECK_CUDA(src); CHECK_CUDA(dst); CHECK_CUDA(mask);
    TORCH_CHECK(src.scalar_type() == at::kFloat && dst.scalar_type() == at::kFloat && src.is_contiguous() && dst.is_contiguous() &&
                src.numel() == dst.numel(), what, ": contiguous fp32 source and destination of one size");
    TORCH_CHECK(mask.scalar_type() == at::kInt && mask.is_contiguous() && mask.numel() * 32 >= n_vote && n_vote <= src.numel(),
                what, ": int32 mask words covering [0, n_vote)");
    if (dst_bf16) {
        CHECK_CUDA(*dst_bf16);
        TORCH_CHECK(dst_bf16->scalar_type() == at::kBFloat16 && dst_bf16->numel() == dst.numel(), what, ": bf16 shadow of the destination's size");
    }
}

void crfl_clip_noise(at::Tensor w_new, at::Tensor w, c10::optional<at::Tensor> w_bf16, at::Tensor mask, int64_t n_vote, double rho,
                     double sigma, int64_t seed, int64_t stream, at::Tensor stats) {
    crfl_check("crfl_clip_noise", w_new, w, w_bf16, mask, n_vote);
    CHECK_CUDA(stats);
    TORCH_CHECK(stats.scalar_type() == at::kDouble && stats.numel() >= 2, "crfl_clip_noise: an fp64 stats[2]");
    c10::cuda::CUDAGuard guard(w.device());
    check(rlr::launch_crfl_clip_noise(w_new.data_ptr<float>(), w.data_ptr<float>(), w_bf16 ? w_bf16->data_ptr() : nullptr,
                                      reinterpret_cast<const uint32_t*>(mask.data_ptr<int>()), n_vote, w.numel(), rho, (float)sigma,
                                      (unsigned long long)seed, (unsigned long long)stream, stats.data_ptr<double>(), num_sms(), cur_stream()),
          "crfl_clip_noise");
}

void crfl_smooth(at::Tensor w, at::Tensor out, c10::optional<at::Tensor> out_bf16, at::Tensor mask, int64_t n_vote, double sigma,
                 int64_t seed, int64_t stream) {
    crfl_check("crfl_smooth", w, out, out_bf16, mask, n_vote);
    c10::cuda::CUDAGuard guard(w.device());
    check(rlr::launch_crfl_smooth(w.data_ptr<float>(), out.data_ptr<float>(), out_bf16 ? out_bf16->data_ptr() : nullptr,
                                  reinterpret_cast<const uint32_t*>(mask.data_ptr<int>()), n_vote, w.numel(), (float)sigma,
                                  (unsigned long long)seed, (unsigned long long)stream, num_sms(), cur_stream()),
          "crfl_smooth");
}

void vote_count(at::Tensor logits, at::Tensor counts, int64_t row0) {
    CHECK_CUDA(logits); CHECK_CUDA(counts);
    TORCH_CHECK(logits.scalar_type() == at::kFloat && logits.dim() == 2 && logits.is_contiguous(), "vote_count: contiguous fp32 logits [rows][classes]");
    TORCH_CHECK(counts.scalar_type() == at::kInt && counts.dim() == 2 && counts.is_contiguous() && counts.size(1) == logits.size(1) &&
                row0 >= 0 && row0 + logits.size(0) <= counts.size(0), "vote_count: int32 counts [inputs][classes] holding rows row0 ..");
    c10::cuda::CUDAGuard guard(logits.device());
    check(rlr::launch_vote_count(logits.data_ptr<float>(), logits.size(0), (int)logits.size(1), counts.data_ptr<int>(), row0, cur_stream()),
          "vote_count");
}

void flare_mmd(at::Tensor z, at::Tensor finite, double inv_s2, at::Tensor out) {
    CHECK_CUDA(z); CHECK_CUDA(finite); CHECK_CUDA(out);
    TORCH_CHECK(z.scalar_type() == at::kFloat && z.dim() == 3 && z.is_contiguous(), "flare_mmd: contiguous fp32 features [K][n][d]");
    const int64_t K = z.size(0);
    TORCH_CHECK(finite.scalar_type() == at::kBool && finite.numel() == K && finite.is_contiguous(), "flare_mmd: bool finite[K]");
    TORCH_CHECK(out.scalar_type() == at::kDouble && out.numel() == K * (K + 1) / 2 && out.is_contiguous(), "flare_mmd: fp64 out[K (K + 1) / 2]");
    TORCH_CHECK(K >= 1 && z.size(1) >= 1 && z.size(2) >= 1 && K < (1LL << 31) && z.size(1) < (1LL << 31) && z.size(2) < (1LL << 31),
                "flare_mmd: empty or oversized features");
    c10::cuda::CUDAGuard guard(z.device());
    check(rlr::launch_flare_mmd(z.data_ptr<float>(), reinterpret_cast<const unsigned char*>(finite.data_ptr()), (int)K, (int)z.size(1),
                                (int)z.size(2), (float)inv_s2, out.data_ptr<double>(), cur_stream()), "flare_mmd");
}

void deepsight_stats(at::Tensor z, at::Tensor zg, at::Tensor slot_ptrs, int64_t wg_ptr, int64_t w_off, int64_t b_off, int64_t S,
                     int64_t d, at::Tensor out) {
    CHECK_CUDA(z); CHECK_CUDA(zg); CHECK_CUDA(slot_ptrs); CHECK_CUDA(out);
    TORCH_CHECK(z.scalar_type() == at::kFloat && z.dim() == 3 && z.is_contiguous(), "deepsight_stats: contiguous fp32 logits [K][S N][P]");
    const int64_t K = z.size(0), SN = z.size(1), P = z.size(2);
    TORCH_CHECK(K >= 1 && S >= 1 && SN >= 1 && SN % S == 0 && K < (1LL << 31) && SN < (1LL << 31) && d >= 1 && d < (1LL << 31),
                "deepsight_stats: empty or oversized logits, or S does not divide their rows");
    TORCH_CHECK(P >= 1 && P <= rlr::kDeepSightMaxClasses, "deepsight_stats: ", P, " classes; the pass takes 1 to ",
                rlr::kDeepSightMaxClasses);
    TORCH_CHECK(zg.scalar_type() == at::kFloat && zg.is_contiguous() && zg.dim() == 2 && zg.size(0) == SN && zg.size(1) == P,
                "deepsight_stats: contiguous fp32 global logits [S N][P]");
    TORCH_CHECK(slot_ptrs.scalar_type() == at::kLong && slot_ptrs.numel() == K, "deepsight_stats: int64 pointer table [K]");
    TORCH_CHECK(wg_ptr && w_off >= 0 && b_off >= 0, "deepsight_stats: global parameters and head offsets");
    TORCH_CHECK(out.scalar_type() == at::kDouble && out.is_contiguous() && out.numel() == K * (S + 2) * P,
                "deepsight_stats: fp64 out[K][(S + 2) P]");
    c10::cuda::CUDAGuard guard(z.device());
    check(rlr::launch_deepsight_stats(z.data_ptr<float>(), zg.data_ptr<float>(), reinterpret_cast<const float* const*>(slot_ptrs.data_ptr()),
                                      reinterpret_cast<const float*>(wg_ptr), w_off, b_off, (int)K, (int)S, (int)(SN / S), (int)P, (int)d,
                                      out.data_ptr<double>(), cur_stream()), "deepsight_stats");
}

void boost_update(at::Tensor slot, at::Tensor w_g, double gamma, int64_t n_vote) {
    CHECK_CUDA(slot); CHECK_CUDA(w_g);
    TORCH_CHECK(slot.scalar_type() == at::kFloat && w_g.scalar_type() == at::kFloat);
    TORCH_CHECK(slot.numel() >= n_vote && w_g.numel() >= n_vote, "boost_update: slot / w_g shorter than n_vote");
    c10::cuda::CUDAGuard guard(slot.device());
    check(rlr::launch_boost_update(slot.data_ptr<float>(), w_g.data_ptr<float>(), n_vote, gamma, num_sms(), cur_stream()), "boost_update");
}

void swap_samples(at::Tensor data, at::Tensor targets, at::Tensor idx, at::Tensor side_data, at::Tensor side_targets) {
    CHECK_CUDA(data); CHECK_CUDA(targets); CHECK_CUDA(idx); CHECK_CUDA(side_data); CHECK_CUDA(side_targets);
    TORCH_CHECK(targets.scalar_type() == at::kLong && idx.scalar_type() == at::kLong && side_targets.scalar_type() == at::kLong,
                "swap_samples: targets, idx and side_targets must be int64");
    TORCH_CHECK(data.scalar_type() == side_data.scalar_type() && data.dim() >= 1 && side_data.dim() >= 1,
                "swap_samples: data and side_data must share a dtype");
    const int64_t n = idx.numel();
    TORCH_CHECK(side_data.size(0) == n && side_targets.numel() == n && targets.numel() == data.size(0),
                "swap_samples: one side row and label per index, one label per data row");
    TORCH_CHECK(data.size(0) > 0 || n == 0, "swap_samples: empty dataset");
    const int64_t row_bytes = data.size(0) > 0 ? data.numel() / data.size(0) * data.element_size() : 0;
    TORCH_CHECK(n == 0 || side_data.numel() / n * side_data.element_size() == row_bytes, "swap_samples: side rows differ in size");
    if (n == 0) return;
    c10::cuda::CUDAGuard guard(data.device());
    check(rlr::launch_swap_samples(data.data_ptr(), reinterpret_cast<long long*>(targets.data_ptr()),
                                   reinterpret_cast<const long long*>(idx.data_ptr()), side_data.data_ptr(),
                                   reinterpret_cast<long long*>(side_targets.data_ptr()), n, row_bytes, num_sms(), cur_stream()),
          "swap_samples");
}

// ---------------------------------------------------------------------------------------------------------------
void softmax_xent(at::Tensor logits, at::Tensor labels, c10::optional<at::Tensor> dlogits, c10::optional<at::Tensor> loss_sum,
                  c10::optional<at::Tensor> correct, double grad_scale) {
    CHECK_CUDA(logits); CHECK_CUDA(labels);
    TORCH_CHECK(logits.dim() == 2 && labels.scalar_type() == at::kLong);
    const int kind = logits.scalar_type() == at::kFloat ? 0 : 1;
    TORCH_CHECK(kind == 0 || logits.scalar_type() == at::kBFloat16);
    c10::cuda::CUDAGuard guard(logits.device());
    check(rlr::launch_softmax_xent(logits.data_ptr(), kind, labels.data_ptr<int64_t>(),
                                   dlogits.has_value() && dlogits->defined() ? dlogits->data_ptr() : nullptr,
                                   ptr_or_null<float>(loss_sum), ptr_or_null<int>(correct), (int)logits.size(0),
                                   (int)logits.size(1), (float)grad_scale, cur_stream()), "softmax_xent");
}

void eval_metrics(at::Tensor logits, at::Tensor labels, at::Tensor loss_sum, at::Tensor confusion) {
    CHECK_CUDA(logits); CHECK_CUDA(labels); CHECK_CUDA(loss_sum); CHECK_CUDA(confusion);
    TORCH_CHECK(loss_sum.scalar_type() == at::kDouble && confusion.scalar_type() == at::kLong);
    const int kind = logits.scalar_type() == at::kFloat ? 0 : 1;
    c10::cuda::CUDAGuard guard(logits.device());
    check(rlr::launch_eval_metrics(logits.data_ptr(), kind, labels.data_ptr<int64_t>(), (int)logits.size(0), (int)logits.size(1),
                                   loss_sum.data_ptr<double>(), reinterpret_cast<long long*>(confusion.data_ptr<int64_t>()),
                                   cur_stream()), "eval_metrics");
}

// ---------------------------------------------------------------------------------------------------------------
// CUDA-IPC symmetric buffers: cudaMalloc'ed slabs whose handles are exchanged through torch.distributed and opened
// by every peer (fallback when torch's symmetric memory / multicast is unavailable).
// ---------------------------------------------------------------------------------------------------------------
std::pair<int64_t, py::bytes> ipc_alloc(int64_t nbytes, int64_t device) {
    c10::cuda::CUDAGuard guard((c10::DeviceIndex)device);
    void* p = nullptr;
    check(cudaMalloc(&p, (size_t)nbytes), "ipc_alloc/cudaMalloc");
    check(cudaMemset(p, 0, (size_t)nbytes), "ipc_alloc/cudaMemset");
    cudaIpcMemHandle_t h;
    check(cudaIpcGetMemHandle(&h, p), "cudaIpcGetMemHandle");
    return {reinterpret_cast<int64_t>(p), py::bytes(reinterpret_cast<const char*>(&h), sizeof(h))};
}
int64_t ipc_open(const std::string& handle, int64_t device) {
    TORCH_CHECK(handle.size() == sizeof(cudaIpcMemHandle_t), "bad IPC handle size");
    c10::cuda::CUDAGuard guard((c10::DeviceIndex)device);
    cudaIpcMemHandle_t h;
    memcpy(&h, handle.data(), sizeof(h));
    void* p = nullptr;
    check(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess), "cudaIpcOpenMemHandle");
    return reinterpret_cast<int64_t>(p);
}
void ipc_close(int64_t ptr) { check(cudaIpcCloseMemHandle(reinterpret_cast<void*>(ptr)), "cudaIpcCloseMemHandle"); }
void ipc_free(int64_t ptr) { check(cudaFree(reinterpret_cast<void*>(ptr)), "cudaFree"); }

at::Tensor tensor_from_ptr(int64_t ptr, std::vector<int64_t> sizes, at::ScalarType dtype, int64_t device) {
    auto opts = at::TensorOptions().dtype(dtype).device(at::kCUDA, (c10::DeviceIndex)device);
    return at::from_blob(reinterpret_cast<void*>(ptr), sizes, [](void*) {}, opts);
}

}  // namespace

void register_gemm_bindings(py::module_& m);  // gemm_binding.cpp

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
    m.doc() = "robust-fl sm_90a kernels";
    m.def("fused_aggregate", &fused_aggregate, py::arg("w_agent_ptrs"), py::arg("weights"), py::arg("scales"), py::arg("total_weight"),
          py::arg("w_global_ptr"), py::arg("out_ptrs"), py::arg("out_bf16_ptrs"), py::arg("use_multimem"), py::arg("begin"), py::arg("end"),
          py::arg("n_vote"), py::arg("mode"), py::arg("theta"), py::arg("server_lr"), py::arg("noise_std"), py::arg("seed"),
          py::arg("noise_stream"), py::arg("flipped"), py::arg("flag_ptrs"), py::arg("local_sync"), py::arg("rank"), py::arg("world"),
          py::arg("epoch"), py::arg("handoff") = false, py::arg("opt") = 0, py::arg("beta1") = 0.0, py::arg("beta2") = 0.0,
          py::arg("tau") = 0.0, py::arg("opt_m") = py::none(), py::arg("opt_v") = py::none(), py::arg("state_base") = 0);
    m.def("aggregate_max_agents", &rlr::aggregate_max_agents);
    m.def("acquire_slices", &acquire_slices);
    m.def("pairwise_sqdist", &pairwise_sqdist);
    m.def("pairwise_gram", &pairwise_gram);
    m.def("history_accumulate", &history_accumulate);
    m.def("history_gram", &history_gram);
    m.def("dnc_gather", &dnc_gather);
    m.def("fld_ring", &fld_ring);
    m.def("fld_hvp", &fld_hvp);
    m.def("fld_predict", &fld_predict);
    m.def("trust_stats", &trust_stats);
    m.def("rfa_sqdist", &rfa_sqdist);
    m.def("collude_stats", &collude_stats);
    m.def("collude_write", &collude_write);
    m.def("gather_normalize", &gather_normalize);
    m.def("gather_im2col", &gather_im2col);
    m.def("stamp_pixels", &stamp_pixels);
    m.def("advance_cursor", &advance_cursor, py::arg("cursor"), py::arg("delta"), py::arg("step") = py::none());
    m.def("memset_zero", &memset_zero);
    m.def("pad_rows", &pad_rows);
    m.def("unpad_add", &unpad_add);
    m.def("round_init", &round_init);
    m.def("sqnorm", &sqnorm, py::arg("x"), py::arg("out"), py::arg("mask") = py::none(), py::arg("n_mask") = 0, py::arg("w") = py::none(),
          py::arg("w0") = py::none(), py::arg("n_pgd") = 0);
    m.def("sgd_step", &sgd_step, py::arg("w"), py::arg("g"), py::arg("m"), py::arg("w0"), py::arg("w_bf16"), py::arg("lr"),
          py::arg("momentum"), py::arg("max_grad_norm"), py::arg("g_sqnorm"), py::arg("d_sqnorm"), py::arg("n_pgd") = 0, py::arg("w_in") = py::none(),
          py::arg("mask") = py::none(), py::arg("objective") = py::none());
    m.def("neurotoxin_mask", &neurotoxin_mask);
    m.def("boost_update", &boost_update);
    m.def("sparsefed", &sparsefed);
    m.def("crfl_clip_noise", &crfl_clip_noise);
    m.def("crfl_smooth", &crfl_smooth);
    m.def("vote_count", &vote_count);
    m.def("flare_mmd", &flare_mmd);
    m.def("deepsight_stats", &deepsight_stats);
    m.def("swap_samples", &swap_samples);
    m.def("pgd_project", &pgd_project, py::arg("w"), py::arg("w0"), py::arg("w_bf16"), py::arg("clip"), py::arg("d_sqnorm"),
          py::arg("n_pgd") = 0, py::arg("mask") = py::none());
    m.def("softmax_xent", &softmax_xent);
    m.def("eval_metrics", &eval_metrics);
    m.def("ipc_alloc", &ipc_alloc);
    m.def("ipc_open", &ipc_open);
    m.def("ipc_close", &ipc_close);
    m.def("ipc_free", &ipc_free);
    m.def("tensor_from_ptr", &tensor_from_ptr);
    register_gemm_bindings(m);
}
