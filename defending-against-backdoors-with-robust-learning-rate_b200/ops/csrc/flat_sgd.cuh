// The fused local-optimizer kernels over flat buffers (elementwise.cu launches them): the norm pass and the clip + momentum-SGD step.
// Templates here, instantiated in two translation units: elementwise.cu holds the plain instantiations (PROX = false) and objective.cu
// the local objective's (PROX = true).  Compiled next to each other, the PROX kernels changed how ptxas scheduled the plain step kernel;
// apart, the plain kernels keep exactly the instructions they had before the objective existed.
#pragma once
#include "common.cuh"

namespace rlr {

// MASK: a gradient mask of bit words over [0, 4 * n4_mask) (bit c % 32 of word c / 32 set = coordinate c reads as zero); the thread of
// float4 q takes the nibble (q % 8) of word q / 8.  The <false> instantiations compile to the same instructions as the unmasked kernels.
__device__ __forceinline__ float4 apply_mask(float4 v, const uint32_t* __restrict__ mask, long long q, long long n4_mask) {
    if (q < n4_mask) {
        const uint32_t nib = (__ldg(mask + (q >> 3)) >> ((q & 7) * 4)) & 0xFu;
        if (nib) {
            if (nib & 1u) v.x = 0.f;
            if (nib & 2u) v.y = 0.f;
            if (nib & 4u) v.z = 0.f;
            if (nib & 8u) v.w = 0.f;
        }
    }
    return v;
}

// d = fp32(w - w0) per lane, the distance of the local objective's pull toward the round's global parameters (FlatSGD, ops/__init__.py)
__device__ __forceinline__ float4 prox_dist(float4 w, float4 o) {
    return make_float4(__fsub_rn(w.x, o.x), __fsub_rn(w.y, o.y), __fsub_rn(w.z, o.z), __fsub_rn(w.w, o.w));
}

// PROX: each CTA writes three partials [S_gg, S_gd, S_dd] instead of one: S_gg as without PROX, and over [0, n4_pgd) S_gd = sum g d and
// S_dd = sum d^2 with d = prox_dist(w, w0), masked like g.  The products of two fp32 values are exact in fp64, so only the fp64 additions
// round.  The <MASK, false> instantiations compile to the same instructions as before PROX existed.
template <bool MASK, bool PROX>
__global__ void __launch_bounds__(256) sqnorm_kernel(const float* __restrict__ x, long long n4, double* part /*[gridDim.x][1 or 3]*/,
                                                     const uint32_t* __restrict__ mask, long long n4_mask, const float* __restrict__ w,
                                                     const float* __restrict__ w0, long long n4_pgd) {
    __shared__ double scratch[32];
    double acc = 0.0, gd = 0.0, dd = 0.0;
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n4; q += (long long)gridDim.x * blockDim.x) {
        float4 v = ld_f4(x + 4 * q);
        if (MASK) v = apply_mask(v, mask, q, n4_mask);
        acc += (double)(v.x * v.x + v.y * v.y) + (double)(v.z * v.z + v.w * v.w);
        if constexpr (PROX) {
            if (q < n4_pgd) {
                float4 d = prox_dist(ld_f4(w + 4 * q), ld_f4(w0 + 4 * q));
                if (MASK) d = apply_mask(d, mask, q, n4_mask);
                gd = fma((double)v.x, (double)d.x, gd); gd = fma((double)v.y, (double)d.y, gd);
                gd = fma((double)v.z, (double)d.z, gd); gd = fma((double)v.w, (double)d.w, gd);
                dd = fma((double)d.x, (double)d.x, dd); dd = fma((double)d.y, (double)d.y, dd);
                dd = fma((double)d.z, (double)d.z, dd); dd = fma((double)d.w, (double)d.w, dd);
            }
        }
    }
    const double tot = block_sum<double>(acc, scratch);
    if constexpr (PROX) {
        const double tgd = block_sum<double>(gd, scratch), tdd = block_sum<double>(dd, scratch);
        if (threadIdx.x == 0) { part[3 * blockIdx.x] = tot; part[3 * blockIdx.x + 1] = tgd; part[3 * blockIdx.x + 2] = tdd; }
    } else {
        if (threadIdx.x == 0) part[blockIdx.x] = tot;
    }
}
template <bool MASK, bool PROX>
__global__ void __launch_bounds__(256) sgd_step_kernel(float* __restrict__ w, const float* __restrict__ g,
                                                         float* __restrict__ m, const float* __restrict__ w0,
                                                         __nv_bfloat16* __restrict__ wb, long long n4, float lr,
                                                         float momentum, float max_grad_norm,
                                                         const double* __restrict__ g_sqnorm, double* d_part /*[gridDim.x]*/,
                                                         long long n4_pgd, const float* __restrict__ w_in, int first,
                                                         const uint32_t* __restrict__ mask, float obj_a, float obj_b, float obj_mu) {
    // MASK: the gradient mask covers [0, n4_pgd) (the model parameters)
    // first = 1: first local step of a round, fused with the round hand-off -- parameters are read from the broadcast buffer w_in
    // (= the round's global parameters) and the momentum is taken as zero (fresh optimizer every round, src/agent.py:37-38), so no
    // separate "w <- w_global, m <- 0" pass exists.  Coordinates >= n4_pgd (BatchNorm running statistics, already updated in w by
    // this step's forward pass) keep their value.
    // PROX: the local objective a CE + b ||d|| + (mu/2) ||d||^2 (FlatSGD, ops/__init__.py): g_sqnorm holds the norm pass's
    // [S_gg, S_gd, S_dd], and the step applies G = fp32(fp32(a g) + fp32(fp32(beta) d)) in place of g, d = prox_dist(w, w0) over
    // [0, n4_pgd) and G = fp32(a g) behind it
    __shared__ double scratch[32];
    float coef = 1.0f;
    if (!PROX && max_grad_norm > 0.f && g_sqnorm) {
        // torch.nn.utils.clip_grad_norm_: coef = max_norm / (total_norm + 1e-6), clamped to 1
        coef = fminf(1.0f, max_grad_norm / ((float)sqrt(*g_sqnorm) + 1e-6f));
    }
    float beta_f = 0.f;
    if constexpr (PROX) {
        // beta = b / ||d|| + mu (b / ||d|| := 0 at ||d|| = 0);  ||G||^2 = a^2 S_gg + 2 a beta S_gd + beta^2 S_dd, floored at 0
        const double S_gg = g_sqnorm[0], S_gd = g_sqnorm[1], S_dd = g_sqnorm[2];
        const double a = obj_a, dn = sqrt(S_dd);
        const double beta = __dadd_rn(dn > 0.0 ? __ddiv_rn((double)obj_b, dn) : 0.0, (double)obj_mu);
        const double G2 = __dadd_rn(__dadd_rn(__dmul_rn(__dmul_rn(a, a), S_gg), __dmul_rn(__dmul_rn(2.0 * a, beta), S_gd)),
                                    __dmul_rn(__dmul_rn(beta, beta), S_dd));
        beta_f = (float)beta;
        if (max_grad_norm > 0.f) coef = fminf(1.0f, max_grad_norm / ((float)sqrt(fmax(G2, 0.0)) + 1e-6f));
    }
    double dacc = 0.0;
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n4; q += (long long)gridDim.x * blockDim.x) {
        if (first && q >= n4_pgd) { st_f4(m + 4 * q, make_float4(0.f, 0.f, 0.f, 0.f)); continue; }
        float4 gv = ld_f4(g + 4 * q);
        if (MASK) gv = apply_mask(gv, mask, q, n4_pgd);
        const float4 mv = first ? make_float4(0.f, 0.f, 0.f, 0.f) : ld_f4(m + 4 * q), wv = ld_f4((first ? w_in : w) + 4 * q);
        if constexpr (PROX) {
            gv = make_float4(__fmul_rn(obj_a, gv.x), __fmul_rn(obj_a, gv.y), __fmul_rn(obj_a, gv.z), __fmul_rn(obj_a, gv.w));
            if (q < n4_pgd) {
                float4 d = prox_dist(wv, ld_f4(w0 + 4 * q));
                if (MASK) d = apply_mask(d, mask, q, n4_pgd);
                gv.x = __fadd_rn(gv.x, __fmul_rn(beta_f, d.x)); gv.y = __fadd_rn(gv.y, __fmul_rn(beta_f, d.y));
                gv.z = __fadd_rn(gv.z, __fmul_rn(beta_f, d.z)); gv.w = __fadd_rn(gv.w, __fmul_rn(beta_f, d.w));
            }
        }
        float4 mn, wn;
        mn.x = momentum * mv.x + coef * gv.x; mn.y = momentum * mv.y + coef * gv.y;
        mn.z = momentum * mv.z + coef * gv.z; mn.w = momentum * mv.w + coef * gv.w;
        wn.x = wv.x - lr * mn.x; wn.y = wv.y - lr * mn.y; wn.z = wv.z - lr * mn.z; wn.w = wv.w - lr * mn.w;
        st_f4(m + 4 * q, mn);
        st_f4(w + 4 * q, wn);
        if (d_part) {
            // PGD radius is measured over the model parameters only ([0, n_pgd): the reference projects parameters_to_vector(),
            // src/agent.py:54-60); BatchNorm running statistics stored behind them never count and are never rescaled
            if (q < n4_pgd) {
                const float4 o = ld_f4(w0 + 4 * q);
                const float d0 = wn.x - o.x, d1 = wn.y - o.y, d2 = wn.z - o.z, d3 = wn.w - o.w;
                dacc += (double)(d0 * d0 + d1 * d1) + (double)(d2 * d2 + d3 * d3);
            }
        } else if (wb) {
            *reinterpret_cast<uint2*>(wb + 4 * q) = make_uint2(pack_bf16x2(wn.x, wn.y), pack_bf16x2(wn.z, wn.w));
        }
    }
    if (d_part) {
        const double tot = block_sum<double>(dacc, scratch);
        if (threadIdx.x == 0) d_part[blockIdx.x] = tot;
    }
}
// the PROX launches (objective.cu); the arguments are the kernels'
void launch_sqnorm_objective(int grid, cudaStream_t st, const float* x, long long n4, double* part, const uint32_t* mask, long long n4_mask,
                             const float* w, const float* w0, long long n4_pgd);
void launch_sgd_step_objective(int grid, cudaStream_t st, float* w, const float* g, float* m, const float* w0, __nv_bfloat16* wb, long long n4,
                               float lr, float momentum, float max_grad_norm, const double* sums, double* d_part, long long n4_pgd,
                               const float* w_in, const uint32_t* mask, float obj_a, float obj_b, float obj_mu);

}  // namespace rlr
