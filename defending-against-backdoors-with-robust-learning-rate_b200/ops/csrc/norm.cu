// Memory-bound layer kernels over NHWC bf16 activations (one 16-byte vector = 8 channels per thread):
// BatchNorm (training statistics, fused normalise + residual add + ReLU, two-pass backward), ReLU backward, 2x2
// max-pool, global average pool, dropout (Philox), space-to-depth for strided convs, filter transpose for dgrad, and
// the tiny classifier heads.  They replace the ATen elementwise / cuDNN-BN calls behind autograd in the reference's
// local step (src/agent.py:46-48) and are what the wgmma conv kernels hand their outputs to.
#include <stdlib.h>

#include "common.cuh"
#include "gemm.h"

namespace rlr {

struct bf8 { float v[8]; };
__device__ __forceinline__ bf8 unpack8(const uint4& u) {
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
    bf8 r;
#pragma unroll
    for (int i = 0; i < 4; ++i) { const float2 f = __bfloat1622float2(h[i]); r.v[2 * i] = f.x; r.v[2 * i + 1] = f.y; }
    return r;
}
__device__ __forceinline__ bf8 load8(const __nv_bfloat16* p) { return unpack8(*reinterpret_cast<const uint4*>(p)); }
__device__ __forceinline__ void store8(__nv_bfloat16* p, const bf8& r) {
    uint4 u;
    u.x = pack_bf16x2(r.v[0], r.v[1]); u.y = pack_bf16x2(r.v[2], r.v[3]);
    u.z = pack_bf16x2(r.v[4], r.v[5]); u.w = pack_bf16x2(r.v[6], r.v[7]);
    *reinterpret_cast<uint4*>(p) = u;
}
static inline int rows_grid(long long M, int rows_per_block, int num_sms, int per_sm) {
    long long want = (M + rows_per_block - 1) / rows_per_block;
    long long cap = (long long)num_sms * per_sm;
    return (int)(want < 1 ? 1 : (want > cap ? cap : want));
}
static inline bool chan_ok(int C) { return C >= 8 && C <= 2048 && (C % 8) == 0 && (256 % (C / 8)) == 0; }

// ---------------------------------------------------------------------------------------------------------------------
// per-channel reductions:  out[0][c] += sum_r a(r,c),  out[1][c] += sum_r b(r,c)
// MODE 0: a = x, b = x^2 (forward statistics)     MODE 1: a = dz, b = dz * xhat (backward)
// ---------------------------------------------------------------------------------------------------------------------
// U rows per thread and iteration, all loads issued before the first use.  The grid (and so the partial-sum layout) is fixed by the
// launchers at kCtasPerSm CTAs per SM; U and the register cap are chosen per residency so that every thread keeps as many 16-byte
// loads in flight as its registers allow.  U never changes a thread's rows or their order of addition.
template <int MODE, bool kRecompute, int U, int kCtasPerSm>
__global__ void __launch_bounds__(256, kCtasPerSm) channel_reduce_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy,
                                                               const __nv_bfloat16* __restrict__ y, const float* __restrict__ mean_rstd,
                                                               float* __restrict__ part /*[gridDim.x][ncols] partial sums*/, long long M, int C, int relu,
                                                               const float* __restrict__ gamma = nullptr, const float* __restrict__ beta = nullptr,
                                                               int out_cols = 0 /*0: both rows (2C values) | C: only the first row (bias gradients)*/) {
    // relu: 0 none | 1 mask = (y > 0) from the stored output | 2 mask recomputed as (x * scale + shift > 0) with exactly the
    // expression of bn_apply_kernel -- BatchNorm + ReLU without a residual: the output tensor is not read at all
    extern __shared__ float sh[];   // [rpi][2][C] per-row-slot partials (16 KB for every C)
    pdl_wait();
    pdl_trigger();
    const int tpr = C / 8, rpi = 256 / tpr;
    const int cg = threadIdx.x % tpr, ry = threadIdx.x / tpr;
    float a[8], b[8], mu[8], rs[8], msc[8], msh[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { a[i] = 0.f; b[i] = 0.f; mu[i] = 0.f; rs[i] = 1.f; msc[i] = 0.f; msh[i] = 1.f; }
    if (MODE == 1) {
#pragma unroll
        for (int i = 0; i < 8; ++i) { mu[i] = mean_rstd[cg * 8 + i]; rs[i] = mean_rstd[C + cg * 8 + i]; }
        if (kRecompute) {
#pragma unroll
            for (int i = 0; i < 8; ++i) { msc[i] = gamma[cg * 8 + i] * rs[i]; msh[i] = beta[cg * 8 + i] - mu[i] * msc[i]; }
        }
    }
    const long long stride = (long long)gridDim.x * rpi;
    for (long long r0 = (long long)blockIdx.x * rpi + ry; r0 < M; r0 += stride * U) {
        uint4 xr[U], dr[U], yr[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const long long r = r0 + u * stride;
            const size_t off = (size_t)(r < M ? r : r0) * C + cg * 8;
            xr[u] = *reinterpret_cast<const uint4*>(x + off);
            if (MODE == 1) {
                dr[u] = *reinterpret_cast<const uint4*>(dy + off);
                if (!kRecompute && relu) yr[u] = *reinterpret_cast<const uint4*>(y + off);
            }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            if (r0 + u * stride >= M) continue;
            const __nv_bfloat162* xh = reinterpret_cast<const __nv_bfloat162*>(&xr[u]);
            const __nv_bfloat162* dh = reinterpret_cast<const __nv_bfloat162*>(&dr[u]);
            const __nv_bfloat162* yh = reinterpret_cast<const __nv_bfloat162*>(&yr[u]);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float2 xv = __bfloat1622float2(xh[i]);
                if (MODE == 0) {
                    a[2 * i] += xv.x; a[2 * i + 1] += xv.y; b[2 * i] += xv.x * xv.x; b[2 * i + 1] += xv.y * xv.y;
                } else {
                    float2 dz = __bfloat1622float2(dh[i]);
                    if (!kRecompute && relu) {
                        const float2 yv = __bfloat1622float2(yh[i]);
                        dz.x = yv.x > 0.f ? dz.x : 0.f; dz.y = yv.y > 0.f ? dz.y : 0.f;
                    } else if (kRecompute) {
                        dz.x = (xv.x * msc[2 * i] + msh[2 * i]) > 0.f ? dz.x : 0.f;
                        dz.y = (xv.y * msc[2 * i + 1] + msh[2 * i + 1]) > 0.f ? dz.y : 0.f;
                    }
                    a[2 * i] += dz.x; a[2 * i + 1] += dz.y;
                    b[2 * i] += dz.x * (xv.x - mu[2 * i]) * rs[2 * i]; b[2 * i + 1] += dz.y * (xv.y - mu[2 * i + 1]) * rs[2 * i + 1];
                }
            }
        }
    }
    // block reduction without atomics: every thread parks its 16 partial sums in its row slot, then each thread sums a few
    // columns over the rpi slots (conflict-free) and stores ONE partial per column and block
    float* mine = sh + (size_t)ry * 2 * C + cg * 8;
#pragma unroll
    for (int i = 0; i < 8; ++i) { mine[i] = a[i]; mine[C + i] = b[i]; }
    __syncthreads();
    const int ncols = out_cols > 0 ? out_cols : 2 * C;
    float* dst = part + (size_t)blockIdx.x * ncols;                  // this CTA's slot; launch_ordered_sum adds the slots into out
    for (int i = threadIdx.x; i < ncols; i += 256) {
        float t = 0.f;
        for (int r = 0; r < rpi; ++r) t += sh[(size_t)r * 2 * C + i];
        dst[i] = t;
    }
}

cudaError_t launch_ordered_sum_f32(float* out, const float* part, int nparts, long long n, cudaStream_t st) {
    return launch_ordered_sum(out, part, nparts, n, st);
}
cudaError_t launch_ordered_sum_f64(double* out, const double* part, int nparts, long long n, cudaStream_t st) {
    return launch_ordered_sum(out, part, nparts, n, st);
}

// The per-CTA partial sums are added into slot 0 of the [nslots][2][C] output in CTA order (deterministic); nslots >= 4 selects
// four CTAs per SM instead of two.
cudaError_t launch_channel_stats(const __nv_bfloat16* x, long long M, int C, float* stats, int num_sms, cudaStream_t st, int only_sum, int nslots) {
    if (!chan_ok(C) || nslots < 1) return cudaErrorInvalidValue;
    const int rpi = 256 / (C / 8);
    const int grid = rows_grid(M, rpi * 8, num_sms, nslots >= 4 ? 4 : 2), ncols = only_sum ? C : 2 * C;
    Scratch part((size_t)grid * ncols * sizeof(float), st);
    const size_t smem = (size_t)rpi * 2 * C * sizeof(float);
    auto kernel = nslots >= 4 ? channel_reduce_kernel<0, false, 4, 4> : channel_reduce_kernel<0, false, 8, 2>;
    RLR_CUDA_CHECK(launch_kernel(kernel, dim3(grid), dim3(256), smem, st, x, nullptr, nullptr, nullptr, part.as<float>(), M, C, 0, nullptr,
                                 nullptr, only_sum ? C : 0));
    return launch_ordered_sum(stats, part.as<float>(), grid, (long long)ncols, st);
}
cudaError_t launch_bn_bwd_reduce(const __nv_bfloat16* dy, const __nv_bfloat16* y, const __nv_bfloat16* x, const float* mean_rstd,
                                 float* dsum, long long M, int C, int relu, int num_sms, cudaStream_t st, const float* gamma,
                                 const float* beta, int nslots) {
    if (!chan_ok(C) || (relu == 2 && (!gamma || !beta)) || (relu == 1 && !y) || nslots < 1) return cudaErrorInvalidValue;
    const int rpi = 256 / (C / 8);
    const bool three = nslots >= 3;
    const int grid = rows_grid(M, rpi * 8, num_sms, three ? 3 : 2);
    const size_t smem = (size_t)rpi * 2 * C * sizeof(float);
    Scratch part((size_t)grid * 2 * C * sizeof(float), st);
    if (relu == 2)
        RLR_CUDA_CHECK(launch_kernel(three ? channel_reduce_kernel<1, true, 2, 3> : channel_reduce_kernel<1, true, 4, 2>, dim3(grid), dim3(256), smem,
                                     st, x, dy, y, mean_rstd, part.as<float>(), M, C, relu, gamma, beta, 0));
    else
        RLR_CUDA_CHECK(launch_kernel(three ? channel_reduce_kernel<1, false, 2, 3> : channel_reduce_kernel<1, false, 4, 2>, dim3(grid), dim3(256), smem,
                                     st, x, dy, y, mean_rstd, part.as<float>(), M, C, relu, nullptr, nullptr, 0));
    return launch_ordered_sum(dsum, part.as<float>(), grid, 2LL * C, st);
}

__global__ void bn_finalize_kernel(const float* __restrict__ stats, int slots, float* __restrict__ mean_rstd, float* running_mean,
                                   float* running_var, int C, float count, float eps, float momentum, int train) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    if (train) {
        float s1 = 0.f, s2 = 0.f;
        for (int k = 0; k < slots; ++k) { s1 += stats[(size_t)k * 2 * C + c]; s2 += stats[(size_t)k * 2 * C + C + c]; }
        const float mean = s1 / count;
        const float var = fmaxf(s2 / count - mean * mean, 0.f);
        mean_rstd[c] = mean;
        mean_rstd[C + c] = rsqrtf(var + eps);
        running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * mean;
        const float unbiased = count > 1.f ? var * count / (count - 1.f) : var;
        running_var[c] = (1.f - momentum) * running_var[c] + momentum * unbiased;
    } else {
        mean_rstd[c] = running_mean[c];
        mean_rstd[C + c] = rsqrtf(running_var[c] + eps);
    }
}
cudaError_t launch_bn_finalize(const float* stats, int slots, float* mean_rstd, float* running_mean, float* running_var, int C,
                               float count, float eps, float momentum, int train, cudaStream_t st) {
    bn_finalize_kernel<<<(C + 127) / 128, 128, 0, st>>>(stats, slots, mean_rstd, running_mean, running_var, C, count, eps, momentum, train);
    return cudaGetLastError();
}

// fin.mode 0: mean/rstd are given.  1 (training): derive them from the raw per-channel sums `fin.stats` ([slots][2][C]); CTA 0 also
// stores mean/rstd for the backward pass and updates the running statistics -- this replaces the separate bn_finalize launch.
// 2 (evaluation): derive them from the running statistics.
struct BnFinalize {
    int mode;
    const float* stats; int slots;
    float count, eps, momentum;
    float* running_mean; float* running_var;
};

// The two BatchNorm apply passes are elementwise once their per-channel constants are fixed, and stream 3-5 bytes of HBM per byte of
// arithmetic input, so they are organised for memory-level parallelism:
//  - every CTA derives the per-channel constants ONCE into shared memory (one thread per channel), then each thread copies its 8;
//  - the grid is the resident one (kApplyCtasPerSm / kBwdCtasPerSm CTAs per SM, the __launch_bounds__ register caps) and every
//    thread keeps U independent 16-byte loads per tensor in flight;
//  - the rows are walked as 4 KB tiles of rpi rows (256 threads x 16 bytes) from the END of the tensor backwards: the pass that read
//    the same tensors just before (channel statistics forward, the backward reduction backward) walked them forwards, so the tail it
//    read last is what is still in L2 when this pass starts.
// Traversal and unrolling do not touch the per-element and per-channel expressions, so the results are bit-identical to a one-row-
// at-a-time loop in any order.
constexpr int kApplyU = 4, kApplyCtasPerSm = 3;
constexpr int kBwdU = 4, kBwdCtasPerSm = 2;

// Tile t of the reversed walk, rows [(nt - 1 - t) * rpi, +rpi); `ok` is false past the end (t >= nt, or a row of the ragged last tile).
__device__ __forceinline__ long long rev_tile_row(int t, int nt, int rpi, int ry, long long M, bool& ok) {
    const long long r = (long long)(nt - 1 - t) * rpi + ry;
    ok = t < nt && r < M;
    return r;
}
static inline int apply_grid(long long M, int rpi, int U, int num_sms, int per_sm) {
    const long long nt = (M + rpi - 1) / rpi;
    return rows_grid(nt, U, num_sms, per_sm);
}

template <int U>
__global__ void __launch_bounds__(256, kApplyCtasPerSm) bn_apply_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ res,
                                                         __nv_bfloat16* __restrict__ y, const float* __restrict__ gamma,
                                                         const float* __restrict__ beta, float* __restrict__ mean_rstd,
                                                         long long M, int C, int relu, BnFinalize fin) {
    extern __shared__ float2 apply_cst[];     // [C] (scale, shift)
    pdl_wait();
    pdl_trigger();
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        float mean, rstd;
        if (fin.mode == 1) {
            float s1 = 0.f, s2 = 0.f;
            for (int k = 0; k < fin.slots; ++k) { s1 += fin.stats[(size_t)k * 2 * C + c]; s2 += fin.stats[(size_t)k * 2 * C + C + c]; }
            mean = s1 / fin.count;
            const float var = fmaxf(s2 / fin.count - mean * mean, 0.f);
            rstd = rsqrtf(var + fin.eps);
            if (blockIdx.x == 0) {
                mean_rstd[c] = mean; mean_rstd[C + c] = rstd;
                fin.running_mean[c] = (1.f - fin.momentum) * fin.running_mean[c] + fin.momentum * mean;
                const float unbiased = fin.count > 1.f ? var * fin.count / (fin.count - 1.f) : var;
                fin.running_var[c] = (1.f - fin.momentum) * fin.running_var[c] + fin.momentum * unbiased;
            }
        } else if (fin.mode == 2) {
            mean = fin.running_mean[c]; rstd = rsqrtf(fin.running_var[c] + fin.eps);
        } else {
            mean = mean_rstd[c]; rstd = mean_rstd[C + c];
        }
        const float scale = gamma[c] * rstd;
        apply_cst[c] = make_float2(scale, beta[c] - mean * scale);
    }
    __syncthreads();
    const int tpr = C / 8, rpi = 256 / tpr;
    const int cg = threadIdx.x % tpr, ry = threadIdx.x / tpr;
    float sc[8], sh[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { const float2 k = apply_cst[cg * 8 + i]; sc[i] = k.x; sh[i] = k.y; }
    const int nt = (int)((M + rpi - 1) / rpi), G = gridDim.x;
    for (int t0 = blockIdx.x; t0 < nt; t0 += G * U) {
        uint4 xr[U], rr[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            bool ok;
            const long long r = rev_tile_row(t0 + u * G, nt, rpi, ry, M, ok);
            if (ok) {
                const size_t off = (size_t)r * C + cg * 8;
                xr[u] = *reinterpret_cast<const uint4*>(x + off);
                if (res) rr[u] = *reinterpret_cast<const uint4*>(res + off);
            }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            bool ok;
            const long long r = rev_tile_row(t0 + u * G, nt, rpi, ry, M, ok);
            if (!ok) continue;
            const __nv_bfloat162* xh = reinterpret_cast<const __nv_bfloat162*>(&xr[u]);
            const __nv_bfloat162* rh = reinterpret_cast<const __nv_bfloat162*>(&rr[u]);
            bf8 v;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float2 xv = __bfloat1622float2(xh[i]);
                v.v[2 * i] = xv.x * sc[2 * i] + sh[2 * i]; v.v[2 * i + 1] = xv.y * sc[2 * i + 1] + sh[2 * i + 1];
                if (res) { const float2 q = __bfloat1622float2(rh[i]); v.v[2 * i] += q.x; v.v[2 * i + 1] += q.y; }
                if (relu) { v.v[2 * i] = fmaxf(v.v[2 * i], 0.f); v.v[2 * i + 1] = fmaxf(v.v[2 * i + 1], 0.f); }
            }
            store8(y + (size_t)r * C + cg * 8, v);
        }
    }
}
cudaError_t launch_bn_apply(const __nv_bfloat16* x, const __nv_bfloat16* res, __nv_bfloat16* y, const float* gamma, const float* beta,
                            float* mean_rstd, long long M, int C, int relu, int fin_mode, const float* stats, int slots, float count,
                            float eps, float momentum, float* running_mean, float* running_var, int num_sms, cudaStream_t st) {
    if (!chan_ok(C)) return cudaErrorInvalidValue;
    const int rpi = 256 / (C / 8);
    BnFinalize fin{fin_mode, stats, slots, count, eps, momentum, running_mean, running_var};
    return launch_kernel(bn_apply_kernel<kApplyU>, dim3(apply_grid(M, rpi, kApplyU, num_sms, kApplyCtasPerSm)), dim3(256),
                         (size_t)C * sizeof(float2), st, x, res, y, gamma, beta, mean_rstd, M, C, relu, fin);
}

template <bool kRecompute, int U>
__global__ void __launch_bounds__(256, kBwdCtasPerSm) bn_bwd_apply_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ y,
                                                             const __nv_bfloat16* __restrict__ x, const float* __restrict__ gamma,
                                                             const float* __restrict__ mean_rstd, const float* __restrict__ dsum,
                                                             __nv_bfloat16* __restrict__ dx, __nv_bfloat16* __restrict__ dres,
                                                             float* dgamma, float* dbeta, long long M, int C, int relu,
                                                             const float* __restrict__ beta = nullptr, int nslots = 1) {
    extern __shared__ float bwd_cst[];        // [6][C]: mean, rstd, g = gamma * rstd, k1, k2, msh
    pdl_wait();
    pdl_trigger();
    const float invM = 1.0f / (float)M;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        const float mu = mean_rstd[c], rs = mean_rstd[C + c], g = gamma[c] * rs;
        float s0 = 0.f, s1 = 0.f;
        for (int k = 0; k < nslots; ++k) { s0 += dsum[(size_t)k * 2 * C + c]; s1 += dsum[(size_t)k * 2 * C + C + c]; }
        const float k1 = s0 * invM, k2 = s1 * invM;
        bwd_cst[c] = mu; bwd_cst[C + c] = rs; bwd_cst[2 * C + c] = g; bwd_cst[3 * C + c] = k1; bwd_cst[4 * C + c] = k2;
        bwd_cst[5 * C + c] = kRecompute ? beta[c] - mu * g : 0.f;     // g = gamma * rstd is bn_apply's scale, msh its shift
        if (blockIdx.x == 0) { dbeta[c] = k1 * (float)M; dgamma[c] = k2 * (float)M; }
    }
    __syncthreads();
    const int tpr = C / 8, rpi = 256 / tpr;
    const int cg = threadIdx.x % tpr, ry = threadIdx.x / tpr;
    float mu[8], rs[8], g[8], k1[8], k2[8], msh[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int c = cg * 8 + i;
        mu[i] = bwd_cst[c]; rs[i] = bwd_cst[C + c]; g[i] = bwd_cst[2 * C + c]; k1[i] = bwd_cst[3 * C + c]; k2[i] = bwd_cst[4 * C + c];
        msh[i] = bwd_cst[5 * C + c];
    }
    const bool need_y = !kRecompute && relu;
    const int nt = (int)((M + rpi - 1) / rpi), G = gridDim.x;
    for (int t0 = blockIdx.x; t0 < nt; t0 += G * U) {
        uint4 dr[U], xr[U], yr[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            bool ok;
            const long long r = rev_tile_row(t0 + u * G, nt, rpi, ry, M, ok);
            if (ok) {
                const size_t off = (size_t)r * C + cg * 8;
                dr[u] = *reinterpret_cast<const uint4*>(dy + off);
                xr[u] = *reinterpret_cast<const uint4*>(x + off);
                if (need_y) yr[u] = *reinterpret_cast<const uint4*>(y + off);
            }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            bool ok;
            const long long r = rev_tile_row(t0 + u * G, nt, rpi, ry, M, ok);
            if (!ok) continue;
            const size_t off = (size_t)r * C + cg * 8;
            bf8 dz = unpack8(dr[u]);
            const bf8 xv = unpack8(xr[u]);
            if (need_y) {
                const bf8 yv = unpack8(yr[u]);
#pragma unroll
                for (int i = 0; i < 8; ++i) dz.v[i] = yv.v[i] > 0.f ? dz.v[i] : 0.f;
            } else if (kRecompute) {
#pragma unroll
                for (int i = 0; i < 8; ++i) dz.v[i] = (xv.v[i] * g[i] + msh[i]) > 0.f ? dz.v[i] : 0.f;
            }
            if (dres) store8(dres + off, dz);
            bf8 o;
#pragma unroll
            for (int i = 0; i < 8; ++i) o.v[i] = g[i] * (dz.v[i] - k1[i] - (xv.v[i] - mu[i]) * rs[i] * k2[i]);
            store8(dx + off, o);
        }
    }
}
cudaError_t launch_bn_bwd_apply(const __nv_bfloat16* dy, const __nv_bfloat16* y, const __nv_bfloat16* x, const float* gamma,
                                const float* mean_rstd, const float* dsum, __nv_bfloat16* dx, __nv_bfloat16* dres, float* dgamma,
                                float* dbeta, long long M, int C, int relu, int num_sms, cudaStream_t st, const float* beta, int nslots) {
    if (!chan_ok(C) || (relu == 2 && !beta) || (relu == 1 && !y) || nslots < 1) return cudaErrorInvalidValue;
    const int rpi = 256 / (C / 8);
    const dim3 grid(apply_grid(M, rpi, kBwdU, num_sms, kBwdCtasPerSm));
    const size_t smem = (size_t)6 * C * sizeof(float);
    if (relu == 2)
        return launch_kernel(bn_bwd_apply_kernel<true, kBwdU>, grid, dim3(256), smem, st, dy, y, x, gamma, mean_rstd, dsum, dx, dres, dgamma, dbeta, M,
                             C, relu, beta, nslots);
    return launch_kernel(bn_bwd_apply_kernel<false, kBwdU>, grid, dim3(256), smem, st, dy, y, x, gamma, mean_rstd, dsum, dx, dres, dgamma, dbeta, M, C,
                         relu, nullptr, nslots);
}

// ---------------------------------------------------------------------------------------------------------------------
// dy <- dy * (y > 0) * scale.  scale != 1: the layer's output went through fused dropout (y = relu(z) * keep / (1 - p)): y > 0 exactly where
// the element was kept AND z > 0, so the ReLU mask and the dropout mask are read off y together and no mask is stored or recomputed.
__global__ void __launch_bounds__(256) relu_bwd_kernel(__nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ y, long long n8, float scale) {
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n8; q += (long long)gridDim.x * blockDim.x) {
        bf8 d = load8(dy + 8 * q);
        const bf8 yv = load8(y + 8 * q);
#pragma unroll
        for (int i = 0; i < 8; ++i) d.v[i] = yv.v[i] > 0.f ? d.v[i] * scale : 0.f;
        store8(dy + 8 * q, d);
    }
}
cudaError_t launch_relu_bwd(__nv_bfloat16* dy, const __nv_bfloat16* y, long long n, int num_sms, cudaStream_t st, float scale) {
    if (n % 8) return cudaErrorInvalidValue;
    relu_bwd_kernel<<<rows_grid(n / 8, 256, num_sms, 8), 256, 0, st>>>(dy, y, n / 8, scale);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------------------
// 2x2 / stride-2 max-pool (floor mode, like nn.MaxPool2d(2,2)); idx = 2*dy+dx of the first maximum
// ---------------------------------------------------------------------------------------------------------------------
// drop.thr != 0: dropout fused into the pooling epilogue -- the pooled value is scaled / zeroed by the Philox keep-mask of its output
// element (dropout_keep8); the backward kernel re-evaluates the same mask, nothing is stored.
__global__ void __launch_bounds__(256) maxpool2_fwd_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y,
                                                             uint8_t* __restrict__ idx, int B, int H, int W, int C, DropSpec drop) {
    const int Ho = H / 2, Wo = W / 2, cg_n = C / 8;
    const long long total = (long long)B * Ho * Wo * cg_n;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const int cg = (int)(t % cg_n);
        long long r = t / cg_n;
        const int wo = (int)(r % Wo); r /= Wo;
        const int ho = (int)(r % Ho);
        const int b = (int)(r / Ho);
        const __nv_bfloat16* base = x + (((size_t)b * H + 2 * ho) * W + 2 * wo) * C + cg * 8;
        bf8 best = load8(base);
        uint8_t bi[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
        for (int k = 1; k < 4; ++k) {
            const bf8 v = load8(base + ((size_t)(k >> 1) * W + (k & 1)) * C);
#pragma unroll
            for (int i = 0; i < 8; ++i) if (v.v[i] > best.v[i]) { best.v[i] = v.v[i]; bi[i] = (uint8_t)k; }
        }
        const size_t o = (((size_t)b * Ho + ho) * Wo + wo) * C + cg * 8;
        if (drop.thr) {
            const uint32_t keep = dropout_keep8(drop, (long long)(o >> 3));
#pragma unroll
            for (int i = 0; i < 8; ++i) best.v[i] = (keep >> i & 1) ? best.v[i] * drop.scale : 0.f;
        }
        store8(y + o, best);
        uint2 pk;
        pk.x = bi[0] | (bi[1] << 8) | (bi[2] << 16) | (bi[3] << 24);
        pk.y = bi[4] | (bi[5] << 8) | (bi[6] << 16) | (bi[7] << 24);
        *reinterpret_cast<uint2*>(idx + o) = pk;
    }
}
// One thread per POOLED element x 8 channels: reads dy / the arg-max index (/ the pooled output) once and writes the four input pixels of its
// window (zeros except at the arg-max); rows / columns of an odd-sized input that no window covers are zeroed by the last windows.
// ``zmask`` (optional) = the pooled forward output: the producer's fused ReLU is back-propagated here -- the arg-max element is positive iff
// the pooled value is (ReLU'(0) = 0, like torch), so the separate relu_bwd pass over the 4x larger tensor disappears.
__global__ void __launch_bounds__(256) maxpool2_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const uint8_t* __restrict__ idx,
                                                             __nv_bfloat16* __restrict__ dx, const __nv_bfloat16* __restrict__ zmask,
                                                             int B, int H, int W, int C, DropSpec drop) {
    const int Ho = H / 2, Wo = W / 2, cg_n = C / 8;
    const long long total = (long long)B * Ho * Wo * cg_n;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const int cg = (int)(t % cg_n);
        long long r = t / cg_n;
        const int wo = (int)(r % Wo); r /= Wo;
        const int ho = (int)(r % Ho);
        const int b = (int)(r / Ho);
        const size_t src = (size_t)t * 8;                       // == (((b * Ho + ho) * Wo + wo) * C + cg * 8
        bf8 g = load8(dy + src);
        if (drop.thr) {     // gradient of the fused dropout: the forward's keep-mask of this pooled element, recomputed
            const uint32_t keep = dropout_keep8(drop, (long long)(src >> 3));
#pragma unroll
            for (int i = 0; i < 8; ++i) g.v[i] = (keep >> i & 1) ? g.v[i] * drop.scale : 0.f;
        }
        if (zmask) {
            const bf8 z = load8(zmask + src);
#pragma unroll
            for (int i = 0; i < 8; ++i) g.v[i] = z.v[i] > 0.f ? g.v[i] : 0.f;
        }
        const uint2 pk = *reinterpret_cast<const uint2*>(idx + src);
        bf8 zero;
#pragma unroll
        for (int i = 0; i < 8; ++i) zero.v[i] = 0.f;
#pragma unroll
        for (int me = 0; me < 4; ++me) {
            bf8 o;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int k = ((i < 4 ? pk.x : pk.y) >> (8 * (i & 3))) & 0xff;
                o.v[i] = (k == me) ? g.v[i] : 0.f;
            }
            store8(dx + (((size_t)b * H + 2 * ho + (me >> 1)) * W + 2 * wo + (me & 1)) * C + cg * 8, o);
        }
        const bool last_w = (W & 1) && wo == Wo - 1, last_h = (H & 1) && ho == Ho - 1;
        if (last_w) {
            store8(dx + (((size_t)b * H + 2 * ho) * W + W - 1) * C + cg * 8, zero);
            store8(dx + (((size_t)b * H + 2 * ho + 1) * W + W - 1) * C + cg * 8, zero);
        }
        if (last_h) {
            store8(dx + (((size_t)b * H + H - 1) * W + 2 * wo) * C + cg * 8, zero);
            store8(dx + (((size_t)b * H + H - 1) * W + 2 * wo + 1) * C + cg * 8, zero);
            if (last_w) store8(dx + (((size_t)b * H + H - 1) * W + W - 1) * C + cg * 8, zero);
        }
    }
}
static DropSpec make_drop(float p, uint64_t seed, const long long* step, uint64_t stream) {
    DropSpec d{};
    if (p > 0.f && step) { d.thr = (uint32_t)(p * 65536.0f); d.scale = 1.0f / (1.0f - p); d.seed = seed; d.stream = stream; d.step = step; }
    return d;
}
cudaError_t launch_maxpool2_fwd(const __nv_bfloat16* x, __nv_bfloat16* y, uint8_t* idx, int B, int H, int W, int C, cudaStream_t st, float drop_p,
                                uint64_t seed, const long long* step, uint64_t stream) {
    if (C % 8) return cudaErrorInvalidValue;
    const long long total = (long long)B * (H / 2) * (W / 2) * (C / 8);
    maxpool2_fwd_kernel<<<rows_grid(total, 256, 132, 8), 256, 0, st>>>(x, y, idx, B, H, W, C, make_drop(drop_p, seed, step, stream));
    return cudaGetLastError();
}
cudaError_t launch_maxpool2_bwd(const __nv_bfloat16* dy, const uint8_t* idx, __nv_bfloat16* dx, int B, int H, int W, int C, cudaStream_t st, float drop_p,
                                uint64_t seed, const long long* step, uint64_t stream, const __nv_bfloat16* zmask) {
    if (C % 8 || H < 2 || W < 2) return cudaErrorInvalidValue;
    const long long total = (long long)B * (H / 2) * (W / 2) * (C / 8);
    maxpool2_bwd_kernel<<<rows_grid(total, 256, 132, 8), 256, 0, st>>>(dy, idx, dx, zmask, B, H, W, C, make_drop(drop_p, seed, step, stream));
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------------------
__global__ void avgpool_fwd_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, int B, int HW, int C) {
    const int cg_n = C / 8;
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= B * cg_n) return;
    const int b = t / cg_n, cg = t % cg_n;
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int p = 0; p < HW; ++p) {
        const bf8 v = load8(x + ((size_t)b * HW + p) * C + cg * 8);
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] += v.v[i];
    }
    bf8 o;
#pragma unroll
    for (int i = 0; i < 8; ++i) o.v[i] = acc[i] / (float)HW;
    store8(y + (size_t)b * C + cg * 8, o);
}
__global__ void avgpool_bwd_kernel(const __nv_bfloat16* __restrict__ dy, __nv_bfloat16* __restrict__ dx, int B, int HW, int C) {
    const int cg_n = C / 8;
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)B * HW * cg_n) return;
    const int cg = (int)(t % cg_n);
    const long long bp = t / cg_n;
    const int b = (int)(bp / HW);
    bf8 g = load8(dy + (size_t)b * C + cg * 8);
#pragma unroll
    for (int i = 0; i < 8; ++i) g.v[i] /= (float)HW;
    store8(dx + (size_t)bp * C + cg * 8, g);
}
cudaError_t launch_avgpool_fwd(const __nv_bfloat16* x, __nv_bfloat16* y, int B, int HW, int C, cudaStream_t st) {
    if (C % 8) return cudaErrorInvalidValue;
    avgpool_fwd_kernel<<<(B * (C / 8) + 127) / 128, 128, 0, st>>>(x, y, B, HW, C);
    return cudaGetLastError();
}
cudaError_t launch_avgpool_bwd(const __nv_bfloat16* dy, __nv_bfloat16* dx, int B, int HW, int C, cudaStream_t st) {
    if (C % 8) return cudaErrorInvalidValue;
    const long long total = (long long)B * HW * (C / 8);
    avgpool_bwd_kernel<<<(int)((total + 255) / 256), 256, 0, st>>>(dy, dx, B, HW, C);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------------------
// dropout: keep-mask from Philox4x32-10 keyed by (seed; element/8, step ^ stream); 16 random bits per element
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) dropout_fwd_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y,
                                                            uint8_t* __restrict__ mask, long long n8, float p, uint64_t seed,
                                                            const long long* __restrict__ step, uint64_t stream) {
    DropSpec d{(uint32_t)(p * 65536.0f), 1.0f / (1.0f - p), seed, stream, step};
    const float scale = d.scale;
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n8; q += (long long)gridDim.x * blockDim.x) {
        const uint32_t keep = dropout_keep8(d, q);
        bf8 v = load8(x + 8 * q);
        uint8_t m[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            m[i] = keep >> i & 1;
            v.v[i] = m[i] ? v.v[i] * scale : 0.f;
        }
        store8(y + 8 * q, v);
        uint2 pk;
        pk.x = m[0] | (m[1] << 8) | (m[2] << 16) | (m[3] << 24);
        pk.y = m[4] | (m[5] << 8) | (m[6] << 16) | (m[7] << 24);
        *reinterpret_cast<uint2*>(mask + 8 * q) = pk;
    }
}
__global__ void __launch_bounds__(256) dropout_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const uint8_t* __restrict__ mask,
                                                            __nv_bfloat16* __restrict__ dx, long long n8, float scale) {
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n8; q += (long long)gridDim.x * blockDim.x) {
        bf8 g = load8(dy + 8 * q);
        const uint2 pk = *reinterpret_cast<const uint2*>(mask + 8 * q);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int k = ((i < 4 ? pk.x : pk.y) >> (8 * (i & 3))) & 0xff;
            g.v[i] = k ? g.v[i] * scale : 0.f;
        }
        store8(dx + 8 * q, g);
    }
}
cudaError_t launch_dropout_fwd(const __nv_bfloat16* x, __nv_bfloat16* y, uint8_t* mask, long long n, float p, uint64_t seed,
                               const long long* step, uint64_t stream, cudaStream_t st) {
    if (n % 8) return cudaErrorInvalidValue;
    dropout_fwd_kernel<<<rows_grid(n / 8, 256, 132, 8), 256, 0, st>>>(x, y, mask, n / 8, p, seed, step, stream);
    return cudaGetLastError();
}
cudaError_t launch_dropout_bwd(const __nv_bfloat16* dy, const uint8_t* mask, __nv_bfloat16* dx, long long n, float p, cudaStream_t st) {
    if (n % 8) return cudaErrorInvalidValue;
    dropout_bwd_kernel<<<rows_grid(n / 8, 256, 132, 8), 256, 0, st>>>(dy, mask, dx, n / 8, 1.0f / (1.0f - p));
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------------------
// space-to-depth: x[NB][H][W][C] -> y[4][NB][H/2][W/2][C], plane = (h&1)*2 + (w&1)
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) space_to_depth_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y,
                                                               int NB, int H, int W, int C) {
    const int cg_n = C / 8, H2 = H / 2, W2 = W / 2;
    const long long total = (long long)NB * H * W * cg_n;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const int cg = (int)(t % cg_n);
        long long r = t / cg_n;
        const int w = (int)(r % W); r /= W;
        const int h = (int)(r % H);
        const int n = (int)(r / H);
        const int plane = (h & 1) * 2 + (w & 1);
        const uint4 v = *reinterpret_cast<const uint4*>(x + (((size_t)n * H + h) * W + w) * C + cg * 8);
        *reinterpret_cast<uint4*>(y + ((((size_t)plane * NB + n) * H2 + (h >> 1)) * W2 + (w >> 1)) * C + cg * 8) = v;
    }
}
cudaError_t launch_space_to_depth(const __nv_bfloat16* x, __nv_bfloat16* y, int NB, int H, int W, int C, int num_sms, cudaStream_t st) {
    if (C % 8 || H % 2 || W % 2) return cudaErrorInvalidValue;
    const long long total = (long long)NB * H * W * (C / 8);
    space_to_depth_kernel<<<rows_grid(total, 256, num_sms, 8), 256, 0, st>>>(x, y, NB, H, W, C);
    return cudaGetLastError();
}

// Small-K im2col for stem convolutions (C * k * k <= 64, stride 1): A[(b,ho,wo)][j] = x[b][ho + dy - pad][wo + dx - pad][c] with
// j = (dy * k + dx) * C + c, zero outside the image and for j >= C*k*k.  The stem conv then is ONE 64-deep k-block of the plain
// GEMM (instead of k*k channel-padded ones) and its weight gradient a [Cout x 64] GEMM over the same matrix.
__global__ void __launch_bounds__(256) im2col_small_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ A, int NB, int H,
                                                             int W, int C, int Ho, int Wo, int k, int pad) {
    const long long total = (long long)NB * Ho * Wo * 8;          // 8 chunks of 8 bf16 per 64-wide row
    const int kkc = k * k * C;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const int chunk = (int)(t & 7);
        const long long pix = t >> 3;
        const int wo = (int)(pix % Wo), ho = (int)((pix / Wo) % Ho), b = (int)(pix / ((long long)Wo * Ho));
        __align__(16) __nv_bfloat16 v[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            const int j = chunk * 8 + e;
            float val = 0.f;
            if (j < kkc) {
                const int tap = j / C, c = j - tap * C;
                const int dy = tap / k, dx = tap - dy * k;
                const int h = ho + dy - pad, w = wo + dx - pad;
                if (h >= 0 && h < H && w >= 0 && w < W) val = __bfloat162float(x[(((long long)b * H + h) * W + w) * C + c]);
            }
            v[e] = __float2bfloat16(val);
        }
        *reinterpret_cast<uint4*>(A + pix * 64 + chunk * 8) = *reinterpret_cast<const uint4*>(v);
    }
}
cudaError_t launch_im2col_small(const __nv_bfloat16* x, __nv_bfloat16* A, int NB, int H, int W, int C, int Ho, int Wo, int k, int pad,
                                int num_sms, cudaStream_t st) {
    if (C * k * k > 64 || k < 1) return cudaErrorInvalidValue;
    const long long total = (long long)NB * Ho * Wo * 8;
    im2col_small_kernel<<<rows_grid(total, 256, num_sms, 8), 256, 0, st>>>(x, A, NB, H, W, C, Ho, Wo, k, pad);
    return cudaGetLastError();
}

// inverse of space_to_depth with optional accumulation; planes missing from `plane_mask` count as zero
__global__ void __launch_bounds__(256) depth_to_space_kernel(const __nv_bfloat16* __restrict__ x4, __nv_bfloat16* __restrict__ y, int NB,
                                                               int H, int W, int C, int accumulate, int plane_mask) {
    const int cg_n = C / 8, H2 = H / 2, W2 = W / 2;
    const long long total = (long long)NB * H * W * cg_n;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const int cg = (int)(t % cg_n);
        long long r = t / cg_n;
        const int w = (int)(r % W); r /= W;
        const int h = (int)(r % H);
        const int n = (int)(r / H);
        const int plane = (h & 1) * 2 + (w & 1);
        __nv_bfloat16* dst = y + (((size_t)n * H + h) * W + w) * C + cg * 8;
        bf8 v;
        if ((plane_mask >> plane) & 1) {
            v = load8(x4 + ((((size_t)plane * NB + n) * H2 + (h >> 1)) * W2 + (w >> 1)) * C + cg * 8);
        } else {
            if (accumulate) continue;
#pragma unroll
            for (int i = 0; i < 8; ++i) v.v[i] = 0.f;
        }
        if (accumulate) {
            const bf8 o = load8(dst);
#pragma unroll
            for (int i = 0; i < 8; ++i) v.v[i] += o.v[i];
        }
        store8(dst, v);
    }
}
cudaError_t launch_depth_to_space(const __nv_bfloat16* x4, __nv_bfloat16* y, int NB, int H, int W, int C, int accumulate, int plane_mask,
                                  int num_sms, cudaStream_t st) {
    if (C % 8 || H % 2 || W % 2) return cudaErrorInvalidValue;
    const long long total = (long long)NB * H * W * (C / 8);
    depth_to_space_kernel<<<rows_grid(total, 256, num_sms, 8), 256, 0, st>>>(x4, y, NB, H, W, C, accumulate, plane_mask);
    return cudaGetLastError();
}

// wt[ci][s][co] = w[co][taps[s]][ci]   (sub-filter of a strided conv's data gradient, one per input parity plane)
struct TapList { int n; int t[9]; };
__global__ void filter_gather_transpose_kernel(const __nv_bfloat16* __restrict__ w, __nv_bfloat16* __restrict__ wt, int Cout, int T,
                                               int Cin, TapList taps) {
    const long long total = (long long)Cout * taps.n * Cin;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int co = (int)(i % Cout);
        const long long r = i / Cout;
        const int s = (int)(r % taps.n);
        const int ci = (int)(r / taps.n);
        wt[i] = w[((size_t)co * T + taps.t[s]) * Cin + ci];
    }
}
cudaError_t launch_filter_gather_transpose(const __nv_bfloat16* w, __nv_bfloat16* wt, int Cout, int T, int Cin, int nsub, const int* taps,
                                           cudaStream_t st) {
    if (nsub < 1 || nsub > 9) return cudaErrorInvalidValue;
    TapList tl; tl.n = nsub;
    for (int i = 0; i < nsub; ++i) tl.t[i] = taps[i];
    const long long total = (long long)Cout * nsub * Cin;
    const long long blocks = (total + 255) / 256;
    filter_gather_transpose_kernel<<<(int)(blocks > 132 * 16 ? 132 * 16 : blocks), 256, 0, st>>>(w, wt, Cout, T, Cin, tl);
    return cudaGetLastError();
}

// wt[ci][T-1-t][co] = w[co][t][ci]
__global__ void filter_transpose_kernel(const __nv_bfloat16* __restrict__ w, __nv_bfloat16* __restrict__ wt, int Cout, int T, int Cin) {
    const long long total = (long long)Cout * T * Cin;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int co = (int)(i % Cout);
        const long long r = i / Cout;
        const int tt = (int)(r % T);
        const int ci = (int)(r / T);
        wt[i] = w[((size_t)co * T + (T - 1 - tt)) * Cin + ci];   // writes coalesced over co
    }
}
cudaError_t launch_filter_transpose(const __nv_bfloat16* w, __nv_bfloat16* wt, int Cout, int ntaps, int Cin, cudaStream_t st) {
    const long long total = (long long)Cout * ntaps * Cin;
    filter_transpose_kernel<<<(int)((total + 255) / 256 > 132 * 16 ? 132 * 16 : (total + 255) / 256), 256, 0, st>>>(w, wt, Cout, ntaps, Cin);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------------------
// small dense layers (classifier heads, N <= 32): CUDA cores, fp32 accumulation
// ---------------------------------------------------------------------------------------------------------------------
// forward: one warp per sample row, lanes stride over K, NMAX accumulators in registers
template <int NMAX>
__global__ void __launch_bounds__(128) linear_small_fwd_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ w,
                                                                 const float* __restrict__ bias, __nv_bfloat16* __restrict__ y,
                                                                 int B, int K, int N, int relu) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= B) return;
    float acc[NMAX];
#pragma unroll
    for (int n = 0; n < NMAX; ++n) acc[n] = 0.f;
    for (int k = lane * 2; k < K; k += 64) {   // K is even for every head in the zoo
        const float2 xv = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(x + (size_t)warp * K + k));
#pragma unroll
        for (int n = 0; n < NMAX; ++n)
            if (n < N) {
                const float2 wv = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(w + (size_t)n * K + k));
                acc[n] += xv.x * wv.x + xv.y * wv.y;
            }
    }
#pragma unroll
    for (int n = 0; n < NMAX; ++n) {
        if (n < N) {
            float v = warp_sum(acc[n]);
            if (lane == 0) {
                v += bias ? bias[n] : 0.f;
                if (relu) v = fmaxf(v, 0.f);
                y[(size_t)warp * N + n] = __float2bfloat16(v);
            }
        }
    }
}
cudaError_t launch_linear_small_fwd(const __nv_bfloat16* x, const __nv_bfloat16* w, const float* bias, __nv_bfloat16* y, int B, int K,
                                    int N, int relu, cudaStream_t st) {
    if (N > 32 || (K & 1)) return cudaErrorInvalidValue;
    const int blocks = (B * 32 + 127) / 128;
    if (N <= 16) linear_small_fwd_kernel<16><<<blocks, 128, 0, st>>>(x, w, bias, y, B, K, N, relu);
    else linear_small_fwd_kernel<32><<<blocks, 128, 0, st>>>(x, w, bias, y, B, K, N, relu);
    return cudaGetLastError();
}

// backward: grid.x = K/64 column chunks (+1 block for dx rows); dW/db: 256 threads = 64 k x 4 batch slices, partials via smem
__global__ void __launch_bounds__(256) linear_small_bwd_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy,
                                                                 const __nv_bfloat16* __restrict__ w, __nv_bfloat16* __restrict__ dx,
                                                                 float* __restrict__ dw, float* __restrict__ db, int B, int K, int N,
                                                                 int accumulate_dx) {
    __shared__ float part[4][32][64];   // [batch slice][n][k in chunk]  (N <= 32)
    const int kchunks = (K + 63) / 64;
    if ((int)blockIdx.x < kchunks) {
        const int kk = threadIdx.x & 63, sl = threadIdx.x >> 6, k = blockIdx.x * 64 + kk;
        float acc[32];
#pragma unroll
        for (int n = 0; n < 32; ++n) acc[n] = 0.f;
        if (k < K) {
            for (int b = sl; b < B; b += 4) {
                const float xv = __bfloat162float(x[(size_t)b * K + k]);
#pragma unroll
                for (int n = 0; n < 32; ++n) if (n < N) acc[n] += xv * __bfloat162float(dy[(size_t)b * N + n]);
            }
        }
#pragma unroll
        for (int n = 0; n < 32; ++n) if (n < N) part[sl][n][kk] = acc[n];
        __syncthreads();
        for (int i = threadIdx.x; i < N * 64; i += 256) {
            const int n = i >> 6, c = i & 63;
            if (blockIdx.x * 64 + c < K) dw[(size_t)n * K + blockIdx.x * 64 + c] = part[0][n][c] + part[1][n][c] + part[2][n][c] + part[3][n][c];
        }
        if (blockIdx.x == 0 && db && threadIdx.x < N) {   // db[n] = sum_b dy[b][n]
            float a = 0.f;
            for (int b = 0; b < B; ++b) a += __bfloat162float(dy[(size_t)b * N + threadIdx.x]);
            db[threadIdx.x] = a;
        }
    } else if (dx) {                                       // dx[b][k] = sum_n dy[b][n] w[n][k]
        const long long total = (long long)B * K;
        for (long long t = (long long)(blockIdx.x - kchunks) * 256 + threadIdx.x; t < total; t += (long long)(gridDim.x - kchunks) * 256) {
            const int b = (int)(t / K), k = (int)(t % K);
            float acc = 0.f;
            for (int n = 0; n < N; ++n) acc += __bfloat162float(dy[(size_t)b * N + n]) * __bfloat162float(w[(size_t)n * K + k]);
            if (accumulate_dx) acc += __bfloat162float(dx[t]);
            dx[t] = __float2bfloat16(acc);
        }
    }
}
// v2 (RLR_HEAD_V2): the weight/bias gradient of the classifier head is spread over (K/64) x (B/16) blocks that stage their
// 16 dy rows in shared memory; block (kc, bs) stores its partial sums in slot bs of `pw` ([B/16][N][K]) / `pb` ([B/16][N]) and
// launch_linear_small_bwd2 adds the slots into dW / db in a fixed order.  v1 used K/64 blocks that each walked the whole batch (30 us for a 256 x 512 x 10 layer).
__global__ void __launch_bounds__(256) linear_small_bwd2_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy,
                                                                  const __nv_bfloat16* __restrict__ w, __nv_bfloat16* __restrict__ dx,
                                                                  float* __restrict__ pw, float* __restrict__ pb, int B, int K, int N,
                                                                  int accumulate_dx, int kchunks, int bsplit) {
    pdl_wait();
    pdl_trigger();
    __shared__ float sdy[16][32];
    __shared__ float sred[4][64];
    const int wblocks = kchunks * bsplit;
    if ((int)blockIdx.x < wblocks) {
        const int kc = blockIdx.x % kchunks, bs = blockIdx.x / kchunks;
        const int b0 = bs * 16;
        for (int i = threadIdx.x; i < 16 * 32; i += 256) {
            const int r = i >> 5, n = i & 31;
            sdy[r][n] = (b0 + r < B && n < N) ? __bfloat162float(dy[(size_t)(b0 + r) * N + n]) : 0.f;
        }
        __syncthreads();
        // 256 threads = 64 columns x 4 row groups of 4 samples
        const int kk = threadIdx.x & 63, rg = threadIdx.x >> 6, k = kc * 64 + kk;
        float xv[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int b = b0 + rg * 4 + r;
            xv[r] = (k < K && b < B) ? __bfloat162float(x[(size_t)b * K + k]) : 0.f;
        }
        for (int n = 0; n < N; ++n) {
            float a = 0.f;
#pragma unroll
            for (int r = 0; r < 4; ++r) a += xv[r] * sdy[rg * 4 + r][n];
            sred[rg][kk] = a;
            __syncthreads();
            if (rg == 0 && k < K) pw[((size_t)bs * N + n) * K + k] = ((sred[0][kk] + sred[1][kk]) + sred[2][kk]) + sred[3][kk];
            __syncthreads();
        }
        if (kc == 0 && pb && threadIdx.x < N) {
            float a = 0.f;
#pragma unroll
            for (int r = 0; r < 16; ++r) a += sdy[r][threadIdx.x];
            pb[(size_t)bs * N + threadIdx.x] = a;
        }
    } else if (dx) {                                       // dx[b][k] = sum_n dy[b][n] w[n][k], two columns per thread
        const long long total2 = (long long)B * (K / 2);
        const int nb = gridDim.x - wblocks;
        for (long long t = (long long)(blockIdx.x - wblocks) * 256 + threadIdx.x; t < total2; t += (long long)nb * 256) {
            const int b = (int)(t / (K / 2)), k = (int)(t % (K / 2)) * 2;
            float a0 = 0.f, a1 = 0.f;
            for (int n = 0; n < N; ++n) {
                const float d = __bfloat162float(dy[(size_t)b * N + n]);
                const float2 wv = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(w + (size_t)n * K + k));
                a0 += d * wv.x; a1 += d * wv.y;
            }
            __nv_bfloat162* o = reinterpret_cast<__nv_bfloat162*>(dx + (size_t)b * K + k);
            if (accumulate_dx) { const float2 old = __bfloat1622float2(*o); a0 += old.x; a1 += old.y; }
            *o = __floats2bfloat162_rn(a0, a1);
        }
    }
}
cudaError_t launch_linear_small_bwd2(const __nv_bfloat16* x, const __nv_bfloat16* dy, const __nv_bfloat16* w, __nv_bfloat16* dx,
                                     float* dw, float* db, int B, int K, int N, int accumulate_dx, cudaStream_t st) {
    if (N > 32 || (K & 1)) return cudaErrorInvalidValue;
    const int kchunks = (K + 63) / 64, bsplit = (B + 15) / 16;
    long long dxb = dx ? ((long long)B * (K / 2) + 255) / 256 : 0;
    if (dxb > 592) dxb = 592;
    Scratch part(((size_t)bsplit * N * K + (size_t)bsplit * N) * sizeof(float), st);
    float* pw = part.as<float>();
    float* pb = db ? pw + (size_t)bsplit * N * K : nullptr;
    RLR_CUDA_CHECK(launch_kernel(linear_small_bwd2_kernel, dim3(kchunks * bsplit + (int)dxb), dim3(256), (size_t)0, st, x, dy, w, dx, pw, pb, B,
                                 K, N, accumulate_dx, kchunks, bsplit));
    RLR_CUDA_CHECK(launch_ordered_sum(dw, pw, bsplit, (long long)N * K, st));
    return db ? launch_ordered_sum(db, pb, bsplit, (long long)N, st) : cudaSuccess;
}

// v2 forward: 8 samples per 256-thread block, one warp per sample, the whole weight matrix staged in shared memory once per block
// (N * K bf16 <= 32 KB) and the k loop unrolled so the loads of a row are all in flight together.
__global__ void __launch_bounds__(256) linear_small_fwd2_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ w,
                                                                  const float* __restrict__ bias, __nv_bfloat16* __restrict__ y,
                                                                  int B, int K, int N, int relu) {
    pdl_wait();
    pdl_trigger();
    extern __shared__ __nv_bfloat16 sw[];                 // [N][K]
    for (int i = threadIdx.x * 8; i < N * K; i += 256 * 8) *reinterpret_cast<uint4*>(sw + i) = *reinterpret_cast<const uint4*>(w + i);
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int b = blockIdx.x * 8 + warp;
    if (b >= B) return;
    float acc[32];
#pragma unroll
    for (int n = 0; n < 32; ++n) acc[n] = 0.f;
#pragma unroll 4
    for (int k = lane * 2; k < K; k += 64) {
        const float2 xv = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(x + (size_t)b * K + k));
#pragma unroll
        for (int n = 0; n < 32; ++n)
            if (n < N) {
                const float2 wv = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(sw + (size_t)n * K + k));
                acc[n] += xv.x * wv.x + xv.y * wv.y;
            }
    }
#pragma unroll
    for (int n = 0; n < 32; ++n) {
        if (n < N) {
            float v = warp_sum(acc[n]);
            if (lane == 0) {
                v += bias ? bias[n] : 0.f;
                if (relu) v = fmaxf(v, 0.f);
                y[(size_t)b * N + n] = __float2bfloat16(v);
            }
        }
    }
}
cudaError_t launch_linear_small_fwd2(const __nv_bfloat16* x, const __nv_bfloat16* w, const float* bias, __nv_bfloat16* y, int B, int K,
                                     int N, int relu, cudaStream_t st) {
    if (N > 32 || (K & 1) || (N * K) % 8 || (size_t)N * K * 2 > 48 * 1024) return cudaErrorInvalidValue;
    return launch_kernel(linear_small_fwd2_kernel, dim3((B + 7) / 8), dim3(256), (size_t)N * K * 2, st, x, w, bias, y, B, K, N, relu);
}

cudaError_t launch_linear_small_bwd(const __nv_bfloat16* x, const __nv_bfloat16* dy, const __nv_bfloat16* w, __nv_bfloat16* dx,
                                    float* dw, float* db, int B, int K, int N, int accumulate_dx, cudaStream_t st) {
    if (N > 32) return cudaErrorInvalidValue;
    const int kchunks = (K + 63) / 64;
    long long dxb = dx ? ((long long)B * K + 255) / 256 : 0;
    if (dxb > 592) dxb = 592;
    linear_small_bwd_kernel<<<kchunks + (int)dxb, 256, 0, st>>>(x, dy, w, dx, dw, db, B, K, N, accumulate_dx);
    return cudaGetLastError();
}

}  // namespace rlr
