// GroupNorm over NHWC bf16 activations with fp32 math: forward (normalise + affine + residual add + ReLU) and backward, for the
// GroupNorm variants of the ResNet / VGG models (models/zoo.py).  Semantics: torch.nn.GroupNorm(groups, C, eps, affine=True) --
// per sample, group g covers channels [g*C/groups, (g+1)*C/groups) over all H x W pixels, biased variance, per-channel affine.
//
// Groups are independent, so a CTA owns one sample n and a slice of S whole-group channels (grid B x C/S): the group statistics
// and the parameter-gradient partials need no cross-CTA reduction inside the kernel.  Every CTA-wide sum goes through shared
// memory in a fixed order (thread row slots, then the channels of a group), and the per-sample affine-gradient partials
// ([2][B][C]) are added across samples by launch_ordered_sum -- no float atomics, bitwise reproducible results.
//
// Thread layout per CTA (256 threads): tpr = S/8 threads per pixel (16-byte vector = 8 channels each), rpi = 256/tpr pixels per
// iteration; threads beyond rpi*tpr only take part in the reductions.  Where the CTA's tile fits (kStage) it is kept in shared
// memory after the first read -- forward: x; backward: dz and x -- otherwise the later passes read it again from global memory
// (L2).  Both variants are correct for any H x W.
#include "common.cuh"
#include "gemm.h"

namespace rlr {
namespace {

constexpr int kThreads = 256;
constexpr int kRedFloats = 2048;                 // [rpi][S] row-slot partials: rpi * S = rpi * tpr * 8 <= 2048
constexpr int kTileTarget = 32 * 1024;           // slice width: grow S while one tensor's tile stays below this ...
constexpr int kStageMax = 96 * 1024;             // ... and stage the tile(s) in shared memory up to this size

struct f8 { float v[8]; };
__device__ __forceinline__ f8 unpack8(const uint4& u) {
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
    f8 r;
#pragma unroll
    for (int i = 0; i < 4; ++i) { const float2 f = __bfloat1622float2(h[i]); r.v[2 * i] = f.x; r.v[2 * i + 1] = f.y; }
    return r;
}
__device__ __forceinline__ uint4 pack8(const f8& r) {
    uint4 u;
    u.x = pack_bf16x2(r.v[0], r.v[1]); u.y = pack_bf16x2(r.v[2], r.v[3]);
    u.z = pack_bf16x2(r.v[4], r.v[5]); u.w = pack_bf16x2(r.v[6], r.v[7]);
    return u;
}

// Visits the rows p = first, first + step, ... < HW of the calling thread with U loads issued before the first use.
template <int U, typename Load, typename Body>
__device__ __forceinline__ void for_rows(int first, int step, int HW, Load load, Body body) {
    for (int p0 = first; p0 < HW; p0 += step * U) {
        decltype(load(0)) v[U];
#pragma unroll
        for (int u = 0; u < U; ++u) { const int p = p0 + u * step; v[u] = load(p < HW ? p : p0); }
#pragma unroll
        for (int u = 0; u < U; ++u) { const int p = p0 + u * step; if (p < HW) body(p, v[u]); }
    }
}

// out[c] = sum over the CTA's row slots of v (channel c = cg*8 + i of the slice), added in slot order.  Ends with a barrier.
__device__ __forceinline__ void slice_sums(const float (&v)[8], bool active, int ry, int cg, int S, int rpi, float* red, float* out) {
    if (active) {
#pragma unroll
        for (int i = 0; i < 8; ++i) red[ry * S + cg * 8 + i] = v[i];
    }
    __syncthreads();
    for (int c = threadIdx.x; c < S; c += kThreads) {
        float t = 0.f;
        for (int r = 0; r < rpi; ++r) t += red[r * S + c];
        out[c] = t;
    }
    __syncthreads();
}

struct GnBwdRow { uint4 dz, x; };

}  // namespace

// y = [ReLU]((x - mean_g) * rstd_g * gamma_c + beta_c [+ res]);  mean_rstd[n][0][g] = mean, mean_rstd[n][1][g] = rstd
template <bool kStage>
__global__ void __launch_bounds__(kThreads) gn_fwd_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ res,
                                                          __nv_bfloat16* __restrict__ y, const float* __restrict__ gamma,
                                                          const float* __restrict__ beta, float* __restrict__ mean_rstd, int HW, int C,
                                                          int G, int S, float eps, int relu) {
    extern __shared__ float4 gn_smem[];
    float* red = reinterpret_cast<float*>(gn_smem);
    float* chs = red + kRedFloats;                    // [S] channel sums
    float* mu = chs + S;                              // [S] group mean of each channel
    float* rs = mu + S;                               // [S] group rstd of each channel
    uint4* tile = reinterpret_cast<uint4*>(rs + 2 * S);     // [HW][tpr] (kStage); header is a multiple of 16 bytes (S % 8 == 0)
    pdl_wait();
    pdl_trigger();
    const int tpr = S / 8, rpi = kThreads / tpr;
    const int cg = threadIdx.x % tpr, ry = threadIdx.x / tpr;
    const bool active = ry < rpi;
    const int n = blockIdx.x, c0 = blockIdx.y * S, cpg = C / G;
    const float invM = 1.f / ((float)HW * (float)cpg);
    const size_t base = (size_t)n * HW * C + c0 + cg * 8;
    auto gload = [&](int p) { return *reinterpret_cast<const uint4*>(x + base + (size_t)p * C); };
    auto tload = [&](int p) { return kStage ? tile[p * tpr + cg] : *reinterpret_cast<const uint4*>(x + base + (size_t)p * C); };

    // pass 1: mean
    float a[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) a[i] = 0.f;
    if (active)
        for_rows<4>(ry, rpi, HW, gload, [&](int p, const uint4& u) {
            if (kStage) tile[p * tpr + cg] = u;
            const f8 f = unpack8(u);
#pragma unroll
            for (int i = 0; i < 8; ++i) a[i] += f.v[i];
        });
    slice_sums(a, active, ry, cg, S, rpi, red, chs);
    for (int gl = threadIdx.x; gl < S / cpg; gl += kThreads) {
        float t = 0.f;
        for (int j = 0; j < cpg; ++j) t += chs[gl * cpg + j];
        const float m = t * invM;
        for (int j = 0; j < cpg; ++j) mu[gl * cpg + j] = m;
    }
    __syncthreads();

    // pass 2: centred variance
    float m8[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { m8[i] = mu[cg * 8 + i]; a[i] = 0.f; }
    if (active)
        for_rows<4>(ry, rpi, HW, tload, [&](int, const uint4& u) {
            const f8 f = unpack8(u);
#pragma unroll
            for (int i = 0; i < 8; ++i) { const float d = f.v[i] - m8[i]; a[i] += d * d; }
        });
    slice_sums(a, active, ry, cg, S, rpi, red, chs);
    const int g0 = c0 / cpg;
    for (int gl = threadIdx.x; gl < S / cpg; gl += kThreads) {
        float t = 0.f;
        for (int j = 0; j < cpg; ++j) t += chs[gl * cpg + j];
        const float r = rsqrtf(t * invM + eps);
        for (int j = 0; j < cpg; ++j) rs[gl * cpg + j] = r;
        mean_rstd[((size_t)n * 2) * G + g0 + gl] = mu[gl * cpg];
        mean_rstd[((size_t)n * 2 + 1) * G + g0 + gl] = r;
    }
    __syncthreads();

    // pass 3: normalise, affine, residual, ReLU
    if (!active) return;
    float sc[8], sh[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int c = c0 + cg * 8 + i;
        sc[i] = rs[cg * 8 + i] * gamma[c];
        sh[i] = beta[c] - m8[i] * sc[i];
    }
    for_rows<4>(ry, rpi, HW, tload, [&](int p, const uint4& u) {
        f8 f = unpack8(u);
        const size_t off = base + (size_t)p * C;
        f8 r{};
        if (res) r = unpack8(*reinterpret_cast<const uint4*>(res + off));
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            float v = f.v[i] * sc[i] + sh[i];
            if (res) v += r.v[i];
            f.v[i] = relu ? fmaxf(v, 0.f) : v;
        }
        *reinterpret_cast<uint4*>(y + off) = pack8(f);
    });
}

// dz = dy * [y > 0] (ReLU fused) ; dres = dz (residual fused)
// per (n, group): s_a = sum dz*gamma, s_b = sum dz*gamma*xhat ; dx = rstd * (dz*gamma - s_a/M - xhat * s_b/M)
// part[0][n][c] = sum_pixels dz*xhat (dgamma partial of sample n), part[1][n][c] = sum_pixels dz (dbeta partial)
template <bool kStage>
__global__ void __launch_bounds__(kThreads) gn_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ y,
                                                          const __nv_bfloat16* __restrict__ x, const float* __restrict__ gamma,
                                                          const float* __restrict__ mean_rstd, __nv_bfloat16* __restrict__ dx,
                                                          __nv_bfloat16* __restrict__ dres, float* __restrict__ part, int B, int HW,
                                                          int C, int G, int S, int relu) {
    extern __shared__ float4 gn_smem[];
    float* red = reinterpret_cast<float*>(gn_smem);
    float* sa = red + kRedFloats;                     // [S] channel sums of dz, then per channel s_a / M of its group
    float* sb = sa + S;                               // [S] channel sums of dz * xhat, then s_b / M
    uint4* tile = reinterpret_cast<uint4*>(sb + 2 * S);     // [HW][tpr] dz, then [HW][tpr] x (kStage)
    pdl_wait();
    pdl_trigger();
    const int tpr = S / 8, rpi = kThreads / tpr;
    const int cg = threadIdx.x % tpr, ry = threadIdx.x / tpr;
    const bool active = ry < rpi;
    const int n = blockIdx.x, c0 = blockIdx.y * S, cpg = C / G;
    const float invM = 1.f / ((float)HW * (float)cpg);
    const size_t base = (size_t)n * HW * C + c0 + cg * 8;
    uint4* xtile = tile + (size_t)HW * tpr;
    float m8[8], r8[8], g8[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int c = c0 + cg * 8 + i, g = c / cpg;
        m8[i] = mean_rstd[((size_t)n * 2) * G + g];
        r8[i] = mean_rstd[((size_t)n * 2 + 1) * G + g];
        g8[i] = gamma[c];
    }
    // dz (masked) and x of row p from global memory
    auto gload = [&](int p) {
        const size_t off = base + (size_t)p * C;
        GnBwdRow r;
        r.dz = *reinterpret_cast<const uint4*>(dy + off);
        r.x = *reinterpret_cast<const uint4*>(x + off);
        if (relu) {      // bf16 -> fp32 -> bf16 is exact: dz keeps the bits of dy where y > 0
            f8 d = unpack8(r.dz);
            const f8 yv = unpack8(*reinterpret_cast<const uint4*>(y + off));
#pragma unroll
            for (int i = 0; i < 8; ++i) d.v[i] = yv.v[i] > 0.f ? d.v[i] : 0.f;
            r.dz = pack8(d);
        }
        return r;
    };
    auto tload = [&](int p) {
        if (!kStage) return gload(p);
        GnBwdRow r;
        r.dz = tile[p * tpr + cg];
        r.x = xtile[p * tpr + cg];
        return r;
    };

    // pass 1: channel sums of dz and dz * xhat; store dres
    float a[8], b[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { a[i] = 0.f; b[i] = 0.f; }
    if (active)
        for_rows<2>(ry, rpi, HW, gload, [&](int p, const GnBwdRow& r) {
            if (kStage) { tile[p * tpr + cg] = r.dz; xtile[p * tpr + cg] = r.x; }
            if (dres) *reinterpret_cast<uint4*>(dres + base + (size_t)p * C) = r.dz;
            const f8 dz = unpack8(r.dz), xv = unpack8(r.x);
#pragma unroll
            for (int i = 0; i < 8; ++i) { a[i] += dz.v[i]; b[i] += dz.v[i] * (xv.v[i] - m8[i]) * r8[i]; }
        });
    slice_sums(a, active, ry, cg, S, rpi, red, sa);
    slice_sums(b, active, ry, cg, S, rpi, red, sb);
    for (int c = threadIdx.x; c < S; c += kThreads) {
        part[(size_t)n * C + c0 + c] = sb[c];                        // dgamma partial
        part[((size_t)B + n) * C + c0 + c] = sa[c];                  // dbeta partial
    }
    __syncthreads();
    for (int gl = threadIdx.x; gl < S / cpg; gl += kThreads) {
        float ta = 0.f, tb = 0.f;
        for (int j = 0; j < cpg; ++j) {
            const float gm = gamma[c0 + gl * cpg + j];
            ta += gm * sa[gl * cpg + j];
            tb += gm * sb[gl * cpg + j];
        }
        for (int j = 0; j < cpg; ++j) { sa[gl * cpg + j] = ta * invM; sb[gl * cpg + j] = tb * invM; }
    }
    __syncthreads();

    // pass 2: data gradient
    if (!active) return;
    float k1[8], k2[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { k1[i] = sa[cg * 8 + i]; k2[i] = sb[cg * 8 + i]; }
    for_rows<2>(ry, rpi, HW, tload, [&](int p, const GnBwdRow& r) {
        const f8 dz = unpack8(r.dz), xv = unpack8(r.x);
        f8 o;
#pragma unroll
        for (int i = 0; i < 8; ++i) o.v[i] = r8[i] * (dz.v[i] * g8[i] - k1[i] - (xv.v[i] - m8[i]) * r8[i] * k2[i]);
        *reinterpret_cast<uint4*>(dx + base + (size_t)p * C) = pack8(o);
    });
}

namespace {

int gcd_int(int a, int b) { while (b) { const int t = a % b; a = b; b = t; } return a; }

// Slice width S (channels per CTA): whole groups and whole 16-byte vectors (a multiple of lcm(8, C/G)), widened by doubling while
// one tensor's tile stays under kTileTarget and the grid keeps at least two CTAs per SM.  0 if no slice fits the thread layout.
int gn_slice(int B, int HW, int C, int G, int num_sms) {
    const int cpg = C / G;
    int S = 8 / gcd_int(8, cpg) * cpg;
    if (S > 8 * kThreads || C % S) return 0;
    while (C % (2 * S) == 0 && 2 * S <= 8 * kThreads && (long long)HW * 2 * S * 2 <= kTileTarget &&
           (long long)B * (C / (2 * S)) >= 2LL * num_sms)
        S *= 2;
    return S;
}

bool gn_shape_ok(int B, int HW, int C, int G) { return B >= 1 && HW >= 1 && C % 8 == 0 && G >= 1 && C % G == 0; }

// largest dynamic shared memory of any launch: row slots + four [S] arrays at S = 2048 + the staged tile(s)
constexpr int kSmemMax = (kRedFloats + 4 * 8 * kThreads) * (int)sizeof(float) + kStageMax;

cudaError_t gn_configure() {
    static bool configured = false;
    if (!configured) {
        RLR_CUDA_CHECK(cudaFuncSetAttribute(gn_fwd_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemMax));
        RLR_CUDA_CHECK(cudaFuncSetAttribute(gn_fwd_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemMax));
        RLR_CUDA_CHECK(cudaFuncSetAttribute(gn_bwd_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemMax));
        RLR_CUDA_CHECK(cudaFuncSetAttribute(gn_bwd_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemMax));
        configured = true;
    }
    return cudaSuccess;
}

}  // namespace

cudaError_t launch_gn_fwd(const __nv_bfloat16* x, const __nv_bfloat16* res, __nv_bfloat16* y, const float* gamma, const float* beta,
                          float* mean_rstd, int B, int HW, int C, int G, float eps, int relu, int num_sms, cudaStream_t st) {
    if (!gn_shape_ok(B, HW, C, G)) return cudaErrorInvalidValue;
    const int S = gn_slice(B, HW, C, G, num_sms);
    if (!S) return cudaErrorInvalidValue;
    const size_t head = (size_t)(kRedFloats + 4 * S) * sizeof(float), tile = (size_t)HW * S * 2;
    const dim3 grid(B, C / S);
    RLR_CUDA_CHECK(gn_configure());
    if (tile <= kStageMax)
        return launch_kernel(gn_fwd_kernel<true>, grid, dim3(kThreads), head + tile, st, x, res, y, gamma, beta, mean_rstd, HW, C, G, S,
                             eps, relu);
    return launch_kernel(gn_fwd_kernel<false>, grid, dim3(kThreads), head, st, x, res, y, gamma, beta, mean_rstd, HW, C, G, S, eps, relu);
}

cudaError_t launch_gn_bwd(const __nv_bfloat16* dy, const __nv_bfloat16* y, const __nv_bfloat16* x, const float* gamma,
                          const float* mean_rstd, __nv_bfloat16* dx, __nv_bfloat16* dres, float* dgamma, float* dbeta, int B, int HW,
                          int C, int G, int relu, int num_sms, cudaStream_t st) {
    if (!gn_shape_ok(B, HW, C, G) || (relu && !y)) return cudaErrorInvalidValue;
    const int S = gn_slice(B, HW, C, G, num_sms);
    if (!S) return cudaErrorInvalidValue;
    const size_t head = (size_t)(kRedFloats + 4 * S) * sizeof(float), tiles = (size_t)HW * S * 2 * 2;
    const dim3 grid(B, C / S);
    RLR_CUDA_CHECK(gn_configure());
    Scratch part((size_t)2 * B * C * sizeof(float), st);          // [2][B][C]: dgamma / dbeta partials of every sample
    if (tiles <= kStageMax) {
        RLR_CUDA_CHECK(launch_kernel(gn_bwd_kernel<true>, grid, dim3(kThreads), head + tiles, st, dy, y, x, gamma, mean_rstd, dx, dres,
                                     part.as<float>(), B, HW, C, G, S, relu));
    } else {
        RLR_CUDA_CHECK(launch_kernel(gn_bwd_kernel<false>, grid, dim3(kThreads), head, st, dy, y, x, gamma, mean_rstd, dx, dres,
                                     part.as<float>(), B, HW, C, G, S, relu));
    }
    RLR_CUDA_CHECK(launch_ordered_sum(dgamma, part.as<float>(), B, (long long)C, st));
    return launch_ordered_sum(dbeta, part.as<float>() + (size_t)B * C, B, (long long)C, st);
}

}  // namespace rlr
