// Memory-bound kernels of the local-training loop: batch gather+normalise from the device-resident dataset,
// trojan stamping, fused clip-grad-norm + momentum-SGD (+ PGD projection) over the FLAT parameter buffers, and the
// loss / evaluation reductions.  Reference call sites: src/agent.py:41-60 (step), src/utils.py:52-54 (per-sample
// host transforms), :160-178 (poisoning), :128-157 (evaluation).
#include "common.cuh"
#include "flat_sgd.cuh"
#include "kernels.h"

#include <cstdlib>

namespace rlr {

// ---- programmatic dependent launch switch (common.cuh) -------------------------------------------------------------------------
int g_pdl = -1;
void set_pdl(int on) { g_pdl = on ? 1 : 0; }
bool pdl_enabled() {
    if (g_pdl < 0) { const char* e = getenv("RLR_PDL"); g_pdl = (e && atoi(e) > 0) ? 1 : 0; }
    return g_pdl > 0;
}

// ------------------------------------------------------------------------------------------------------------
// batch = normalize(dataset[perm[cursor : cursor+B]])   (uint8/float NHWC  ->  fp32/bf16, NCHW or padded NHWC)
// AUG: the raw image is random-cropped / flipped first (augment_draw, common.cuh); AUG = false is the plain gather, and the
// launchers pick it whenever crop pad and flip are both off, so un-augmented batches keep exactly the arithmetic they always had.
// ------------------------------------------------------------------------------------------------------------
template <typename TIn, typename TOut, bool AUG>
__global__ void gather_normalize_kernel(const TIn* __restrict__ data, const int64_t* __restrict__ idx,
                                        const int* __restrict__ cursor, const int64_t* __restrict__ targets,
                                        TOut* __restrict__ out, int64_t* __restrict__ out_labels, int B, int H, int W, int C,
                                        int c_pad, int nchw, float4 mean, float4 inv_std, float in_scale, AugSpec aug) {
    const int HW = H * W;
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= B * HW) return;
    const int b = t / HW, px = t - b * HW;
    const int64_t src = idx[(cursor ? *cursor : 0) + b];
    if (px == 0 && out_labels) out_labels[b] = targets[src];
    const TIn* in = data + (src * HW + px) * C;
    bool inside = true;
    if constexpr (AUG) {
        const AugDraw d = augment_draw(aug, (cursor ? (long long)*cursor : aug.start) + b);
        const int h = px / W, w = px - h * W;
        const int sh = h + d.oy - aug.pad, sw = (d.flip ? W - 1 - w : w) + d.ox - aug.pad;
        inside = sh >= 0 && sh < H && sw >= 0 && sw < W;
        in = data + (src * HW + (inside ? sh * W + sw : 0)) * C;
    }
    auto raw = [&](int c) { return (AUG && !inside) ? 0.f : (float)in[c]; };
    const float mu[4] = {mean.x, mean.y, mean.z, mean.w};
    const float is[4] = {inv_std.x, inv_std.y, inv_std.z, inv_std.w};
    if (nchw) {
        for (int c = 0; c < C; ++c)
            out[((int64_t)b * C + c) * HW + px] = (TOut)((raw(c) * in_scale - mu[c]) * is[c]);
    } else {
        TOut* o = out + ((int64_t)b * HW + px) * c_pad;
        for (int c = 0; c < C; ++c) o[c] = (TOut)((raw(c) * in_scale - mu[c]) * is[c]);
        for (int c = C; c < c_pad; ++c) o[c] = (TOut)0.f;
    }
}

// Padded NHWC output (c_pad % 8 == 0, bf16): c_pad/8 threads per pixel, one 16-byte store each -> fully coalesced rows.
template <typename TIn, bool AUG>
__global__ void __launch_bounds__(256) gather_normalize_padded_kernel(const TIn* __restrict__ data, const int64_t* __restrict__ idx,
                                                                        const int* __restrict__ cursor, const int64_t* __restrict__ targets,
                                                                        __nv_bfloat16* __restrict__ out, int64_t* __restrict__ out_labels, int B,
                                                                        int H, int W, int C, int c_pad, float4 mean, float4 inv_std, float in_scale,
                                                                        AugSpec aug) {
    const int HW = H * W;
    const int cpp = c_pad >> 3;                                  // chunks per pixel
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)B * HW * cpp) return;
    const long long pix = t / cpp;
    const int chunk = (int)(t - pix * cpp);
    const int b = (int)(pix / HW), px = (int)(pix - (long long)b * HW);
    const int64_t src = idx[(cursor ? *cursor : 0) + b];
    if (px == 0 && chunk == 0 && out_labels) out_labels[b] = targets[src];
    uint4 v = make_uint4(0, 0, 0, 0);
    if (chunk == 0) {
        const TIn* in = data + (src * HW + px) * C;
        bool inside = true;
        if constexpr (AUG) {
            const AugDraw d = augment_draw(aug, (cursor ? (long long)*cursor : aug.start) + b);
            const int h = px / W, w = px - h * W;
            const int sh = h + d.oy - aug.pad, sw = (d.flip ? W - 1 - w : w) + d.ox - aug.pad;
            inside = sh >= 0 && sh < H && sw >= 0 && sw < W;
            in = data + (src * HW + (inside ? sh * W + sw : 0)) * C;
        }
        const float mu[4] = {mean.x, mean.y, mean.z, mean.w};
        const float is[4] = {inv_std.x, inv_std.y, inv_std.z, inv_std.w};
        float f[4] = {0.f, 0.f, 0.f, 0.f};
        for (int c = 0; c < C; ++c) f[c] = (((AUG && !inside) ? 0.f : (float)in[c]) * in_scale - mu[c]) * is[c];
        v.x = pack_bf16x2(f[0], f[1]); v.y = pack_bf16x2(f[2], f[3]);
    }
    *reinterpret_cast<uint4*>(out + pix * c_pad + chunk * 8) = v;
}

// Gather + normalise + im2col for tiny-K first layers (C*k*k <= 64): row m = (b, ho, wo) of A[B*Ho*Wo][64] holds the k x k x C patch
// of the NORMALISED image around output pixel (ho, wo) in (tap, channel) order -- the K-major operand of the stem convolution as a
// plain 64-deep GEMM -- with zeros for padding pixels and for columns >= k*k*C.  Eight threads per row, one 16-byte store each.
// Replaces batch assembly (src/utils.py:52-54) + the first layer's implicit im2col (src/models.py:23,48) in one pass over the raw images.
// One block per (image b, output row ho): the k input rows that output row needs are normalised ONCE into shared memory (zero
// border included), then every thread assembles one 16-byte chunk of one im2col row from shared memory -- the global side is k
// coalesced row reads per block and fully coalesced 128-byte row writes (a first version gathered bytes straight from global
// memory: 67 us per 256-image batch, L1-wavefront bound; this one streams at the store rate).
// CT / KT > 0: channel count / filter size known at compile time (index arithmetic becomes multiply-shift); 0 = run-time values.
// AUG: the tile holds rows of the cropped / flipped image -- only the source coordinate of the staging loop moves, crop-padding
// pixels are stored value 0 normalised (-mean/std), and the convolution's own zero border stays 0.
template <typename TIn, int CT, int KT, bool AUG>
__global__ void __launch_bounds__(256) gather_im2col_kernel(const TIn* __restrict__ data, const int64_t* __restrict__ idx,
                                                              const int* __restrict__ cursor, const int64_t* __restrict__ targets,
                                                              __nv_bfloat16* __restrict__ A, int64_t* __restrict__ out_labels, int B, int H, int W,
                                                              int C_rt, int k_rt, int pad, int Ho, int Wo, float4 mean, float4 inv_std, float in_scale,
                                                              AugSpec aug) {
    extern __shared__ float tile[];                               // [k][W + 2 pad][C] normalised input rows, zero outside the image
    const int C = CT > 0 ? CT : C_rt, k = KT > 0 ? KT : k_rt;
    const int ho = blockIdx.x, b = blockIdx.y;
    const int Wp = W + 2 * pad;
    const int64_t src = idx[(cursor ? *cursor : 0) + b];
    if (ho == 0 && threadIdx.x == 0 && out_labels) out_labels[b] = targets[src];
    const float mu[4] = {mean.x, mean.y, mean.z, mean.w};
    const float is[4] = {inv_std.x, inv_std.y, inv_std.z, inv_std.w};
    const TIn* img = data + src * (int64_t)H * W * C;
    AugDraw d{0, 0, 0};
    if constexpr (AUG) {            // one draw per block: in every warp the Philox rounds doubled the kernel's instruction count
        __shared__ AugDraw sdraw;
        if (threadIdx.x == 0) sdraw = augment_draw(aug, (cursor ? (long long)*cursor : aug.start) + b);
        __syncthreads();
        d = sdraw;
    }
    for (int i = threadIdx.x; i < k * Wp * C; i += blockDim.x) {
        const int dy = i / (Wp * C), r = i - dy * (Wp * C);
        const int wp = r / C, ch = r - wp * C;
        const int hh = ho + dy - pad, ww = wp - pad;
        float v = 0.f;
        if (hh >= 0 && hh < H && ww >= 0 && ww < W) {
            const float m = ch == 0 ? mu[0] : ch == 1 ? mu[1] : ch == 2 ? mu[2] : mu[3];
            const float s_ = ch == 0 ? is[0] : ch == 1 ? is[1] : ch == 2 ? is[2] : is[3];
            if constexpr (AUG) {
                const int sh = hh + d.oy - aug.pad, sw = (d.flip ? W - 1 - ww : ww) + d.ox - aug.pad;
                const float x = (sh >= 0 && sh < H && sw >= 0 && sw < W) ? (float)img[(sh * W + sw) * C + ch] : 0.f;
                v = (x * in_scale - m) * s_;
            } else {
                v = ((float)img[(hh * W + ww) * C + ch] * in_scale - m) * s_;
            }
        }
        tile[i] = v;
    }
    __syncthreads();
    const int kvalid = k * k * C;
    for (int t = threadIdx.x; t < Wo * 8; t += blockDim.x) {
        const int wo = t >> 3, chunk = t & 7;
        float f[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int kk = chunk * 8 + j;
            f[j] = 0.f;
            if (kk < kvalid) {
                const int tap = kk / C, ch = kk - tap * C;
                const int dy = tap / k, dx = tap - dy * k;
                f[j] = tile[(dy * Wp + wo + dx) * C + ch];
            }
        }
        *reinterpret_cast<uint4*>(A + (((int64_t)b * Ho + ho) * Wo + wo) * 64 + chunk * 8) =
            make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]), pack_bf16x2(f[6], f[7]));
    }
}

static inline bool make_aug(AugSpec& a, int H, int W, int crop_pad, int flip, long long seed, const long long* stream, long long start) {
    a = AugSpec{stream, (unsigned long long)seed, start, crop_pad, flip ? 1 : 0};
    return crop_pad >= 0 && crop_pad < H && crop_pad < W && (!(crop_pad > 0 || flip) || stream);
}

cudaError_t launch_gather_im2col(const void* data, int in_is_float, const int64_t* idx, const int* cursor, const int64_t* targets,
                                 __nv_bfloat16* A, int64_t* out_labels, int B, int H, int W, int C, int k, int pad, const float* mean,
                                 const float* stdv, int crop_pad, int flip, long long seed, const long long* aug_stream, long long start,
                                 cudaStream_t st) {
    if (C > 4 || B <= 0 || k * k * C > 64) return cudaErrorInvalidValue;
    AugSpec aug;
    if (!make_aug(aug, H, W, crop_pad, flip, seed, aug_stream, start)) return cudaErrorInvalidValue;
    float mu[4] = {0, 0, 0, 0}, is[4] = {1, 1, 1, 1};
    for (int c = 0; c < C; ++c) { mu[c] = mean[c]; is[c] = 1.0f / stdv[c]; }
    const float4 m4 = make_float4(mu[0], mu[1], mu[2], mu[3]), s4 = make_float4(is[0], is[1], is[2], is[3]);
    const int Ho = H + 2 * pad - k + 1, Wo = W + 2 * pad - k + 1;
    const dim3 grid(Ho, B);
    const size_t smem = (size_t)k * (W + 2 * pad) * C * sizeof(float);
    if (smem > 40 * 1024) return cudaErrorInvalidValue;
    const int threads = Wo * 8 >= 256 ? 256 : ((Wo * 8 + 31) / 32) * 32;
#define RLR_GI(TI, CT, KT, SC)                                                                                                        \
    do {                                                                                                                               \
        if (crop_pad > 0 || flip)                                                                                                      \
            gather_im2col_kernel<TI, CT, KT, true><<<grid, threads, smem, st>>>((const TI*)data, idx, cursor, targets, A, out_labels,  \
                                                                                B, H, W, C, k, pad, Ho, Wo, m4, s4, SC, aug);          \
        else                                                                                                                           \
            gather_im2col_kernel<TI, CT, KT, false><<<grid, threads, smem, st>>>((const TI*)data, idx, cursor, targets, A, out_labels, \
                                                                                 B, H, W, C, k, pad, Ho, Wo, m4, s4, SC, aug);         \
    } while (0)
    if (in_is_float) {
        if (C == 1 && k == 3) RLR_GI(float, 1, 3, 1.0f); else if (C == 3 && k == 3) RLR_GI(float, 3, 3, 1.0f); else RLR_GI(float, 0, 0, 1.0f);
    } else {
        if (C == 1 && k == 3) RLR_GI(uint8_t, 1, 3, 1.0f / 255.0f); else if (C == 3 && k == 3) RLR_GI(uint8_t, 3, 3, 1.0f / 255.0f);
        else RLR_GI(uint8_t, 0, 0, 1.0f / 255.0f);
    }
#undef RLR_GI
    return cudaGetLastError();
}

cudaError_t launch_gather_normalize(const void* data, int in_is_float, const int64_t* idx, const int* cursor,
                                    const int64_t* targets, void* out, int out_kind, int64_t* out_labels, int B, int H,
                                    int W, int C, int c_pad, int nchw, const float* mean, const float* stdv,
                                    int crop_pad, int flip, long long seed, const long long* aug_stream, long long start,
                                    cudaStream_t st) {
    if (C > 4 || B <= 0) return cudaErrorInvalidValue;
    AugSpec aug;
    if (!make_aug(aug, H, W, crop_pad, flip, seed, aug_stream, start)) return cudaErrorInvalidValue;
    const bool on = crop_pad > 0 || flip;
    float mu[4] = {0, 0, 0, 0}, is[4] = {1, 1, 1, 1};
    for (int c = 0; c < C; ++c) { mu[c] = mean[c]; is[c] = 1.0f / stdv[c]; }
    const float4 m4 = make_float4(mu[0], mu[1], mu[2], mu[3]), s4 = make_float4(is[0], is[1], is[2], is[3]);
    const int HW = H * W, total = B * HW, threads = 256, blocks = (total + threads - 1) / threads;
    const float sc = in_is_float ? 1.0f : (1.0f / 255.0f);
    if (!nchw && out_kind == 1 && c_pad > C && c_pad % 8 == 0) {      // channel-padded bf16 NHWC (stem input of the wgmma conv)
        const long long tot = (long long)total * (c_pad / 8);
        const int nb = (int)((tot + 255) / 256);
#define RLR_GP(TI, A_)                                                                                                                 \
        gather_normalize_padded_kernel<TI, A_><<<nb, 256, 0, st>>>((const TI*)data, idx, cursor, targets, (__nv_bfloat16*)out,        \
                                                                    out_labels, B, H, W, C, c_pad, m4, s4, sc, aug)
        if (in_is_float) { if (on) RLR_GP(float, true); else RLR_GP(float, false); }
        else             { if (on) RLR_GP(uint8_t, true); else RLR_GP(uint8_t, false); }
#undef RLR_GP
        return cudaGetLastError();
    }
#define RLR_GN(TI, TO)                                                                                                    \
    do {                                                                                                                  \
        if (on) gather_normalize_kernel<TI, TO, true><<<blocks, threads, 0, st>>>((const TI*)data, idx, cursor, targets,  \
                                                                                   (TO*)out, out_labels, B, H, W, C,      \
                                                                                   c_pad, nchw, m4, s4, sc, aug);         \
        else gather_normalize_kernel<TI, TO, false><<<blocks, threads, 0, st>>>((const TI*)data, idx, cursor, targets,    \
                                                                                 (TO*)out, out_labels, B, H, W, C,        \
                                                                                 c_pad, nchw, m4, s4, sc, aug);           \
    } while (0)
    if (in_is_float) { if (out_kind == 0) RLR_GN(float, float); else RLR_GN(float, __nv_bfloat16); }
    else             { if (out_kind == 0) RLR_GN(uint8_t, float); else RLR_GN(uint8_t, __nv_bfloat16); }
#undef RLR_GN
    return cudaGetLastError();
}

// end of a local step: the batch cursor moves on and (optionally) the Philox step counter of the dropout masks is bumped --
// one single-thread node instead of a torch `+= 1` inside the captured step
__global__ void advance_cursor_kernel(int* cursor, int delta, long long* step) {
    *cursor += delta;
    if (step) *step += 1;
}
cudaError_t launch_advance_cursor(int* cursor, int delta, long long* step, cudaStream_t st) {
    advance_cursor_kernel<<<1, 1, 0, st>>>(cursor, delta, step);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------------------
// row padding for tiny-K operands: dst[r][0..Kp) = src[r][0..K) followed by zeros (bf16).  Used for the stem conv's channel-
// padded input / filter and the im2col filter matrix ([Cout][k*k*Cin] -> [Cout][64]); the inverse adds the valid columns of an
// fp32 [R][Kp] gradient into the [R][K] slice of the flat gradient.
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) pad_rows_kernel(const __nv_bfloat16* __restrict__ src, __nv_bfloat16* __restrict__ dst,
                                                         long long R, int K, int Kp) {
    // one thread per 8 output columns (Kp % 8 == 0): 16-byte stores; the <= K valid columns of a chunk are gathered one by one
    const int cpr = Kp >> 3;
    const long long n = R * cpr;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / cpr;
        const int c0 = (int)(i - r * cpr) * 8;
        uint32_t h[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) h[j] = (c0 + j < K) ? (uint32_t)__bfloat16_as_ushort(src[r * K + c0 + j]) : 0u;
        *reinterpret_cast<uint4*>(dst + r * Kp + c0) = make_uint4(h[0] | (h[1] << 16), h[2] | (h[3] << 16), h[4] | (h[5] << 16), h[6] | (h[7] << 16));
    }
}
cudaError_t launch_pad_rows(const __nv_bfloat16* src, __nv_bfloat16* dst, long long R, int K, int Kp, int num_sms, cudaStream_t st) {
    if (K > Kp || R <= 0 || (Kp & 7)) return cudaErrorInvalidValue;
    const long long want = (R * (Kp >> 3) + 255) / 256;
    const int grid = (int)(want > (long long)num_sms * 8 ? (long long)num_sms * 8 : want);
    pad_rows_kernel<<<grid, 256, 0, st>>>(src, dst, R, K, Kp);
    return cudaGetLastError();
}
__global__ void __launch_bounds__(256) unpad_add_kernel(const float* __restrict__ src, float* __restrict__ dst, long long R, int K, int Kp) {
    const long long n = R * K;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / K;
        dst[i] += src[r * Kp + (i - r * K)];
    }
}
cudaError_t launch_unpad_add(const float* src, float* dst, long long R, int K, int Kp, int num_sms, cudaStream_t st) {
    if (K > Kp || R <= 0) return cudaErrorInvalidValue;
    const long long want = (R * K + 255) / 256;
    const int grid = (int)(want > (long long)num_sms * 8 ? (long long)num_sms * 8 : want);
    unpad_add_kernel<<<grid, 256, 0, st>>>(src, dst, R, K, Kp);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------------------
// trojan stamping: apply a compiled pixel program to selected images in place (SURVEY.md 2.2)
// mode 0: set (all channels) | 1: uint8 wrap-around add | 2: float subtract
// ------------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void stamp_pixels_kernel(T* __restrict__ data, const int64_t* __restrict__ sel, int S,
                                    const int* __restrict__ rows, const int* __restrict__ cols,
                                    const float* __restrict__ vals, int P, int H, int W, int C, int mode) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (int64_t)S * P * C) return;
    const int c = (int)(t % C);
    const int pi = (int)((t / C) % P);
    const int64_t s = t / ((int64_t)C * P);
    T* px = data + ((sel[s] * H + rows[pi]) * W + cols[pi]) * C + c;
    const float v = vals[pi];
    if (mode == 0) *px = (T)v;
    else if (mode == 1) *px = (T)(uint8_t)((unsigned)(*px) + (unsigned)v);  // wraps mod 256 like numpy uint8
    else *px = (T)((float)(*px) - v);
}

cudaError_t launch_stamp_pixels(void* data, int is_float, const int64_t* sel, int S, const int* rows, const int* cols,
                                const float* vals, int P, int H, int W, int C, int mode, cudaStream_t st) {
    if (S <= 0 || P <= 0) return cudaSuccess;
    const int64_t total = (int64_t)S * P * C;
    const int threads = 256;
    const int blocks = (int)((total + threads - 1) / threads);
    if (is_float) stamp_pixels_kernel<float><<<blocks, threads, 0, st>>>((float*)data, sel, S, rows, cols, vals, P, H, W, C, mode);
    else stamp_pixels_kernel<uint8_t><<<blocks, threads, 0, st>>>((uint8_t*)data, sel, S, rows, cols, vals, P, H, W, C, mode);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------------------
// round start: w_local <- w_global (the "broadcast" consumer), bf16 operand shadow, momentum <- 0
// (reference: deepcopy + vector_to_parameters src/federated.py:72; fresh optimizer src/agent.py:37-38)
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) round_init_kernel(const float* __restrict__ wg, float* __restrict__ wl,
                                                           __nv_bfloat16* __restrict__ wb, float* __restrict__ mom,
                                                           long long n4) {
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n4; q += (long long)gridDim.x * blockDim.x) {
        const float4 v = ld_f4(wg + 4 * q);
        if (wl) st_f4(wl + 4 * q, v);
        if (wb) *reinterpret_cast<uint2*>(wb + 4 * q) = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
        if (mom) st_f4(mom + 4 * q, make_float4(0.f, 0.f, 0.f, 0.f));
    }
}
static inline int grid_for(long long n4, int threads, int num_sms, int per_sm) {
    long long want = (n4 + threads - 1) / threads;
    long long cap = (long long)num_sms * per_sm;
    return (int)(want < 1 ? 1 : (want > cap ? cap : want));
}
cudaError_t launch_round_init(const float* w_global, float* w_local, __nv_bfloat16* w_bf16, float* mom, long long n,
                              cudaStream_t st) {
    if (n & 3) return cudaErrorInvalidValue;
    round_init_kernel<<<grid_for(n / 4, 256, 132, 8), 256, 0, st>>>(w_global, w_local, w_bf16, mom, n / 4);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------------------
// fused clip_grad_norm_(.,max) + SGD(momentum) [+ ||w-w0||^2 for PGD] over flat buffers   (src/agent.py:50-60)
// ------------------------------------------------------------------------------------------------------------
// the norm pass and the step are templates in flat_sgd.cuh; a local objective's launches go to objective.cu
cudaError_t launch_sqnorm(const float* x, long long n, double* out, int num_sms, cudaStream_t st, const uint32_t* mask,
                          long long n_mask, const float* w, const float* w0, long long n_pgd) {
    if ((n & 3) || (mask && ((n_mask & 3) || n_mask < 0 || n_mask > n))) return cudaErrorInvalidValue;
    if (w0 && (!w || (n_pgd & 3) || n_pgd <= 0 || n_pgd > n)) return cudaErrorInvalidValue;
    const int grid = grid_for(n / 4, 256, num_sms, 4);
    const long long nout = w0 ? 3 : 1;
    Scratch part((size_t)grid * nout * sizeof(double), st);
    if (w0) launch_sqnorm_objective(grid, st, x, n / 4, part.as<double>(), mask, n_mask / 4, w, w0, n_pgd / 4);
    else if (mask) sqnorm_kernel<true, false><<<grid, 256, 0, st>>>(x, n / 4, part.as<double>(), mask, n_mask / 4, nullptr, nullptr, 0);
    else sqnorm_kernel<false, false><<<grid, 256, 0, st>>>(x, n / 4, part.as<double>(), nullptr, 0, nullptr, nullptr, 0);
    RLR_CUDA_CHECK(cudaGetLastError());
    RLR_CUDA_CHECK(launch_ordered_sum(out, part.as<double>(), grid, nout, st));
    return cudaGetLastError();
}

cudaError_t launch_sgd_step(float* w, const float* g, float* m, const float* w0, __nv_bfloat16* w_bf16, long long n,
                            float lr, float momentum, float max_grad_norm, const double* g_sqnorm, double* d_sqnorm,
                            int num_sms, cudaStream_t st, long long n_pgd, const float* w_in, const uint32_t* mask,
                            const float* objective) {
    if ((n & 3) || (n_pgd & 3)) return cudaErrorInvalidValue;
    if (objective && (!w0 || !g_sqnorm)) return cudaErrorInvalidValue;
    if (n_pgd <= 0 || n_pgd > n) n_pgd = n;
    const int grid = grid_for(n / 4, 256, num_sms, 4);
    auto step = [&](double* dp) {
        if (objective)
            launch_sgd_step_objective(grid, st, w, g, m, w0, w_bf16, n / 4, lr, momentum, max_grad_norm, g_sqnorm, dp, n_pgd / 4, w_in,
                                      mask, objective[0], objective[1], objective[2]);
        else if (mask)
            sgd_step_kernel<true, false><<<grid, 256, 0, st>>>(w, g, m, w0, w_bf16, n / 4, lr, momentum, max_grad_norm, g_sqnorm, dp,
                                                               n_pgd / 4, w_in, w_in ? 1 : 0, mask, 1.f, 0.f, 0.f);
        else
            sgd_step_kernel<false, false><<<grid, 256, 0, st>>>(w, g, m, w0, w_bf16, n / 4, lr, momentum, max_grad_norm, g_sqnorm, dp,
                                                                n_pgd / 4, w_in, w_in ? 1 : 0, nullptr, 1.f, 0.f, 0.f);
        return cudaGetLastError();
    };
    if (!d_sqnorm) return step(nullptr);
    // PGD: per-CTA ||w - w0||^2 partials, added into d_sqnorm in CTA order (as launch_sqnorm), so the radius pgd_project reads is
    // the same sum on every run
    Scratch part((size_t)grid * sizeof(double), st);
    RLR_CUDA_CHECK(step(part.as<double>()));
    RLR_CUDA_CHECK(launch_ordered_sum(d_sqnorm, part.as<double>(), grid, 1LL, st));
    return cudaGetLastError();
}

// PGD: w <- w0 + (w - w0) / max(1, ||w - w0|| / clip)   (src/agent.py:54-60), no host sync for the norm
// MASK: masked coordinates (never moved from w0 by a masked step) keep their bits, -0 included
template <bool MASK>
__global__ void __launch_bounds__(256) pgd_project_kernel(float* __restrict__ w, const float* __restrict__ w0,
                                                            __nv_bfloat16* __restrict__ wb, long long n4, float clip,
                                                            const double* __restrict__ d_sqnorm, long long n4_pgd,
                                                            const uint32_t* __restrict__ mask) {
    const float denom = fmaxf(1.0f, (float)sqrt(*d_sqnorm) / clip);
    const float inv = 1.0f / denom;
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n4; q += (long long)gridDim.x * blockDim.x) {
        float4 wv = ld_f4(w + 4 * q);
        if (denom > 1.0f && q < n4_pgd) {
            const float4 o = ld_f4(w0 + 4 * q);
            float4 pv;
            pv.x = o.x + (wv.x - o.x) * inv; pv.y = o.y + (wv.y - o.y) * inv;
            pv.z = o.z + (wv.z - o.z) * inv; pv.w = o.w + (wv.w - o.w) * inv;
            if (MASK) {
                const uint32_t nib = (__ldg(mask + (q >> 3)) >> ((q & 7) * 4)) & 0xFu;
                if (!(nib & 1u)) wv.x = pv.x;
                if (!(nib & 2u)) wv.y = pv.y;
                if (!(nib & 4u)) wv.z = pv.z;
                if (!(nib & 8u)) wv.w = pv.w;
            } else {
                wv = pv;
            }
            st_f4(w + 4 * q, wv);
        }
        if (wb) *reinterpret_cast<uint2*>(wb + 4 * q) = make_uint2(pack_bf16x2(wv.x, wv.y), pack_bf16x2(wv.z, wv.w));
    }
}
cudaError_t launch_pgd_project(float* w, const float* w0, __nv_bfloat16* w_bf16, long long n, float clip,
                               const double* d_sqnorm, int num_sms, cudaStream_t st, long long n_pgd, const uint32_t* mask) {
    if ((n & 3) || (n_pgd & 3)) return cudaErrorInvalidValue;
    if (n_pgd <= 0 || n_pgd > n) n_pgd = n;
    const int grid = grid_for(n / 4, 256, num_sms, 4);
    if (mask) pgd_project_kernel<true><<<grid, 256, 0, st>>>(w, w0, w_bf16, n / 4, clip, d_sqnorm, n_pgd / 4, mask);
    else pgd_project_kernel<false><<<grid, 256, 0, st>>>(w, w0, w_bf16, n / 4, clip, d_sqnorm, n_pgd / 4, nullptr);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------------------
// softmax cross-entropy forward+backward (mean reduction): one thread per row, C <= 32
// ------------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void softmax_xent_kernel(const T* __restrict__ logits, const int64_t* __restrict__ labels, T* __restrict__ dlogits,
                                    float* loss_part /*[gridDim.x]*/, int* correct, int B, int C, float grad_scale) {
    __shared__ float scratch[32];
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    float loss = 0.f;
    int ok = 0;
    if (b < B) {
        float v[32];
        float mx = -INFINITY;
        int arg = 0;
        for (int c = 0; c < C; ++c) {
            v[c] = (float)logits[(int64_t)b * C + c];
            if (v[c] > mx) { mx = v[c]; arg = c; }
        }
        float se = 0.f;
        for (int c = 0; c < C; ++c) { v[c] = __expf(v[c] - mx); se += v[c]; }
        const int y = (int)labels[b];
        const float inv = 1.0f / se;
        // -log p_y while p_y is far above underflow (the 1e-30 guard is then below rounding).  Below 2^-64 the label lies ~44 or more
        // below the max, and -log(p_y + 1e-30) would saturate at 69.08 once p_y underflows: there the loss is the stable
        // log(se) - (x_y - mx) of eval_metrics, from the label's logit itself
        const float q = v[y] * inv + 1e-30f;
        loss = q >= 0x1p-64f ? -(__logf(q)) : logf(se) - ((float)logits[(int64_t)b * C + y] - mx);
        ok = (arg == y);
        if (dlogits)
            for (int c = 0; c < C; ++c) dlogits[(int64_t)b * C + c] = (T)((v[c] * inv - (c == y ? 1.f : 0.f)) * grad_scale);
    }
    const float tot = block_sum<float>(loss, scratch);
    if (threadIdx.x == 0 && loss_part) loss_part[blockIdx.x] = tot;
    if (correct) {
        const int nok = __syncthreads_count(ok);
        if (threadIdx.x == 0 && nok) atomicAdd(correct, nok);
    }
}
cudaError_t launch_softmax_xent(const void* logits, int kind, const int64_t* labels, void* dlogits, float* loss_sum,
                                int* correct, int B, int C, float grad_scale, cudaStream_t st) {
    if (C > 32 || B <= 0) return cudaErrorInvalidValue;
    const int threads = 128, blocks = (B + threads - 1) / threads;
    Scratch part((size_t)blocks * sizeof(float), st);                 // per-block loss sums, added into loss_sum in block order
    float* lp = loss_sum ? part.as<float>() : nullptr;
    if (kind == 0) softmax_xent_kernel<float><<<blocks, threads, 0, st>>>((const float*)logits, labels, (float*)dlogits, lp, correct, B, C, grad_scale);
    else softmax_xent_kernel<__nv_bfloat16><<<blocks, threads, 0, st>>>((const __nv_bfloat16*)logits, labels, (__nv_bfloat16*)dlogits, lp, correct, B, C, grad_scale);
    RLR_CUDA_CHECK(cudaGetLastError());
    if (loss_sum) RLR_CUDA_CHECK(launch_ordered_sum(loss_sum, part.as<float>(), blocks, 1LL, st));
    return cudaGetLastError();
}

// evaluation: sum of per-sample losses + confusion matrix, all on device (reference loops over samples on the
// host with .item() syncs, src/utils.py:144-152)
template <typename T>
__global__ void eval_metrics_kernel(const T* __restrict__ logits, const int64_t* __restrict__ labels, int B, int C,
                                    double* loss_part /*[gridDim.x]*/, long long* confusion) {
    __shared__ double scratch[32];
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    double loss = 0.0;
    if (b < B) {
        float mx = -INFINITY;
        int arg = 0;
        for (int c = 0; c < C; ++c) {
            const float v = (float)logits[(int64_t)b * C + c];
            if (v > mx) { mx = v; arg = c; }
        }
        float se = 0.f;
        for (int c = 0; c < C; ++c) se += expf((float)logits[(int64_t)b * C + c] - mx);
        const int y = (int)labels[b];
        loss = (double)(logf(se) - ((float)logits[(int64_t)b * C + y] - mx));
        atomicAdd((unsigned long long*)(confusion + (int64_t)y * C + arg), 1ull);
    }
    const double tot = block_sum<double>(loss, scratch);
    if (threadIdx.x == 0) loss_part[blockIdx.x] = tot;
}
cudaError_t launch_eval_metrics(const void* logits, int kind, const int64_t* labels, int B, int C, double* loss_sum,
                                long long* confusion, cudaStream_t st) {
    if (B <= 0) return cudaSuccess;
    const int threads = 128, blocks = (B + threads - 1) / threads;
    Scratch part((size_t)blocks * sizeof(double), st);                // per-block loss sums, added into loss_sum in block order
    double* lp = part.as<double>();
    if (kind == 0) eval_metrics_kernel<float><<<blocks, threads, 0, st>>>((const float*)logits, labels, B, C, lp, confusion);
    else eval_metrics_kernel<__nv_bfloat16><<<blocks, threads, 0, st>>>((const __nv_bfloat16*)logits, labels, B, C, lp, confusion);
    RLR_CUDA_CHECK(cudaGetLastError());
    RLR_CUDA_CHECK(launch_ordered_sum(loss_sum, lp, blocks, 1LL, st));
    return cudaGetLastError();
}

}  // namespace rlr
