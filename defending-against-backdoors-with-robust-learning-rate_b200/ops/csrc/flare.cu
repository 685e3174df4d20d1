// FLARE's MMD pass (Wang, Xiao, Chen, Hu, Lou, Hou, ASIA CCS 2022; DESIGN.md section 3): the kernel sums between the penultimate-layer
// representations of every pair of candidate models on the server's root set,
//   S[i][j] = sum_{a in Z_i, b in Z_j} exp(-||a - b||^2 / sigma^2),   i <= j,
// with Z_k the [n][d] fp32 features of candidate k.  The host forms M_ij = max(0, (S_ii + S_jj - 2 S_ij) / n^2) from them.
//
// Each squared distance is accumulated in fp32 from direct differences (a - b)^2 (one FMA per coordinate), over the feature dimension in
// ascending order.  The expansion ||a||^2 + ||b||^2 - 2 a.b would be a GEMM, but its cancellation moves exactly the nearby points whose
// kernel values are close to 1 and dominate the sums.  kappa = expf(-dist * (1 / sigma^2)).
//
// Work decomposition: one CTA per (pair, 64 x 64 tile of the n x n sample pairs); the pairs (i <= j) are numbered row by row and a CTA
// decodes its own, so one launch covers every pair for any number of candidates.  A CTA stages 32-coordinate slices of its 64 rows of
// Z_i and 64 rows of Z_j in shared memory, transposed (coordinate-major), and each of its 256 threads keeps a 4 x 4 block of distances in
// registers.  A pair with a non-finite candidate (mask 0) writes 0 without reading its features.  Each thread adds its kappas in fp64
// in a fixed order, the warp shuffles and then warp 0 add the threads' sums in a fixed order, and the CTA writes its value to the
// workspace slot [tile][pair]; launch_ordered_sum adds the tiles of every pair in tile order.  No atomics: two launches are bitwise equal.
#include "common.cuh"
#include "kernels.h"

namespace rlr {

namespace {

constexpr int kFlareThreads = 256;
constexpr int kFlareTile = 64;                   // samples of Z_i (rows) and of Z_j (columns) per CTA
constexpr int kFlareChunk = 32;                  // feature coordinates staged per step
constexpr int kFlarePitch = kFlareTile + 4;      // staged row pitch in floats (16-byte aligned, spreads the transposed stores)

struct FlareKernelParams {
    const float* z;                              // [K][n][d]
    const unsigned char* finite;                 // [K]: 1 = every feature of the candidate is finite
    int K, n, d, tiles_1d;                       // tiles_1d = ceil(n / 64)
    long long pairs;                             // K (K + 1) / 2
    float inv_s2;                                // 1 / sigma^2 (fp32)
    double* ws;                                  // [tiles_1d^2][pairs]
};

__device__ __forceinline__ void decode_pair(long long p, int K, int& i, int& j) {
    int r = 0;
    long long len = K;
    while (p >= len) {                           // row r holds the pairs (r, r), (r, r + 1), ..., (r, K - 1)
        p -= len;
        ++r;
        --len;
    }
    i = r;
    j = r + (int)p;
}

__global__ void __launch_bounds__(kFlareThreads) flare_mmd_kernel(FlareKernelParams kp) {
    __shared__ __align__(16) float sa[kFlareChunk][kFlarePitch];
    __shared__ __align__(16) float sb[kFlareChunk][kFlarePitch];
    __shared__ double wsum[kFlareThreads / kWarp];
    const int tid = threadIdx.x;
    const long long tiles = (long long)kp.tiles_1d * kp.tiles_1d;
    const long long pair = (long long)blockIdx.x / tiles;
    const int tile = (int)((long long)blockIdx.x - pair * tiles);
    int ci, cj;
    decode_pair(pair, kp.K, ci, cj);
    double* const out = kp.ws + (size_t)tile * kp.pairs + pair;
    if (!kp.finite[ci] || !kp.finite[cj]) {
        if (tid == 0) *out = 0.0;
        return;
    }
    const int n = kp.n, d = kp.d;
    const int a0 = (tile / kp.tiles_1d) * kFlareTile, b0 = (tile % kp.tiles_1d) * kFlareTile;
    const float* const za = kp.z + ((size_t)ci * n + a0) * d;
    const float* const zb = kp.z + ((size_t)cj * n + b0) * d;
    const int ty = tid / 16, tx = tid % 16;      // this thread's rows a0 + 4 ty .. + 3, columns b0 + 4 tx .. + 3

    float acc[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int s = 0; s < 4; ++s) acc[r][s] = 0.f;

    for (int c0 = 0; c0 < d; c0 += kFlareChunk) {
        const int cw = min(kFlareChunk, d - c0);
        __syncthreads();                                             // the previous slice has been consumed
        // stage: 64 rows x 32 coordinates of each side; consecutive threads read consecutive coordinates of one row
        for (int e = tid; e < kFlareTile * kFlareChunk; e += kFlareThreads) {
            const int row = e / kFlareChunk, c = e % kFlareChunk;
            const bool in_c = c < cw;
            sa[c][row] = (in_c && a0 + row < n) ? za[(size_t)row * d + c0 + c] : 0.f;
            sb[c][row] = (in_c && b0 + row < n) ? zb[(size_t)row * d + c0 + c] : 0.f;
        }
        __syncthreads();
        for (int c = 0; c < cw; ++c) {                               // ascending coordinates
            const float4 av = *reinterpret_cast<const float4*>(&sa[c][4 * ty]);
            const float4 bv = *reinterpret_cast<const float4*>(&sb[c][4 * tx]);
            const float a[4] = {av.x, av.y, av.z, av.w}, b[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
            for (int r = 0; r < 4; ++r)
#pragma unroll
                for (int s = 0; s < 4; ++s) {
                    const float df = __fsub_rn(a[r], b[s]);
                    acc[r][s] = __fmaf_rn(df, df, acc[r][s]);
                }
        }
    }

    // kappa of every valid sample pair, added in fp64 in (row, column) order
    double sum = 0.0;
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int s = 0; s < 4; ++s)
            if (a0 + 4 * ty + r < n && b0 + 4 * tx + s < n) sum += (double)expf(-acc[r][s] * kp.inv_s2);
#pragma unroll
    for (int o = kWarp / 2; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if ((tid & (kWarp - 1)) == 0) wsum[tid / kWarp] = sum;
    __syncthreads();
    if (tid == 0) {
        double t = wsum[0];
        for (int w = 1; w < kFlareThreads / kWarp; ++w) t += wsum[w];
        *out = t;
    }
}

}  // namespace

cudaError_t launch_flare_mmd(const float* z, const unsigned char* finite, int K, int n, int d, float inv_s2, double* out,
                             cudaStream_t st) {
    if (K < 1 || n < 1 || d < 1 || !z || !finite || !out) return cudaErrorInvalidValue;
    FlareKernelParams kp{};
    kp.z = z;
    kp.finite = finite;
    kp.K = K;
    kp.n = n;
    kp.d = d;
    kp.tiles_1d = (n + kFlareTile - 1) / kFlareTile;
    kp.pairs = (long long)K * (K + 1) / 2;
    kp.inv_s2 = inv_s2;
    const long long tiles = (long long)kp.tiles_1d * kp.tiles_1d;
    const long long grid = kp.pairs * tiles;
    if (grid > 0x7fffffffLL) return cudaErrorInvalidValue;
    Scratch ws((size_t)(tiles * kp.pairs) * sizeof(double), st);
    kp.ws = ws.as<double>();
    RLR_CUDA_CHECK(cudaMemsetAsync(out, 0, (size_t)kp.pairs * sizeof(double), st));
    flare_mmd_kernel<<<dim3((unsigned)grid), kFlareThreads, 0, st>>>(kp);
    RLR_CUDA_CHECK(cudaGetLastError());
    return launch_ordered_sum(out, kp.ws, (int)tiles, kp.pairs, st);
}

}  // namespace rlr
