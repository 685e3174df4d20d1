// Shared device helpers for the sm_90a kernels of robust-fl.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

#include "dropspec.h"
#include "kernels.h"

#define RLR_CUDA_CHECK(expr)                                                                     \
    do {                                                                                         \
        cudaError_t _e = (expr);                                                                 \
        if (_e != cudaSuccess) return _e;                                                        \
    } while (0)

namespace rlr {

constexpr int kWarp = 32;

// ---- programmatic dependent launch (PDL) ------------------------------------------------------------------------------------
// Kernels launched through launch_kernel() with PDL enabled (RLR_PDL=1 / set_pdl) may start while their predecessor in the stream
// is still draining: they run their prologue (barrier init, tensor-map prefetch, index arithmetic) and then block
// in pdl_wait() until the predecessor grid has completed and its memory is visible.  Rules every such kernel follows: NO global
// memory access before pdl_wait(); pdl_wait() is executed by every thread; pdl_trigger() (lets the successor start launching)
// comes after it.  Without the launch attribute both instructions are no-ops, so the same kernels serve plain launches.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

extern int g_pdl;             // -1: read RLR_PDL on first use (default off); defined in elementwise.cu
bool pdl_enabled();

template <typename... KArgs, typename... Args>
inline cudaError_t launch_kernel(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
    if (!pdl_enabled()) {
        kernel<<<grid, block, smem, st>>>(static_cast<KArgs>(args)...);
        return cudaGetLastError();
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// ---- deterministic cross-CTA reductions ---------------------------------------------------------------------------------------
// A reduction over CTAs never adds into its output with float atomics (their order, and so the rounding, changes from run to run):
// every CTA writes its partial result to a slot of a scratch buffer and launch_ordered_sum adds the slots in a fixed order.
// Scratch memory comes from the framework's stream-ordered caching allocator (gemm_binding.cpp), so it is safe to release right
// after the launches that use it and it is captured with the rest of a CUDA graph.
void* scratch_alloc(size_t bytes, cudaStream_t st);
void scratch_free(void* p);
struct Scratch {
    void* p;
    Scratch(size_t bytes, cudaStream_t st) : p(scratch_alloc(bytes, st)) {}
    ~Scratch() { scratch_free(p); }
    Scratch(const Scratch&) = delete;
    Scratch& operator=(const Scratch&) = delete;
    template <typename T> T* as() const { return static_cast<T*>(p); }
};
// out[i] += part[0][i] + part[1][i] + ... + part[nparts-1][i]   (part = [nparts][n])
template <typename T>
__global__ void __launch_bounds__(256) ordered_sum_kernel(T* __restrict__ out, const T* __restrict__ part, int nparts, long long n) {
    pdl_wait();
    pdl_trigger();
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
        T s = part[i];
        for (int j = 1; j < nparts; ++j) s += part[(size_t)j * n + i];
        out[i] += s;
    }
}

// Same sums as ordered_sum_kernel for many partials (the per-CTA slots of a grid-wide reduction: hundreds of parts of a few hundred
// columns).  One thread per element walking hundreds of dependent-order loads leaves a handful of CTAs latency-bound, so here a CTA
// takes 32 columns: all eight warps stage 64 parts at a time into shared memory with independent coalesced loads, and warp 0 adds
// the staged rows in part order -- the additions, and so the rounding, are exactly those of ordered_sum_kernel.
template <typename T>
__global__ void __launch_bounds__(256) ordered_sum_cols_kernel(T* __restrict__ out, const T* __restrict__ part, int nparts, long long n) {
    constexpr int kRows = 64, kPerWarp = kRows / 8;
    __shared__ T tile[kRows][33];
    pdl_wait();
    pdl_trigger();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long col = (long long)blockIdx.x * 32 + lane;
    T s = T(0);
    for (int j0 = 0; j0 < nparts; j0 += kRows) {
        T v[kPerWarp];
#pragma unroll
        for (int q = 0; q < kPerWarp; ++q) {
            const int j = j0 + warp + 8 * q;
            v[q] = (j < nparts && col < n) ? part[(size_t)j * n + col] : T(0);
        }
#pragma unroll
        for (int q = 0; q < kPerWarp; ++q) tile[warp + 8 * q][lane] = v[q];
        __syncthreads();
        if (warp == 0) {
            const int rows = nparts - j0 < kRows ? nparts - j0 : kRows;
            int r = 0;
            if (j0 == 0) { s = tile[0][lane]; r = 1; }
            for (; r < rows; ++r) s += tile[r][lane];
        }
        __syncthreads();
    }
    if (warp == 0 && col < n) out[col] += s;
}

// Same sums again, for few columns (the BatchNorm / GroupNorm statistics: 2C <= 2048 columns of 256-528 parts).  There the staged
// kernel runs on 4-32 CTAs and its chain is load latency, then warp 0's additions, then the next load: this one spreads the columns
// over 4x more CTAs (8 columns each) and double-buffers 256-part chunks, so the loads of chunk k + 1 are in flight while lanes 0-7
// of warp 0 add chunk k in part order.  Additions and rounding are those of ordered_sum_kernel.
template <typename T>
__global__ void __launch_bounds__(256) ordered_sum_narrow_kernel(T* __restrict__ out, const T* __restrict__ part, int nparts, long long n) {
    constexpr int kCols = 8, kRows = 256 * 8 / kCols, kPerThread = kRows * kCols / 256;
    __shared__ T tile[2][kRows][kCols];
    pdl_wait();
    pdl_trigger();
    const int c = threadIdx.x % kCols, r0 = threadIdx.x / kCols;          // element q of a thread: part row r0 + 32 q, column c
    const long long col = (long long)blockIdx.x * kCols + c;
    const int nchunks = (nparts + kRows - 1) / kRows;
    T v[kPerThread];
    auto load = [&](int chunk) {
#pragma unroll
        for (int q = 0; q < kPerThread; ++q) {
            const int j = chunk * kRows + r0 + (256 / kCols) * q;
            v[q] = (j < nparts && col < n) ? part[(size_t)j * n + col] : T(0);
        }
    };
    auto stage = [&](int buf) {
#pragma unroll
        for (int q = 0; q < kPerThread; ++q) tile[buf][r0 + (256 / kCols) * q][c] = v[q];
    };
    load(0);
    stage(0);
    __syncthreads();
    T s = T(0);
    for (int k = 0; k < nchunks; ++k) {
        if (k + 1 < nchunks) load(k + 1);
        if (threadIdx.x < kCols) {
            const int rows = nparts - k * kRows < kRows ? nparts - k * kRows : kRows;
            int r = 0;
            if (k == 0) { s = tile[0][0][threadIdx.x]; r = 1; }
#pragma unroll 8
            for (; r < rows; ++r) s += tile[k & 1][r][threadIdx.x];
        }
        if (k + 1 < nchunks) stage((k + 1) & 1);
        __syncthreads();
    }
    if (threadIdx.x < kCols && col < n) out[col] += s;
}

__device__ __forceinline__ unsigned long long gtimer() {     // nanosecond timer common to all SMs
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ unsigned long long warp_sum(unsigned long long v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ int warp_sum(int v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Column sums of a 32(lanes) x 32(values) tile held one row per lane: after the call lane l returns sum_over_lanes v[l].
// Butterfly that halves the live values per stage: 31 shuffles instead of 32 x 5.
__device__ __forceinline__ float warp_transpose_sum32(float (&v)[32], int lane) {
#define RLR_TSTAGE(O, N)                                                         \
    {                                                                            \
        const bool up = (lane & (O)) != 0;                                       \
        _Pragma("unroll") for (int i = 0; i < (N); ++i) {                        \
            const float send = up ? v[i] : v[i + (N)];                           \
            const float keep = up ? v[i + (N)] : v[i];                           \
            v[i] = keep + __shfl_xor_sync(0xffffffffu, send, (O));               \
        }                                                                        \
    }
    RLR_TSTAGE(16, 16) RLR_TSTAGE(8, 8) RLR_TSTAGE(4, 4) RLR_TSTAGE(2, 2) RLR_TSTAGE(1, 1)
#undef RLR_TSTAGE
    return v[0];
}

// Block-wide sum; result valid in thread 0. `scratch` must hold >= 32 elements.
template <typename T>
__device__ __forceinline__ T block_sum(T v, T* scratch) {
    v = warp_sum(v);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (lane == 0) scratch[wid] = v;
    __syncthreads();
    const int nw = (blockDim.x + 31) >> 5;
    v = (threadIdx.x < nw) ? scratch[threadIdx.x] : T(0);
    if (wid == 0) v = warp_sum(v);
    __syncthreads();
    return v;
}

// ---- streaming 128-bit global accesses (read-once / write-once data) --------------------------------
__device__ __forceinline__ float4 ld_stream_f4(const float* p) {
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}
// Peer (NVLink) / freshly written data: plain relaxed load, never the non-coherent path.
__device__ __forceinline__ float4 ld_f4(const float* p) {
    float4 r;
    asm volatile("ld.global.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ float ld_f1(const float* p) {
    float r;
    asm volatile("ld.global.f32 %0, [%1];" : "=f"(r) : "l"(p));
    return r;
}
__device__ __forceinline__ void st_f4(float* p, float4 v) {
    asm volatile("st.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
// NVLS multicast store: one store lands in every GPU bound to the multicast object.
__device__ __forceinline__ void multimem_st_f4(float* mc, float4 v) {
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc), "f"(v.x), "f"(v.y),
                 "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ void multimem_st_b2(uint2* mc, uint2 v) {  // 4 packed bf16
    asm volatile("multimem.st.relaxed.sys.global.v2.f32 [%0], {%1,%2};" ::"l"(mc), "f"(__uint_as_float(v.x)),
                 "f"(__uint_as_float(v.y)) : "memory");
}

// ---- cross-GPU flags (system scope) ------------------------------------------------------------------
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_gpu(uint32_t* p, uint32_t v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_gpu(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

// Cross-GPU barrier executed by the first `world` threads of ONE block (barrier_in below, the aggregate kernel's barrier-out).
__device__ __forceinline__ void xgpu_barrier(uint32_t* const* flag_ptrs, int slot_base, int rank, int world, uint32_t epoch) {
    const int t = threadIdx.x;
    if (t < world) {
        st_release_sys(flag_ptrs[t] + slot_base + rank, epoch);           // tell peer t "rank is here"
        const uint32_t* mine = flag_ptrs[rank] + slot_base + t;           // wait for peer t
        while ((int32_t)(ld_acquire_sys(mine) - epoch) < 0) { __nanosleep(64); }
    }
}

// Barrier-in of the server step's passes (aggregate, distances, trust statistics) on the fused multi-GPU path: every rank's participant
// slots are final before any peer slot is read.  Every thread calls it.  The `leader` CTA runs the cross-GPU barrier and then releases
// the other CTAs of this GPU through the ready flag, so every CTA of the grid has to be resident (the launchers cap their grids).
__device__ __forceinline__ void barrier_in(const Gate& g, bool leader) {
    if (g.world > 1) {
        if (leader) {
            xgpu_barrier(g.flag_ptrs, 0, g.rank, g.world, g.epoch);
            __syncthreads();
            if (threadIdx.x == 0) st_release_gpu(g.local_sync, g.epoch);
        } else if (threadIdx.x == 0) {
            while ((int32_t)(ld_acquire_gpu(g.local_sync) - g.epoch) < 0) { __nanosleep(32); }
        }
    }
    __syncthreads();
}
// Host check of a launch's gate: the multi-GPU form needs the flag words and the intra-GPU sync words.
inline bool gate_ok(const Gate& g) { return g.world <= 1 || (g.flag_ptrs && g.local_sync); }

// Coordinate splits of a participant pass: about two waves of CTAs, one wave when world > 1 (every CTA has to be resident while the
// leader waits in barrier_in), at least 4096 coordinates per split, at most `max_splits` (a workspace bound), and at least one.
inline long long coord_splits(long long len, long long ctas_per_split, long long resident, int world,
                              long long max_splits = 1LL << 62) {
    long long splits = (world > 1 ? resident : 2 * resident) / ctas_per_split;
    splits = splits < len / 4096 ? splits : len / 4096;
    splits = splits < max_splits ? splits : max_splits;
    return splits < 1 ? 1 : splits;
}

// ---- Philox4x32-10 counter RNG (Salmon et al.), used for dropout masks and server noise ---------------
struct Philox {
    uint32_t k0, k1;
    __device__ __forceinline__ Philox(uint64_t seed) : k0((uint32_t)seed), k1((uint32_t)(seed >> 32)) {}
    __device__ __forceinline__ uint4 operator()(uint64_t ctr, uint64_t stream) const {
        uint32_t c0 = (uint32_t)ctr, c1 = (uint32_t)(ctr >> 32), c2 = (uint32_t)stream, c3 = (uint32_t)(stream >> 32);
        uint32_t a = k0, b = k1;
#pragma unroll
        for (int r = 0; r < 10; ++r) {
            const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
            const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
            const uint32_t n0 = hi1 ^ c1 ^ a, n2 = hi0 ^ c3 ^ b;
            c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
            a += 0x9E3779B9u; b += 0xBB67AE85u;
        }
        return make_uint4(c0, c1, c2, c3);
    }
};
__device__ __forceinline__ float u32_to_unit(uint32_t x) {  // (0,1]
    return ((float)(x >> 8) + 1.0f) * (1.0f / 16777216.0f);
}
__device__ __forceinline__ float4 philox_normal4(const Philox& ph, uint64_t ctr, uint64_t stream) {
    const uint4 u = ph(ctr, stream);
    const float r0 = sqrtf(-2.0f * logf(u32_to_unit(u.x))), r1 = sqrtf(-2.0f * logf(u32_to_unit(u.z)));
    float s0, c0, s1, c1;
    sincospif(2.0f * u32_to_unit(u.y), &s0, &c0);
    sincospif(2.0f * u32_to_unit(u.w), &s1, &c1);
    return make_float4(r0 * c0, r0 * s0, r1 * c1, r1 * s1);
}

// ---- training augmentation (RandomCrop(padding = pad, fill 0) + RandomHorizontalFlip) ----------------------------------------------
// The sample at position p of an agent's epoch order (cursor + b, not its dataset index) draws u = Philox(seed)(p, *stream), where
// *stream is a device word the trainer sets once per epoch (ops.augment_stream).  Augmented pixel (h, w) reads stored pixel
// (h + oy - pad, w' + ox - pad), w' = W-1-w when flipped, and stored value 0 outside the image.  ops.philox4x32 is the host twin.
struct AugSpec {
    const long long* stream;
    unsigned long long seed;
    long long start;                 // position of batch row 0 when no cursor is given
    int pad, flip;
};
struct AugDraw { int oy, ox, flip; };
__device__ __forceinline__ AugDraw augment_draw(const AugSpec& a, long long pos) {
    const uint4 u = Philox(a.seed)((uint64_t)pos, (uint64_t)*a.stream);
    const uint32_t n = 2u * (uint32_t)a.pad + 1u;
    return {(int)(u.x % n), (int)(u.y % n), a.flip ? (int)(u.z & 1u) : 0};
}

// ---- fused dropout --------------------------------------------------------------------------------------------------------------
// Keep-mask of a tensor viewed as a flat array of elements: the 8 elements [8 q, 8 q + 8) share ONE Philox4x32-10 call keyed by
// (seed; counter q, stream = (step << 20) ^ node), 16 random bits per element, keep iff bits >= p * 65536.  Every kernel that produces
// or back-propagates through a dropped tensor (maxpool / GEMM epilogues, their backward kernels, the stand-alone dropout kernels)
// evaluates THIS function, so no mask tensor is ever written.  Reference: nn.Dropout2d(p=.5) on 2-D activations (src/models.py:17-19,
// 40-44) = element-wise dropout; bit-parity with torch's Philox stream is not a goal (SURVEY.md 4), mask statistics are tested.
__device__ __forceinline__ uint32_t dropout_keep8(const DropSpec& d, long long q) {     // bit i = element 8 q + i is kept
    const Philox ph(d.seed);
    const uint4 u = ph((uint64_t)q, ((uint64_t)(*d.step) << 20) ^ d.stream);
    const uint32_t r[4] = {u.x, u.y, u.z, u.w};
    uint32_t keep = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) keep |= (uint32_t)(((r[i >> 1] >> (16 * (i & 1))) & 0xffffu) >= d.thr) << i;
    return keep;
}

template <typename T>
inline cudaError_t launch_ordered_sum(T* out, const T* part, int nparts, long long n, cudaStream_t st) {
    if (nparts >= 16 && n <= 2048)
        return launch_kernel(ordered_sum_narrow_kernel<T>, dim3((unsigned)((n + 7) / 8)), dim3(256), (size_t)0, st, out, part, nparts, n);
    if (nparts >= 16)
        return launch_kernel(ordered_sum_cols_kernel<T>, dim3((unsigned)((n + 31) / 32)), dim3(256), (size_t)0, st, out, part, nparts, n);
    long long blocks = (n + 255) / 256;
    if (blocks > 1024) blocks = 1024;
    if (blocks < 1) blocks = 1;
    return launch_kernel(ordered_sum_kernel<T>, dim3((unsigned)blocks), dim3(256), (size_t)0, st, out, part, nparts, n);
}

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
    __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
}

}  // namespace rlr
