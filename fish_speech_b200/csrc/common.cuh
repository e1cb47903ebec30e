// fishb200 — common device/host helpers for the sm_90a kernels.
// Everything here is written for H100 (Hopper) only (compile with
// -gencode arch=compute_90a,code=sm_90a); there is no other backend.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

namespace fsb {

// ---------------------------------------------------------------------------------------------
// Error plumbing. Every C-ABI entry point returns 0 on success; the message of the last failure
// on this host thread is kept for fsb_last_error().
// ---------------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
const char* get_error();
extern thread_local int g_launch_count;  // kernels launched by this thread (bench: gpu_launches)

#define FSB_CUDA(expr)                                                                            \
    do {                                                                                          \
        cudaError_t _e = (expr);                                                                  \
        if (_e != cudaSuccess) {                                                                  \
            ::fsb::set_error("%s:%d: %s failed: %s", __FILE__, __LINE__, #expr,                   \
                             cudaGetErrorString(_e));                                             \
            return 1;                                                                             \
        }                                                                                         \
    } while (0)

#define FSB_CHECK(cond, ...)                                                                      \
    do {                                                                                          \
        if (!(cond)) {                                                                            \
            ::fsb::set_error(__VA_ARGS__);                                                        \
            return 1;                                                                             \
        }                                                                                         \
    } while (0)

#define FSB_TRY(expr)                                                                             \
    do {                                                                                          \
        int _r = (expr);                                                                          \
        if (_r != 0) return _r;                                                                   \
    } while (0)

// Launch-check: catches bad configurations at the call site (works during stream capture too).
#define FSB_LAUNCH_CHECK()                                                                        \
    do {                                                                                          \
        ::fsb::g_launch_count++;                                                                  \
        FSB_CUDA(cudaGetLastError());                                                             \
    } while (0)

// Launch with the programmatic-stream-serialization attribute (PDL): the kernel may start while its
// predecessor in the stream is still running; every kernel launched this way executes
// griddepcontrol.wait before it touches anything a predecessor produces (or still reads).
template <typename... Args>
static inline cudaError_t launch_pdl(const void* kernel, dim3 grid, dim3 block, size_t smem,
                                     cudaStream_t st, Args... args) {
    void* kargs[] = {reinterpret_cast<void*>(&args)...};
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelExC(&cfg, kernel, kargs);
}
#define FSB_LAUNCH(kernel, grid, block, smem, st, ...)                                            \
    do {                                                                                          \
        ::fsb::g_launch_count++;                                                                  \
        FSB_CUDA(::fsb::launch_pdl(reinterpret_cast<const void*>(kernel), grid, block, smem, st,  \
                                   __VA_ARGS__));                                                 \
    } while (0)

static inline int cdiv(int a, int b) { return (a + b - 1) / b; }
static inline long long cdivll(long long a, long long b) { return (a + b - 1) / b; }

#ifdef __CUDACC__
// ---------------------------------------------------------------------------------------------
// bf16 helpers. The reference keeps activations in bf16 between ops (every nn.Linear / norm /
// elementwise result is rounded to bf16); the kernels reproduce those rounding points with rbf().
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float bf2f(__nv_bfloat16 v) { return __bfloat162float(v); }
__device__ __forceinline__ __nv_bfloat16 f2bf(float v) { return __float2bfloat16_rn(v); }
// round an fp32 value to the nearest bf16 and return it as fp32
__device__ __forceinline__ float rbf(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }

__device__ __forceinline__ float bf_lo(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float bf_hi(uint32_t w) { return __uint_as_float(w & 0xffff0000u); }
__device__ __forceinline__ uint32_t pack_bf2(float lo, float hi) {
    __nv_bfloat162 p = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&p);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// Block-wide sum for blockDim.x <= 1024; `red` is a __shared__ float[33]. All threads get the sum.
__device__ __forceinline__ float block_sum(float v, float* red) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    v = warp_sum(v);
    __syncthreads();
    if (lane == 0) red[w] = v;
    __syncthreads();
    if (w == 0) {
        float t = lane < nw ? red[lane] : 0.f;
        t = warp_sum(t);
        if (lane == 0) red[32] = t;
    }
    __syncthreads();
    return red[32];
}
__device__ __forceinline__ float block_max(float v, float* red) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    v = warp_max(v);
    __syncthreads();
    if (lane == 0) red[w] = v;
    __syncthreads();
    if (w == 0) {
        float t = lane < nw ? red[lane] : -INFINITY;
        t = warp_max(t);
        if (lane == 0) red[32] = t;
    }
    __syncthreads();
    return red[32];
}

// ---------------------------------------------------------------------------------------------
// PTX wrappers: mbarrier, TMA (cp.async.bulk.tensor).  The wgmma wrappers are in wgmma.cuh.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ bool elect_one() {
    uint32_t pred = 0;
    asm volatile(
        "{\n\t.reg .pred P;\n\telect.sync _|P, 0xffffffff;\n\tselp.b32 %0, 1, 0, P;\n\t}\n"
        : "=r"(pred));
    return pred != 0;
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred P;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, P;\n\t}\n"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded wait: a protocol bug becomes a trap (launch failure) instead of a hung GPU box.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    // ~2 s at ~2 GHz: a lost arrival or TMA completion traps instead of hanging. No printf here: a function call
    // between wgmma issue and wgmma wait makes ptxas serialize every wgmma of the kernel (warning C7510).
    while (!mbar_try_wait(bar, parity))
        if (clock64() - t0 > 4000000000ll) __trap();
}

constexpr uint64_t kEvictNormal = 0x1000000000000000ull;
constexpr uint64_t kEvictFirst = 0x12F0000000000000ull;
constexpr uint64_t kEvictLast = 0x14F0000000000000ull;

__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
// 3-D tiled TMA load global -> shared, completion on an mbarrier, with an L2 eviction hint.
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const void* tmap, uint32_t bar, int c0,
                                            int c1, int c2, uint64_t hint) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
        ".L2::cache_hint [%0], [%1, {%3, %4, %5}], [%2], %6;"
        ::"r"(dst), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(bar), "r"(c0), "r"(c1), "r"(c2),
        "l"(hint)
        : "memory");
}

// TMA store of a {64, rows, 1} box from shared memory (SWIZZLE_128B tile) to global memory; rows / columns outside
// the tensor are clipped.  Part of the calling thread's current bulk async-group.
__device__ __forceinline__ void tma_store_3d(const void* tmap, uint32_t src, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
                 ::"l"(reinterpret_cast<uint64_t>(tmap)), "r"(src), "r"(c0), "r"(c1), "r"(c2)
                 : "memory");
}
// Prefetch of the line at `p` into L2 only.
__device__ __forceinline__ void prefetch_l2(const void* p) {
    asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
}

// Programmatic dependent launch: wait for the producing grid / allow the dependent grid to start.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() {
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
#endif  // __CUDACC__

}  // namespace fsb
