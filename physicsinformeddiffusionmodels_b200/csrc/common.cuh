// Shared device/host helpers for libpidm (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#define PIDM_F32 0
#define PIDM_BF16 1

namespace pidm {

// ---- error plumbing (thread-local last-error string, returned through pidm_last_error) ----------
extern thread_local char g_last_error[512];
int set_error(int code, const char* fmt, ...);

#define PIDM_REQUIRE(cond, ...)                                   \
    do {                                                          \
        if (!(cond)) return ::pidm::set_error(2, __VA_ARGS__);    \
    } while (0)

#define PIDM_LAUNCH_CHECK(name)                                                              \
    do {                                                                                     \
        cudaError_t e__ = cudaGetLastError();                                                \
        if (e__ != cudaSuccess)                                                              \
            return ::pidm::set_error(3, "%s: launch failed: %s", name, cudaGetErrorString(e__)); \
    } while (0)

#define PIDM_CUDA(call)                                                                      \
    do {                                                                                     \
        cudaError_t e__ = (call);                                                            \
        if (e__ != cudaSuccess)                                                              \
            return ::pidm::set_error(4, "%s: %s", #call, cudaGetErrorString(e__));           \
    } while (0)

// ---- scalar type traits -------------------------------------------------------------------------
template <typename T> struct Act;
template <> struct Act<float> {
    static __device__ __forceinline__ float ld(const float* p) { return *p; }
    static __device__ __forceinline__ void st(float* p, float v) { *p = v; }
};
template <> struct Act<__nv_bfloat16> {
    static __device__ __forceinline__ float ld(const __nv_bfloat16* p) { return __bfloat162float(*p); }
    static __device__ __forceinline__ void st(__nv_bfloat16* p, float v) { *p = __float2bfloat16_rn(v); }
};

// 4-wide vector load/store of activations (p must be 4-element aligned)
__device__ __forceinline__ void ld4(const float* p, float v[4]) {
    float4 t = *reinterpret_cast<const float4*>(p);
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
}
__device__ __forceinline__ void ld4(const __nv_bfloat16* p, float v[4]) {
    uint2 t = *reinterpret_cast<const uint2*>(p);
    __nv_bfloat162 a = *reinterpret_cast<__nv_bfloat162*>(&t.x);
    __nv_bfloat162 b = *reinterpret_cast<__nv_bfloat162*>(&t.y);
    v[0] = __low2float(a); v[1] = __high2float(a); v[2] = __low2float(b); v[3] = __high2float(b);
}
__device__ __forceinline__ void st4(float* p, const float v[4]) {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
}
__device__ __forceinline__ void st4(__nv_bfloat16* p, const float v[4]) {
    __nv_bfloat162 a = __floats2bfloat162_rn(v[0], v[1]);
    __nv_bfloat162 b = __floats2bfloat162_rn(v[2], v[3]);
    uint2 t;
    t.x = *reinterpret_cast<uint32_t*>(&a);
    t.y = *reinterpret_cast<uint32_t*>(&b);
    *reinterpret_cast<uint2*>(p) = t;
}
// 8-wide
__device__ __forceinline__ void ld8(const float* p, float v[8]) { ld4(p, v); ld4(p + 4, v + 4); }
__device__ __forceinline__ void ld8(const __nv_bfloat16* p, float v[8]) {
    uint4 t = *reinterpret_cast<const uint4*>(p);
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&t);
#pragma unroll
    for (int i = 0; i < 4; ++i) { v[2 * i] = __low2float(h[i]); v[2 * i + 1] = __high2float(h[i]); }
}
__device__ __forceinline__ void st8(float* p, const float v[8]) { st4(p, v); st4(p + 4, v + 4); }
__device__ __forceinline__ void st8(__nv_bfloat16* p, const float v[8]) {
    uint4 t;
    __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&t);
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
    *reinterpret_cast<uint4*>(p) = t;
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

// Threads are laid out as (row = tid / oct, octet = tid % oct).  When oct is a power of two < 32, lanes that own
// the same channel octet sit `oct` apart inside a warp: sum them by shuffles so that only the first `oct` lanes of
// each warp touch shared-memory atomics (cuts same-address ATOMS traffic by 32/oct).  Returns true for the lanes
// that must publish their (now warp-reduced) values.
template <int NV>
__device__ __forceinline__ bool reduce_same_octet(float (&v)[NV], int oct) {
    if (oct >= 32 || (oct & (oct - 1)) != 0) return true;
    for (int off = oct; off < 32; off <<= 1) {
#pragma unroll
        for (int k = 0; k < NV; ++k) v[k] += __shfl_xor_sync(0xffffffffu, v[k], off);
    }
    return (threadIdx.x & 31) < oct;
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarriers (TMA completion in the tensor-core kernels and the Darcy sample staging) ----------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
// make the initialised barriers visible to the async proxy (TMA) before any copy completes on them
__device__ __forceinline__ void mbar_init_fence() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
    } while (!ok);
}

__device__ __forceinline__ float silu_f(float z) { return z / (1.f + __expf(-z)); }
__device__ __forceinline__ float silu_grad_f(float z) {
    float s = 1.f / (1.f + __expf(-z));
    return s * (1.f + z * (1.f - s));
}
// GELU, exact erf form (nn.GELU()); each translation unit compiles it under its own arithmetic flags
__device__ __forceinline__ float gelu_erf_f(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }
__device__ __forceinline__ float gelu_erf_grad_f(float x) {
    return 0.5f * (1.f + erff(x * 0.70710678118654752f)) + x * 0.3989422804014327f * expf(-0.5f * x * x);
}

static inline int ceil_div(long long a, long long b) { return (int)((a + b - 1) / b); }

// streaming multiprocessors of the current device (queried once; sizes persistent grids and one-wave splits)
int num_sms();

// Opt a kernel into `bytes` of dynamic shared memory (needed above 48 KB).  The attribute is set only when `bytes`
// exceeds what was last set for that kernel, so a call before every launch costs a lookup; safe from several host
// threads (the autograd worker and the main thread) at once.
cudaError_t allow_smem(const void* kernel, size_t bytes);
template <typename... KArgs>
static inline cudaError_t allow_smem(void (*kernel)(KArgs...), size_t bytes) {
    return allow_smem((const void*)kernel, bytes);
}

// ---- programmatic dependent launch (PDL) -----------------------------------------------------------------------
// The step is a chain of ~420 dependent kernels, many of them a few microseconds long: the kernel-to-kernel launch
// latency is a first-order cost.  Kernels launched through launch_pdl() may start while their predecessor is still
// draining: they run their prologue (barrier init, tensor-map prefetch, parameter loads that do not
// depend on the predecessor) and then block in pdl_wait() until the predecessor grid has completed and flushed.
// Every kernel calls pdl_trigger() first so that ITS successor can be scheduled as early as possible.  Both
// instructions are no-ops for kernels launched without the attribute.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// Only the prologue-heavy persistent kernels (convolutions, weight gradients, normalisations) are launched with the
// attribute.  The attention, element-wise, linear, optimizer and residual kernels go through launch_plain(): a kernel
// whose first instruction is the wait gains nothing, and its early-scheduled CTAs only take SM slots from the forked
// weight-gradient stream.
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                     Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

template <typename... KArgs, typename... Args>
static inline cudaError_t launch_plain(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                       Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

// dispatch on activation dtype code
#define PIDM_DISPATCH_DTYPE(dtype, ...)                                       \
    do {                                                                      \
        if ((dtype) == PIDM_F32) { using T = float; __VA_ARGS__; }            \
        else if ((dtype) == PIDM_BF16) { using T = __nv_bfloat16; __VA_ARGS__; } \
        else return ::pidm::set_error(2, "unknown dtype code %d", (int)(dtype)); \
    } while (0)

}  // namespace pidm
