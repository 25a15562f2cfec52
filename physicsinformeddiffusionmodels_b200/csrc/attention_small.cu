// Linear attention (reference unet_model.py:286-297) for the LOW-RESOLUTION levels of the U-Net (N = H*W <= 256
// tokens: the 16x16 and 8x8 levels), bf16 activations, dim_head = 32:  ONE kernel per direction, one CTA per
// (sample, head), everything in shared memory.
//
//   k~[n,d] = exp(k[n,d] - M_d) / Z_d            (softmax over the N tokens, per column d)
//   p[n,d]  = softmax_d(q[n,:])[d] * s            (softmax over the 32 channels, per token; s = 32^-0.5)
//   ctx[d][e] = sum_n k~[n,d] v[n,e] / N ;   out[n,e] = sum_d p[n,d] ctx[d][e]
//
// Why: at these sizes a (sample, head) problem is 64..256 tokens x 96 channels = 12..48 KB, and the streaming
// formulation (column statistics -> context -> output, and dcontext -> per-token gradients for the backward: 3 + 2
// dependent kernels plus two memsets, each a grid-wide pass) is pure launch / dependency latency for 6..25 MB of
// traffic.  Here the whole chain runs inside one CTA on
// CUDA cores (the products are 32-wide: 2 MFLOP per CTA), 256 CTAs = one wave.
// (A one-CTA backward was built and measured too: no faster than the streaming backward at 64 tokens, slower at 256.)
#include "common.cuh"
#include "pidm.h"

namespace pidm {

constexpr int LS_D = 32;            // dim_head
constexpr int LS_PITCH = LS_D + 1;  // fp32 row pitch: a thread that owns a token walks its row without bank conflicts
constexpr int LS_BPITCH = LS_D + 2;  // bf16 row pitch of the read-only planes (v, dout): 17 words, odd -> conflict-free rows
constexpr int LS_THREADS = 256;
constexpr int LS_MAXN = 256;       // kernels are written for N <= 256; the dispatcher only routes N <= 64 here (see below)

// dynamic shared memory layout: fp32 planes [N][LS_PITCH] for the operands that are transformed in place (q -> p,
// k -> k~), bf16 planes [N][LS_BPITCH] for the read-only ones (v, dout: they ARE bf16, nothing is lost), small vectors
struct LsLayout {
    int plane;        // floats per fp32 plane
    int bplane;       // floats (4-byte units) per bf16 plane
    __host__ __device__ explicit LsLayout(int N) : plane(N * LS_PITCH), bplane((N * LS_BPITCH + 1) / 2) {}
};

// load one [N][32] head slice (row stride `stride` elements) into an fp32 plane
__device__ __forceinline__ void ls_load_plane(float* dst, const __nv_bfloat16* __restrict__ src, size_t stride, int N) {
    for (int i = threadIdx.x; i < N * 4; i += blockDim.x) {          // 4 x 16-byte vectors per row
        const int n = i >> 2, o = i & 3;
        float v[8];
        ld8(src + (size_t)n * stride + o * 8, v);
#pragma unroll
        for (int k = 0; k < 8; ++k) dst[n * LS_PITCH + o * 8 + k] = v[k];
    }
}

// same, raw bf16 copy (4-byte units: the 68-byte rows are only 4-byte aligned)
__device__ __forceinline__ void ls_load_bplane(__nv_bfloat16* dst, const __nv_bfloat16* __restrict__ src, size_t stride, int N) {
    for (int i = threadIdx.x; i < N * 4; i += blockDim.x) {
        const int n = i >> 2, o = i & 3;
        const uint4 t = *reinterpret_cast<const uint4*>(src + (size_t)n * stride + o * 8);
        uint32_t* d = reinterpret_cast<uint32_t*>(dst + n * LS_BPITCH + o * 8);
        d[0] = t.x; d[1] = t.y; d[2] = t.z; d[3] = t.w;
    }
}
__device__ __forceinline__ float2 ls_b2(const __nv_bfloat16* p) {          // two consecutive bf16 (4-byte aligned)
    return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p));
}

// column softmax over the tokens, in place: plane[n][d] <- exp(plane[n][d] - M_d) / Z_d.  red: [8][32] scratch.
// Returns nothing; M_d and 1/Z_d are left in colM / colZi (shared, [32]).
__device__ __forceinline__ void ls_col_softmax(float* plane, float* red, float* colM, float* colZi, int N) {
    const int d = threadIdx.x & 31, seg = threadIdx.x >> 5;          // 8 segments of tokens per column
    float m = -INFINITY;
    for (int n = seg; n < N; n += 8) m = fmaxf(m, plane[n * LS_PITCH + d]);
    red[seg * 32 + d] = m;
    __syncthreads();
    if (threadIdx.x < 32) {
        float mm = red[d];
#pragma unroll
        for (int s = 1; s < 8; ++s) mm = fmaxf(mm, red[s * 32 + d]);
        colM[d] = mm;
    }
    __syncthreads();
    const float M = colM[d];
    float z = 0.f;
    for (int n = seg; n < N; n += 8) {
        const float e = __expf(plane[n * LS_PITCH + d] - M);
        plane[n * LS_PITCH + d] = e;
        z += e;
    }
    __syncthreads();                                                 // all reads of red (max) are done
    red[seg * 32 + d] = z;
    __syncthreads();
    if (threadIdx.x < 32) {
        float zz = 0.f;
#pragma unroll
        for (int s = 0; s < 8; ++s) zz += red[s * 32 + d];
        colZi[d] = 1.f / zz;
    }
    __syncthreads();
    const float zi = colZi[d];
    for (int n = seg; n < N; n += 8) plane[n * LS_PITCH + d] *= zi;
    __syncthreads();
}

// row softmax over the 32 channels, in place (no scale): one thread per token
__device__ __forceinline__ void ls_row_softmax(float* plane, int N) {
    for (int n = threadIdx.x; n < N; n += blockDim.x) {
        float* r = plane + n * LS_PITCH;
        float m = -INFINITY;
#pragma unroll
        for (int d = 0; d < LS_D; ++d) m = fmaxf(m, r[d]);
        float s = 0.f;
#pragma unroll
        for (int d = 0; d < LS_D; ++d) { const float e = __expf(r[d] - m); r[d] = e; s += e; }
        const float inv = 1.f / s;
#pragma unroll
        for (int d = 0; d < LS_D; ++d) r[d] *= inv;
    }
}

// C[d][e] = mul * sum_n A[n][d] * Bm[n][e]   (32 x 32 outputs; thread t owns d = t / 8 and the 4 columns (t % 8) * 4 ...)
__device__ __forceinline__ void ls_outer_sum(float* C, const float* A, const __nv_bfloat16* Bm, int N, float mul) {
    const int d = threadIdx.x >> 3, e0 = (threadIdx.x & 7) * 4;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll 4
    for (int n = 0; n < N; ++n) {
        const float a = A[n * LS_PITCH + d];
        const float2 b01 = ls_b2(Bm + n * LS_BPITCH + e0), b23 = ls_b2(Bm + n * LS_BPITCH + e0 + 2);
        a0 += a * b01.x; a1 += a * b01.y; a2 += a * b23.x; a3 += a * b23.y;
    }
    C[d * LS_D + e0] = a0 * mul; C[d * LS_D + e0 + 1] = a1 * mul; C[d * LS_D + e0 + 2] = a2 * mul; C[d * LS_D + e0 + 3] = a3 * mul;
}

// ---- forward -------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(LS_THREADS) la_small_fwd_kernel(const __nv_bfloat16* __restrict__ qkv,
                                                                  __nv_bfloat16* __restrict__ out, float* __restrict__ ctx_out,
                                                                  float* __restrict__ kmax, float* __restrict__ kzinv,
                                                                  int N, int heads, float scale) {
    pdl_trigger();
    pdl_wait();
    extern __shared__ __align__(16) float sm[];
    const LsLayout L(N);
    float* Q = sm;
    float* K = Q + L.plane;
    float* ctx = K + L.plane;                  // [32][32]
    float* red = ctx + LS_D * LS_D;            // [8][32]
    float* colM = red + 8 * 32;
    float* colZi = colM + 32;
    __nv_bfloat16* V = reinterpret_cast<__nv_bfloat16*>(colZi + 32);
    const int h = blockIdx.x, b = blockIdx.y, HID = heads * LS_D;
    const size_t stride = 3 * (size_t)HID;
    const __nv_bfloat16* base = qkv + (size_t)b * N * stride + h * LS_D;
    ls_load_plane(Q, base, stride, N);
    ls_load_plane(K, base + HID, stride, N);
    ls_load_bplane(V, base + 2 * HID, stride, N);
    __syncthreads();
    ls_col_softmax(K, red, colM, colZi, N);                        // K <- k~
    ls_outer_sum(ctx, K, V, N, 1.f / (float)N);                    // ctx = k~^T (v / N)
    ls_row_softmax(Q, N);                                          // Q <- softmax_d(q)
    __syncthreads();
    for (int i = threadIdx.x; i < LS_D * LS_D; i += blockDim.x) ctx_out[((size_t)b * heads + h) * LS_D * LS_D + i] = ctx[i];
    if (threadIdx.x < 32) {
        kmax[(size_t)b * HID + h * LS_D + threadIdx.x] = colM[threadIdx.x];
        kzinv[(size_t)b * HID + h * LS_D + threadIdx.x] = colZi[threadIdx.x];
    }
    // out[n][e] = s * sum_d p[n][d] ctx[d][e]: thread = (token, 8-column octet)
    for (int w = threadIdx.x; w < N * 4; w += blockDim.x) {
        const int n = w >> 2, e0 = (w & 3) * 8;
        const float* p = Q + n * LS_PITCH;
        float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int d = 0; d < LS_D; ++d) {
            const float pv = p[d];
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[k] += pv * ctx[d * LS_D + e0 + k];
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] *= scale;
        st8(out + ((size_t)b * N + n) * HID + h * LS_D + e0, acc);
    }
}

static size_t ls_smem(int N, bool bwd) {
    const LsLayout L(N);
    return (size_t)(2 * L.plane + (bwd ? 2 : 1) * LS_D * LS_D + 8 * 32 + 3 * 32 + (bwd ? 2 : 1) * L.bplane) * sizeof(float);
}

// entry points used by attention.cu
// At 256 tokens the 32-wide products (0.7 GFLOP per layer) are CUDA-core FLOP-bound here while the streaming kernels
// run them on mma.sync, so only the 8x8 level takes this path, and only where it wins (forward).
bool la_small_supported(int N, int dtype) { return dtype == PIDM_BF16 && N >= 32 && N <= 64; }

int la_small_fwd(const void* qkv, void* out, float* ctx, float* kmax, float* kzinv, int B, int N, int heads, float scale,
                 cudaStream_t st) {
    PIDM_CUDA(allow_smem(la_small_fwd_kernel, ls_smem(LS_MAXN, false)));
    PIDM_CUDA(launch_plain(la_small_fwd_kernel, dim3(heads, B), dim3(LS_THREADS), ls_smem(N, false), st, (const __nv_bfloat16*)qkv,
                           (__nv_bfloat16*)out, ctx, kmax, kzinv, N, heads, scale));
    PIDM_LAUNCH_CHECK("la_small_fwd");
    return 0;
}

}  // namespace pidm
