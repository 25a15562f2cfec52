// Linear attention of the U-Net (SpatialLinearAttention core, reference unet_model.py:286-297) on NHWC activations,
// dim_head = 32: pidm_linattn_fwd / _bwd / _plan and the three paths they choose between.  qkv[B, N, 3*HID],
// HID = heads*32, channel = which*HID + head*32 + d:
//         q~ = softmax_d(q) * 32^-1/2 ;  k~ = softmax_n(k) ;  v~ = v / N
//         ctx[b,h,d,e] = sum_n k~[n,d] v~[n,e] ;   out[n, h*32+e] = sum_d ctx[d,e] q~[n,d]
// The k-softmax is a reduction over all N pixels: pass 1 computes per-chunk (max, sum-exp) per column, pass 2 merges
// them and accumulates the 32x32 context per (sample, head), pass 3 applies it per pixel.  Backward uses the identity
//         sum_n k~[n,d] dk~[n,d] = sum_e dctx[d,e] ctx[d,e]
// so no extra pass over N is needed for the k-softmax Jacobian.
//   (1) SIMT: the three passes on CUDA cores, fp32 math, any head count and either activation type;
//   (2) one CTA per (sample, head) for the 8x8 level's forward;
//   (3) mma.sync: passes 2 and 3 and the backward on the tensor cores for bf16 activations and 8 heads.
#include "common.cuh"
#include "mma_util.cuh"
#include "pidm.h"

namespace pidm {

// ==== (1) SIMT =======================================================================================================
constexpr int LA_TN = 64;         // pixel tile of the context kernels

// ---- pass 1: per-chunk column statistics of k -----------------------------------------------------------
// part[b][chunk][c] = (max_n k[n,c], sum_n exp(k[n,c] - max)) over the rows of the chunk.  Thread = (row group,
// channel octet): 16-byte loads, a max pass and an exp-sum pass (the chunk stays in L1/L2 between them) instead of
// the serial online-softmax recurrence per row; the row groups are combined through shared memory.
template <typename T>
__global__ void la_kstats_kernel(const T* __restrict__ qkv, float* __restrict__ part /*[B][chunks][HID][2]*/, int N,
                                 int HID, int rows_per_chunk) {
    pdl_trigger();
    pdl_wait();
    extern __shared__ float skm[];                 // [groups][HID] max, then [groups][HID] sums
    const int b = blockIdx.y, chunk = blockIdx.x;
    const int oct = HID / 8;
    const int o = threadIdx.x % oct, rg = threadIdx.x / oct, groups = blockDim.x / oct;
    const int n0 = chunk * rows_per_chunk;
    int n1 = n0 + rows_per_chunk;
    if (n1 > N) n1 = N;
    const T* base = qkv + ((size_t)b * N) * 3 * HID + HID + o * 8;
    float m[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) m[k] = -INFINITY;
    for (int n = n0 + rg; n < n1; n += groups) {
        float v[8];
        ld8(base + (size_t)n * 3 * HID, v);
#pragma unroll
        for (int k = 0; k < 8; ++k) m[k] = fmaxf(m[k], v[k]);
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) skm[rg * HID + o * 8 + k] = m[k];
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        float mm = -INFINITY;
        for (int g = 0; g < groups; ++g) mm = fmaxf(mm, skm[g * HID + o * 8 + k]);
        m[k] = mm;
    }
    float s[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int n = n0 + rg; n < n1; n += groups) {
        float v[8];
        ld8(base + (size_t)n * 3 * HID, v);
#pragma unroll
        for (int k = 0; k < 8; ++k) s[k] += __expf(v[k] - m[k]);
    }
    float* ssum = skm + groups * HID;
#pragma unroll
    for (int k = 0; k < 8; ++k) ssum[rg * HID + o * 8 + k] = s[k];
    __syncthreads();
    for (int c = threadIdx.x; c < HID; c += blockDim.x) {
        float mm = -INFINITY, t = 0.f;
        for (int g = 0; g < groups; ++g) { mm = fmaxf(mm, skm[g * HID + c]); t += ssum[g * HID + c]; }
        float* op = part + (((size_t)b * gridDim.x + chunk) * HID + c) * 2;
        op[0] = mm; op[1] = t;
    }
}

// ---- pass 2: context accumulation.  MODE 0: w = exp(k - M) (ctx, scaled by 1/(Z*N) at the end);
//              MODE 1: w = softmax_d(q)*scale, v := dout  (dctx, unscaled)
template <typename T, int MODE>
__global__ void __launch_bounds__(256) la_context_kernel(const T* __restrict__ qkv, const T* __restrict__ dout,
                                                         const float* __restrict__ part, int n_stat_chunks,
                                                         float* __restrict__ kmax, float* __restrict__ kzinv,
                                                         float* __restrict__ ctx, int N, int heads,
                                                         int rows_per_chunk, float scale) {
    pdl_trigger();
    pdl_wait();
    __shared__ float sM[DH], sZi[DH];
    __shared__ __align__(16) float Wt[LA_TN][DH + 1];
    __shared__ __align__(16) float Vt[LA_TN][DH];
    const int HID = heads * DH;
    const int b = blockIdx.z, h = blockIdx.y, chunk = blockIdx.x, tid = threadIdx.x;
    if (MODE == 0) {
        if (tid < DH) {
            float M = -INFINITY;
            for (int i = 0; i < n_stat_chunks; ++i)
                M = fmaxf(M, part[(((size_t)b * n_stat_chunks + i) * HID + h * DH + tid) * 2]);
            float Z = 0.f;
            for (int i = 0; i < n_stat_chunks; ++i) {
                const float* p = part + (((size_t)b * n_stat_chunks + i) * HID + h * DH + tid) * 2;
                Z += p[1] * __expf(p[0] - M);
            }
            sM[tid] = M;
            sZi[tid] = 1.f / Z;
            if (chunk == 0) {
                kmax[((size_t)b * heads + h) * DH + tid] = M;
                kzinv[((size_t)b * heads + h) * DH + tid] = 1.f / Z;
            }
        }
        __syncthreads();
    }
    const int n0 = chunk * rows_per_chunk;
    int n1 = n0 + rows_per_chunk;
    if (n1 > N) n1 = N;
    const int lrow = tid >> 2, lpart = (tid & 3) * 8;
    const int d = tid >> 3, e0 = (tid & 7) * 4;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    const size_t row_stride = (size_t)3 * HID;
    for (int t0 = n0; t0 < n1; t0 += LA_TN) {
        int n = t0 + lrow;
        float w[8], v[8];
        if (n < n1) {
            const T* rowp = qkv + ((size_t)b * N + n) * row_stride;
            if (MODE == 0) {
                ld8(rowp + HID + h * DH + lpart, w);
                ld8(rowp + 2 * HID + h * DH + lpart, v);
#pragma unroll
                for (int k = 0; k < 8; ++k) w[k] = __expf(w[k] - sM[lpart + k]);
            } else {
                ld8(rowp + h * DH + lpart, w);
                ld8(dout + ((size_t)b * N + n) * HID + h * DH + lpart, v);
            }
        } else {
#pragma unroll
            for (int k = 0; k < 8; ++k) { w[k] = (MODE == 0) ? 0.f : -INFINITY; v[k] = 0.f; }
        }
        __syncthreads();   // previous tile fully consumed
#pragma unroll
        for (int k = 0; k < 8; ++k) { Wt[lrow][lpart + k] = w[k]; Vt[lrow][lpart + k] = v[k]; }
        __syncthreads();
        if (MODE == 1) {
            if (tid < LA_TN) {   // row-wise softmax over d
                float mx = -INFINITY;
#pragma unroll
                for (int k = 0; k < DH; ++k) mx = fmaxf(mx, Wt[tid][k]);
                float sum = 0.f;
                if (mx == -INFINITY) {
#pragma unroll
                    for (int k = 0; k < DH; ++k) Wt[tid][k] = 0.f;
                } else {
#pragma unroll
                    for (int k = 0; k < DH; ++k) { float ex = __expf(Wt[tid][k] - mx); Wt[tid][k] = ex; sum += ex; }
                    float inv = scale / sum;
#pragma unroll
                    for (int k = 0; k < DH; ++k) Wt[tid][k] *= inv;
                }
            }
            __syncthreads();
        }
#pragma unroll 8
        for (int r = 0; r < LA_TN; ++r) {
            float wv = Wt[r][d];
            float4 vv = *reinterpret_cast<const float4*>(&Vt[r][e0]);
            acc[0] += wv * vv.x; acc[1] += wv * vv.y; acc[2] += wv * vv.z; acc[3] += wv * vv.w;
        }
    }
    float f = (MODE == 0) ? sZi[d] / (float)N : 1.f;
    float* o = ctx + (((size_t)b * heads + h) * DH + d) * DH + e0;
#pragma unroll
    for (int k = 0; k < 4; ++k) atomicAdd(o + k, acc[k] * f);
}

// ---- pass 3: out[n, h*32+e] = sum_d ctx[h][d][e] * softmax_d(q[n,h,:])[d] * scale -------------------------
// block = 32 pixels x heads (one warp per head -> ctx reads are warp-uniform broadcasts)
template <typename T>
__global__ void la_out_kernel(const T* __restrict__ qkv, const float* __restrict__ ctx, T* __restrict__ out, int N,
                              int heads, float scale) {
    pdl_trigger();
    pdl_wait();
    extern __shared__ __align__(16) float sctx[];   // [heads][32][32]
    const int HID = heads * DH;
    const long long pix0 = (long long)blockIdx.x * 32;
    const int b = (int)(pix0 / N);
    for (int i = threadIdx.x; i < heads * DH * DH; i += blockDim.x) sctx[i] = ctx[(size_t)b * heads * DH * DH + i];
    __syncthreads();
    const int lane = threadIdx.x & 31, h = threadIdx.x >> 5;
    const long long pix = pix0 + lane;
    float q[DH];
    const T* qp = qkv + (size_t)pix * 3 * HID + h * DH;
#pragma unroll
    for (int k = 0; k < DH; k += 8) ld8(qp + k, q + k);
    float mx = q[0];
#pragma unroll
    for (int k = 1; k < DH; ++k) mx = fmaxf(mx, q[k]);
    float sum = 0.f;
#pragma unroll
    for (int k = 0; k < DH; ++k) { q[k] = __expf(q[k] - mx); sum += q[k]; }
    const float inv = scale / sum;
    float o[DH];
#pragma unroll
    for (int e = 0; e < DH; ++e) o[e] = 0.f;
    const float* cx = sctx + h * DH * DH;
#pragma unroll
    for (int d = 0; d < DH; ++d) {
        float qd = q[d] * inv;
#pragma unroll
        for (int e = 0; e < DH; e += 4) {
            float4 c4 = *reinterpret_cast<const float4*>(cx + d * DH + e);
            o[e] += qd * c4.x; o[e + 1] += qd * c4.y; o[e + 2] += qd * c4.z; o[e + 3] += qd * c4.w;
        }
    }
    T* op = out + (size_t)pix * HID + h * DH;
#pragma unroll
    for (int k = 0; k < DH; k += 8) st8(op + k, o + k);
}

// ---- backward, per pixel: dq, dk, dv from dout, ctx, dctx and the saved column statistics -----------------
// block = 32 pixels x HB heads (grid.y covers heads/HB)
constexpr int LA_HB = 4;
template <typename T>
__global__ void __launch_bounds__(32 * LA_HB) la_bwd_pixel_kernel(const T* __restrict__ qkv, const T* __restrict__ dout,
                                                                  const float* __restrict__ ctx,
                                                                  const float* __restrict__ dctx,
                                                                  const float* __restrict__ kmax,
                                                                  const float* __restrict__ kzinv,
                                                                  T* __restrict__ dqkv, int N, int heads, float scale) {
    pdl_trigger();
    pdl_wait();
    __shared__ __align__(16) float sctx[LA_HB][DH][DH];
    __shared__ __align__(16) float sdctx[LA_HB][DH][DH];
    __shared__ float scd[LA_HB][DH], sM[LA_HB][DH], sZi[LA_HB][DH];
    const int HID = heads * DH;
    const long long pix0 = (long long)blockIdx.x * 32;
    const int b = (int)(pix0 / N);
    const int h0 = blockIdx.y * LA_HB;
    for (int i = threadIdx.x; i < LA_HB * DH * DH; i += blockDim.x) {
        int hh = i / (DH * DH), r = i % (DH * DH);
        (&sctx[0][0][0])[i] = ctx[((size_t)b * heads + h0 + hh) * DH * DH + r];
        (&sdctx[0][0][0])[i] = dctx[((size_t)b * heads + h0 + hh) * DH * DH + r];
    }
    for (int i = threadIdx.x; i < LA_HB * DH; i += blockDim.x) {
        int hh = i / DH, d = i % DH;
        (&sM[0][0])[i] = kmax[((size_t)b * heads + h0 + hh) * DH + d];
        (&sZi[0][0])[i] = kzinv[((size_t)b * heads + h0 + hh) * DH + d];
    }
    __syncthreads();
    for (int i = threadIdx.x; i < LA_HB * DH; i += blockDim.x) {
        int hh = i / DH, d = i % DH;
        float s = 0.f;
#pragma unroll
        for (int e = 0; e < DH; ++e) s += sdctx[hh][d][e] * sctx[hh][d][e];
        scd[hh][d] = s;
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, hh = threadIdx.x >> 5, h = h0 + hh;
    const long long pix = pix0 + lane;
    const T* row = qkv + (size_t)pix * 3 * HID;
    T* drow = dqkv + (size_t)pix * 3 * HID;
    float g[DH];   // dout
    const T* gp = dout + (size_t)pix * HID + h * DH;
#pragma unroll
    for (int k = 0; k < DH; k += 8) ld8(gp + k, g + k);
    float a[DH], r[DH];
    // ---- dq
#pragma unroll
    for (int k = 0; k < DH; k += 8) ld8(row + h * DH + k, a + k);
    {
        float mx = a[0];
#pragma unroll
        for (int k = 1; k < DH; ++k) mx = fmaxf(mx, a[k]);
        float sum = 0.f;
#pragma unroll
        for (int k = 0; k < DH; ++k) { a[k] = __expf(a[k] - mx); sum += a[k]; }
        float inv = 1.f / sum, dot = 0.f;
#pragma unroll
        for (int d = 0; d < DH; ++d) {
            a[d] *= inv;                               // p[d]
            float s = 0.f;
#pragma unroll
            for (int e = 0; e < DH; e += 4) {
                float4 c4 = *reinterpret_cast<const float4*>(&sctx[hh][d][e]);
                s += g[e] * c4.x + g[e + 1] * c4.y + g[e + 2] * c4.z + g[e + 3] * c4.w;
            }
            r[d] = s * scale;                          // dp[d]
            dot += a[d] * r[d];
        }
#pragma unroll
        for (int d = 0; d < DH; ++d) r[d] = a[d] * (r[d] - dot);
#pragma unroll
        for (int k = 0; k < DH; k += 8) st8(drow + h * DH + k, r + k);
    }
    // ---- dk, dv
    float v[DH];
#pragma unroll
    for (int k = 0; k < DH; k += 8) { ld8(row + HID + h * DH + k, a + k); ld8(row + 2 * HID + h * DH + k, v + k); }
    const float invN = 1.f / (float)N;
#pragma unroll
    for (int e = 0; e < DH; ++e) r[e] = 0.f;          // dv accumulator
#pragma unroll
    for (int d = 0; d < DH; ++d) {
        float kt = __expf(a[d] - sM[hh][d]) * sZi[hh][d];   // k~[n,d]
        float s = 0.f;
#pragma unroll
        for (int e = 0; e < DH; e += 4) {
            float4 c4 = *reinterpret_cast<const float4*>(&sdctx[hh][d][e]);
            s += v[e] * c4.x + v[e + 1] * c4.y + v[e + 2] * c4.z + v[e + 3] * c4.w;
            r[e] += kt * c4.x; r[e + 1] += kt * c4.y; r[e + 2] += kt * c4.z; r[e + 3] += kt * c4.w;
        }
        a[d] = kt * (s * invN - scd[hh][d]);           // dk[n,d]
    }
#pragma unroll
    for (int e = 0; e < DH; ++e) r[e] *= invN;
#pragma unroll
    for (int k = 0; k < DH; k += 8) { st8(drow + HID + h * DH + k, a + k); st8(drow + 2 * HID + h * DH + k, r + k); }
}

// ==== (2) one CTA per (sample, head) =================================================================================
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
constexpr int LS_PITCH = DH + 1;  // fp32 row pitch: a thread that owns a token walks its row without bank conflicts
constexpr int LS_BPITCH = DH + 2;  // bf16 row pitch of the read-only planes (v, dout): 17 words, odd -> conflict-free rows
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
        for (int d = 0; d < DH; ++d) m = fmaxf(m, r[d]);
        float s = 0.f;
#pragma unroll
        for (int d = 0; d < DH; ++d) { const float e = __expf(r[d] - m); r[d] = e; s += e; }
        const float inv = 1.f / s;
#pragma unroll
        for (int d = 0; d < DH; ++d) r[d] *= inv;
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
    C[d * DH + e0] = a0 * mul; C[d * DH + e0 + 1] = a1 * mul; C[d * DH + e0 + 2] = a2 * mul; C[d * DH + e0 + 3] = a3 * mul;
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
    float* red = ctx + DH * DH;            // [8][32]
    float* colM = red + 8 * 32;
    float* colZi = colM + 32;
    __nv_bfloat16* V = reinterpret_cast<__nv_bfloat16*>(colZi + 32);
    const int h = blockIdx.x, b = blockIdx.y, HID = heads * DH;
    const size_t stride = 3 * (size_t)HID;
    const __nv_bfloat16* base = qkv + (size_t)b * N * stride + h * DH;
    ls_load_plane(Q, base, stride, N);
    ls_load_plane(K, base + HID, stride, N);
    ls_load_bplane(V, base + 2 * HID, stride, N);
    __syncthreads();
    ls_col_softmax(K, red, colM, colZi, N);                        // K <- k~
    ls_outer_sum(ctx, K, V, N, 1.f / (float)N);                    // ctx = k~^T (v / N)
    ls_row_softmax(Q, N);                                          // Q <- softmax_d(q)
    __syncthreads();
    for (int i = threadIdx.x; i < DH * DH; i += blockDim.x) ctx_out[((size_t)b * heads + h) * DH * DH + i] = ctx[i];
    if (threadIdx.x < 32) {
        kmax[(size_t)b * HID + h * DH + threadIdx.x] = colM[threadIdx.x];
        kzinv[(size_t)b * HID + h * DH + threadIdx.x] = colZi[threadIdx.x];
    }
    // out[n][e] = s * sum_d p[n][d] ctx[d][e]: thread = (token, 8-column octet)
    for (int w = threadIdx.x; w < N * 4; w += blockDim.x) {
        const int n = w >> 2, e0 = (w & 3) * 8;
        const float* p = Q + n * LS_PITCH;
        float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int d = 0; d < DH; ++d) {
            const float pv = p[d];
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[k] += pv * ctx[d * DH + e0 + k];
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] *= scale;
        st8(out + ((size_t)b * N + n) * HID + h * DH + e0, acc);
    }
}

static size_t ls_smem(int N, bool bwd) {
    const LsLayout L(N);
    return (size_t)(2 * L.plane + (bwd ? 2 : 1) * DH * DH + 8 * 32 + 3 * 32 + (bwd ? 2 : 1) * L.bplane) * sizeof(float);
}

// At 256 tokens the 32-wide products (0.7 GFLOP per layer) are CUDA-core FLOP-bound here while the streaming kernels
// run them on mma.sync, so only the 8x8 level takes this path, and only where it wins (forward).
static bool la_small_supported(int N, int dtype) { return dtype == PIDM_BF16 && N >= 32 && N <= 64; }

static int la_small_fwd(const void* qkv, void* out, float* ctx, float* kmax, float* kzinv, int B, int N, int heads,
                        float scale, cudaStream_t st) {
    PIDM_CUDA(allow_smem(la_small_fwd_kernel, ls_smem(LS_MAXN, false)));
    PIDM_CUDA(launch_plain(la_small_fwd_kernel, dim3(heads, B), dim3(LS_THREADS), ls_smem(N, false), st, (const __nv_bfloat16*)qkv,
                           (__nv_bfloat16*)out, ctx, kmax, kzinv, N, heads, scale));
    PIDM_LAUNCH_CHECK("la_small_fwd");
    return 0;
}

// ==== (3) mma.sync ===================================================================================================
// Linear attention (reference unet_model.py:286-297) on the tensor cores for bf16 activations, heads = 8, dim_head = 32.
//
// The per-(sample, head) products are 32x32 blocks -- too small for wgmma (M = 64 per warpgroup) and HBM-bound anyway
// (the whole qkv row of a pixel, 8 heads x 3 x 32 channels = 1536 B, is streamed once), so these kernels use
// warp-level mma.sync m16n8k16 (bf16 in, fp32 accumulate) with ldmatrix-fed fragments.  One warp per head, and the
// eight warps of a CTA are fully DECOUPLED: every warp streams its own head's 64-byte slice of each pixel row through
// a private cp.async ring in shared memory, transforms it in place (one lane per pixel row) and feeds the tensor cores;
// only __syncwarp is used in the loops.  (The first version staged whole 512-byte rows for all heads behind two
// __syncthreads per tile, which left every warp stalled on the barriers.)
//   la_ctx_mma<0>: ctx[h][d][e]  += sum_n exp(k[n,d]-M_d) v[n,e]      (scaled by 1/(Z_d N) in the epilogue)
//   la_ctx_mma<1>: dctx[h][d][e] += sum_n softmax_d(q[n,:])[d]*s * dout[n,e]
//   la_out_mma   : out[n,h,e]     = sum_d softmax_d(q[n,:])[d]*s * ctx[h][d][e]
//   la_bwd_mma   : dq, dk, dv per pixel from dout, ctx, dctx and the saved column statistics
// ---- context / dcontext ---------------------------------------------------------------------------------------------
//   MODE 0: ctx[h][d][e]  += sum_n exp(k[n,d] - M_d) v[n,e]        (scaled by 1/(Z_d N) in the epilogue)
//   MODE 1: dctx[h][d][e] += sum_n softmax_d(q[n,:])[d] * s * dout[n,e]
// grid (pixel chunks, B); warp h owns head h; per-warp ring of LC_STAGES x (W | V) 32-pixel tiles.
constexpr int LC_STAGES = 3;
template <int MODE>
__global__ void __launch_bounds__(256) la_ctx_mma_kernel(const __nv_bfloat16* __restrict__ qkv,
                                                         const __nv_bfloat16* __restrict__ dout,
                                                         const float* __restrict__ part, int n_stat_chunks,
                                                         float* __restrict__ kmax, float* __restrict__ kzinv,
                                                         float* __restrict__ ctx, int N, int chunk_px, float scale) {
    pdl_trigger();
    pdl_wait();
    extern __shared__ __align__(16) unsigned char raw[];
    const int b = blockIdx.y, chunk = blockIdx.x, lane = threadIdx.x & 31, h = threadIdx.x >> 5;
    float* sM = reinterpret_cast<float*>(raw + (size_t)LM_HEADS * LC_STAGES * 2 * LW_TILE * 2) + h * 2 * DH;
    float* sZi = sM + DH;
    const int n_begin = chunk * chunk_px, n_end = min(N, n_begin + chunk_px);
    const int n_tiles = (n_end - n_begin) / 32;
    const size_t pix0 = (size_t)b * N + n_begin;
    const __nv_bfloat16* wsrc = qkv + pix0 * 3 * LM_HID + (MODE == 0 ? LM_HID : 0) + h * DH;
    const __nv_bfloat16* vsrc = (MODE == 0) ? qkv + pix0 * 3 * LM_HID + 2 * LM_HID + h * DH : dout + pix0 * LM_HID + h * DH;
    const size_t vstride = (MODE == 0) ? 3 * LM_HID : LM_HID;
    const CpRing<LC_STAGES, 2 * LW_TILE> ring{reinterpret_cast<__nv_bfloat16*>(raw) + (size_t)h * (LC_STAGES * 2 * LW_TILE),
                                              n_tiles};
    auto load = [&](__nv_bfloat16* buf, int it) {
        lw_issue<32>(buf, wsrc + (size_t)it * 32 * 3 * LM_HID, 3 * LM_HID, lane);
        lw_issue<32>(buf + LW_TILE, vsrc + (size_t)it * 32 * vstride, vstride, lane);
    };
    ring.prime(load);
    if (MODE == 0) {                               // lane = channel d of this head: combine the per-chunk statistics
        const int c = h * DH + lane;
        float M = -INFINITY;
        for (int i = 0; i < n_stat_chunks; ++i) M = fmaxf(M, part[(((size_t)b * n_stat_chunks + i) * LM_HID + c) * 2]);
        float Z = 0.f;
        for (int i = 0; i < n_stat_chunks; ++i) {
            const float* p = part + (((size_t)b * n_stat_chunks + i) * LM_HID + c) * 2;
            Z += p[1] * __expf(p[0] - M);
        }
        sM[lane] = M;
        sZi[lane] = 1.f / Z;
        if (chunk == 0) { kmax[(size_t)b * LM_HID + c] = M; kzinv[(size_t)b * LM_HID + c] = 1.f / Z; }
        __syncwarp();
    }
    float acc[2][4][4];
    zero(acc);
    for (int it = 0; it < n_tiles; ++it) {
        __nv_bfloat16* Ws = ring.wait(it, load);
        const __nv_bfloat16* Vs = Ws + LW_TILE;
        {   // in-place transform of the W tile, one lane per pixel row
            float v[32];
            row_load32(Ws + lane * LW_PITCH, v);
            if (MODE == 0) {
#pragma unroll
                for (int j = 0; j < 32; j += 4) {
                    const float4 m4 = *reinterpret_cast<const float4*>(sM + j);
                    v[j] = __expf(v[j] - m4.x); v[j + 1] = __expf(v[j + 1] - m4.y);
                    v[j + 2] = __expf(v[j + 2] - m4.z); v[j + 3] = __expf(v[j + 3] - m4.w);
                }
            } else {
                row_softmax32(v, scale);
            }
            row_store32(Ws + lane * LW_PITCH, v);
        }
        __syncwarp();
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) {
            uint32_t a0[4], a1[4], b01[4], b23[4];
            frag_a_kmajor(a0, Ws, LW_PITCH, ks * 16, 0, lane);
            frag_a_kmajor(a1, Ws, LW_PITCH, ks * 16, 16, lane);
            frag_b_krows(b01, Vs, LW_PITCH, ks * 16, 0, lane);
            frag_b_krows(b23, Vs, LW_PITCH, ks * 16, 16, lane);
            mma_bf16(acc[0][0], a0, b01[0], b01[1]); mma_bf16(acc[0][1], a0, b01[2], b01[3]);
            mma_bf16(acc[0][2], a0, b23[0], b23[1]); mma_bf16(acc[0][3], a0, b23[2], b23[3]);
            mma_bf16(acc[1][0], a1, b01[0], b01[1]); mma_bf16(acc[1][1], a1, b01[2], b01[3]);
            mma_bf16(acc[1][2], a1, b23[0], b23[1]); mma_bf16(acc[1][3], a1, b23[2], b23[3]);
        }
        ring.release(it, load);
    }
    ctx_atomic_add(ctx + ((size_t)b * LM_HEADS + h) * DH * DH, acc,
                   [&](int d) { return (MODE == 0) ? sZi[d] / (float)N : 1.f; }, lane);
}

// ---- out[n,h,e] = sum_d softmax_d(q[n,:])[d] * s * ctx[h][d][e] ---------------------------------------------------------
constexpr int LO_STAGES = 4;
__global__ void __launch_bounds__(256) la_out_mma_kernel(const __nv_bfloat16* __restrict__ qkv,
                                                         const float* __restrict__ ctx, __nv_bfloat16* __restrict__ out,
                                                         int N, int chunk_px, float scale) {
    pdl_trigger();
    pdl_wait();
    extern __shared__ __align__(16) unsigned char raw[];
    const int b = blockIdx.y, chunk = blockIdx.x, lane = threadIdx.x & 31, h = threadIdx.x >> 5;
    const int n_begin = chunk * chunk_px, n_end = min(N, n_begin + chunk_px);
    const int n_tiles = (n_end - n_begin) / 32;
    const size_t pix0 = (size_t)b * N + n_begin;
    const __nv_bfloat16* qsrc = qkv + pix0 * 3 * LM_HID + h * DH;
    __nv_bfloat16* odst = out + pix0 * LM_HID + h * DH;
    const CpRing<LO_STAGES, LW_TILE> ring{reinterpret_cast<__nv_bfloat16*>(raw) + (size_t)h * (LO_STAGES * LW_TILE),
                                          n_tiles};
    auto load = [&](__nv_bfloat16* buf, int it) {
        lw_issue<32>(buf, qsrc + (size_t)it * 32 * 3 * LM_HID, 3 * LM_HID, lane);
    };
    ring.prime(load);
    uint32_t bf[2][4][2];                          // B[k = d][n = e] = ctx[d][e], straight from global fp32
    frags_b_global<true>(bf, ctx + ((size_t)b * LM_HEADS + h) * DH * DH, lane);
    for (int it = 0; it < n_tiles; ++it) {
        __nv_bfloat16* Qs = ring.wait(it, load);
        {
            float v[32];
            row_load32(Qs + lane * LW_PITCH, v);
            row_softmax32(v, scale);
            row_store32(Qs + lane * LW_PITCH, v);
        }
        __syncwarp();
        uint32_t a[2][2][4];
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int ks = 0; ks < 2; ++ks) frag_a_rowmajor(a[mt][ks], Qs, LW_PITCH, mt * 16, ks * 16, lane);
        __syncwarp();                              // the q tile is in registers: the buffer becomes the output staging
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
            float c[4][4];
            zero(c);
#pragma unroll
            for (int ks = 0; ks < 2; ++ks)
#pragma unroll
                for (int nt = 0; nt < 4; ++nt) mma_bf16(c[nt], a[mt][ks], bf[ks][nt][0], bf[ks][nt][1]);
            store_rows_bf16(Qs + (size_t)(mt * 16) * LW_PITCH, LW_PITCH, c, lane);
        }
        __syncwarp();
        lw_store<32>(odst + (size_t)it * 32 * LM_HID, LM_HID, Qs, lane);
        ring.release(it, load);
    }
}

// ---- backward per pixel ---------------------------------------------------------------------------------------------
// Per warp: ring of LB_STAGES raw 16-pixel tiles (dout | q | k | v head slices).  The landed tile is transformed in
// place (q -> softmax p, k -> k~), multiplied against the head's ctx / dctx blocks (B fragments live in registers),
// and dq | dk | dv overwrite p | k~ | v in the same buffer before they are stored with 16-byte vectors.
constexpr int LB_ROWS = 16;
constexpr int LB_STAGES = 3;
constexpr int LB_TILE = 4 * LB_ROWS * LW_PITCH;          // dout, q, k, v
__global__ void __launch_bounds__(256) la_bwd_mma_kernel(const __nv_bfloat16* __restrict__ qkv,
                                                         const __nv_bfloat16* __restrict__ dout,
                                                         const float* __restrict__ ctx, const float* __restrict__ dctx,
                                                         const float* __restrict__ kmax, const float* __restrict__ kzinv,
                                                         __nv_bfloat16* __restrict__ dqkv, int N, int chunk_px, float scale) {
    pdl_trigger();
    pdl_wait();
    extern __shared__ __align__(16) unsigned char raw[];
    const int b = blockIdx.y, chunk = blockIdx.x, lane = threadIdx.x & 31, h = threadIdx.x >> 5;
    float* sM = reinterpret_cast<float*>(raw + (size_t)LM_HEADS * LB_STAGES * LB_TILE * 2) + h * 3 * DH;
    float* sZi = sM + DH;
    float* scd = sZi + DH;
    const int n_begin = chunk * chunk_px, n_end = min(N, n_begin + chunk_px);
    const int n_tiles = (n_end - n_begin) / LB_ROWS;
    const size_t pix0 = (size_t)b * N + n_begin;
    const __nv_bfloat16* qsrc = qkv + pix0 * 3 * LM_HID + h * DH;
    const __nv_bfloat16* gsrc = dout + pix0 * LM_HID + h * DH;
    __nv_bfloat16* ddst = dqkv + pix0 * 3 * LM_HID + h * DH;
    const CpRing<LB_STAGES, LB_TILE> ring{reinterpret_cast<__nv_bfloat16*>(raw) + (size_t)h * (LB_STAGES * LB_TILE),
                                          n_tiles};
    auto load = [&](__nv_bfloat16* buf, int it) {
        const __nv_bfloat16* q = qsrc + (size_t)it * LB_ROWS * 3 * LM_HID;
        lw_issue<LB_ROWS>(buf, gsrc + (size_t)it * LB_ROWS * LM_HID, LM_HID, lane);
        lw_issue<LB_ROWS>(buf + LB_ROWS * LW_PITCH, q, 3 * LM_HID, lane);
        lw_issue<LB_ROWS>(buf + 2 * LB_ROWS * LW_PITCH, q + LM_HID, 3 * LM_HID, lane);
        lw_issue<LB_ROWS>(buf + 3 * LB_ROWS * LW_PITCH, q + 2 * LM_HID, 3 * LM_HID, lane);
    };
    ring.prime(load);
    const float* cg = ctx + ((size_t)b * LM_HEADS + h) * DH * DH;
    const float* dg = dctx + ((size_t)b * LM_HEADS + h) * DH * DH;
    sM[lane] = kmax[(size_t)b * LM_HID + h * DH + lane];
    sZi[lane] = kzinv[(size_t)b * LM_HID + h * DH + lane];
    scd[lane] = ctx_dot_row(cg, dg, lane);
    uint32_t bc[2][4][2], bd[2][4][2], bt[2][4][2];
    frags_b_global<false>(bc, cg, lane);           // B[k=e][n=d] = ctx[d][e]
    frags_b_global<false>(bd, dg, lane);           // B[k=e][n=d] = dctx[d][e]
    frags_b_global<true>(bt, dg, lane);            // B[k=d][n=e] = dctx[d][e]
    __syncwarp();
    const int g = lane >> 2, t = lane & 3;
    const float invN = 1.f / (float)N;
    for (int it = 0; it < n_tiles; ++it) {
        __nv_bfloat16* buf = ring.wait(it, load);
        __nv_bfloat16* T0 = buf;                           // dout
        __nv_bfloat16* T1 = buf + LB_ROWS * LW_PITCH;      // q  -> p  -> dq
        __nv_bfloat16* T2 = buf + 2 * LB_ROWS * LW_PITCH;  // k  -> k~ -> dk
        __nv_bfloat16* T3 = buf + 3 * LB_ROWS * LW_PITCH;  // v        -> dv
        {   // lanes 0-15: softmax of a q row; lanes 16-31: k~ = exp(k - M) * Zinv of a k row
            const int row = lane & 15;
            float v[32];
            if (lane < 16) {
                row_load32(T1 + row * LW_PITCH, v);
                row_softmax32(v, 1.f);
                row_store32(T1 + row * LW_PITCH, v);
            } else {
                row_load32(T2 + row * LW_PITCH, v);
#pragma unroll
                for (int j = 0; j < 32; ++j) v[j] = __expf(v[j] - sM[j]) * sZi[j];
                row_store32(T2 + row * LW_PITCH, v);
            }
        }
        __syncwarp();
        float cq[4][4], ck[4][4], cv[4][4];
        zero(cq);
        zero(ck);
        zero(cv);
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) {
            uint32_t ag[4], av[4], ak[4];
            frag_a_rowmajor(ag, T0, LW_PITCH, 0, ks * 16, lane);      // dout [px][e]
            frag_a_rowmajor(av, T3, LW_PITCH, 0, ks * 16, lane);      // v    [px][e]
            frag_a_rowmajor(ak, T2, LW_PITCH, 0, ks * 16, lane);      // k~   [px][d]
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                mma_bf16(cq[nt], ag, bc[ks][nt][0], bc[ks][nt][1]);
                mma_bf16(ck[nt], av, bd[ks][nt][0], bd[ks][nt][1]);
                mma_bf16(cv[nt], ak, bt[ks][nt][0], bt[ks][nt][1]);
            }
        }
        // dq = p * (dp - sum_d p dp), dp = scale * (dout ctx^T);  dk = k~ * (dk~ - cd), dk~ = (v/N) dctx^T;  dv = (k~ dctx)/N
        // each thread rewrites exactly the elements it has just read (p, k~) -- v is dead after the last mma above
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const int row = g + half * 8;
            float pv[4][2], dot = 0.f;
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                const __nv_bfloat162 p2 = *reinterpret_cast<const __nv_bfloat162*>(T1 + row * LW_PITCH + nt * 8 + 2 * t);
                pv[nt][0] = __low2float(p2); pv[nt][1] = __high2float(p2);
                dot += pv[nt][0] * cq[nt][half * 2] + pv[nt][1] * cq[nt][half * 2 + 1];
            }
            dot = quad_sum(dot);
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                const int col = nt * 8 + 2 * t;
                const int o = row * LW_PITCH + col;
                const __nv_bfloat162 k2 = *reinterpret_cast<const __nv_bfloat162*>(T2 + o);
                *reinterpret_cast<uint32_t*>(T1 + o) = pack_bf16(scale * pv[nt][0] * (cq[nt][half * 2] - dot),
                                                                scale * pv[nt][1] * (cq[nt][half * 2 + 1] - dot));
                *reinterpret_cast<uint32_t*>(T2 + o) = pack_bf16(__low2float(k2) * (ck[nt][half * 2] * invN - scd[col]),
                                                                __high2float(k2) * (ck[nt][half * 2 + 1] * invN - scd[col + 1]));
                *reinterpret_cast<uint32_t*>(T3 + o) = pack_bf16(cv[nt][half * 2] * invN, cv[nt][half * 2 + 1] * invN);
            }
        }
        __syncwarp();
        __nv_bfloat16* d = ddst + (size_t)it * LB_ROWS * 3 * LM_HID;
        lw_store<LB_ROWS>(d, 3 * LM_HID, T1, lane);
        lw_store<LB_ROWS>(d + LM_HID, 3 * LM_HID, T2, lane);
        lw_store<LB_ROWS>(d + 2 * LM_HID, 3 * LM_HID, T3, lane);
        ring.release(it, load);
    }
}

constexpr size_t LA_CTX_SMEM = (size_t)LM_HEADS * LC_STAGES * 2 * LW_TILE * 2 + (size_t)LM_HEADS * 2 * DH * 4;
constexpr size_t LA_OUT_SMEM = (size_t)LM_HEADS * LO_STAGES * LW_TILE * 2;
constexpr size_t LA_BWD_SMEM = (size_t)LM_HEADS * LB_STAGES * LB_TILE * 2 + (size_t)LM_HEADS * 3 * DH * 4;

// host launchers of the bf16 / 8-head case: about two CTAs per SM
static int la_mma_ctx(int mode, const void* qkv, const void* dout, const float* part, int n_stat_chunks, float* kmax,
                      float* kzinv, float* ctx, int B, int N, float scale, cudaStream_t st) {
    const int cpx = chunk_px(B, N, 2);
    dim3 grid((N + cpx - 1) / cpx, B);
    if (mode == 0) {
        PIDM_CUDA(allow_smem(la_ctx_mma_kernel<0>, LA_CTX_SMEM));
        PIDM_CUDA(launch_plain(la_ctx_mma_kernel<0>, dim3(grid), dim3(256), (size_t)(LA_CTX_SMEM), st, (const __nv_bfloat16*)qkv, nullptr, part, n_stat_chunks, kmax,
                                                              kzinv, ctx, N, cpx, scale));
    } else {
        PIDM_CUDA(allow_smem(la_ctx_mma_kernel<1>, LA_CTX_SMEM));
        PIDM_CUDA(launch_plain(la_ctx_mma_kernel<1>, dim3(grid), dim3(256), (size_t)(LA_CTX_SMEM), st, (const __nv_bfloat16*)qkv, (const __nv_bfloat16*)dout, nullptr,
                                                              0, nullptr, nullptr, ctx, N, cpx, scale));
    }
    PIDM_LAUNCH_CHECK("la_ctx_mma");
    return 0;
}
static int la_mma_out(const void* qkv, const float* ctx, void* out, int B, int N, float scale, cudaStream_t st) {
    const int cpx = chunk_px(B, N, 2);
    dim3 grid((N + cpx - 1) / cpx, B);
    PIDM_CUDA(allow_smem(la_out_mma_kernel, LA_OUT_SMEM));
    PIDM_CUDA(launch_plain(la_out_mma_kernel, dim3(grid), dim3(256), (size_t)(LA_OUT_SMEM), st, (const __nv_bfloat16*)qkv, ctx, (__nv_bfloat16*)out, N, cpx, scale));
    PIDM_LAUNCH_CHECK("la_out_mma");
    return 0;
}
static int la_mma_bwd(const void* qkv, const void* dout, const float* ctx, const float* dctx, const float* kmax,
                      const float* kzinv, void* dqkv, int B, int N, float scale, cudaStream_t st) {
    const int cpx = chunk_px(B, N, 2);
    dim3 grid((N + cpx - 1) / cpx, B);
    PIDM_CUDA(allow_smem(la_bwd_mma_kernel, LA_BWD_SMEM));
    PIDM_CUDA(launch_plain(la_bwd_mma_kernel, dim3(grid), dim3(256), (size_t)(LA_BWD_SMEM), st, (const __nv_bfloat16*)qkv, (const __nv_bfloat16*)dout, ctx, dctx, kmax,
                                                       kzinv, (__nv_bfloat16*)dqkv, N, cpx, scale));
    PIDM_LAUNCH_CHECK("la_bwd_mma");
    return 0;
}

// ==== path choice ====================================================================================================
// block = whole row groups of HID/8 threads, about 256 threads
static int la_kstats_block(int HID) {
    const int oct = HID / 8;
    int groups = 256 / oct;
    if (groups < 1) groups = 1;
    return groups * oct;
}
static size_t la_kstats_smem(int HID) { return (size_t)2 * (la_kstats_block(HID) / (HID / 8)) * HID * sizeof(float); }

static int la_chunks(int N) {
    int c = N / 128;
    if (c < 1) c = 1;
    if (c > 32) c = 32;
    return c;
}

// forward path: one CTA per (sample, head) | mma.sync ctx / out | SIMT kstats -> context -> out
enum { LA_FWD_SMALL = 0, LA_FWD_MMA = 1, LA_FWD_SIMT = 2 };
static int la_fwd_path(int N, int heads, int dtype) {
    if (la_small_supported(N, dtype)) return LA_FWD_SMALL;
    return (dtype == PIDM_BF16 && heads == 8 && N % 64 == 0) ? LA_FWD_MMA : LA_FWD_SIMT;
}
static bool la_bwd_mma(int N, int heads, int dtype) { return dtype == PIDM_BF16 && heads == 8 && N % 64 == 0; }

// statistics rows per chunk (the last chunk may be shorter)
static int la_stat_rows(int N) { return (N + la_chunks(N) - 1) / la_chunks(N); }

// SIMT context kernels: at most 16 pixel chunks, each a whole number of LA_TN-row tiles (the last may be ragged)
static int la_ctx_rows(int N) {
    const int cchunks = (N + 255) / 256 > 16 ? 16 : (N + 255) / 256;
    return ((N + cchunks - 1) / cchunks + LA_TN - 1) / LA_TN * LA_TN;
}

}  // namespace pidm
using namespace pidm;

// workspace floats: part [B*chunks*HID*2];  ctx [B,heads,32,32], kmax/kzinv [B,heads,32] are outputs kept for backward.
extern "C" int pidm_linattn_fwd(const void* qkv, void* out, float* ctx, float* kmax, float* kzinv, float* workspace,
                                int B, int N, int heads, int dtype, void* stream) {
    PIDM_REQUIRE(N % 32 == 0 && heads >= 1 && heads * DH <= 1024, "linattn: N%%32==0 and heads*32<=1024 required");
    cudaStream_t st = (cudaStream_t)stream;
    const int HID = heads * DH;
    const int chunks = la_chunks(N);
    const int rpc = la_stat_rows(N);
    const int path = la_fwd_path(N, heads, dtype);
    if (path == LA_FWD_SMALL)     // 8x8 level: the whole (sample, head) problem in one CTA, one launch
        return la_small_fwd(qkv, out, ctx, kmax, kzinv, B, N, heads, ATTN_SCALE, st);
    PIDM_CUDA(cudaMemsetAsync(ctx, 0, (size_t)B * heads * DH * DH * sizeof(float), st));
    if (path == LA_FWD_MMA) {
        PIDM_CUDA(launch_plain(la_kstats_kernel<__nv_bfloat16>, dim3(dim3(chunks, B)), dim3(256), (size_t)(la_kstats_smem(HID)), st, (const __nv_bfloat16*)qkv, workspace, N, HID, rpc));
        if (int e = la_mma_ctx(0, qkv, nullptr, workspace, chunks, kmax, kzinv, ctx, B, N, ATTN_SCALE, st)) return e;
        if (int e = la_mma_out(qkv, ctx, out, B, N, ATTN_SCALE, st)) return e;
        PIDM_LAUNCH_CHECK("linattn_fwd");
        return 0;
    }
    const int crpc = la_ctx_rows(N);
    PIDM_DISPATCH_DTYPE(dtype, {
        PIDM_CUDA(launch_plain(la_kstats_kernel<T>, dim3(dim3(chunks, B)), dim3(la_kstats_block(HID)), (size_t)(la_kstats_smem(HID)), st, (const T*)qkv, workspace, N, HID, rpc));
        PIDM_CUDA(launch_plain(la_context_kernel<T, 0>, dim3(dim3((N + crpc - 1) / crpc, heads, B)), dim3(256), (size_t)(0), st, (const T*)qkv, nullptr, workspace, chunks, kmax, kzinv, ctx, N, heads, crpc, ATTN_SCALE));
        PIDM_CUDA(launch_plain(la_out_kernel<T>, dim3((unsigned)((long long)B * N / 32)), dim3(32 * heads), (size_t)(heads * DH * DH * sizeof(float)), st, (const T*)qkv, ctx, (T*)out, N, heads, ATTN_SCALE));
    });
    PIDM_LAUNCH_CHECK("linattn_fwd");
    return 0;
}

extern "C" int pidm_linattn_workspace_floats(int B, int N, int heads) {
    return B * la_chunks(N) * heads * DH * 2;
}

// dctx [B,heads,32,32] is scratch (zeroed here).
extern "C" int pidm_linattn_bwd(const void* qkv, const void* dout, const float* ctx, const float* kmax,
                                const float* kzinv, void* dqkv, float* dctx, int B, int N, int heads, int dtype,
                                void* stream) {
    PIDM_REQUIRE(N % 32 == 0 && heads % LA_HB == 0, "linattn_bwd: N%%32==0 and heads%%4==0 required");
    cudaStream_t st = (cudaStream_t)stream;
    PIDM_CUDA(cudaMemsetAsync(dctx, 0, (size_t)B * heads * DH * DH * sizeof(float), st));
    if (la_bwd_mma(N, heads, dtype)) {
        if (int e = la_mma_ctx(1, qkv, dout, nullptr, 0, nullptr, nullptr, dctx, B, N, ATTN_SCALE, st)) return e;
        return la_mma_bwd(qkv, dout, ctx, dctx, kmax, kzinv, dqkv, B, N, ATTN_SCALE, st);
    }
    const int crpc = la_ctx_rows(N);
    PIDM_DISPATCH_DTYPE(dtype, {
        PIDM_CUDA(launch_plain(la_context_kernel<T, 1>, dim3(dim3((N + crpc - 1) / crpc, heads, B)), dim3(256), (size_t)(0), st, (const T*)qkv, (const T*)dout, nullptr, 0, nullptr, nullptr, dctx, N, heads, crpc, ATTN_SCALE));
        PIDM_CUDA(launch_plain(la_bwd_pixel_kernel<T>, dim3(dim3((unsigned)((long long)B * N / 32), heads / LA_HB)), dim3(32 * LA_HB), (size_t)(0), st, (const T*)qkv, (const T*)dout, ctx, dctx, kmax, kzinv, (T*)dqkv, N, heads, ATTN_SCALE));
    });
    PIDM_LAUNCH_CHECK("linattn_bwd");
    return 0;
}

// What pidm_linattn_fwd / _bwd launch for a shape (test aid), see pidm.h.
extern "C" int pidm_linattn_plan(int B, int N, int heads, int dtype, int* out) {
    PIDM_REQUIRE(B > 0 && N > 0 && N % 32 == 0 && heads >= 1 && heads * DH <= 1024,
                 "linattn: N%%32==0 and heads*32<=1024 required");
    PIDM_REQUIRE(dtype == PIDM_BF16 || dtype == PIDM_F32, "unknown dtype code %d", dtype);
    const int fwd = la_fwd_path(N, heads, dtype);
    const int bwd = heads % LA_HB != 0 ? -1 : la_bwd_mma(N, heads, dtype) ? 0 : 1;
    const int crpc = la_ctx_rows(N);
    const int cpx = chunk_px(B, N, 2);
    const int v[8] = {fwd, bwd, la_chunks(N), la_stat_rows(N), crpc, (N + crpc - 1) / crpc, cpx, (N + cpx - 1) / cpx};
    for (int i = 0; i < 8; ++i) out[i] = v[i];
    return 0;
}
