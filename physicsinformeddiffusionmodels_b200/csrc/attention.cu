// Attention blocks of the U-Net on NHWC activations (dim_head = 32, fp32 math):
//
// (1) SpatialLinearAttention core (reference unet_model.py:286-297), on qkv[B, N, 3*HID], HID = heads*32,
//     channel = which*HID + head*32 + d:
//         q~ = softmax_d(q) * 32^-1/2 ;  k~ = softmax_n(k) ;  v~ = v / N
//         ctx[b,h,d,e] = sum_n k~[n,d] v~[n,e] ;   out[n, h*32+e] = sum_d ctx[d,e] q~[n,d]
//     The k-softmax is a reduction over all N pixels: pass 1 computes per-chunk (max, sum-exp) per column,
//     pass 2 merges them and accumulates the 32x32 context per (sample, head) from pixel tiles staged in
//     shared memory, pass 3 applies it per pixel.  Backward uses the identity
//         sum_n k~[n,d] dk~[n,d] = sum_e dctx[d,e] ctx[d,e]
//     so no extra pass over N is needed for the k-softmax Jacobian.
// (2) Mid-block softmax attention over <= 64 tokens (Attention.forward, unet_model.py:341-367): one CTA per
//     (sample, head), everything in shared memory.
#include "common.cuh"
#include "pidm.h"

namespace pidm {

constexpr int DH = 32;            // dim_head
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

// ---- mid-block softmax attention over NT <= 64 tokens, one CTA per (head, sample) -----------------------------
constexpr int AT_N = 64;
struct AttnSmemF {
    float q[AT_N][DH + 1], k[AT_N][DH + 1], v[AT_N][DH + 1];
    float s[AT_N][AT_N + 1];
};
struct AttnSmemB {
    float q[AT_N][DH + 1], k[AT_N][DH + 1], v[AT_N][DH + 1], g[AT_N][DH + 1];
    float s[AT_N][AT_N + 1], ds[AT_N][AT_N + 1];
};

template <typename T, typename S>
__device__ __forceinline__ void attn_load_scores(const T* __restrict__ qkv, S& sm, int b, int h, int n, int HID,
                                                 float scale) {
    const int tid = threadIdx.x;
    for (int i = tid; i < AT_N * DH; i += blockDim.x) {
        int tok = i / DH, d = i % DH;
        float qv = 0.f, kv = 0.f, vv = 0.f;
        if (tok < n) {
            const T* row = qkv + ((size_t)b * n + tok) * 3 * HID + h * DH + d;
            qv = Act<T>::ld(row); kv = Act<T>::ld(row + HID); vv = Act<T>::ld(row + 2 * HID);
        }
        sm.q[tok][d] = qv * scale; sm.k[tok][d] = kv; sm.v[tok][d] = vv;
    }
    __syncthreads();
    {   // S = (q*scale) k^T ; thread -> row i, 16 columns
        const int i = tid >> 2, j0 = (tid & 3) * 16;
        for (int j = j0; j < j0 + 16; ++j) {
            float s = 0.f;
#pragma unroll
            for (int d = 0; d < DH; ++d) s += sm.q[i][d] * sm.k[j][d];
            sm.s[i][j] = (j < n) ? s : -INFINITY;
        }
    }
    __syncthreads();
    {   // row softmax: warp per row
        const int warp = tid >> 5, lane = tid & 31;
        for (int i = warp; i < AT_N; i += (blockDim.x >> 5)) {
            float a = sm.s[i][lane], c = sm.s[i][lane + 32];
            float mx = warp_max(fmaxf(a, c));
            a = __expf(a - mx); c = __expf(c - mx);
            float inv = 1.f / warp_sum(a + c);
            sm.s[i][lane] = a * inv; sm.s[i][lane + 32] = c * inv;
        }
    }
    __syncthreads();
}

template <typename T>
__global__ void __launch_bounds__(256) attn_fwd_kernel(const T* __restrict__ qkv, T* __restrict__ out, int n, int heads,
                                                       float scale) {
    pdl_trigger();
    pdl_wait();
    extern __shared__ __align__(16) unsigned char raw[];
    AttnSmemF& sm = *reinterpret_cast<AttnSmemF*>(raw);
    const int h = blockIdx.x, b = blockIdx.y, HID = heads * DH, tid = threadIdx.x;
    attn_load_scores(qkv, sm, b, h, n, HID, scale);
    const int i = tid >> 2, d0 = (tid & 3) * 8;
    float o[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int j = 0; j < AT_N; ++j) {
        float p = sm.s[i][j];
#pragma unroll
        for (int k = 0; k < 8; ++k) o[k] += p * sm.v[j][d0 + k];
    }
    if (i < n) st8(out + ((size_t)b * n + i) * HID + h * DH + d0, o);
}

template <typename T>
__global__ void __launch_bounds__(256) attn_bwd_kernel(const T* __restrict__ qkv, const T* __restrict__ dout,
                                                       T* __restrict__ dqkv, int n, int heads, float scale) {
    pdl_trigger();
    pdl_wait();
    extern __shared__ __align__(16) unsigned char raw[];
    AttnSmemB& sm = *reinterpret_cast<AttnSmemB*>(raw);
    const int h = blockIdx.x, b = blockIdx.y, HID = heads * DH, tid = threadIdx.x;
    for (int i = tid; i < AT_N * DH; i += blockDim.x) {
        int tok = i / DH, d = i % DH;
        sm.g[tok][d] = (tok < n) ? Act<T>::ld(dout + ((size_t)b * n + tok) * HID + h * DH + d) : 0.f;
    }
    attn_load_scores(qkv, sm, b, h, n, HID, scale);      // sm.q already holds q*scale; sm.s = P
    const int i = tid >> 2;
    {   // dP = g v^T ; dS = P * (dP - rowdot)
        const int j0 = (tid & 3) * 16;
        float part = 0.f;
        for (int j = j0; j < j0 + 16; ++j) {
            float s = 0.f;
#pragma unroll
            for (int d = 0; d < DH; ++d) s += sm.g[i][d] * sm.v[j][d];
            sm.ds[i][j] = s;
            part += s * sm.s[i][j];
        }
        part += __shfl_xor_sync(0xffffffffu, part, 1);
        part += __shfl_xor_sync(0xffffffffu, part, 2);
        for (int j = j0; j < j0 + 16; ++j) sm.ds[i][j] = sm.s[i][j] * (sm.ds[i][j] - part);
    }
    __syncthreads();
    const int d0 = (tid & 3) * 8;
    float dq[8] = {0, 0, 0, 0, 0, 0, 0, 0}, dk[8] = {0, 0, 0, 0, 0, 0, 0, 0}, dv[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int j = 0; j < AT_N; ++j) {
        float dsij = sm.ds[i][j];        // row i (queries)
        float dsji = sm.ds[j][i];        // column i (keys)
        float pji = sm.s[j][i];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            dq[k] += dsij * sm.k[j][d0 + k];
            dk[k] += dsji * sm.q[j][d0 + k];      // q is pre-scaled
            dv[k] += pji * sm.g[j][d0 + k];
        }
    }
    if (i < n) {
#pragma unroll
        for (int k = 0; k < 8; ++k) dq[k] *= scale;
        T* row = dqkv + ((size_t)b * n + i) * 3 * HID + h * DH + d0;
        st8(row, dq); st8(row + HID, dk); st8(row + 2 * HID, dv);
    }
}

// tensor-core (mma.sync) versions for bf16 activations and 8 heads (attention_mma.cu)
// attention_small.cu: whole (sample, head) problem in one CTA for N <= 256 tokens
bool la_small_supported(int N, int dtype);
int la_small_fwd(const void* qkv, void* out, float* ctx, float* kmax, float* kzinv, int B, int N, int heads, float scale,
                 cudaStream_t st);
// attention_mid.cu: the 64-token softmax attention on mma.sync (bf16)
bool attn_mid_supported(int n_tokens, int dtype);
int attn_mid_fwd(const void* qkv, void* out, int B, int heads, float scale, cudaStream_t st);
int attn_mid_bwd(const void* qkv, const void* dout, void* dqkv, int B, int heads, float scale, cudaStream_t st);
int la_mma_ctx(int mode, const void* qkv, const void* dout, const float* part, int n_stat_chunks, float* kmax,
               float* kzinv, float* ctx, int B, int N, float scale, cudaStream_t st);
int la_mma_out(const void* qkv, const float* ctx, void* out, int B, int N, float scale, cudaStream_t st);
int la_mma_bwd(const void* qkv, const void* dout, const float* ctx, const float* dctx, const float* kmax,
               const float* kzinv, void* dqkv, int B, int N, float scale, cudaStream_t st);
int la_mma_chunk_px(int B, int N);

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
    const float scale = 0.17677669529663687f;   // 32^-0.5
    const int path = la_fwd_path(N, heads, dtype);
    if (path == LA_FWD_SMALL)     // 8x8 level: the whole (sample, head) problem in one CTA, one launch
        return la_small_fwd(qkv, out, ctx, kmax, kzinv, B, N, heads, scale, st);
    PIDM_CUDA(cudaMemsetAsync(ctx, 0, (size_t)B * heads * DH * DH * sizeof(float), st));
    if (path == LA_FWD_MMA) {
        PIDM_CUDA(launch_plain(la_kstats_kernel<__nv_bfloat16>, dim3(dim3(chunks, B)), dim3(256), (size_t)(la_kstats_smem(HID)), st, (const __nv_bfloat16*)qkv, workspace, N, HID, rpc));
        if (int e = la_mma_ctx(0, qkv, nullptr, workspace, chunks, kmax, kzinv, ctx, B, N, scale, st)) return e;
        if (int e = la_mma_out(qkv, ctx, out, B, N, scale, st)) return e;
        PIDM_LAUNCH_CHECK("linattn_fwd");
        return 0;
    }
    const int crpc = la_ctx_rows(N);
    PIDM_DISPATCH_DTYPE(dtype, {
        PIDM_CUDA(launch_plain(la_kstats_kernel<T>, dim3(dim3(chunks, B)), dim3(la_kstats_block(HID)), (size_t)(la_kstats_smem(HID)), st, (const T*)qkv, workspace, N, HID, rpc));
        PIDM_CUDA(launch_plain(la_context_kernel<T, 0>, dim3(dim3((N + crpc - 1) / crpc, heads, B)), dim3(256), (size_t)(0), st, (const T*)qkv, nullptr, workspace, chunks, kmax, kzinv, ctx, N, heads, crpc, scale));
        PIDM_CUDA(launch_plain(la_out_kernel<T>, dim3((unsigned)((long long)B * N / 32)), dim3(32 * heads), (size_t)(heads * DH * DH * sizeof(float)), st, (const T*)qkv, ctx, (T*)out, N, heads, scale));
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
    const float scale = 0.17677669529663687f;
    PIDM_CUDA(cudaMemsetAsync(dctx, 0, (size_t)B * heads * DH * DH * sizeof(float), st));
    if (la_bwd_mma(N, heads, dtype)) {
        if (int e = la_mma_ctx(1, qkv, dout, nullptr, 0, nullptr, nullptr, dctx, B, N, scale, st)) return e;
        return la_mma_bwd(qkv, dout, ctx, dctx, kmax, kzinv, dqkv, B, N, scale, st);
    }
    const int crpc = la_ctx_rows(N);
    PIDM_DISPATCH_DTYPE(dtype, {
        PIDM_CUDA(launch_plain(la_context_kernel<T, 1>, dim3(dim3((N + crpc - 1) / crpc, heads, B)), dim3(256), (size_t)(0), st, (const T*)qkv, (const T*)dout, nullptr, 0, nullptr, nullptr, dctx, N, heads, crpc, scale));
        PIDM_CUDA(launch_plain(la_bwd_pixel_kernel<T>, dim3(dim3((unsigned)((long long)B * N / 32), heads / LA_HB)), dim3(32 * LA_HB), (size_t)(0), st, (const T*)qkv, (const T*)dout, ctx, dctx, kmax, kzinv, (T*)dqkv, N, heads, scale));
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
    const int cpx = la_mma_chunk_px(B, N);
    const int v[8] = {fwd, bwd, la_chunks(N), la_stat_rows(N), crpc, (N + crpc - 1) / crpc, cpx, (N + cpx - 1) / cpx};
    for (int i = 0; i < 8; ++i) out[i] = v[i];
    return 0;
}

extern "C" int pidm_attn_fwd(const void* qkv, void* out, int B, int n_tokens, int heads, int dtype, void* stream) {
    PIDM_REQUIRE(n_tokens >= 1 && n_tokens <= AT_N, "attn: at most %d tokens supported (got %d)", AT_N, n_tokens);
    const float scale = 0.17677669529663687f;
    if (attn_mid_supported(n_tokens, dtype)) return attn_mid_fwd(qkv, out, B, heads, scale, (cudaStream_t)stream);
    PIDM_DISPATCH_DTYPE(dtype, {
        PIDM_CUDA(allow_smem(attn_fwd_kernel<T>, sizeof(AttnSmemF)));
        PIDM_CUDA(launch_plain(attn_fwd_kernel<T>, dim3(dim3(heads, B)), dim3(256), (size_t)(sizeof(AttnSmemF)), (cudaStream_t)stream, (const T*)qkv, (T*)out,
                                                                                              n_tokens, heads, scale));
    });
    PIDM_LAUNCH_CHECK("attn_fwd");
    return 0;
}

extern "C" int pidm_attn_bwd(const void* qkv, const void* dout, void* dqkv, int B, int n_tokens, int heads, int dtype,
                             void* stream) {
    PIDM_REQUIRE(n_tokens >= 1 && n_tokens <= AT_N, "attn: at most %d tokens supported (got %d)", AT_N, n_tokens);
    const float scale = 0.17677669529663687f;
    if (attn_mid_supported(n_tokens, dtype)) return attn_mid_bwd(qkv, dout, dqkv, B, heads, scale, (cudaStream_t)stream);
    PIDM_DISPATCH_DTYPE(dtype, {
        PIDM_CUDA(allow_smem(attn_bwd_kernel<T>, sizeof(AttnSmemB)));
        PIDM_CUDA(launch_plain(attn_bwd_kernel<T>, dim3(dim3(heads, B)), dim3(256), (size_t)(sizeof(AttnSmemB)), (cudaStream_t)stream, (const T*)qkv, (const T*)dout, (T*)dqkv, n_tokens, heads, scale));
    });
    PIDM_LAUNCH_CHECK("attn_bwd");
    return 0;
}
