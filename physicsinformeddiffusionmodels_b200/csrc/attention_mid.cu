// Softmax attention over the 64 tokens of the 8x8 level (reference unet_model.py:300-334, the `mid_spatial_attn` of the
// U-Net), bf16 activations, dim_head = 32, on mma.sync tensor-core tiles: one CTA of four warps per (sample, head),
// warp w owns the 16 query rows [16w, 16w + 16).
//
//   S = s q k^T     P = softmax_j(S)     out = P v
//   dP = dout v^T   dS = P * (dP - sum_j P dP)      dq = s dS k     dk = s dS^T q     dv = P^T dout
//
// The CUDA-core version of these kernels (attention.cu: attn_fwd_kernel / attn_bwd_kernel, still used for fp32
// activations and for fewer than 64 tokens) spends ~3.8 k shared-memory loads per thread on five 64x64x32 products;
// here the five products are 40 MMAs per warp, the probabilities
// never leave the registers in forward, and backward stages P and dS once (bf16) for the two key-side products.
#include "common.cuh"
#include "mma_util.cuh"
#include "pidm.h"

namespace pidm {

constexpr int AM_N = 64;                      // tokens
constexpr int AM_D = 32;                      // dim_head
constexpr int AM_PITCH = LW_PITCH;            // bf16 per [token][32] row: 80 B, conflict-free ldmatrix
constexpr int AM_SPITCH = AM_N + 8;           // bf16 per [query][64] row of the staged P / dS: 144 B
constexpr int AM_THREADS = 128;

// [64 tokens][32] head slice (row stride `stride` elements) -> smem [64][AM_PITCH]
__device__ __forceinline__ void am_load(__nv_bfloat16* dst, const __nv_bfloat16* __restrict__ src, size_t stride) {
    for (int i = threadIdx.x; i < AM_N * 4; i += AM_THREADS) {
        const int n = i >> 2, o = (i & 3) * 8;
        *reinterpret_cast<uint4*>(dst + n * AM_PITCH + o) = *reinterpret_cast<const uint4*>(src + (size_t)n * stride + o);
    }
}

// acc[nt] (nt = 0..7: columns nt*8 + 2t, +1 of rows g / g + 8) = A(rows m0..m0+15 of X [64][32]) * Y^T, Y [64][32]
__device__ __forceinline__ void am_rows_times_rows_t(float (&acc)[8][4], const __nv_bfloat16* X, const __nv_bfloat16* Y,
                                                     int m0, int lane) {
#pragma unroll
    for (int nt = 0; nt < 8; ++nt)
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[nt][i] = 0.f;
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
        uint32_t a[4];
        frag_a_rowmajor(a, X, AM_PITCH, m0, ks * 16, lane);
#pragma unroll
        for (int np = 0; np < 4; ++np) {          // pairs of n-tiles: tokens np*16 .. np*16 + 15
            uint32_t b[4];
            frag_b_nrows(b, Y, AM_PITCH, np * 16, ks * 16, lane);
            mma_bf16(acc[2 * np], a, b[0], b[1]);
            mma_bf16(acc[2 * np + 1], a, b[2], b[3]);
        }
    }
}

// accumulator fragments [16][64] -> the four A fragments (k16 steps over the 64 columns) of the same matrix, bf16
__device__ __forceinline__ void am_c_to_a(uint32_t (&a)[4][4], const float (&c)[8][4]) {
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
        a[ks][0] = pack_bf16(c[2 * ks][0], c[2 * ks][1]);
        a[ks][1] = pack_bf16(c[2 * ks][2], c[2 * ks][3]);
        a[ks][2] = pack_bf16(c[2 * ks + 1][0], c[2 * ks + 1][1]);
        a[ks][3] = pack_bf16(c[2 * ks + 1][2], c[2 * ks + 1][3]);
    }
}

// o[nt] (nt = 0..3: channels) = A(16 x 64, fragments a) * Y, Y [64 tokens][32] (rows = K index)
__device__ __forceinline__ void am_frag_times_rows(float (&o)[4][4], const uint32_t (&a)[4][4], const __nv_bfloat16* Y, int lane) {
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
        for (int i = 0; i < 4; ++i) o[nt][i] = 0.f;
#pragma unroll
    for (int ks = 0; ks < 4; ++ks)
#pragma unroll
        for (int np = 0; np < 2; ++np) {
            uint32_t b[4];
            frag_b_krows(b, Y, AM_PITCH, ks * 16, np * 16, lane);
            mma_bf16(o[2 * np], a[ks], b[0], b[1]);
            mma_bf16(o[2 * np + 1], a[ks], b[2], b[3]);
        }
}

// in-place softmax over the 64 columns of the two rows (g, g + 8) a thread shares with its quad; s = scale * s first
__device__ __forceinline__ void am_softmax(float (&s)[8][4], float scale) {
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        float mx = -INFINITY;
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
            s[nt][half * 2] *= scale; s[nt][half * 2 + 1] *= scale;
            mx = fmaxf(mx, fmaxf(s[nt][half * 2], s[nt][half * 2 + 1]));
        }
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        float z = 0.f;
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
            s[nt][half * 2] = __expf(s[nt][half * 2] - mx);
            s[nt][half * 2 + 1] = __expf(s[nt][half * 2 + 1] - mx);
            z += s[nt][half * 2] + s[nt][half * 2 + 1];
        }
        z += __shfl_xor_sync(0xffffffffu, z, 1);
        z += __shfl_xor_sync(0xffffffffu, z, 2);
        const float inv = 1.f / z;
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) { s[nt][half * 2] *= inv; s[nt][half * 2 + 1] *= inv; }
    }
}

// rows g / g + 8 of a [16][32] accumulator tile -> global rows (64-byte head slices), bf16
__device__ __forceinline__ void am_store(__nv_bfloat16* __restrict__ dst, size_t stride, const float (&o)[4][4], float mul,
                                         int lane) {
    const int g = lane >> 2, t = lane & 3;
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
        *reinterpret_cast<uint32_t*>(dst + (size_t)g * stride + nt * 8 + 2 * t) = pack_bf16(o[nt][0] * mul, o[nt][1] * mul);
        *reinterpret_cast<uint32_t*>(dst + (size_t)(g + 8) * stride + nt * 8 + 2 * t) = pack_bf16(o[nt][2] * mul, o[nt][3] * mul);
    }
}

__global__ void __launch_bounds__(AM_THREADS) attn_mid_fwd_kernel(const __nv_bfloat16* __restrict__ qkv,
                                                                  __nv_bfloat16* __restrict__ out, int heads, float scale) {
    pdl_trigger();
    pdl_wait();
    __shared__ __align__(16) __nv_bfloat16 Q[AM_N * AM_PITCH], K[AM_N * AM_PITCH], V[AM_N * AM_PITCH];
    const int h = blockIdx.x, b = blockIdx.y, HID = heads * AM_D, lane = threadIdx.x & 31, m0 = (threadIdx.x >> 5) * 16;
    const size_t stride = 3 * (size_t)HID;
    const __nv_bfloat16* base = qkv + (size_t)b * AM_N * stride + h * AM_D;
    am_load(Q, base, stride);
    am_load(K, base + HID, stride);
    am_load(V, base + 2 * HID, stride);
    __syncthreads();
    float s[8][4];
    am_rows_times_rows_t(s, Q, K, m0, lane);
    am_softmax(s, scale);
    uint32_t p[4][4];
    am_c_to_a(p, s);
    float o[4][4];
    am_frag_times_rows(o, p, V, lane);
    am_store(out + ((size_t)b * AM_N + m0) * HID + h * AM_D, (size_t)HID, o, 1.f, lane);
}

__global__ void __launch_bounds__(AM_THREADS) attn_mid_bwd_kernel(const __nv_bfloat16* __restrict__ qkv,
                                                                  const __nv_bfloat16* __restrict__ dout,
                                                                  __nv_bfloat16* __restrict__ dqkv, int heads, float scale) {
    pdl_trigger();
    pdl_wait();
    __shared__ __align__(16) __nv_bfloat16 Q[AM_N * AM_PITCH], K[AM_N * AM_PITCH], V[AM_N * AM_PITCH], G[AM_N * AM_PITCH];
    __shared__ __align__(16) __nv_bfloat16 Ps[AM_N * AM_SPITCH], Ds[AM_N * AM_SPITCH];
    const int h = blockIdx.x, b = blockIdx.y, HID = heads * AM_D, lane = threadIdx.x & 31, m0 = (threadIdx.x >> 5) * 16;
    const int g = lane >> 2, t = lane & 3;
    const size_t stride = 3 * (size_t)HID;
    const __nv_bfloat16* base = qkv + (size_t)b * AM_N * stride + h * AM_D;
    am_load(Q, base, stride);
    am_load(K, base + HID, stride);
    am_load(V, base + 2 * HID, stride);
    am_load(G, dout + (size_t)b * AM_N * HID + h * AM_D, (size_t)HID);
    __syncthreads();
    float s[8][4], dp[8][4];
    am_rows_times_rows_t(s, Q, K, m0, lane);          // S
    am_softmax(s, scale);                             // P
    am_rows_times_rows_t(dp, G, V, m0, lane);         // dP = dout v^T
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        float dot = 0.f;
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) dot += s[nt][half * 2] * dp[nt][half * 2] + s[nt][half * 2 + 1] * dp[nt][half * 2 + 1];
        dot += __shfl_xor_sync(0xffffffffu, dot, 1);
        dot += __shfl_xor_sync(0xffffffffu, dot, 2);
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {              // dp <- dS
            dp[nt][half * 2] = s[nt][half * 2] * (dp[nt][half * 2] - dot);
            dp[nt][half * 2 + 1] = s[nt][half * 2 + 1] * (dp[nt][half * 2 + 1] - dot);
        }
    }
    // stage P and dS (bf16, [query][key]) for the key-side products of all four warps
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
        *reinterpret_cast<uint32_t*>(Ps + (m0 + g) * AM_SPITCH + nt * 8 + 2 * t) = pack_bf16(s[nt][0], s[nt][1]);
        *reinterpret_cast<uint32_t*>(Ps + (m0 + g + 8) * AM_SPITCH + nt * 8 + 2 * t) = pack_bf16(s[nt][2], s[nt][3]);
        *reinterpret_cast<uint32_t*>(Ds + (m0 + g) * AM_SPITCH + nt * 8 + 2 * t) = pack_bf16(dp[nt][0], dp[nt][1]);
        *reinterpret_cast<uint32_t*>(Ds + (m0 + g + 8) * AM_SPITCH + nt * 8 + 2 * t) = pack_bf16(dp[nt][2], dp[nt][3]);
    }
    __nv_bfloat16* drow = dqkv + ((size_t)b * AM_N + m0) * stride + h * AM_D;
    {   // dq = s dS k  (query rows of this warp)
        uint32_t a[4][4];
        am_c_to_a(a, dp);
        float o[4][4];
        am_frag_times_rows(o, a, K, lane);
        am_store(drow, stride, o, scale, lane);
    }
    __syncthreads();
    // key rows j = m0 .. m0 + 15:  dk[j][:] = s sum_i dS[i][j] q[i][:],  dv[j][:] = sum_i P[i][j] dout[i][:]
    float dk[4][4], dv[4][4];
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
        for (int i = 0; i < 4; ++i) { dk[nt][i] = 0.f; dv[nt][i] = 0.f; }
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {                  // 16 queries per step
        uint32_t ad[4], ap[4];
        frag_a_kmajor(ad, Ds, AM_SPITCH, ks * 16, m0, lane);
        frag_a_kmajor(ap, Ps, AM_SPITCH, ks * 16, m0, lane);
#pragma unroll
        for (int np = 0; np < 2; ++np) {
            uint32_t bq[4], bg[4];
            frag_b_krows(bq, Q, AM_PITCH, ks * 16, np * 16, lane);
            frag_b_krows(bg, G, AM_PITCH, ks * 16, np * 16, lane);
            mma_bf16(dk[2 * np], ad, bq[0], bq[1]);
            mma_bf16(dk[2 * np + 1], ad, bq[2], bq[3]);
            mma_bf16(dv[2 * np], ap, bg[0], bg[1]);
            mma_bf16(dv[2 * np + 1], ap, bg[2], bg[3]);
        }
    }
    am_store(drow + HID, stride, dk, scale, lane);
    am_store(drow + 2 * HID, stride, dv, 1.f, lane);
}

// entry points used by attention.cu
bool attn_mid_supported(int n_tokens, int dtype) { return dtype == PIDM_BF16 && n_tokens == AM_N; }

int attn_mid_fwd(const void* qkv, void* out, int B, int heads, float scale, cudaStream_t st) {
    PIDM_CUDA(launch_plain(attn_mid_fwd_kernel, dim3(heads, B), dim3(AM_THREADS), (size_t)0, st, (const __nv_bfloat16*)qkv,
                           (__nv_bfloat16*)out, heads, scale));
    PIDM_LAUNCH_CHECK("attn_mid_fwd");
    return 0;
}

int attn_mid_bwd(const void* qkv, const void* dout, void* dqkv, int B, int heads, float scale, cudaStream_t st) {
    PIDM_CUDA(launch_plain(attn_mid_bwd_kernel, dim3(heads, B), dim3(AM_THREADS), (size_t)0, st, (const __nv_bfloat16*)qkv,
                           (const __nv_bfloat16*)dout, (__nv_bfloat16*)dqkv, heads, scale));
    PIDM_LAUNCH_CHECK("attn_mid_bwd");
    return 0;
}

}  // namespace pidm
