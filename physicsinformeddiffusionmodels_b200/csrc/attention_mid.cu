// Softmax attention over the 64 tokens of the 8x8 level (reference unet_model.py:300-334, the `mid_spatial_attn` of the
// U-Net), bf16 activations, dim_head = 32, on mma.sync tensor-core tiles: one CTA of four warps per (sample, head),
// warp w owns the 16 query rows [16w, 16w + 16).
//
//   S = s q k^T     P = softmax_j(S)     out = P v
//   dP = dout v^T   dS = P * (dP - sum_j P dP)      dq = s dS k     dk = s dS^T q     dv = P^T dout
//
// The CUDA-core version of these kernels (attn_fwd_kernel / attn_bwd_kernel below, still used for fp32 activations
// and for fewer than 64 tokens) spends ~3.8 k shared-memory loads per thread on five 64x64x32 products;
// here the five products are 40 MMAs per warp, the probabilities
// never leave the registers in forward, and backward stages P and dS once (bf16) for the two key-side products.
#include "common.cuh"
#include "mma_util.cuh"
#include "pidm.h"

namespace pidm {

constexpr int AT_N = 64;                      // tokens: the most either pair of kernels takes
constexpr int AM_PITCH = LW_PITCH;            // bf16 per [token][32] row: 80 B, conflict-free ldmatrix
constexpr int AM_SPITCH = AT_N + 8;           // bf16 per [query][64] row of the staged P / dS: 144 B
constexpr int AM_THREADS = 128;

// [64 tokens][32] head slice (row stride `stride` elements) -> smem [64][AM_PITCH]
__device__ __forceinline__ void mid_load(__nv_bfloat16* dst, const __nv_bfloat16* __restrict__ src, size_t stride) {
    for (int i = threadIdx.x; i < AT_N * 4; i += AM_THREADS) {
        const int n = i >> 2, o = (i & 3) * 8;
        *reinterpret_cast<uint4*>(dst + n * AM_PITCH + o) = *reinterpret_cast<const uint4*>(src + (size_t)n * stride + o);
    }
}

// acc[nt] (nt = 0..7: columns nt*8 + 2t, +1 of rows g / g + 8) = A(rows m0..m0+15 of X [64][32]) * Y^T, Y [64][32]
__device__ __forceinline__ void mid_rows_times_rows_t(float (&acc)[8][4], const __nv_bfloat16* X, const __nv_bfloat16* Y,
                                                     int m0, int lane) {
    zero(acc);
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

// o[nt] (nt = 0..3: channels) = A(16 x 64, fragments a) * Y, Y [64 tokens][32] (rows = K index)
__device__ __forceinline__ void mid_frag_times_rows(float (&o)[4][4], const uint32_t (&a)[4][4], const __nv_bfloat16* Y,
                                                    int lane) {
    zero(o);
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

// S = scale * S, then the softmax of its rows g, g + 8 over the 64 keys
__device__ __forceinline__ void scale_then_softmax(float (&s)[8][4], float scale) {
#pragma unroll
    for (int nt = 0; nt < 8; ++nt)
#pragma unroll
        for (int i = 0; i < 4; ++i) s[nt][i] *= scale;
    frag_softmax(s, 1.f);
}

__global__ void __launch_bounds__(AM_THREADS) attn_mid_fwd_kernel(const __nv_bfloat16* __restrict__ qkv,
                                                                  __nv_bfloat16* __restrict__ out, int heads, float scale) {
    pdl_trigger();
    pdl_wait();
    __shared__ __align__(16) __nv_bfloat16 Q[AT_N * AM_PITCH], K[AT_N * AM_PITCH], V[AT_N * AM_PITCH];
    const int h = blockIdx.x, b = blockIdx.y, HID = heads * DH, lane = threadIdx.x & 31, m0 = (threadIdx.x >> 5) * 16;
    const size_t stride = 3 * (size_t)HID;
    const __nv_bfloat16* base = qkv + (size_t)b * AT_N * stride + h * DH;
    mid_load(Q, base, stride);
    mid_load(K, base + HID, stride);
    mid_load(V, base + 2 * HID, stride);
    __syncthreads();
    float s[8][4];
    mid_rows_times_rows_t(s, Q, K, m0, lane);
    scale_then_softmax(s, scale);
    uint32_t p[4][4];
    c_to_a(p, s);
    float o[4][4];
    mid_frag_times_rows(o, p, V, lane);
    store_rows_bf16(out + ((size_t)b * AT_N + m0) * HID + h * DH, (size_t)HID, o, lane);
}

__global__ void __launch_bounds__(AM_THREADS) attn_mid_bwd_kernel(const __nv_bfloat16* __restrict__ qkv,
                                                                  const __nv_bfloat16* __restrict__ dout,
                                                                  __nv_bfloat16* __restrict__ dqkv, int heads, float scale) {
    pdl_trigger();
    pdl_wait();
    __shared__ __align__(16) __nv_bfloat16 Q[AT_N * AM_PITCH], K[AT_N * AM_PITCH], V[AT_N * AM_PITCH], G[AT_N * AM_PITCH];
    __shared__ __align__(16) __nv_bfloat16 Ps[AT_N * AM_SPITCH], Ds[AT_N * AM_SPITCH];
    const int h = blockIdx.x, b = blockIdx.y, HID = heads * DH, lane = threadIdx.x & 31, m0 = (threadIdx.x >> 5) * 16;
    const size_t stride = 3 * (size_t)HID;
    const __nv_bfloat16* base = qkv + (size_t)b * AT_N * stride + h * DH;
    mid_load(Q, base, stride);
    mid_load(K, base + HID, stride);
    mid_load(V, base + 2 * HID, stride);
    mid_load(G, dout + (size_t)b * AT_N * HID + h * DH, (size_t)HID);
    __syncthreads();
    float s[8][4], dp[8][4];
    mid_rows_times_rows_t(s, Q, K, m0, lane);          // S
    scale_then_softmax(s, scale);                     // P
    mid_rows_times_rows_t(dp, G, V, m0, lane);         // dP = dout v^T
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        float dot = 0.f;
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) dot += s[nt][half * 2] * dp[nt][half * 2] + s[nt][half * 2 + 1] * dp[nt][half * 2 + 1];
        dot = quad_sum(dot);
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {              // dp <- dS
            dp[nt][half * 2] = s[nt][half * 2] * (dp[nt][half * 2] - dot);
            dp[nt][half * 2 + 1] = s[nt][half * 2 + 1] * (dp[nt][half * 2 + 1] - dot);
        }
    }
    // stage P and dS (bf16, [query][key]) for the key-side products of all four warps
    store_rows_bf16(Ps + m0 * AM_SPITCH, AM_SPITCH, s, lane);
    store_rows_bf16(Ds + m0 * AM_SPITCH, AM_SPITCH, dp, lane);
    __nv_bfloat16* drow = dqkv + ((size_t)b * AT_N + m0) * stride + h * DH;
    {   // dq = s dS k  (query rows of this warp)
        uint32_t a[4][4];
        c_to_a(a, dp);
        float o[4][4];
        mid_frag_times_rows(o, a, K, lane);
        store_rows_bf16(drow, stride, o, lane, scale);
    }
    __syncthreads();
    // key rows j = m0 .. m0 + 15:  dk[j][:] = s sum_i dS[i][j] q[i][:],  dv[j][:] = sum_i P[i][j] dout[i][:]
    float dk[4][4], dv[4][4];
    zero(dk);
    zero(dv);
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
    store_rows_bf16(drow + HID, stride, dk, lane, scale);
    store_rows_bf16(drow + 2 * HID, stride, dv, lane);
}

// ---- CUDA-core softmax attention over n <= 64 tokens, fp32 math, one CTA per (head, sample) --------------------
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

// host launchers of the mma.sync kernels
static bool attn_mid_supported(int n_tokens, int dtype) { return dtype == PIDM_BF16 && n_tokens == AT_N; }

static int attn_mid_fwd(const void* qkv, void* out, int B, int heads, float scale, cudaStream_t st) {
    PIDM_CUDA(launch_plain(attn_mid_fwd_kernel, dim3(heads, B), dim3(AM_THREADS), (size_t)0, st, (const __nv_bfloat16*)qkv,
                           (__nv_bfloat16*)out, heads, scale));
    PIDM_LAUNCH_CHECK("attn_mid_fwd");
    return 0;
}

static int attn_mid_bwd(const void* qkv, const void* dout, void* dqkv, int B, int heads, float scale, cudaStream_t st) {
    PIDM_CUDA(launch_plain(attn_mid_bwd_kernel, dim3(heads, B), dim3(AM_THREADS), (size_t)0, st, (const __nv_bfloat16*)qkv,
                           (const __nv_bfloat16*)dout, (__nv_bfloat16*)dqkv, heads, scale));
    PIDM_LAUNCH_CHECK("attn_mid_bwd");
    return 0;
}

}  // namespace pidm
using namespace pidm;

extern "C" int pidm_attn_fwd(const void* qkv, void* out, int B, int n_tokens, int heads, int dtype, void* stream) {
    PIDM_REQUIRE(n_tokens >= 1 && n_tokens <= AT_N, "attn: at most %d tokens supported (got %d)", AT_N, n_tokens);
    if (attn_mid_supported(n_tokens, dtype)) return attn_mid_fwd(qkv, out, B, heads, ATTN_SCALE, (cudaStream_t)stream);
    PIDM_DISPATCH_DTYPE(dtype, {
        PIDM_CUDA(allow_smem(attn_fwd_kernel<T>, sizeof(AttnSmemF)));
        PIDM_CUDA(launch_plain(attn_fwd_kernel<T>, dim3(dim3(heads, B)), dim3(256), (size_t)(sizeof(AttnSmemF)), (cudaStream_t)stream, (const T*)qkv, (T*)out,
                                                                                              n_tokens, heads, ATTN_SCALE));
    });
    PIDM_LAUNCH_CHECK("attn_fwd");
    return 0;
}

extern "C" int pidm_attn_bwd(const void* qkv, const void* dout, void* dqkv, int B, int n_tokens, int heads, int dtype,
                             void* stream) {
    PIDM_REQUIRE(n_tokens >= 1 && n_tokens <= AT_N, "attn: at most %d tokens supported (got %d)", AT_N, n_tokens);
    if (attn_mid_supported(n_tokens, dtype)) return attn_mid_bwd(qkv, dout, dqkv, B, heads, ATTN_SCALE, (cudaStream_t)stream);
    PIDM_DISPATCH_DTYPE(dtype, {
        PIDM_CUDA(allow_smem(attn_bwd_kernel<T>, sizeof(AttnSmemB)));
        PIDM_CUDA(launch_plain(attn_bwd_kernel<T>, dim3(dim3(heads, B)), dim3(256), (size_t)(sizeof(AttnSmemB)), (cudaStream_t)stream, (const T*)qkv, (const T*)dout, (T*)dqkv, n_tokens, heads, ATTN_SCALE));
    });
    PIDM_LAUNCH_CHECK("attn_bwd");
    return 0;
}
