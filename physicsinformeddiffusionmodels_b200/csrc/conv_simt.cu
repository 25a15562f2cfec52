// Generic implicit-GEMM convolution on NHWC activations (fp32 accumulate, CUDA cores).
// This is the geometry-complete path: any KHxKW / stride / padding, regular ("gather from input") or
// transposed addressing, forward / dgrad / wgrad, fp32 or bf16 activations.  It is the parity anchor
// for the tensor-core (wgmma) tile kernel in conv_tc.cu (which takes the stride-1 layers that carry the FLOPs) and
// runs the layers that kernel does not cover (7x7 stem, 4x4/s2 down, 4x4/s2 transposed up, wgrad).
//
//   y[m, n] = sum_k A(m, k) * Wp[n, k] (+ bias[n]) (+ residual[m, n]),  m = (b, oh, ow),  k = tap*Cin + c
//   regular    : A(m,k) = x[b, oh*s - p + r, ow*s - p + q, c]
//   transposed : A(m,k) = x[b, (oh + p - r)/s, (ow + p - q)/s, c]   when divisible and in range
// Forward conv = regular; its dgrad = transposed over dy.  ConvTranspose forward = transposed; its dgrad =
// regular over dy.  Packed weights Wp[n][tap*Cin + c] are produced by pidm_pack_weights.
#include "common.cuh"
#include "pidm.h"

namespace pidm {

struct ConvGeom {
    int B, H, W, Cin;     // input  [B,H,W,Cin]
    int Ho, Wo, Cout;     // output [B,Ho,Wo,Cout]
    int KH, KW, stride, pad, transposed;
};

constexpr int CS_BM = 64, CS_BN = 64, CS_BK = 16, CS_THREADS = 256;

template <typename T>
__device__ __forceinline__ void gather_a4(const T* __restrict__ x, const ConvGeom& g, bool m_ok, int b, int oh, int ow,
                                          int k, int K, float v[4]) {
    v[0] = v[1] = v[2] = v[3] = 0.f;
    if (!m_ok || k >= K) return;
    int tap = k / g.Cin, c = k - tap * g.Cin;
    int r = tap / g.KW, q = tap - r * g.KW;
    int ih, iw;
    if (!g.transposed) {
        ih = oh * g.stride - g.pad + r;
        iw = ow * g.stride - g.pad + q;
        if (ih < 0 || ih >= g.H || iw < 0 || iw >= g.W) return;
    } else {
        int th = oh + g.pad - r, tw = ow + g.pad - q;
        if (th < 0 || tw < 0) return;
        if (g.stride > 1) {
            if ((th % g.stride) || (tw % g.stride)) return;
            ih = th / g.stride; iw = tw / g.stride;
        } else { ih = th; iw = tw; }
        if (ih >= g.H || iw >= g.W) return;
    }
    ld4(x + (((size_t)b * g.H + ih) * g.W + iw) * g.Cin + c, v);
}

template <typename T>
__global__ void __launch_bounds__(CS_THREADS) conv_simt_kernel(const T* __restrict__ x, const T* __restrict__ wp,
                                                               const float* __restrict__ bias,
                                                               const T* __restrict__ residual, T* __restrict__ y,
                                                               ConvGeom g) {
    __shared__ __align__(16) float As[CS_BK][CS_BM + 4];
    __shared__ __align__(16) float Bs[CS_BK][CS_BN + 4];
    const int tid = threadIdx.x;
    const long long M = (long long)g.B * g.Ho * g.Wo;
    const int K = g.KH * g.KW * g.Cin;
    const long long m0 = (long long)blockIdx.x * CS_BM;
    const int n0 = blockIdx.y * CS_BN;
    // loader coordinates
    const int lrow = tid >> 2, lk = (tid & 3) * 4;
    const long long lm = m0 + lrow;
    const bool m_ok = lm < M;
    int lb = 0, loh = 0, low = 0;
    if (m_ok) {
        lb = (int)(lm / (g.Ho * g.Wo));
        int rem = (int)(lm - (long long)lb * g.Ho * g.Wo);
        loh = rem / g.Wo; low = rem - loh * g.Wo;
    }
    const int ln = n0 + lrow;
    const bool n_ok = ln < g.Cout;
    const int ty = tid >> 4, tx = tid & 15;
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    for (int k0 = 0; k0 < K; k0 += CS_BK) {
        float a[4], w[4];
        gather_a4(x, g, m_ok, lb, loh, low, k0 + lk, K, a);
        if (n_ok && k0 + lk < K) ld4(wp + (size_t)ln * K + k0 + lk, w);
        else w[0] = w[1] = w[2] = w[3] = 0.f;
        __syncthreads();
#pragma unroll
        for (int j = 0; j < 4; ++j) { As[lk + j][lrow] = a[j]; Bs[lk + j][lrow] = w[j]; }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < CS_BK; ++kk) {
            float4 av = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
            float4 bv = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
            float aa[4] = {av.x, av.y, av.z, av.w}, bb[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] += aa[i] * bb[j];
        }
    }
    const int n = n0 + tx * 4;
    if (n < g.Cout) {
        float bv[4] = {0.f, 0.f, 0.f, 0.f};
        if (bias) { bv[0] = bias[n]; bv[1] = bias[n + 1]; bv[2] = bias[n + 2]; bv[3] = bias[n + 3]; }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            long long m = m0 + ty * 4 + i;
            if (m >= M) continue;
            float o[4] = {acc[i][0] + bv[0], acc[i][1] + bv[1], acc[i][2] + bv[2], acc[i][3] + bv[3]};
            if (residual) {
                float r[4];
                ld4(residual + m * g.Cout + n, r);
                o[0] += r[0]; o[1] += r[1]; o[2] += r[2]; o[3] += r[3];
            }
            st4(y + m * g.Cout + n, o);
        }
    }
}

// wgrad: dW[n][tap][c] += sum_m dy[m][n] * A(m, tap*Cin + c); written (atomicAdd) into the framework weight
// layout through strides:  index = n*s_n + c*s_c + tap.   dbias[n] += sum_m dy[m][n].
template <typename T>
__global__ void __launch_bounds__(CS_THREADS) conv_wgrad_simt_kernel(const T* __restrict__ x, const T* __restrict__ dy,
                                                                     float* __restrict__ dw, float* __restrict__ dbias,
                                                                     ConvGeom g, int c_real, long long s_n,
                                                                     long long s_c, int m_per_split) {
    __shared__ __align__(16) float Ds[CS_BK][CS_BN + 4];   // [mm][co]
    __shared__ __align__(16) float As[CS_BK][CS_BM + 4];   // [mm][k]
    const int tid = threadIdx.x;
    const long long M = (long long)g.B * g.Ho * g.Wo;
    const int K = g.KH * g.KW * g.Cin;
    const int k0 = blockIdx.x * CS_BM;      // k tile (64 wide)
    const int n0 = blockIdx.y * CS_BN;      // co tile
    const long long m_begin = (long long)blockIdx.z * m_per_split;
    long long m_end = m_begin + m_per_split;
    if (m_end > M) m_end = M;
    const int lmm = tid >> 4, lq = (tid & 15) * 4;
    const int ty = tid >> 4, tx = tid & 15;
    float acc[4][4];
    float bacc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    for (long long mb = m_begin; mb < m_end; mb += CS_BK) {
        long long m = mb + lmm;
        bool m_ok = m < m_end;
        int b = 0, oh = 0, ow = 0;
        if (m_ok) {
            b = (int)(m / (g.Ho * g.Wo));
            int rem = (int)(m - (long long)b * g.Ho * g.Wo);
            oh = rem / g.Wo; ow = rem - oh * g.Wo;
        }
        float a[4], d[4];
        gather_a4(x, g, m_ok, b, oh, ow, k0 + lq, K, a);
        if (m_ok && n0 + lq < g.Cout) ld4(dy + m * g.Cout + n0 + lq, d);
        else d[0] = d[1] = d[2] = d[3] = 0.f;
        __syncthreads();
        *reinterpret_cast<float4*>(&As[lmm][lq]) = make_float4(a[0], a[1], a[2], a[3]);
        *reinterpret_cast<float4*>(&Ds[lmm][lq]) = make_float4(d[0], d[1], d[2], d[3]);
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < CS_BK; ++kk) {
            float4 dv = *reinterpret_cast<const float4*>(&Ds[kk][ty * 4]);
            float4 av = *reinterpret_cast<const float4*>(&As[kk][tx * 4]);
            float dd[4] = {dv.x, dv.y, dv.z, dv.w}, aa[4] = {av.x, av.y, av.z, av.w};
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                bacc[i] += dd[i];
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] += dd[i] * aa[j];
            }
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        int n = n0 + ty * 4 + i;
        if (n >= g.Cout) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            int k = k0 + tx * 4 + j;
            if (k >= K) continue;
            int tap = k / g.Cin, c = k - tap * g.Cin;
            if (c < c_real) atomicAdd(dw + (long long)n * s_n + (long long)c * s_c + tap, acc[i][j]);
        }
        if (dbias && blockIdx.x == 0 && tx == 0) atomicAdd(dbias + n, bacc[i]);
    }
}

// ---- weight packing (framework fp32 layout -> Wp[n][tap*Cpad + c] in the activation dtype) ----------------
struct PackEntry {
    const float* src;
    void* dst;
    long long s_n, s_c;     // src index = n*s_n + c*s_c + tap_src
    int N, C, Cpad, taps;
    int flip, pad_;         // flip: tap_src = taps-1-tap (180-degree rotated kernel for stride-1 dgrad)
};

// two consecutive packed channels per thread (Cpad is even): 32-bit index arithmetic (the 64-bit divisions of the first
// version cost more than the memory traffic), one 4- or 8-byte store
template <typename T>
__global__ void pack_weights_kernel(const PackEntry* __restrict__ table) {
    const PackEntry e = table[blockIdx.y];
    const unsigned total2 = (unsigned)((long long)e.N * e.taps * e.Cpad / 2);
    const unsigned cpad = (unsigned)e.Cpad, taps = (unsigned)e.taps;
    T* dst = reinterpret_cast<T*>(e.dst);
    for (unsigned i2 = blockIdx.x * blockDim.x + threadIdx.x; i2 < total2; i2 += gridDim.x * blockDim.x) {
        const unsigned i = 2u * i2;
        const unsigned r = i / cpad, c = i - r * cpad;
        const unsigned n = r / taps, tap = r - n * taps;
        const unsigned ts = e.flip ? taps - 1u - tap : tap;
        const float* sp = e.src + (long long)n * e.s_n + ts;
        const float v0 = ((int)c < e.C) ? sp[(long long)c * e.s_c] : 0.f;
        const float v1 = ((int)c + 1 < e.C) ? sp[(long long)(c + 1) * e.s_c] : 0.f;
        if (sizeof(T) == 2) {
            *reinterpret_cast<__nv_bfloat162*>(reinterpret_cast<__nv_bfloat16*>(dst) + i) = __floats2bfloat162_rn(v0, v1);
        } else {
            *reinterpret_cast<float2*>(reinterpret_cast<float*>(dst) + i) = make_float2(v0, v1);
        }
    }
}

// ---- weight packing, both operand variants from ONE read ---------------------------------------------------------
// For layers with Cin, Cout multiples of 32 and <= 16 taps a CTA owns a 32 (co) x 32 (ci) x taps block of the fp32
// master weights: it reads the block as 32 contiguous runs of 32 * taps floats, keeps it in shared memory in the
// activation dtype and writes the forward operand Wp_f[co][tap * Cin + ci] and the dgrad operand
// Wp_d[ci][tap' * Cout + co] (tap' = taps - 1 - tap for stride-1 layers) as 64 / 128-byte row segments.  The generic
// kernel above reads every source element twice with a stride of `taps` floats between neighbouring threads; this one
// moves 41.5 MB in and 2 x 20.8 MB out once.
struct PackPairEntry {
    const float* src;
    void* dst_f;
    void* dst_d;             // null: no dgrad operand
    long long s_co, s_ci;    // src index = co * s_co + ci * s_ci + tap; the inner one equals taps
    int Cout, Cin, taps, flip;
    int tile0, pad_;         // index of this entry's first 32 x 32 block in the launch's block list
};

template <typename T>
__device__ __forceinline__ void pack_store2(T* p, T a, T b);
template <>
__device__ __forceinline__ void pack_store2<__nv_bfloat16>(__nv_bfloat16* p, __nv_bfloat16 a, __nv_bfloat16 b) {
    __nv_bfloat162 v; v.x = a; v.y = b;
    *reinterpret_cast<__nv_bfloat162*>(p) = v;
}
template <>
__device__ __forceinline__ void pack_store2<float>(float* p, float a, float b) { *reinterpret_cast<float2*>(p) = make_float2(a, b); }
template <typename T>
__device__ __forceinline__ T pack_cvt(float v);
template <>
__device__ __forceinline__ __nv_bfloat16 pack_cvt<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
template <>
__device__ __forceinline__ float pack_cvt<float>(float v) { return v; }

template <typename T>
__global__ void __launch_bounds__(256) pack_pair_kernel(const PackPairEntry* __restrict__ table,
                                                        const int* __restrict__ tile_map /*[all tiles] -> entry*/,
                                                        int tile_base) {
    extern __shared__ __align__(16) unsigned char pack_raw[];
    T* tile = reinterpret_cast<T*>(pack_raw);        // [32 co][32 ci][taps], pitches p_i (odd) and p_o = 32 * p_i + 2
    const int tile_id = (int)blockIdx.x + tile_base;
    const PackPairEntry e = table[tile_map[tile_id]];
    const int local = tile_id - e.tile0;
    const int tiles_ci = e.Cin >> 5;
    const int co0 = (local / tiles_ci) << 5, ci0 = (local % tiles_ci) << 5;
    const int taps = e.taps, run = 32 * taps, total = 32 * run;
    const int p_i = taps | 1, p_o = 32 * p_i + 2;
    // x / taps and x / run by multiply-high with a rounded-up reciprocal (exact for x * d < 2^32): with plain integer
    // divisions the index arithmetic (~35 instructions each, 4-5 per element) cost 3x the memory time of the whole kernel
    const uint32_t inv_taps = (uint32_t)(((1ull << 32) + (uint32_t)taps - 1) / (uint32_t)taps);
    const uint32_t inv_run = (uint32_t)(((1ull << 32) + (uint32_t)run - 1) / (uint32_t)run);
    auto div_taps = [&](int x) { return taps == 1 ? x : (int)__umulhi((uint32_t)x, inv_taps); };
    auto div_run = [&](int x) { return (int)__umulhi((uint32_t)x, inv_run); };
    const bool ci_inner = e.s_ci == (long long)taps;   // Conv layout [co][ci][tap]; otherwise ConvTranspose [ci][co][tap]
    const long long s_outer = ci_inner ? e.s_co : e.s_ci;
    const float* src0 = e.src + (long long)(ci_inner ? co0 : ci0) * s_outer + (long long)(ci_inner ? ci0 : co0) * taps;
    // 32 runs of 32 * taps contiguous floats; eight loads in flight per thread (a plain loop serialises on the load latency)
    for (int base = threadIdx.x; base < total; base += 8 * 256) {
        float v[8];
        int uu[8], rr[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            const int idx = base + q * 256;
            uu[q] = div_run(idx);
            rr[q] = idx - uu[q] * run;
            v[q] = idx < total ? __ldg(src0 + (long long)uu[q] * s_outer + rr[q]) : 0.f;
        }
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            if (base + q * 256 < total) {
                const int w = div_taps(rr[q]), t = rr[q] - w * taps;
                tile[ci_inner ? (uu[q] * p_o + w * p_i + t) : (w * p_o + uu[q] * p_i + t)] = pack_cvt<T>(v[q]);
            }
        }
    }
    __syncthreads();
    T* df = reinterpret_cast<T*>(e.dst_f);
    for (int idx = threadIdx.x; idx < run * 16; idx += 256) {            // (co, tap) rows of 32 ci: 16 pairs each
        const int i2 = idx & 15, r = idx >> 4;
        const int o = div_taps(r), t = r - o * taps;
        const T* sp = tile + o * p_o + (2 * i2) * p_i + t;
        pack_store2<T>(df + (size_t)(co0 + o) * ((size_t)taps * e.Cin) + (size_t)t * e.Cin + ci0 + 2 * i2, sp[0], sp[p_i]);
    }
    if (e.dst_d != nullptr) {
        T* dd = reinterpret_cast<T*>(e.dst_d);
        for (int idx = threadIdx.x; idx < run * 16; idx += 256) {        // (ci, tap) rows of 32 co
            const int o2 = idx & 15, r = idx >> 4;
            const int i = div_taps(r), t = r - i * taps;
            const int td = e.flip ? taps - 1 - t : t;
            const T* sp = tile + (2 * o2) * p_o + i * p_i + t;
            pack_store2<T>(dd + (size_t)(ci0 + i) * ((size_t)taps * e.Cout) + (size_t)td * e.Cout + co0 + 2 * o2, sp[0], sp[p_o]);
        }
    }
}

static int check_geom(const ConvGeom& g) {
    PIDM_REQUIRE(g.Cin % 4 == 0 && g.Cout % 4 == 0, "conv: Cin and Cout must be multiples of 4 (Cin=%d Cout=%d)", g.Cin,
                 g.Cout);
    PIDM_REQUIRE(g.B > 0 && g.H > 0 && g.W > 0 && g.Ho > 0 && g.Wo > 0 && g.stride >= 1, "conv: bad geometry");
    return 0;
}

}  // namespace pidm
using namespace pidm;

extern "C" int pidm_conv2d_simt(const void* x, const void* w_packed, const float* bias, const void* residual, void* y,
                                int B, int H, int W, int Cin, int Ho, int Wo, int Cout, int KH, int KW, int stride,
                                int pad, int transposed, int dtype, void* stream) {
    ConvGeom g{B, H, W, Cin, Ho, Wo, Cout, KH, KW, stride, pad, transposed};
    if (int e = check_geom(g)) return e;
    long long M = (long long)B * Ho * Wo;
    dim3 grid(ceil_div(M, CS_BM), ceil_div(Cout, CS_BN));
    PIDM_DISPATCH_DTYPE(dtype, (conv_simt_kernel<T><<<grid, CS_THREADS, 0, (cudaStream_t)stream>>>(
                                   (const T*)x, (const T*)w_packed, bias, (const T*)residual, (T*)y, g)));
    PIDM_LAUNCH_CHECK("conv2d_simt");
    return 0;
}

// dw / dbias are ACCUMULATED (atomicAdd).  (x, geometry) describe the A-operand gather exactly as in the
// forward call whose weights are being differentiated; dy is [B,Ho,Wo,Cout].
extern "C" int pidm_conv2d_wgrad_simt(const void* x, const void* dy, float* dw, float* dbias, int B, int H, int W,
                                      int Cin, int Cin_real, int Ho, int Wo, int Cout, int KH, int KW, int stride,
                                      int pad, int transposed, long long w_stride_n, long long w_stride_c, int dtype,
                                      void* stream) {
    ConvGeom g{B, H, W, Cin, Ho, Wo, Cout, KH, KW, stride, pad, transposed};
    if (int e = check_geom(g)) return e;
    long long M = (long long)B * Ho * Wo;
    int K = KH * KW * Cin;
    int tiles = ceil_div(K, CS_BM) * ceil_div(Cout, CS_BN);
    int splits = (num_sms() * 4 + tiles - 1) / tiles;
    long long max_splits = (M + 255) / 256;
    if (splits > max_splits) splits = (int)max_splits;
    if (splits < 1) splits = 1;
    int m_per_split = (int)(((M + splits - 1) / splits + CS_BK - 1) / CS_BK * CS_BK);
    splits = (int)((M + m_per_split - 1) / m_per_split);
    dim3 grid(ceil_div(K, CS_BM), ceil_div(Cout, CS_BN), splits);
    PIDM_DISPATCH_DTYPE(dtype, (conv_wgrad_simt_kernel<T><<<grid, CS_THREADS, 0, (cudaStream_t)stream>>>(
                                   (const T*)x, (const T*)dy, dw, dbias, g, Cin_real, w_stride_n, w_stride_c,
                                   m_per_split)));
    PIDM_LAUNCH_CHECK("conv2d_wgrad_simt");
    return 0;
}

// table: device array of n_entries PackEntry records (see pidm.h for the layout).
extern "C" int pidm_pack_weights(const void* table_dev, int n_entries, int dtype, void* stream) {
    if (n_entries <= 0) return 0;
    dim3 grid(32, n_entries);
    PIDM_DISPATCH_DTYPE(dtype, (pack_weights_kernel<T><<<grid, 256, 0, (cudaStream_t)stream>>>(
                                   (const PackEntry*)table_dev)));
    PIDM_LAUNCH_CHECK("pack_weights");
    return 0;
}

extern "C" int pidm_pack_entry_size(void) { return (int)sizeof(PackEntry); }

// table: device array of PackPairEntry records (Cin % 32 == 0, Cout % 32 == 0, taps <= 16); tile_map[i] = entry that owns
// the i-th 32 x 32 channel block (entry e owns blocks [tile0, tile0 + (Cout / 32) * (Cin / 32))); max_taps over the table.
// The launch packs blocks [tile_base, tile_base + n_tiles): a caller can pack the layers it needs first in a first launch.
extern "C" int pidm_pack_weights_pairs(const void* table_dev, const int* tile_map_dev, int tile_base, int n_tiles, int max_taps,
                                       int dtype, void* stream) {
    if (n_tiles <= 0) return 0;
    PIDM_REQUIRE(max_taps >= 1 && max_taps <= 16, "pack_weights_pairs: taps must be 1..16 (got %d)", max_taps);
    const size_t esz = dtype == PIDM_BF16 ? 2 : 4;
    const size_t smem = (size_t)32 * (32 * (max_taps | 1) + 2) * esz;
    PIDM_CUDA(allow_smem(pack_pair_kernel<float>, 32 * (32 * 17 + 2) * 4));
    PIDM_DISPATCH_DTYPE(dtype, (pack_pair_kernel<T><<<n_tiles, 256, smem, (cudaStream_t)stream>>>((const PackPairEntry*)table_dev,
                                                                                                    tile_map_dev, tile_base)));
    PIDM_LAUNCH_CHECK("pack_weights_pairs");
    return 0;
}

extern "C" int pidm_pack_pair_entry_size(void) { return (int)sizeof(PackPairEntry); }
