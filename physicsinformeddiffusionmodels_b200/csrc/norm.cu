// Normalisations of the U-Net on NHWC activations, all statistics in fp32:
//   * GroupNorm(G) -> (scale+1, shift) FiLM -> SiLU      (Block.forward, reference unet_model.py:233-241)
//   * channel LayerNorm (gain only, biased variance)     (LayerNorm.forward, unet_model.py:201-210)
// Forward = one reduction kernel (sum, sum-of-squares per (sample, group), one atomic per CTA per group)
// + one vectorised apply kernel.  Backward = reduction over pixels of (dz, dz*xhat) per (sample, channel),
// a tiny per-sample kernel that turns those into parameter / FiLM gradients and group means, and an
// element-wise dx kernel.  Nothing but the conv output x and the raw sums is saved for backward.
#include "common.cuh"
#include "pidm.h"
#include <cooperative_groups.h>

namespace pidm {

constexpr int NORM_THREADS = 256;

// ------------------------------------------------------------------------------------------------
// GroupNorm statistics: sums[b][g][0] += sum x, sums[b][g][1] += sum x^2
// thread = (row r, octet o); rows advance by rows_per_pass; grid = (chunks, B)
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void gn_stats_kernel(const T* __restrict__ x, float* __restrict__ sums, int HW, int C, int G) {
    extern __shared__ float sg[];  // [G][2]
    const int oct = C / 8, cpg = C / G;
    const int b = blockIdx.y;
    const int o = threadIdx.x % oct, r0 = threadIdx.x / oct;
    const int rows_per_pass = blockDim.x / oct;
    for (int i = threadIdx.x; i < 2 * G; i += blockDim.x) sg[i] = 0.f;
    __syncthreads();
    float s[2] = {0.f, 0.f}, ss[2] = {0.f, 0.f};   // two half-octets (cpg may be 4)
    const T* xb = x + (size_t)b * HW * C;
    for (int p = blockIdx.x * rows_per_pass + r0; p < HW; p += gridDim.x * rows_per_pass) {
        float v[8];
        ld8(xb + (size_t)p * C + o * 8, v);
#pragma unroll
        for (int k = 0; k < 8; ++k) { s[k >> 2] += v[k]; ss[k >> 2] += v[k] * v[k]; }
    }
    float red[4] = {s[0], s[1], ss[0], ss[1]};
    if (reduce_same_octet(red, oct)) {
        int g = (o * 8) / cpg;
        if (cpg >= 8) {
            atomicAdd(&sg[2 * g], red[0] + red[1]);
            atomicAdd(&sg[2 * g + 1], red[2] + red[3]);
        } else {  // cpg == 4
            atomicAdd(&sg[2 * g], red[0]); atomicAdd(&sg[2 * g + 1], red[2]);
            atomicAdd(&sg[2 * g + 2], red[1]); atomicAdd(&sg[2 * g + 3], red[3]);
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 2 * G; i += blockDim.x) atomicAdd(&sums[(size_t)b * 2 * G + i], sg[i]);
}

__device__ __forceinline__ void gn_mean_rstd(const float* sums, int b, int g, int G, float inv_n, float eps, float& mean,
                                             float& rstd) {
    float s = sums[((size_t)b * G + g) * 2], ss = sums[((size_t)b * G + g) * 2 + 1];
    mean = s * inv_n;
    float var = fmaxf(ss * inv_n - mean * mean, 0.f);
    rstd = rsqrtf(var + eps);
}

// 16-byte vector of activations: 8 bf16 or 4 fp32 channels
template <typename T> struct Vec { static constexpr int N = 16 / (int)sizeof(T); };
template <typename T> __device__ __forceinline__ void ldv(const T* p, float* v);
template <> __device__ __forceinline__ void ldv<float>(const float* p, float* v) { ld4(p, v); }
template <> __device__ __forceinline__ void ldv<__nv_bfloat16>(const __nv_bfloat16* p, float* v) { ld8(p, v); }
template <typename T> __device__ __forceinline__ void stv(T* p, const float* v);
template <> __device__ __forceinline__ void stv<float>(float* p, const float* v) { st4(p, v); }
template <> __device__ __forceinline__ void stv<__nv_bfloat16>(__nv_bfloat16* p, const float* v) { st8(p, v); }

// y = silu( ((x-mean)*rstd*gamma + beta) * (scale+1) + shift ) (+ res)
// grid (chunks, B).  A thread owns ONE 16-byte channel vector position (o) and walks pixels: its per-channel constants
// (group mean, rstd*gamma, beta, 1+scale, shift) are loaded once into registers, the pixel loop is 3 FMAs + SiLU per
// element with GN_APPLY_UNR independent 16-byte loads in flight.  (The first version re-derived mean/rstd and re-read
// gamma/beta/scale/shift from global memory for every vector: ~30 loads per 8 outputs, 2.2 TB/s at 64x64x32.)
constexpr int GN_APPLY_UNR = 4;
template <typename T>
__global__ void __launch_bounds__(NORM_THREADS) gn_apply_kernel(
        const T* __restrict__ x, const float* __restrict__ sums, const float* __restrict__ gamma,
        const float* __restrict__ beta, const float* __restrict__ ss /*[B,2C] or null*/,
        const T* __restrict__ res /*added after the SiLU, or null*/, T* __restrict__ y, int HW, int C, int G, float eps) {
    constexpr int VE = Vec<T>::N;
    const int ov = C / VE, cpg = C / G;
    const int b = blockIdx.y;
    const int o = threadIdx.x % ov, r0 = threadIdx.x / ov;
    const int rpp = blockDim.x / ov;
    const float inv_n = 1.f / ((float)cpg * (float)HW);
    pdl_trigger();
    // parameters do not depend on the predecessor kernel: load them before the grid dependency resolves
    float a[VE], bt[VE], s1p[VE], sh[VE], mean[VE];
#pragma unroll
    for (int k = 0; k < VE; ++k) { a[k] = gamma[o * VE + k]; bt[k] = beta[o * VE + k]; }
    pdl_wait();
#pragma unroll
    for (int k = 0; k < VE; k += 4) {          // cpg is 4 or a multiple of 8: 4 consecutive channels share a group
        float m, r;
        gn_mean_rstd(sums, b, (o * VE + k) / cpg, G, inv_n, eps, m, r);
#pragma unroll
        for (int j = 0; j < 4; ++j) { mean[k + j] = m; a[k + j] *= r; }
    }
#pragma unroll
    for (int k = 0; k < VE; ++k) {
        const int c = o * VE + k;
        s1p[k] = ss ? ss[(size_t)b * 2 * C + c] + 1.f : 1.f;
        sh[k] = ss ? ss[(size_t)b * 2 * C + C + c] : 0.f;
    }
    const size_t base = (size_t)b * HW * C + (size_t)o * VE;
    const int stride = gridDim.x * rpp;
    for (int p0 = blockIdx.x * rpp + r0; p0 < HW; p0 += stride * GN_APPLY_UNR) {
        float v[GN_APPLY_UNR][VE], rr[GN_APPLY_UNR][VE];
#pragma unroll
        for (int u = 0; u < GN_APPLY_UNR; ++u) {
            const int p = p0 + u * stride;
            if (p < HW) {
                ldv<T>(x + base + (size_t)p * C, v[u]);
                if (res) ldv<T>(res + base + (size_t)p * C, rr[u]);
            }
        }
#pragma unroll
        for (int u = 0; u < GN_APPLY_UNR; ++u) {
            const int p = p0 + u * stride;
            if (p < HW) {
#pragma unroll
                for (int k = 0; k < VE; ++k) {
                    const float z = ((v[u][k] - mean[k]) * a[k] + bt[k]) * s1p[k] + sh[k];
                    v[u][k] = silu_f(z);
                    if (res) v[u][k] += rr[u][k];
                }
                stv<T>(y + base + (size_t)p * C, v[u]);
            }
        }
    }
}

// raw 16-byte activation vector <-> floats
template <typename T> __device__ __forceinline__ void unpack_vec(const uint4& r, float* v);
template <> __device__ __forceinline__ void unpack_vec<float>(const uint4& r, float* v) {
    v[0] = __uint_as_float(r.x); v[1] = __uint_as_float(r.y); v[2] = __uint_as_float(r.z); v[3] = __uint_as_float(r.w);
}
template <> __device__ __forceinline__ void unpack_vec<__nv_bfloat16>(const uint4& r, float* v) {
    const __nv_bfloat162* hp = reinterpret_cast<const __nv_bfloat162*>(&r);
#pragma unroll
    for (int k = 0; k < 4; ++k) { v[2 * k] = __low2float(hp[k]); v[2 * k + 1] = __high2float(hp[k]); }
}

// The piece kernel for pieces of 3..NV vectors per thread: ALL x / dy vectors of the thread are fetched up front and
// stay in registers PACKED (NV x 2 x 4 registers), so the kernel pays one memory latency instead of one per chunk and
// per phase, and nothing is read twice.  Used with NV = 4 only (see the dispatch for the measurement).  Both phases unpack and recompute xhat / dz (a few FMAs and one SiLU' per element).
// Per-channel constants are folded (z = xhat * A + Bc; mean / rstd / group means per half-vector) to stay inside 128
// registers.  Same arguments and shared-memory layout as gn_bwd_piece_kernel.
template <typename T, int NV>
__global__ void __launch_bounds__(NORM_THREADS, 2) gn_bwd_piece_packed_kernel(
        const T* __restrict__ x, const T* __restrict__ dy, const float* __restrict__ sums, const float* __restrict__ gamma,
        const float* __restrict__ beta, const float* __restrict__ ss, T* __restrict__ dx, float* __restrict__ dss,
        float* __restrict__ dgamma, float* __restrict__ dbeta, float* __restrict__ dbias, int HW, int C, int G, float eps,
        int S /*channels per slab*/, int CL /*CTAs per (sample, slab)*/, int rows_per_cta) {
    namespace cg = cooperative_groups;
    constexpr int VE = Vec<T>::N, NH = VE / 4;
    extern __shared__ float rsm[];
    float* part = rsm;                 // [S][2] partial sums of this CTA
    float* Sf = part + 2 * S;          // [S][2] sums over the whole (sample, slab)
    float* gm = Sf + 2 * S;            // [S / cpg][2]
    float* cs = gm + 2 * (S / (C / G));// [S] column sums of dx
    volatile float* AB = cs + S;       // [2][S] folded per-channel constants A | Bc (re-read where used: they would cost
                                       // 16 registers next to the 64 that hold the packed data)
    const int cpg = C / G, so = S / VE, nslab = C / S;
    const int piece = blockIdx.x / CL, rank = blockIdx.x - piece * CL;
    const int b = piece / nslab, slab = piece - b * nslab;
    const int c0 = slab * S;
    const int o = threadIdx.x % so, r0 = threadIdx.x / so;
    const int rpp = blockDim.x / so;
    const int row_begin = rank * rows_per_cta;
    const int row_end = min(HW, row_begin + rows_per_cta);
    const float inv_n = 1.f / ((float)cpg * (float)HW);
    pdl_trigger();
    for (int i = threadIdx.x; i < 5 * S + 2 * (S / cpg); i += blockDim.x) rsm[i] = 0.f;
    pdl_wait();
    const size_t base = (size_t)b * HW * C + c0 + (size_t)o * VE;
    uint4 xr[NV], dr[NV];
#pragma unroll
    for (int u = 0; u < NV; ++u) {
        const int p = row_begin + r0 + u * rpp;
        if (p < row_end) {
            xr[u] = *reinterpret_cast<const uint4*>(x + base + (size_t)p * C);
            dr[u] = *reinterpret_cast<const uint4*>(dy + base + (size_t)p * C);
        }
    }
    float rs[NH], mr[NH];
#pragma unroll
    for (int h = 0; h < NH; ++h) {
        float m, r;
        gn_mean_rstd(sums, b, (c0 + o * VE + 4 * h) / cpg, G, inv_n, eps, m, r);
        rs[h] = r; mr[h] = m * r;
    }
    if (r0 == 0) {
#pragma unroll
        for (int k = 0; k < VE; ++k) {
            const int c = c0 + o * VE + k;
            const float s1p = ss ? ss[(size_t)b * 2 * C + c] + 1.f : 1.f;
            const float sh = ss ? ss[(size_t)b * 2 * C + C + c] : 0.f;
            AB[o * VE + k] = gamma[c] * s1p; AB[S + o * VE + k] = beta[c] * s1p + sh;
        }
    }
    __syncthreads();                                           // constants and the zero-fill of the shared sums are visible
    // ---- phase 1
    float a1[VE], a2[VE];
#pragma unroll
    for (int k = 0; k < VE; ++k) { a1[k] = 0.f; a2[k] = 0.f; }
#pragma unroll
    for (int u = 0; u < NV; ++u) {
        if (row_begin + r0 + u * rpp < row_end) {
            float xv[VE], dv[VE];
            unpack_vec<T>(xr[u], xv);
            unpack_vec<T>(dr[u], dv);
#pragma unroll
            for (int k = 0; k < VE; ++k) {
                const float xh = xv[k] * rs[k >> 2] - mr[k >> 2];
                const float dz = dv[k] * silu_grad_f(xh * AB[o * VE + k] + AB[S + o * VE + k]);
                a1[k] += dz; a2[k] += dz * xh;
            }
        }
    }
    const bool pub1 = reduce_same_octet(a1, so);
    reduce_same_octet(a2, so);
    if (pub1) {
#pragma unroll
        for (int k = 0; k < VE; ++k) { atomicAdd(&part[(o * VE + k) * 2], a1[k]); atomicAdd(&part[(o * VE + k) * 2 + 1], a2[k]); }
    }
    if (CL > 1) {
        cg::cluster_group cluster = cg::this_cluster();
        cluster.sync();
        for (int i = threadIdx.x; i < 2 * S; i += blockDim.x) {
            float t = 0.f;
            for (int r = 0; r < CL; ++r) t += cluster.map_shared_rank(part, r)[i];
            Sf[i] = t;
        }
        cluster.sync();
    } else {
        __syncthreads();
        for (int i = threadIdx.x; i < 2 * S; i += blockDim.x) Sf[i] = part[i];
        __syncthreads();
    }
    for (int cl = threadIdx.x; cl < S; cl += blockDim.x) {
        const int c = c0 + cl;
        const float s1 = Sf[cl * 2], s2 = Sf[cl * 2 + 1];
        const float f = ss ? ss[(size_t)b * 2 * C + c] + 1.f : 1.f;
        atomicAdd(&gm[(cl / cpg) * 2], gamma[c] * f * s1);
        atomicAdd(&gm[(cl / cpg) * 2 + 1], gamma[c] * f * s2);
        if (rank == 0) {
            if (dss) {
                dss[(size_t)b * 2 * C + c] = gamma[c] * s2 + beta[c] * s1;   // d scale
                dss[(size_t)b * 2 * C + C + c] = s1;                          // d shift
            }
            atomicAdd(&dgamma[c], f * s2);
            atomicAdd(&dbeta[c], f * s1);
        }
    }
    __syncthreads();
    // ---- phase 2
    float m1[NH], m2[NH];
#pragma unroll
    for (int h = 0; h < NH; ++h) {
        const int gl = (o * VE + 4 * h) / cpg;
        m1[h] = gm[gl * 2] * inv_n; m2[h] = gm[gl * 2 + 1] * inv_n;
    }
    float colsum[VE];
#pragma unroll
    for (int k = 0; k < VE; ++k) colsum[k] = 0.f;
#pragma unroll
    for (int u = 0; u < NV; ++u) {
        const int p = row_begin + r0 + u * rpp;
        if (p < row_end) {
            float xv[VE], dv[VE], g[VE];
            unpack_vec<T>(xr[u], xv);
            unpack_vec<T>(dr[u], dv);
#pragma unroll
            for (int k = 0; k < VE; ++k) {
                const float xh = xv[k] * rs[k >> 2] - mr[k >> 2];
                const float ak = AB[o * VE + k];
                const float dz = dv[k] * silu_grad_f(xh * ak + AB[S + o * VE + k]);
                g[k] = rs[k >> 2] * (ak * dz - m1[k >> 2] - xh * m2[k >> 2]);
                colsum[k] += g[k];
            }
            stv<T>(dx + base + (size_t)p * C, g);
        }
    }
    if (dbias) {
        if (reduce_same_octet(colsum, so)) {
#pragma unroll
            for (int k = 0; k < VE; ++k) atomicAdd(&cs[o * VE + k], colsum[k]);
        }
        __syncthreads();
        for (int i = threadIdx.x; i < S; i += blockDim.x) atomicAdd(&dbias[c0 + i], cs[i]);
    }
}

// The piece kernel for pieces of MORE than 4 vectors per thread (the 64x64 levels): x and dy are streamed twice (the second
// pass hits L2).  Compared with gn_bwd_piece_kernel<T, 2, false>, which it replaces, the loops are written for instruction
// count -- that variant spends 29 instructions per element and phase, a third of them 64-bit address arithmetic and
// predicate bookkeeping.  Here a thread walks its vectors with three running
// pointers, per-channel constants are folded (xhat = x * rs - mr, z = xhat * A + Bc, dx = dz * Ap - m1p - xhat * m2p), the
// next two vector pairs are fetched (raw, 16 registers) while the current two are processed, and the first pass parks dz in
// the dx buffer (activation dtype) so that the second pass needs no SiLU' (it reads x and dz, overwrites dz with dx).
// SiLU'(z) for the streaming kernel: bf16 activations take the one-MUFU form through tanh.approx (abs. error ~5e-4, below
// the bf16 resolution of the stored result; the exp + rcp form costs two MUFU operations per element and the kernel is
// bound by the XU pipe as much as by issue slots), fp32 activations keep the exact form.
template <typename T> __device__ __forceinline__ float silu_grad_t(float z) { return silu_grad_f(z); }
template <> __device__ __forceinline__ float silu_grad_t<__nv_bfloat16>(float z) {
    float t;
    asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(0.5f * z));
    const float sg = fmaf(0.5f, t, 0.5f);                 // sigmoid(z)
    return sg * fmaf(z, fmaf(-0.5f, t, 0.5f), 1.f);       // s * (1 + z * (1 - s))
}

template <typename T>
__global__ void __launch_bounds__(NORM_THREADS, 2) gn_bwd_piece_stream_kernel(
        const T* __restrict__ x, const T* __restrict__ dy, const float* __restrict__ sums, const float* __restrict__ gamma,
        const float* __restrict__ beta, const float* __restrict__ ss, T* __restrict__ dx, float* __restrict__ dss,
        float* __restrict__ dgamma, float* __restrict__ dbeta, float* __restrict__ dbias, int HW, int C, int G, float eps,
        int S /*channels per slab*/, int CL /*CTAs per (sample, slab)*/, int rows_per_cta) {
    namespace cg = cooperative_groups;
    constexpr int VE = Vec<T>::N, NH = VE / 4;
    extern __shared__ float rsm[];
    float* part = rsm;                 // [S][2] partial sums of this CTA
    float* Sf = part + 2 * S;          // [S][2] sums over the whole (sample, slab)
    float* gm = Sf + 2 * S;            // [S / cpg][2]
    float* cs = gm + 2 * (S / (C / G));// [S] column sums of dx
    const int cpg = C / G, so = S / VE, nslab = C / S;
    const int piece = blockIdx.x / CL, rank = blockIdx.x - piece * CL;
    const int b = piece / nslab, slab = piece - b * nslab;
    const int c0 = slab * S;
    const int o = threadIdx.x % so, r0 = threadIdx.x / so;
    const int rpp = blockDim.x / so;
    const int row_begin = rank * rows_per_cta;
    const int row_end = min(HW, row_begin + rows_per_cta);
    const float inv_n = 1.f / ((float)cpg * (float)HW);
    pdl_trigger();
    for (int i = threadIdx.x; i < 5 * S + 2 * (S / cpg); i += blockDim.x) rsm[i] = 0.f;
    pdl_wait();
    // vectors of this thread: rows row_begin + r0 + i * rpp, i = 0 .. nvec - 1
    const int first = row_begin + r0;
    const int nvec = first < row_end ? (row_end - first + rpp - 1) / rpp : 0;
    const size_t off0 = (size_t)b * HW * C + c0 + (size_t)o * VE + (size_t)first * C;
    const size_t vstride = (size_t)rpp * C;
    const uint4 zero4 = make_uint4(0u, 0u, 0u, 0u);
    auto ldr = [](const T* p) { return *reinterpret_cast<const uint4*>(p); };
    const T* xp = x + off0;
    const T* dp = dy + off0;
    uint4 cx0 = zero4, cd0 = zero4, cx1 = zero4, cd1 = zero4;
    if (nvec > 0) { cx0 = ldr(xp); cd0 = ldr(dp); }
    if (nvec > 1) { cx1 = ldr(xp + vstride); cd1 = ldr(dp + vstride); }
    float A[VE], Bc[VE], rs[NH], mr[NH];
#pragma unroll
    for (int h = 0; h < NH; ++h) {
        float m, r;
        gn_mean_rstd(sums, b, (c0 + o * VE + 4 * h) / cpg, G, inv_n, eps, m, r);
        rs[h] = r; mr[h] = m * r;
    }
#pragma unroll
    for (int k = 0; k < VE; ++k) {
        const int c = c0 + o * VE + k;
        const float s1p = ss ? ss[(size_t)b * 2 * C + c] + 1.f : 1.f;
        const float sh = ss ? ss[(size_t)b * 2 * C + C + c] : 0.f;
        A[k] = gamma[c] * s1p; Bc[k] = beta[c] * s1p + sh;
    }
    // ---- phase 1: sums of dz and dz * xhat
    float a1[VE], a2[VE];
#pragma unroll
    for (int k = 0; k < VE; ++k) { a1[k] = 0.f; a2[k] = 0.f; }
    T* op = dx + off0;                                         // phase 1 parks dz here, phase 2 overwrites it with dx
    for (int i = 0; i < nvec; i += 2) {
        xp += 2 * vstride; dp += 2 * vstride;
        uint4 nx0 = zero4, nd0 = zero4, nx1 = zero4, nd1 = zero4;
        if (i + 2 < nvec) { nx0 = ldr(xp); nd0 = ldr(dp); }
        if (i + 3 < nvec) { nx1 = ldr(xp + vstride); nd1 = ldr(dp + vstride); }
        const bool two = i + 1 < nvec;
        {
            float xv[VE], dv[VE];
            unpack_vec<T>(cx0, xv); unpack_vec<T>(cd0, dv);
#pragma unroll
            for (int k = 0; k < VE; ++k) {
                const float xh = fmaf(xv[k], rs[k >> 2], -mr[k >> 2]);
                dv[k] *= silu_grad_t<T>(fmaf(xh, A[k], Bc[k]));
                a1[k] += dv[k]; a2[k] = fmaf(dv[k], xh, a2[k]);
            }
            stv<T>(op, dv);
        }
        if (two) {
            float xv[VE], dv[VE];
            unpack_vec<T>(cx1, xv); unpack_vec<T>(cd1, dv);
#pragma unroll
            for (int k = 0; k < VE; ++k) {
                const float xh = fmaf(xv[k], rs[k >> 2], -mr[k >> 2]);
                dv[k] *= silu_grad_t<T>(fmaf(xh, A[k], Bc[k]));
                a1[k] += dv[k]; a2[k] = fmaf(dv[k], xh, a2[k]);
            }
            stv<T>(op + vstride, dv);
        }
        op += 2 * vstride;
        cx0 = nx0; cd0 = nd0; cx1 = nx1; cd1 = nd1;
    }
    // the second pass re-reads x (L2) and the parked dz (written by this very thread): issue its first loads before the
    // reduction chain
    xp = x + off0;
    const T* zp = dx + off0;
    if (nvec > 0) { cx0 = ldr(xp); cd0 = ldr(zp); }
    if (nvec > 1) { cx1 = ldr(xp + vstride); cd1 = ldr(zp + vstride); }
    __syncthreads();                                           // zero-fill of the shared sums is complete
    const bool pub1 = reduce_same_octet(a1, so);
    reduce_same_octet(a2, so);
    if (pub1) {
#pragma unroll
        for (int k = 0; k < VE; ++k) { atomicAdd(&part[(o * VE + k) * 2], a1[k]); atomicAdd(&part[(o * VE + k) * 2 + 1], a2[k]); }
    }
    if (CL > 1) {
        cg::cluster_group cluster = cg::this_cluster();
        cluster.sync();
        for (int i = threadIdx.x; i < 2 * S; i += blockDim.x) {
            float t = 0.f;
            for (int r = 0; r < CL; ++r) t += cluster.map_shared_rank(part, r)[i];
            Sf[i] = t;
        }
        cluster.sync();
    } else {
        __syncthreads();
        for (int i = threadIdx.x; i < 2 * S; i += blockDim.x) Sf[i] = part[i];
        __syncthreads();
    }
    for (int cl = threadIdx.x; cl < S; cl += blockDim.x) {
        const int c = c0 + cl;
        const float s1 = Sf[cl * 2], s2 = Sf[cl * 2 + 1];
        const float f = ss ? ss[(size_t)b * 2 * C + c] + 1.f : 1.f;
        atomicAdd(&gm[(cl / cpg) * 2], gamma[c] * f * s1);
        atomicAdd(&gm[(cl / cpg) * 2 + 1], gamma[c] * f * s2);
        if (rank == 0) {
            if (dss) {
                dss[(size_t)b * 2 * C + c] = gamma[c] * s2 + beta[c] * s1;   // d scale
                dss[(size_t)b * 2 * C + C + c] = s1;                          // d shift
            }
            atomicAdd(&dgamma[c], f * s2);
            atomicAdd(&dbeta[c], f * s1);
        }
    }
    __syncthreads();
    // ---- phase 2: dx = rstd * (A dz - mean(A dz) - xhat mean(A dz xhat)), folded
    float Ap[VE], m1p[NH], m2p[NH];
#pragma unroll
    for (int h = 0; h < NH; ++h) {
        const int gl = (o * VE + 4 * h) / cpg;
        m1p[h] = rs[h] * gm[gl * 2] * inv_n; m2p[h] = rs[h] * gm[gl * 2 + 1] * inv_n;
    }
#pragma unroll
    for (int k = 0; k < VE; ++k) Ap[k] = rs[k >> 2] * A[k];
    float colsum[VE];
#pragma unroll
    for (int k = 0; k < VE; ++k) colsum[k] = 0.f;
    op = dx + off0;
    for (int i = 0; i < nvec; i += 2) {
        xp += 2 * vstride; zp += 2 * vstride;
        uint4 nx0 = zero4, nd0 = zero4, nx1 = zero4, nd1 = zero4;
        if (i + 2 < nvec) { nx0 = ldr(xp); nd0 = ldr(zp); }
        if (i + 3 < nvec) { nx1 = ldr(xp + vstride); nd1 = ldr(zp + vstride); }
        const bool two = i + 1 < nvec;
        {
            float xv[VE], dv[VE], g[VE];
            unpack_vec<T>(cx0, xv); unpack_vec<T>(cd0, dv);
#pragma unroll
            for (int k = 0; k < VE; ++k) {
                const float xh = fmaf(xv[k], rs[k >> 2], -mr[k >> 2]);
                g[k] = fmaf(-xh, m2p[k >> 2], fmaf(dv[k], Ap[k], -m1p[k >> 2]));
                colsum[k] += g[k];
            }
            stv<T>(op, g);
        }
        if (two) {
            float xv[VE], dv[VE], g[VE];
            unpack_vec<T>(cx1, xv); unpack_vec<T>(cd1, dv);
#pragma unroll
            for (int k = 0; k < VE; ++k) {
                const float xh = fmaf(xv[k], rs[k >> 2], -mr[k >> 2]);
                g[k] = fmaf(-xh, m2p[k >> 2], fmaf(dv[k], Ap[k], -m1p[k >> 2]));
                colsum[k] += g[k];
            }
            stv<T>(op + vstride, g);
        }
        op += 2 * vstride;
        cx0 = nx0; cd0 = nd0; cx1 = nx1; cd1 = nd1;
    }
    if (dbias) {
        if (reduce_same_octet(colsum, so)) {
#pragma unroll
            for (int k = 0; k < VE; ++k) atomicAdd(&cs[o * VE + k], colsum[k]);
        }
        __syncthreads();
        for (int i = threadIdx.x; i < S; i += blockDim.x) atomicAdd(&dbias[c0 + i], cs[i]);
    }
}

// backward pass 1: S[b][c][0] += sum_pix dz, S[b][c][1] += sum_pix dz*xhat, dz = dy * silu'(z)
template <typename T>
__global__ void gn_bwd_reduce_kernel(const T* __restrict__ x, const T* __restrict__ dy, const float* __restrict__ sums,
                                     const float* __restrict__ gamma, const float* __restrict__ beta,
                                     const float* __restrict__ ss, float* __restrict__ S, int HW, int C, int G,
                                     float eps) {
    extern __shared__ float sc[];  // [C][2]
    const int oct = C / 8, cpg = C / G;
    const int b = blockIdx.y;
    const int o = threadIdx.x % oct, r0 = threadIdx.x / oct;
    const int rows_per_pass = blockDim.x / oct;
    const float inv_n = 1.f / ((float)cpg * (float)HW);
    for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) sc[i] = 0.f;
    __syncthreads();
    float mean[2], rstd[2], gm[8], bt[8], s1p[8], sh[8];
#pragma unroll
    for (int h = 0; h < 2; ++h) gn_mean_rstd(sums, b, (o * 8 + h * 4) / cpg, G, inv_n, eps, mean[h], rstd[h]);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        int c = o * 8 + k;
        gm[k] = gamma[c]; bt[k] = beta[c];
        s1p[k] = ss ? ss[(size_t)b * 2 * C + c] + 1.f : 1.f;
        sh[k] = ss ? ss[(size_t)b * 2 * C + C + c] : 0.f;
    }
    float a1[8], a2[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) { a1[k] = 0.f; a2[k] = 0.f; }
    const size_t base = (size_t)b * HW * C;
    for (int p = blockIdx.x * rows_per_pass + r0; p < HW; p += gridDim.x * rows_per_pass) {
        float v[8], d[8];
        ld8(x + base + (size_t)p * C + o * 8, v);
        ld8(dy + base + (size_t)p * C + o * 8, d);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            float xh = (v[k] - mean[k >> 2]) * rstd[k >> 2];
            float z = (xh * gm[k] + bt[k]) * s1p[k] + sh[k];
            float dz = d[k] * silu_grad_f(z);
            a1[k] += dz; a2[k] += dz * xh;
        }
    }
    const bool pub1 = reduce_same_octet(a1, oct);
    reduce_same_octet(a2, oct);
    if (pub1) {
#pragma unroll
        for (int k = 0; k < 8; ++k) { atomicAdd(&sc[(o * 8 + k) * 2], a1[k]); atomicAdd(&sc[(o * 8 + k) * 2 + 1], a2[k]); }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) atomicAdd(&S[(size_t)b * 2 * C + i], sc[i]);
}

// backward pass 2: dx = rstd * (gamma*(1+scale)*dz - m1 - xhat*m2), grid (chunks, B).
// Every CTA first turns S[b] into the group means m1, m2 (C values: cheap); the chunk-0 CTA of each sample also
// emits the FiLM gradients and the (atomic) parameter gradients.  Optionally accumulates the column sums of dx
// (= bias gradient of the convolution that produced x) -- each thread owns a fixed channel octet.
template <typename T>
__global__ void gn_bwd_dx_kernel(const T* __restrict__ x, const T* __restrict__ dy, const float* __restrict__ sums,
                                 const float* __restrict__ gamma, const float* __restrict__ beta,
                                 const float* __restrict__ ss, const float* __restrict__ S, T* __restrict__ dx,
                                 float* __restrict__ dss, float* __restrict__ dgamma, float* __restrict__ dbeta,
                                 float* __restrict__ dbias, int HW, int C, int G, float eps) {
    extern __shared__ float sm[];   // gm[G][2] | cs[C]
    float* gm = sm;
    float* cs = sm + 2 * G;
    const int oct = C / 8, cpg = C / G;
    const int b = blockIdx.y;
    const int o = threadIdx.x % oct, r0 = threadIdx.x / oct;
    const int rows_per_pass = blockDim.x / oct;
    const float inv_n = 1.f / ((float)cpg * (float)HW);
    for (int i = threadIdx.x; i < 2 * G + C; i += blockDim.x) sm[i] = 0.f;
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        float s1 = S[((size_t)b * C + c) * 2], s2 = S[((size_t)b * C + c) * 2 + 1];
        float f = ss ? ss[(size_t)b * 2 * C + c] + 1.f : 1.f;
        atomicAdd(&gm[(c / cpg) * 2], gamma[c] * f * s1);
        atomicAdd(&gm[(c / cpg) * 2 + 1], gamma[c] * f * s2);
        if (blockIdx.x == 0) {
            if (dss) {
                dss[(size_t)b * 2 * C + c] = gamma[c] * s2 + beta[c] * s1;   // d scale
                dss[(size_t)b * 2 * C + C + c] = s1;                          // d shift
            }
            atomicAdd(&dgamma[c], f * s2);
            atomicAdd(&dbeta[c], f * s1);
        }
    }
    __syncthreads();
    float mean[2], rstd[2], m1[2], m2[2], gmv[8], bt[8], s1p[8], sh[8];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        int g = (o * 8 + h * 4) / cpg;
        gn_mean_rstd(sums, b, g, G, inv_n, eps, mean[h], rstd[h]);
        m1[h] = gm[g * 2] * inv_n;
        m2[h] = gm[g * 2 + 1] * inv_n;
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        int c = o * 8 + k;
        gmv[k] = gamma[c]; bt[k] = beta[c];
        s1p[k] = ss ? ss[(size_t)b * 2 * C + c] + 1.f : 1.f;
        sh[k] = ss ? ss[(size_t)b * 2 * C + C + c] : 0.f;
    }
    float colsum[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    const size_t base = (size_t)b * HW * C;
    for (int p = blockIdx.x * rows_per_pass + r0; p < HW; p += gridDim.x * rows_per_pass) {
        float v[8], d[8];
        ld8(x + base + (size_t)p * C + o * 8, v);
        ld8(dy + base + (size_t)p * C + o * 8, d);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            float xh = (v[k] - mean[k >> 2]) * rstd[k >> 2];
            float z = (xh * gmv[k] + bt[k]) * s1p[k] + sh[k];
            float dz = d[k] * silu_grad_f(z);
            float g = rstd[k >> 2] * (gmv[k] * s1p[k] * dz - m1[k >> 2] - xh * m2[k >> 2]);
            v[k] = g;
            colsum[k] += g;
        }
        st8(dx + base + (size_t)p * C + o * 8, v);
    }
    if (dbias) {
        if (reduce_same_octet(colsum, oct)) {
#pragma unroll
            for (int k = 0; k < 8; ++k) atomicAdd(&cs[o * 8 + k], colsum[k]);
        }
        __syncthreads();
        for (int i = threadIdx.x; i < C; i += blockDim.x) atomicAdd(&dbias[i], cs[i]);
    }
}

// Single-launch backward.  GroupNorm couples only the channels of one group, so the work is cut into (sample, channel
// slab) pieces -- a slab is one or more whole groups and at least 32 bytes of channels per pixel -- and a piece is owned by
// a cluster of CL CTAs that split its pixels (CL = 1 at the low-resolution levels: no cluster launch at all).
//   phase 1: per-channel sums of dz and dz*xhat over the thread's pixels -> warp shuffles -> shared memory
//            (-> distributed shared memory across the CL CTAs of the cluster)
//   phase 2: dx = rstd * (gamma*(1+scale)*dz - m1 - xhat*m2), FiLM / affine / bias gradients
// KEEP = true (<= 2 vectors per thread): xhat and dz stay in REGISTERS between the phases, x and dy are read once.
// KEEP = false: phase 2 re-reads the thread's own vectors (L1 / L2 hits: the CTA touched them a few microseconds
// earlier), two vectors at a time -- holding 4 x 8 x 2 fp32 values per thread costs 156 registers = one CTA per SM.
// Either way the grid has 256..512 CTAs at every level of the U-Net (the first version ran one CTA or one 8-CTA cluster
// per SAMPLE: 32 CTAs for the whole GPU at the 8x8 level, a small fraction of one wave).
// Element-wise arithmetic is the same, in the same order, as in gn_bwd_reduce_kernel + gn_bwd_dx_kernel.
template <typename T, int V, bool KEEP>
__global__ void __launch_bounds__(NORM_THREADS, 2) gn_bwd_piece_kernel(
        const T* __restrict__ x, const T* __restrict__ dy, const float* __restrict__ sums, const float* __restrict__ gamma,
        const float* __restrict__ beta, const float* __restrict__ ss, T* __restrict__ dx, float* __restrict__ dss,
        float* __restrict__ dgamma, float* __restrict__ dbeta, float* __restrict__ dbias, int HW, int C, int G, float eps,
        int S /*channels per slab*/, int CL /*CTAs per (sample, slab)*/, int rows_per_cta, int nchunks) {
    namespace cg = cooperative_groups;
    constexpr int VE = Vec<T>::N;
    extern __shared__ float rsm[];
    float* part = rsm;                 // [S][2] partial sums of this CTA
    float* Sf = part + 2 * S;          // [S][2] sums over the whole (sample, slab)
    float* gm = Sf + 2 * S;            // [S / cpg][2]
    float* cs = gm + 2 * (S / (C / G));// [S] column sums of dx
    const int cpg = C / G, so = S / VE, nslab = C / S;
    const int piece = blockIdx.x / CL, rank = blockIdx.x - piece * CL;
    const int b = piece / nslab, slab = piece - b * nslab;
    const int c0 = slab * S;                                   // first channel of the slab
    const int o = threadIdx.x % so, r0 = threadIdx.x / so;
    const int rpp = blockDim.x / so;
    const int row_begin = rank * rows_per_cta;
    const int row_end = min(HW, row_begin + rows_per_cta);
    const float inv_n = 1.f / ((float)cpg * (float)HW);
    pdl_trigger();
    float gmv[VE], bt[VE];
#pragma unroll
    for (int k = 0; k < VE; ++k) { gmv[k] = gamma[c0 + o * VE + k]; bt[k] = beta[c0 + o * VE + k]; }
    for (int i = threadIdx.x; i < 5 * S + 2 * (S / cpg); i += blockDim.x) rsm[i] = 0.f;
    pdl_wait();
    const size_t base = (size_t)b * HW * C + c0 + (size_t)o * VE;
    float xv[V][VE], dv[V][VE];
    bool ok[V];
    // the first chunk's loads are issued before the parameter loads they do not depend on
#pragma unroll
    for (int u = 0; u < V; ++u) {
        const int p = row_begin + r0 + u * rpp;
        ok[u] = p < row_end;
        if (ok[u]) {
            ldv<T>(x + base + (size_t)p * C, xv[u]);
            ldv<T>(dy + base + (size_t)p * C, dv[u]);
        }
    }
    float mean[VE], rstd[VE], s1p[VE], sh[VE];
#pragma unroll
    for (int k = 0; k < VE; k += 4) {
        float m, r;
        gn_mean_rstd(sums, b, (c0 + o * VE + k) / cpg, G, inv_n, eps, m, r);
#pragma unroll
        for (int j = 0; j < 4; ++j) { mean[k + j] = m; rstd[k + j] = r; }
    }
#pragma unroll
    for (int k = 0; k < VE; ++k) {
        const int c = c0 + o * VE + k;
        s1p[k] = ss ? ss[(size_t)b * 2 * C + c] + 1.f : 1.f;
        sh[k] = ss ? ss[(size_t)b * 2 * C + C + c] : 0.f;
    }
    // ---- phase 1
    float a1[VE], a2[VE];
#pragma unroll
    for (int k = 0; k < VE; ++k) { a1[k] = 0.f; a2[k] = 0.f; }
    for (int it = 0; it < nchunks; ++it) {
        if (it > 0) {
#pragma unroll
            for (int u = 0; u < V; ++u) {
                const int p = row_begin + r0 + (it * V + u) * rpp;
                ok[u] = p < row_end;
                if (ok[u]) {
                    ldv<T>(x + base + (size_t)p * C, xv[u]);
                    ldv<T>(dy + base + (size_t)p * C, dv[u]);
                }
            }
        }
#pragma unroll
        for (int u = 0; u < V; ++u) {
            if (ok[u]) {
#pragma unroll
                for (int k = 0; k < VE; ++k) {
                    const float xh = (xv[u][k] - mean[k]) * rstd[k];
                    const float z = (xh * gmv[k] + bt[k]) * s1p[k] + sh[k];
                    const float dz = dv[u][k] * silu_grad_f(z);
                    a1[k] += dz; a2[k] += dz * xh;
                    if (KEEP) { xv[u][k] = xh; dv[u][k] = dz; }       // keep xhat / dz for phase 2
                }
            }
        }
    }
    __syncthreads();                                           // zero-fill of the shared sums is complete
    const bool pub1 = reduce_same_octet(a1, so);
    reduce_same_octet(a2, so);
    if (pub1) {
#pragma unroll
        for (int k = 0; k < VE; ++k) { atomicAdd(&part[(o * VE + k) * 2], a1[k]); atomicAdd(&part[(o * VE + k) * 2 + 1], a2[k]); }
    }
    if (CL > 1) {
        cg::cluster_group cluster = cg::this_cluster();
        cluster.sync();                                        // all partial vectors of the piece are complete
        for (int i = threadIdx.x; i < 2 * S; i += blockDim.x) {
            float t = 0.f;
            for (int r = 0; r < CL; ++r) t += cluster.map_shared_rank(part, r)[i];
            Sf[i] = t;
        }
        cluster.sync();                                        // nobody reads a peer's `part` after this point
    } else {
        __syncthreads();
        for (int i = threadIdx.x; i < 2 * S; i += blockDim.x) Sf[i] = part[i];
        __syncthreads();
    }
    for (int cl = threadIdx.x; cl < S; cl += blockDim.x) {
        const int c = c0 + cl;
        const float s1 = Sf[cl * 2], s2 = Sf[cl * 2 + 1];
        const float f = ss ? ss[(size_t)b * 2 * C + c] + 1.f : 1.f;
        atomicAdd(&gm[(cl / cpg) * 2], gamma[c] * f * s1);
        atomicAdd(&gm[(cl / cpg) * 2 + 1], gamma[c] * f * s2);
        if (rank == 0) {
            if (dss) {
                dss[(size_t)b * 2 * C + c] = gamma[c] * s2 + beta[c] * s1;   // d scale
                dss[(size_t)b * 2 * C + C + c] = s1;                          // d shift
            }
            atomicAdd(&dgamma[c], f * s2);
            atomicAdd(&dbeta[c], f * s1);
        }
    }
    __syncthreads();
    // ---- phase 2
    float m1[VE], m2[VE];
#pragma unroll
    for (int k = 0; k < VE; k += 4) {
        const int gl = (o * VE + k) / cpg;
#pragma unroll
        for (int j = 0; j < 4; ++j) { m1[k + j] = gm[gl * 2] * inv_n; m2[k + j] = gm[gl * 2 + 1] * inv_n; }
    }
    float colsum[VE];
#pragma unroll
    for (int k = 0; k < VE; ++k) colsum[k] = 0.f;
    for (int it = 0; it < nchunks; ++it) {
        if (!KEEP) {
#pragma unroll
            for (int u = 0; u < V; ++u) {
                const int p = row_begin + r0 + (it * V + u) * rpp;
                ok[u] = p < row_end;
                if (ok[u]) {
                    ldv<T>(x + base + (size_t)p * C, xv[u]);
                    ldv<T>(dy + base + (size_t)p * C, dv[u]);
                }
            }
        }
#pragma unroll
        for (int u = 0; u < V; ++u) {
            if (ok[u]) {
                float g[VE];
#pragma unroll
                for (int k = 0; k < VE; ++k) {
                    float xh, dz;
                    if (KEEP) { xh = xv[u][k]; dz = dv[u][k]; }
                    else {
                        xh = (xv[u][k] - mean[k]) * rstd[k];
                        const float z = (xh * gmv[k] + bt[k]) * s1p[k] + sh[k];
                        dz = dv[u][k] * silu_grad_f(z);
                    }
                    g[k] = rstd[k] * (gmv[k] * s1p[k] * dz - m1[k] - xh * m2[k]);
                    colsum[k] += g[k];
                }
                stv<T>(dx + base + (size_t)(row_begin + r0 + (it * V + u) * rpp) * C, g);
            }
        }
    }
    if (dbias) {
        if (reduce_same_octet(colsum, so)) {
#pragma unroll
            for (int k = 0; k < VE; ++k) atomicAdd(&cs[o * VE + k], colsum[k]);
        }
        __syncthreads();
        for (int i = threadIdx.x; i < S; i += blockDim.x) atomicAdd(&dbias[c0 + i], cs[i]);
    }
}

// ------------------------------------------------------------------------------------------------
// channel LayerNorm: y[m,c] = (x[m,c]-mean_m)/sqrt(var_m+eps)*gamma[c]
// a group of L = min(32, C/8) lanes owns one pixel; lane handles octets lane, lane+L, ...
// ------------------------------------------------------------------------------------------------
template <typename T, bool BWD>
__global__ void ln_kernel(const T* __restrict__ x, const T* __restrict__ dy, const float* __restrict__ gamma,
                          T* __restrict__ out, float* __restrict__ dgamma, const T* __restrict__ res, long long M, int C,
                          float eps) {
    extern __shared__ float sdg[];  // [C] (BWD only)
    const int oct = C / 8;
    int L = 1;
    while (L < 32 && L < oct) L <<= 1;            // power of two
    const int lane = threadIdx.x & 31, sub = lane % L, grp = lane / L, gpw = 32 / L;
    const int warps = blockDim.x >> 5, warp = threadIdx.x >> 5;
    if (BWD) {
        for (int i = threadIdx.x; i < C; i += blockDim.x) sdg[i] = 0.f;
        __syncthreads();
    }
    float dg[4][8];   // up to 4 octets per lane (C <= 1024)
    if (BWD) {
#pragma unroll
        for (int q = 0; q < 4; ++q)
#pragma unroll
            for (int k = 0; k < 8; ++k) dg[q][k] = 0.f;
    }
    const long long stride = (long long)gridDim.x * warps * gpw;
    const long long first = ((long long)blockIdx.x * warps + warp) * gpw + grp;
    const long long iters = (M + stride - 1) / stride;   // uniform trip count (shuffles need all lanes)
    for (long long it = 0; it < iters; ++it) {
        long long m = first + it * stride;
        bool ok = m < M;
        float s = 0.f, ss = 0.f;
        if (ok)
            for (int o = sub; o < oct; o += L) {
                float v[8];
                ld8(x + m * C + o * 8, v);
#pragma unroll
                for (int k = 0; k < 8; ++k) { s += v[k]; ss += v[k] * v[k]; }
            }
        for (int off = L >> 1; off > 0; off >>= 1) {
            s += __shfl_xor_sync(0xffffffffu, s, off);
            ss += __shfl_xor_sync(0xffffffffu, ss, off);
        }
        float mean = s / C;
        float rstd = rsqrtf(fmaxf(ss / C - mean * mean, 0.f) + eps);
        if (!BWD) {
            if (ok)
                for (int o = sub; o < oct; o += L) {
                    float v[8];
                    ld8(x + m * C + o * 8, v);
#pragma unroll
                    for (int k = 0; k < 8; ++k) v[k] = (v[k] - mean) * rstd * gamma[o * 8 + k];
                    st8(out + m * C + o * 8, v);
                }
        } else {
            float a = 0.f, bsum = 0.f;   // sum dxhat, sum dxhat*xhat
            if (ok) {
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const int o = sub + q * L;
                    if (o >= oct) break;
                    float v[8], d[8];
                    ld8(x + m * C + o * 8, v);
                    ld8(dy + m * C + o * 8, d);
#pragma unroll
                    for (int k = 0; k < 8; ++k) {
                        float xh = (v[k] - mean) * rstd;
                        float dxh = d[k] * gamma[o * 8 + k];
                        a += dxh; bsum += dxh * xh;
                        dg[q][k] += d[k] * xh;
                    }
                }
            }
            for (int off = L >> 1; off > 0; off >>= 1) {
                a += __shfl_xor_sync(0xffffffffu, a, off);
                bsum += __shfl_xor_sync(0xffffffffu, bsum, off);
            }
            a /= C; bsum /= C;
            if (ok)
                for (int o = sub; o < oct; o += L) {
                    float v[8], d[8];
                    ld8(x + m * C + o * 8, v);
                    ld8(dy + m * C + o * 8, d);
#pragma unroll
                    for (int k = 0; k < 8; ++k) {
                        float xh = (v[k] - mean) * rstd;
                        v[k] = rstd * (d[k] * gamma[o * 8 + k] - a - xh * bsum);
                    }
                    if (res) {
                        float rr[8];
                        ld8(res + m * C + o * 8, rr);
#pragma unroll
                        for (int k = 0; k < 8; ++k) v[k] += rr[k];
                    }
                    st8(out + m * C + o * 8, v);
                }
        }
    }
    if (BWD) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int o = sub + q * L;
            if (o < oct) {
#pragma unroll
                for (int k = 0; k < 8; ++k) atomicAdd(&sdg[o * 8 + k], dg[q][k]);
            }
        }
        __syncthreads();
        for (int i = threadIdx.x; i < C; i += blockDim.x) atomicAdd(&dgamma[i], sdg[i]);
    }
}

// Fast path for C = 32, 64, 128, 256 (C/8 a power of two <= 32): a group of L = C/8 lanes owns a pixel and every lane
// exactly one channel octet, so x (and dy) are read ONCE into registers; LN_UNR pixels per group are in flight together.
constexpr int LN_UNR = 4;
template <typename T, bool BWD>
__global__ void __launch_bounds__(256) ln1_kernel(const T* __restrict__ x, const T* __restrict__ dy,
                                                  const float* __restrict__ gamma, T* __restrict__ out,
                                                  float* __restrict__ dgamma, const T* __restrict__ res, long long M,
                                                  int C, float eps) {
    extern __shared__ float sdg[];  // [C] (BWD only)
    pdl_trigger();
    pdl_wait();
    const int L = C / 8;
    const int lane = threadIdx.x & 31, sub = lane % L, grp = lane / L, gpw = 32 / L;
    const int warps = blockDim.x >> 5, warp = threadIdx.x >> 5;
    float gmm[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) gmm[k] = gamma[sub * 8 + k];
    if (BWD) {
        for (int i = threadIdx.x; i < C; i += blockDim.x) sdg[i] = 0.f;
        __syncthreads();
    }
    float dg[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    const float inv_c = 1.f / (float)C;
    const long long stride = (long long)gridDim.x * warps * gpw;          // pixels per sweep of the grid
    const long long first = ((long long)blockIdx.x * warps + warp) * gpw + grp;
    const long long iters = (M + stride * LN_UNR - 1) / (stride * LN_UNR);   // uniform trip count (shuffles)
    for (long long it = 0; it < iters; ++it) {
        float v[LN_UNR][8], d[LN_UNR][8];
        bool ok[LN_UNR];
#pragma unroll
        for (int u = 0; u < LN_UNR; ++u) {
            const long long m = first + (it * LN_UNR + u) * stride;
            ok[u] = m < M;
            if (ok[u]) {
                ld8(x + m * C + sub * 8, v[u]);
                if (BWD) ld8(dy + m * C + sub * 8, d[u]);
            } else {
#pragma unroll
                for (int k = 0; k < 8; ++k) { v[u][k] = 0.f; if (BWD) d[u][k] = 0.f; }
            }
        }
#pragma unroll
        for (int u = 0; u < LN_UNR; ++u) {
            const long long m = first + (it * LN_UNR + u) * stride;
            float s = 0.f, ss = 0.f;
#pragma unroll
            for (int k = 0; k < 8; ++k) { s += v[u][k]; ss += v[u][k] * v[u][k]; }
            for (int off = L >> 1; off > 0; off >>= 1) {
                s += __shfl_xor_sync(0xffffffffu, s, off);
                ss += __shfl_xor_sync(0xffffffffu, ss, off);
            }
            const float mean = s * inv_c;
            const float rstd = rsqrtf(fmaxf(ss * inv_c - mean * mean, 0.f) + eps);
            float o[8];
            if (!BWD) {
#pragma unroll
                for (int k = 0; k < 8; ++k) o[k] = (v[u][k] - mean) * rstd * gmm[k];
            } else {
                float a = 0.f, bsum = 0.f, xh[8];
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    xh[k] = (v[u][k] - mean) * rstd;
                    const float dxh = d[u][k] * gmm[k];
                    a += dxh; bsum += dxh * xh[k];
                    dg[k] += d[u][k] * xh[k];
                }
                for (int off = L >> 1; off > 0; off >>= 1) {
                    a += __shfl_xor_sync(0xffffffffu, a, off);
                    bsum += __shfl_xor_sync(0xffffffffu, bsum, off);
                }
                a *= inv_c; bsum *= inv_c;
#pragma unroll
                for (int k = 0; k < 8; ++k) o[k] = rstd * (d[u][k] * gmm[k] - a - xh[k] * bsum);
                if (res != nullptr && ok[u]) {          // gradient of a skip connection that bypasses the norm
                    float rr[8];
                    ld8(res + m * C + sub * 8, rr);
#pragma unroll
                    for (int k = 0; k < 8; ++k) o[k] += rr[k];
                }
            }
            if (ok[u]) st8(out + m * C + sub * 8, o);
        }
    }
    if (BWD) {
        if (reduce_same_octet(dg, L)) {
#pragma unroll
            for (int k = 0; k < 8; ++k) atomicAdd(&sdg[sub * 8 + k], dg[k]);
        }
        __syncthreads();
        for (int i = threadIdx.x; i < C; i += blockDim.x) atomicAdd(&dgamma[i], sdg[i]);
    }
}

static int gn_block(int C) {
    int oct = C / 8;
    int rows = NORM_THREADS / oct;
    if (rows < 1) rows = 1;
    return oct * rows;
}

}  // namespace pidm
using namespace pidm;

static int gn_check(int C, int G) {
    PIDM_REQUIRE(C % 8 == 0 && C / 8 <= 1024 && G > 0 && C % G == 0, "groupnorm: bad C=%d G=%d", C, G);
    int cpg = C / G;
    PIDM_REQUIRE(cpg == 4 || cpg % 8 == 0, "groupnorm: channels per group must be 4 or a multiple of 8 (got %d)", cpg);
    return 0;
}

static void gn_launch_dims(int HW, int C, int& block, int& chunks) {
    block = gn_block(C);
    const int rows = block / (C / 8);
    chunks = ceil_div(HW, rows * 2);          // ~2 pixels per thread: enough CTAs to cover the machine at 64x64
    if (chunks > 32) chunks = 32;
    if (chunks < 1) chunks = 1;
}

// Grid of gn_apply_kernel: a thread owns one 16-byte channel vector position (ov of them per pixel row);
// ~GN_APPLY_UNR vectors per thread, >= 2 waves of CTAs.  `rules` reports which adjustments fired (bit 0 shrink the unroll,
// bit 1 halve, bit 2 one wave and loop).
static int gn_apply_chunks(int B, int HW, int ov, int& rules) {
    const int rpp = NORM_THREADS / ov;
    int ach = ceil_div(HW, rpp * GN_APPLY_UNR);
    rules = 0;
    for (int u = GN_APPLY_UNR; u > 1 && (long long)B * ach < num_sms() * 2; u /= 2) { ach = ceil_div(HW, rpp * (u / 2)); rules |= 1; }
    while (ach > 1 && (long long)B * ach > num_sms() * 8) { ach = (ach + 1) / 2; rules |= 2; }
    // ~123 registers: two CTAs per SM are resident.  Between one and two waves the second wave runs mostly empty
    // (e.g. 512 CTAs at 64x64x32, batch 32): size the grid to one wave and let the CTAs loop
    if ((long long)B * ach > num_sms() * 2 && (long long)B * ach < num_sms() * 4 && B <= num_sms() * 2) { ach = (num_sms() * 2) / B; rules |= 4; }
    return ach;
}

// Plan of pidm_groupnorm_silu_bwd: the single-launch piece kernel (see gn_bwd_piece_kernel) with its channel slab S,
// thread count, cluster size cl, pixel rows per CTA and vectors per thread v, or the two-launch fallback (path 0).
struct GnBwdPlan { int path /*0 fallback, 1 piece<1>, 2 piece<2>, 3 packed<4>, 4 stream*/, S, threads, cl, rows_per_cta, v; };
static GnBwdPlan gn_bwd_plan(int B, int HW, int C, int G, int dtype) {
    GnBwdPlan pl = {0, 0, 0, 0, 0, 0};
    const int esz = dtype == PIDM_BF16 ? 2 : 4, ve = 16 / esz, cpg = C / G;
    int S = cpg;
    while (S * esz < 32 && S * 2 <= C && C % (S * 2) == 0) S *= 2;    // >= 32 bytes of channels per pixel row
    const int so = S / ve;
    const bool shape_ok = S % ve == 0 && so >= 1 && so <= 32 && (so & (so - 1)) == 0 && C % S == 0 && (C * esz) % 16 == 0;
    if (!shape_ok) return pl;
    const int nslab = C / S;
    const long long nv = (long long)HW * so;            // 16-byte vectors per (sample, slab)
    int threads = NORM_THREADS;
    while (threads > 32 && threads / 2 >= nv && (threads / 2) % so == 0) threads /= 2;
    // CTAs per piece.  A CTA of this kernel is a latency chain of a few microseconds whatever its size, a
    // second wave of CTAs doubles the launch and a cluster costs ~1 us extra -- so: no cluster unless a piece
    // has more than 8 vectors per thread, never more CTAs than are resident at once (2 per SM), and otherwise
    // as many CTAs as that allows.
    const int resident = num_sms() * 2;
    int cl = 1;
    while (cl < 8 && nv > (long long)cl * threads * 8) cl *= 2;
    while (cl < 8 && (long long)B * nslab * cl * 2 <= resident && nv > (long long)cl * threads) cl *= 2;
    const int rpp = threads / so;
    int rows_per_cta = ceil_div(HW, cl);
    rows_per_cta = ceil_div(rows_per_cta, rpp) * rpp;
    const int v = rows_per_cta / rpp;                   // vectors per thread
    if ((long long)rows_per_cta * (cl - 1) >= HW) return pl;        // a cluster rank would own no pixel
    // three shapes of a piece: <= 2 vectors per thread stay in registers unpacked between the phases; 3-4 vectors are
    // held packed (with 8 vectors that variant spills); larger pieces are streamed twice
    pl.path = v <= 1 ? 1 : v <= 2 ? 2 : v <= 4 ? 3 : 4;
    pl.S = S; pl.threads = threads; pl.cl = cl; pl.rows_per_cta = rows_per_cta; pl.v = v;
    return pl;
}

// sums [B,G,2] holds (sum, sum of squares) per (sample, group): computed here unless stats_precomputed (then it was
// filled by the producing convolution's epilogue); it must be kept for backward.
extern "C" int pidm_groupnorm_silu_fwd(const void* x, const float* gamma, const float* beta, const float* scale_shift,
                                       const void* residual, void* y, float* sums, int stats_precomputed, int B, int HW,
                                       int C, int G, float eps, int dtype, void* stream) {
    if (int e = gn_check(C, G)) return e;
    cudaStream_t st = (cudaStream_t)stream;
    int block, chunks;
    gn_launch_dims(HW, C, block, chunks);
    if (!stats_precomputed) PIDM_CUDA(cudaMemsetAsync(sums, 0, (size_t)B * G * 2 * sizeof(float), st));
    PIDM_DISPATCH_DTYPE(dtype, {
        if (!stats_precomputed)
            gn_stats_kernel<T><<<dim3(chunks, B), block, 2 * G * sizeof(float), st>>>((const T*)x, sums, HW, C, G);
        const int ov = C / Vec<T>::N;
        PIDM_REQUIRE(ov <= NORM_THREADS && NORM_THREADS % ov == 0, "groupnorm: C=%d is not supported by the apply kernel", C);
        int rules;
        const int ach = gn_apply_chunks(B, HW, ov, rules);
        PIDM_CUDA(launch_pdl(gn_apply_kernel<T>, dim3(ach, B), dim3(NORM_THREADS), 0, st, (const T*)x, (const float*)sums,
                             gamma, beta, scale_shift, (const T*)residual, (T*)y, HW, C, G, eps));
    });
    PIDM_LAUNCH_CHECK("groupnorm_silu_fwd");
    return 0;
}

// workspace: float[B*C*2].  dgamma/dbeta (and dbias_of_producer, if given) are ACCUMULATED (atomicAdd);
// d_scale_shift is overwritten.
extern "C" int pidm_groupnorm_silu_bwd(const void* x, const void* dy, const float* sums, const float* gamma,
                                       const float* beta, const float* scale_shift, void* dx, float* dgamma,
                                       float* dbeta, float* d_scale_shift, float* dbias_of_producer, float* workspace,
                                       int B, int HW, int C, int G, float eps, int dtype, void* stream) {
    if (int e = gn_check(C, G)) return e;
    cudaStream_t st = (cudaStream_t)stream;
    int block, chunks;
    gn_launch_dims(HW, C, block, chunks);
    const GnBwdPlan pl = gn_bwd_plan(B, HW, C, G, dtype);
    if (pl.path) {
        const int S = pl.S, cl = pl.cl, rows_per_cta = pl.rows_per_cta;
        const size_t smem = (size_t)(7 * S + 2 * (S / (C / G))) * sizeof(float);      // + 2 S: constants of the packed variant
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3((unsigned)(B * (C / S) * cl));
        cfg.blockDim = dim3((unsigned)pl.threads);
        cfg.dynamicSmemBytes = smem;
        cfg.stream = st;
        cudaLaunchAttribute attr[2];
        attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[0].val.programmaticStreamSerializationAllowed = 1;
        int na = 1;
        if (cl > 1) {
            attr[na].id = cudaLaunchAttributeClusterDimension;
            attr[na].val.clusterDim.x = (unsigned)cl; attr[na].val.clusterDim.y = 1; attr[na].val.clusterDim.z = 1;
            ++na;
        }
        cfg.attrs = attr; cfg.numAttrs = na;
#define GN_PIECE_ARGS (const T*)x, (const T*)dy, sums, gamma, beta, scale_shift, (T*)dx, d_scale_shift, dgamma, dbeta, \
                      dbias_of_producer, HW, C, G, eps, S, cl, rows_per_cta
        PIDM_DISPATCH_DTYPE(dtype, {
            if (pl.path == 1) PIDM_CUDA(cudaLaunchKernelEx(&cfg, gn_bwd_piece_kernel<T, 1, true>, GN_PIECE_ARGS, 1));
            else if (pl.path == 2) PIDM_CUDA(cudaLaunchKernelEx(&cfg, gn_bwd_piece_kernel<T, 2, true>, GN_PIECE_ARGS, 1));
            else if (pl.path == 3) PIDM_CUDA(cudaLaunchKernelEx(&cfg, gn_bwd_piece_packed_kernel<T, 4>, GN_PIECE_ARGS));
            else PIDM_CUDA(cudaLaunchKernelEx(&cfg, gn_bwd_piece_stream_kernel<T>, GN_PIECE_ARGS));
        });
#undef GN_PIECE_ARGS
        PIDM_LAUNCH_CHECK("groupnorm_silu_bwd(piece)");
        return 0;
    }
    float* S = workspace;
    PIDM_CUDA(cudaMemsetAsync(S, 0, (size_t)B * C * 2 * sizeof(float), st));
    PIDM_DISPATCH_DTYPE(dtype, {
        gn_bwd_reduce_kernel<T><<<dim3(chunks, B), block, 2 * C * sizeof(float), st>>>(
            (const T*)x, (const T*)dy, sums, gamma, beta, scale_shift, S, HW, C, G, eps);
        gn_bwd_dx_kernel<T><<<dim3(chunks, B), block, (2 * G + C) * sizeof(float), st>>>(
            (const T*)x, (const T*)dy, sums, gamma, beta, scale_shift, S, (T*)dx, d_scale_shift, dgamma, dbeta,
            dbias_of_producer, HW, C, G, eps);
    });
    PIDM_LAUNCH_CHECK("groupnorm_silu_bwd");
    return 0;
}

// What the two entry points above launch for a shape (test aid).  out[10] = {statistics chunks, statistics block, apply
// chunks, apply grid rules (bit 0 shrink the unroll, bit 1 halve, bit 2 one wave and loop), backward path (0 two-launch
// fallback, 1 piece<1>, 2 piece<2>, 3 packed<4>, 4 stream), channel slab S, threads, cluster size, pixel rows per CTA,
// vectors per thread}; the last five are 0 on the fallback path.
extern "C" int pidm_groupnorm_plan(int B, int HW, int C, int G, int dtype, int* out) {
    if (int e = gn_check(C, G)) return e;
    PIDM_REQUIRE(dtype == PIDM_BF16 || dtype == PIDM_F32, "unknown dtype code %d", dtype);
    const int ov = C / (dtype == PIDM_BF16 ? 8 : 4);
    PIDM_REQUIRE(ov <= NORM_THREADS && NORM_THREADS % ov == 0, "groupnorm: C=%d is not supported by the apply kernel", C);
    int block, chunks, rules;
    gn_launch_dims(HW, C, block, chunks);
    const int ach = gn_apply_chunks(B, HW, ov, rules);
    const GnBwdPlan pl = gn_bwd_plan(B, HW, C, G, dtype);
    const int v[10] = {chunks, block, ach, rules, pl.path, pl.S, pl.threads, pl.cl, pl.rows_per_cta, pl.v};
    for (int i = 0; i < 10; ++i) out[i] = v[i];
    return 0;
}

extern "C" int pidm_layernorm_c_fwd(const void* x, const float* gamma, void* y, long long M, int C, float eps, int dtype,
                                    void* stream) {
    PIDM_REQUIRE(C % 8 == 0 && C <= 1024, "layernorm: C must be a multiple of 8 and <= 1024 (got %d)", C);
    int oct = C / 8, L = 1;
    while (L < 32 && L < oct) L <<= 1;
    long long groups = (M + (32 / L) * 8 - 1) / ((32 / L) * 8);
    int grid = (int)(groups < num_sms() * 8 ? (groups < 1 ? 1 : groups) : num_sms() * 8);
    if (L == oct) {          // one octet per lane: register-resident kernel
        long long g1 = (M + (32 / L) * 8 * LN_UNR - 1) / ((32 / L) * 8 * LN_UNR);
        int grid1 = (int)(g1 < num_sms() * 8 ? (g1 < 1 ? 1 : g1) : num_sms() * 8);
        PIDM_DISPATCH_DTYPE(dtype, PIDM_CUDA(launch_pdl(ln1_kernel<T, false>, dim3(grid1), dim3(256), 0, (cudaStream_t)stream,
                                                        (const T*)x, (const T*)nullptr, gamma, (T*)y, (float*)nullptr,
                                                        (const T*)nullptr, M, C, eps)));
        PIDM_LAUNCH_CHECK("layernorm_c_fwd");
        return 0;
    }
    PIDM_DISPATCH_DTYPE(dtype, (ln_kernel<T, false><<<grid, 256, 0, (cudaStream_t)stream>>>(
                                   (const T*)x, nullptr, gamma, (T*)y, nullptr, nullptr, M, C, eps)));
    PIDM_LAUNCH_CHECK("layernorm_c_fwd");
    return 0;
}

// dgamma is ACCUMULATED.  dx_residual (optional, same shape as dx) is added to dx: the gradient of a skip connection
// that bypasses the norm, so that the caller needs no separate accumulation kernel.
extern "C" int pidm_layernorm_c_bwd(const void* x, const void* dy, const float* gamma, void* dx, float* dgamma,
                                    const void* dx_residual, long long M, int C, float eps, int dtype, void* stream) {
    PIDM_REQUIRE(C % 8 == 0 && C <= 1024, "layernorm: C must be a multiple of 8 and <= 1024 (got %d)", C);
    int oct = C / 8, L = 1;
    while (L < 32 && L < oct) L <<= 1;
    long long groups = (M + (32 / L) * 8 - 1) / ((32 / L) * 8);
    int grid = (int)(groups < num_sms() * 4 ? (groups < 1 ? 1 : groups) : num_sms() * 4);
    if (L == oct) {
        long long g1 = (M + (32 / L) * 8 * LN_UNR - 1) / ((32 / L) * 8 * LN_UNR);
        int grid1 = (int)(g1 < num_sms() * 4 ? (g1 < 1 ? 1 : g1) : num_sms() * 4);
        PIDM_DISPATCH_DTYPE(dtype, PIDM_CUDA(launch_pdl(ln1_kernel<T, true>, dim3(grid1), dim3(256), C * sizeof(float),
                                                        (cudaStream_t)stream, (const T*)x, (const T*)dy, gamma, (T*)dx,
                                                        dgamma, (const T*)dx_residual, M, C, eps)));
        PIDM_LAUNCH_CHECK("layernorm_c_bwd");
        return 0;
    }
    PIDM_DISPATCH_DTYPE(dtype, (ln_kernel<T, true><<<grid, 256, C * sizeof(float), (cudaStream_t)stream>>>(
                                   (const T*)x, (const T*)dy, gamma, (T*)dx, dgamma, (const T*)dx_residual, M, C, eps)));
    PIDM_LAUNCH_CHECK("layernorm_c_bwd");
    return 0;
}
