// Darcy-flow PDE residual on x0_hat = (p, K):   reference src/residuals_darcy.py:134-183 with the
// second-order finite-difference operators of src/grad_utils.py:64-146 (net semantics: central stencil
// in the interior, one-sided 3-/4-point stencils at the two ends of each axis).
//
//   r[b, i*P+j, 0] = -K (p_00 + p_11) - K_0 p_0 - K_1 p_1 - f_s
//   r[b, i*P+j, 1] = (i==0 ? -p_0 : i==P-1 ? +p_0 : 0)
//   r[b, i*P+j, 2] = (j==0 ? +s p_1 : j==P-1 ? -s p_1 : 0),  s = +1 if reverse_d1 else -1
//
// bcs='periodic' (PIDM_DARCY_PERIODIC; reference grad_utils.py:76-81, circular padding + the interior stencil): every
// kernel has a PER = true instantiation in which every pixel uses the central stencil with wrapped neighbours.  The two
// BC channels keep their rows / columns and signs.  The PER = false instantiations compile to the same SASS as before.
//
// Design: HBM-bound (about 2 flop/byte).  Persistent CTAs; every sample (p-plane + K-plane,
// 2*P*P*4 = 32 KiB contiguous in NCHW) is staged into shared memory by ONE bulk-async (TMA) copy
// that completes on an mbarrier, double-buffered so the copy of sample n+1 overlaps the stencil math
// of sample n.  All stencils read shared memory (the halo is the plane itself: one-sided stencils at
// the boundary), each thread owns 4 consecutive pixels so that the interleaved [P*P,3] residual is
// written with 128-bit coalesced stores (48 contiguous bytes per thread, 1536 per warp).
// Loss-fused variants never materialise r: warp-shuffle + one atomic per CTA for the sums, and the
// gradient is produced in the same pass (transposed stencils gathered from five product planes in smem).
#include "common.cuh"
#include "pidm.h"
#include <stddef.h>

namespace pidm {

constexpr int P = 64;             // pixels per dim (reference: pixels_per_dim = 64, main.py:73)
constexpr int PP = P * P;
constexpr int DARCY_THREADS = 256;

__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

struct DarcyGeom {
    float inv_h0, inv_h1;      // 1/d0, 1/d1 (d1 negative when reverse_d1)
    float inv_h0sq, inv_h1sq;
    float bc1_sign;            // +1 if reverse_d1 else -1
};

// f_s on the pixel-centre grid: +10 on rows/cols [0,8), -10 on [56,64)  (residuals_darcy.py:40-53,95-104)
__device__ __forceinline__ float source_fs(int i, int j, const float* __restrict__ fs) { return fs[i * P + j]; }

// ---- pointwise stencil helpers on a PxP plane in shared memory ------------------------------------
// PER (bcs='periodic', reference grad_utils.py:76-81): the central stencil at every pixel, neighbours wrap around the
// plane.  PER = false is the one-sided-boundary code.
__device__ __forceinline__ int wrap(int x) { return x & (P - 1); }   // P is a power of two

template <bool PER>
__device__ __forceinline__ float d_row(const float* u, int i, int j, float inv_h) {  // d/dx0
    if constexpr (PER) return (u[wrap(i + 1) * P + j] - u[wrap(i - 1) * P + j]) * (0.5f * inv_h);
    if (i == 0) return (-1.5f * u[j] + 2.f * u[P + j] - 0.5f * u[2 * P + j]) * inv_h;
    if (i == P - 1) return (1.5f * u[(P - 1) * P + j] - 2.f * u[(P - 2) * P + j] + 0.5f * u[(P - 3) * P + j]) * inv_h;
    return (u[(i + 1) * P + j] - u[(i - 1) * P + j]) * (0.5f * inv_h);
}
template <bool PER>
__device__ __forceinline__ float d_col(const float* u, int i, int j, float inv_h) {  // d/dx1
    const float* r = u + i * P;
    if constexpr (PER) return (r[wrap(j + 1)] - r[wrap(j - 1)]) * (0.5f * inv_h);
    if (j == 0) return (-1.5f * r[0] + 2.f * r[1] - 0.5f * r[2]) * inv_h;
    if (j == P - 1) return (1.5f * r[P - 1] - 2.f * r[P - 2] + 0.5f * r[P - 3]) * inv_h;
    return (r[j + 1] - r[j - 1]) * (0.5f * inv_h);
}
template <bool PER>
__device__ __forceinline__ float d2_row(const float* u, int i, int j, float inv_h2) {
    if constexpr (PER) return (u[wrap(i + 1) * P + j] - 2.f * u[i * P + j] + u[wrap(i - 1) * P + j]) * inv_h2;
    if (i == 0) return (2.f * u[j] - 5.f * u[P + j] + 4.f * u[2 * P + j] - u[3 * P + j]) * inv_h2;
    if (i == P - 1)
        return (2.f * u[(P - 1) * P + j] - 5.f * u[(P - 2) * P + j] + 4.f * u[(P - 3) * P + j] - u[(P - 4) * P + j]) * inv_h2;
    return (u[(i + 1) * P + j] - 2.f * u[i * P + j] + u[(i - 1) * P + j]) * inv_h2;
}
template <bool PER>
__device__ __forceinline__ float d2_col(const float* u, int i, int j, float inv_h2) {
    const float* r = u + i * P;
    if constexpr (PER) return (r[wrap(j + 1)] - 2.f * r[j] + r[wrap(j - 1)]) * inv_h2;
    if (j == 0) return (2.f * r[0] - 5.f * r[1] + 4.f * r[2] - r[3]) * inv_h2;
    if (j == P - 1) return (2.f * r[P - 1] - 5.f * r[P - 2] + 4.f * r[P - 3] - r[P - 4]) * inv_h2;
    return (r[j + 1] - 2.f * r[j] + r[j - 1]) * inv_h2;
}

// Residual triple for the 4 pixels (i, j0..j0+3) from planes p, K in smem.
template <bool PER>
__device__ __forceinline__ void residual_quad(const float* sp, const float* sk, const float* __restrict__ fs, int i,
                                              int j0, const DarcyGeom& g, float req[4], float rb0[4], float rb1[4]) {
    // row-direction derivatives are row-uniform across the quad: vectorised float4 rows
    float p0[4], p00[4], k0[4];
    {
        float4 a, b, c, d;
        if (i == 0 || i == P - 1) {
            int s = (i == 0) ? 1 : -1;
            a = *reinterpret_cast<const float4*>(sp + i * P + j0);
            b = *reinterpret_cast<const float4*>(sp + (i + s) * P + j0);
            c = *reinterpret_cast<const float4*>(sp + (i + 2 * s) * P + j0);
            d = *reinterpret_cast<const float4*>(sp + (i + 3 * s) * P + j0);
            float sg = (float)s * g.inv_h0;
            p0[0] = (-1.5f * a.x + 2.f * b.x - 0.5f * c.x) * sg;
            p0[1] = (-1.5f * a.y + 2.f * b.y - 0.5f * c.y) * sg;
            p0[2] = (-1.5f * a.z + 2.f * b.z - 0.5f * c.z) * sg;
            p0[3] = (-1.5f * a.w + 2.f * b.w - 0.5f * c.w) * sg;
            p00[0] = (2.f * a.x - 5.f * b.x + 4.f * c.x - d.x) * g.inv_h0sq;
            p00[1] = (2.f * a.y - 5.f * b.y + 4.f * c.y - d.y) * g.inv_h0sq;
            p00[2] = (2.f * a.z - 5.f * b.z + 4.f * c.z - d.z) * g.inv_h0sq;
            p00[3] = (2.f * a.w - 5.f * b.w + 4.f * c.w - d.w) * g.inv_h0sq;
            a = *reinterpret_cast<const float4*>(sk + i * P + j0);
            b = *reinterpret_cast<const float4*>(sk + (i + s) * P + j0);
            c = *reinterpret_cast<const float4*>(sk + (i + 2 * s) * P + j0);
            k0[0] = (-1.5f * a.x + 2.f * b.x - 0.5f * c.x) * sg;
            k0[1] = (-1.5f * a.y + 2.f * b.y - 0.5f * c.y) * sg;
            k0[2] = (-1.5f * a.z + 2.f * b.z - 0.5f * c.z) * sg;
            k0[3] = (-1.5f * a.w + 2.f * b.w - 0.5f * c.w) * sg;
        } else {
            a = *reinterpret_cast<const float4*>(sp + (i - 1) * P + j0);
            b = *reinterpret_cast<const float4*>(sp + i * P + j0);
            c = *reinterpret_cast<const float4*>(sp + (i + 1) * P + j0);
            float hh = 0.5f * g.inv_h0;
            p0[0] = (c.x - a.x) * hh; p0[1] = (c.y - a.y) * hh; p0[2] = (c.z - a.z) * hh; p0[3] = (c.w - a.w) * hh;
            p00[0] = (c.x - 2.f * b.x + a.x) * g.inv_h0sq;
            p00[1] = (c.y - 2.f * b.y + a.y) * g.inv_h0sq;
            p00[2] = (c.z - 2.f * b.z + a.z) * g.inv_h0sq;
            p00[3] = (c.w - 2.f * b.w + a.w) * g.inv_h0sq;
            a = *reinterpret_cast<const float4*>(sk + (i - 1) * P + j0);
            c = *reinterpret_cast<const float4*>(sk + (i + 1) * P + j0);
            k0[0] = (c.x - a.x) * hh; k0[1] = (c.y - a.y) * hh; k0[2] = (c.z - a.z) * hh; k0[3] = (c.w - a.w) * hh;
        }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        int j = j0 + q;
        float kv = sk[i * P + j];
        float p1 = d_col<PER>(sp, i, j, g.inv_h1);
        float p11 = d2_col<PER>(sp, i, j, g.inv_h1sq);
        float k1 = d_col<PER>(sk, i, j, g.inv_h1);
        req[q] = -kv * (p00[q] + p11) - k0[q] * p0[q] - k1 * p1 - source_fs(i, j, fs);
        rb0[q] = (i == 0) ? -p0[q] : ((i == P - 1) ? p0[q] : 0.f);
        rb1[q] = (j == 0) ? g.bc1_sign * p1 : ((j == P - 1) ? -g.bc1_sign * p1 : 0.f);
    }
}

// Periodic: rows i-1 and i+1 wrap, so every row takes the central float4 path.
template <>
__device__ __forceinline__ void residual_quad<true>(const float* sp, const float* sk, const float* __restrict__ fs, int i,
                                                    int j0, const DarcyGeom& g, float req[4], float rb0[4], float rb1[4]) {
    const int im = wrap(i - 1), ip = wrap(i + 1);
    const float hh = 0.5f * g.inv_h0;
    float4 a = *reinterpret_cast<const float4*>(sp + im * P + j0);
    const float4 b = *reinterpret_cast<const float4*>(sp + i * P + j0);
    float4 c = *reinterpret_cast<const float4*>(sp + ip * P + j0);
    const float p0[4] = {(c.x - a.x) * hh, (c.y - a.y) * hh, (c.z - a.z) * hh, (c.w - a.w) * hh};
    const float p00[4] = {(c.x - 2.f * b.x + a.x) * g.inv_h0sq, (c.y - 2.f * b.y + a.y) * g.inv_h0sq,
                          (c.z - 2.f * b.z + a.z) * g.inv_h0sq, (c.w - 2.f * b.w + a.w) * g.inv_h0sq};
    a = *reinterpret_cast<const float4*>(sk + im * P + j0);
    c = *reinterpret_cast<const float4*>(sk + ip * P + j0);
    const float k0[4] = {(c.x - a.x) * hh, (c.y - a.y) * hh, (c.z - a.z) * hh, (c.w - a.w) * hh};
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const int j = j0 + q;
        const float kv = sk[i * P + j];
        const float p1 = d_col<true>(sp, i, j, g.inv_h1);
        const float p11 = d2_col<true>(sp, i, j, g.inv_h1sq);
        const float k1 = d_col<true>(sk, i, j, g.inv_h1);
        req[q] = -kv * (p00[q] + p11) - k0[q] * p0[q] - k1 * p1 - source_fs(i, j, fs);
        rb0[q] = (i == 0) ? -p0[q] : ((i == P - 1) ? p0[q] : 0.f);
        rb1[q] = (j == 0) ? g.bc1_sign * p1 : ((j == P - 1) ? -g.bc1_sign * p1 : 0.f);
    }
}

// ---- adjoint (transposed) 1-D operators, gather form ------------------------------------------------
// (D^T F)[x] for the first-derivative matrix D (central interior rows 1..P-2, one-sided rows 0 and P-1).
// Periodic: D is circulant, D^T F(x) = (F(x-1) - F(x+1)) / 2h and D2^T = D2, indices wrapped.
template <bool PER, typename F>
__device__ __forceinline__ float adj_d1(F f, int x, float inv_h) {
    if constexpr (PER) return (f(wrap(x - 1)) * 0.5f - f(wrap(x + 1)) * 0.5f) * inv_h;
    float acc = 0.f;
    if (x - 1 >= 1) acc += f(x - 1) * 0.5f;           // row x-1 is interior (x-1 <= P-2 always when x<=P-1)
    if (x + 1 <= P - 2) acc -= f(x + 1) * 0.5f;       // row x+1 is interior
    if (x <= 2) acc += f(0) * (x == 0 ? -1.5f : (x == 1 ? 2.f : -0.5f));
    if (x >= P - 3) acc += f(P - 1) * (x == P - 1 ? 1.5f : (x == P - 2 ? -2.f : 0.5f));
    return acc * inv_h;
}
// fix-up: interior rows are 1..P-2, so row x-1 is interior iff 1 <= x-1 <= P-2, row x+1 iff 1 <= x+1 <= P-2.
template <bool PER, typename F>
__device__ __forceinline__ float adj_d2(F f, int x, float inv_h2) {
    if constexpr (PER) return (f(wrap(x - 1)) - 2.f * f(x) + f(wrap(x + 1))) * inv_h2;
    float acc = 0.f;
    if (x - 1 >= 1 && x - 1 <= P - 2) acc += f(x - 1);
    if (x >= 1 && x <= P - 2) acc -= 2.f * f(x);
    if (x + 1 >= 1 && x + 1 <= P - 2) acc += f(x + 1);
    if (x <= 3) acc += f(0) * (x == 0 ? 2.f : (x == 1 ? -5.f : (x == 2 ? 4.f : -1.f)));
    if (x >= P - 4) acc += f(P - 1) * (x == P - 1 ? 2.f : (x == P - 2 ? -5.f : (x == P - 3 ? 4.f : -1.f)));
    return acc * inv_h2;
}

struct DarcySmem {
    uint64_t bar[2];
    float planes[2][2 * PP];   // double-buffered (p, K), 16-byte aligned for the bulk copy
};

// Residual, materialised: persistent CTAs, one bulk-async copy per sample, double-buffered.
template <bool PER>
__global__ void __launch_bounds__(DARCY_THREADS) darcy_fwd_kernel(const float* __restrict__ x0hat /*[B,2,P,P]*/,
                                                                 const float* __restrict__ fs /*[P*P]*/,
                                                                 float* __restrict__ residual /*[B,P*P,3]*/, int B,
                                                                 DarcyGeom geom) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    DarcySmem& S = *reinterpret_cast<DarcySmem*>(smem_raw);
    const int tid = threadIdx.x;
    if (tid == 0) {
        mbar_init(&S.bar[0], 1);
        mbar_init(&S.bar[1], 1);
        mbar_init_fence();
    }
    pdl_trigger();
    __syncthreads();
    pdl_wait();                 // barriers are set up; x0hat is produced by the previous kernel
    const uint32_t bytes = 2 * PP * sizeof(float);
    int n_local = 0;
    if (tid == 0 && (int)blockIdx.x < B) {
        mbar_expect_tx(&S.bar[0], bytes);
        bulk_g2s(S.planes[0], x0hat + (size_t)blockIdx.x * 2 * PP, bytes, &S.bar[0]);
    }
    for (int b = blockIdx.x; b < B; b += gridDim.x, ++n_local) {
        const int buf = n_local & 1;
        const int nb = b + gridDim.x;
        if (tid == 0 && nb < B) {   // prefetch next sample into the other buffer (its readers finished last iteration)
            mbar_expect_tx(&S.bar[buf ^ 1], bytes);
            bulk_g2s(S.planes[buf ^ 1], x0hat + (size_t)nb * 2 * PP, bytes, &S.bar[buf ^ 1]);
        }
        mbar_wait(&S.bar[buf], (n_local >> 1) & 1);
        const float* sp = S.planes[buf];
        const float* sk = sp + PP;
        float* out = residual + (size_t)b * PP * 3;
#pragma unroll 1
        for (int q = tid; q < PP / 4; q += DARCY_THREADS) {
            int i = q / (P / 4), j0 = (q % (P / 4)) * 4;
            float req[4], rb0[4], rb1[4];
            residual_quad<PER>(sp, sk, fs, i, j0, geom, req, rb0, rb1);
            float4* o = reinterpret_cast<float4*>(out + (size_t)(i * P + j0) * 3);
            o[0] = make_float4(req[0], rb0[0], rb1[0], req[1]);
            o[1] = make_float4(rb0[1], rb1[1], req[2], rb0[2]);
            o[2] = make_float4(rb1[2], req[3], rb0[3], rb1[3]);
        }
        __syncthreads();   // all readers of planes[buf] are done before it is refilled
    }
}

// ---- backward / fused loss ------------------------------------------------------------------------------------------
// With g = cotangent of eq_0 the adjoint is a sum of transposed 1-D stencils applied to five per-pixel products:
//   d p = D00^T A + D11^T A + D0^T U0 + D1^T U1,     A = -g K,  U0 = -g K_0 (+ bc_x0 seeds),  U1 = -g K_1 (+ bc_x1 seeds)
//   d K = -g (p_00 + p_11) + D0^T V0 + D1^T V1,       V0 = -g p_0,  V1 = -g p_1
// Phase 1 evaluates the residual of a quad of pixels (all derivatives of p and K are already in registers there) and
// leaves A, U0, U1, V0, V1 in shared-memory planes; phase 2 gathers the <= 5-point adjoint stencils from those planes.
// (The first version re-derived K_0 / K_1 / p_0 / p_1 at every neighbour inside the gather -- ~60 shared-memory loads
// per pixel -- and used 256 threads per sample.)
constexpr int DG_THREADS = 512;
constexpr int DG_QUADS = PP / 4 / DG_THREADS;      // quads per thread per sample (2)

struct DarcyGradSmem {
    uint64_t bar[2];
    float red[3][DG_THREADS / 32];
    float planes[2][2 * PP];   // double-buffered (p, K)
    float aux[5][PP];          // A, U0, U1, V0, V1
};

// residual of a quad + every derivative it is built from
template <bool PER>
__device__ __forceinline__ void residual_quad_full(const float* sp, const float* sk, const float* __restrict__ fs, int i,
                                                   int j0, const DarcyGeom& g, float req[4], float rb0[4], float rb1[4],
                                                   float kv[4], float k0[4], float k1[4], float p0[4], float p1[4],
                                                   float lap[4]) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const int j = j0 + q;
        kv[q] = sk[i * P + j];
        p0[q] = d_row<PER>(sp, i, j, g.inv_h0);
        k0[q] = d_row<PER>(sk, i, j, g.inv_h0);
        p1[q] = d_col<PER>(sp, i, j, g.inv_h1);
        k1[q] = d_col<PER>(sk, i, j, g.inv_h1);
        lap[q] = d2_row<PER>(sp, i, j, g.inv_h0sq) + d2_col<PER>(sp, i, j, g.inv_h1sq);
        // same association as residual_quad: -K (p_00 + p_11) - K_0 p_0 - K_1 p_1 - f_s
        req[q] = -kv[q] * lap[q] - k0[q] * p0[q] - k1[q] * p1[q] - source_fs(i, j, fs);
        rb0[q] = (i == 0) ? -p0[q] : ((i == P - 1) ? p0[q] : 0.f);
        rb1[q] = (j == 0) ? g.bc1_sign * p1[q] : ((j == P - 1) ? -g.bc1_sign * p1[q] : 0.f);
    }
}

// sign(x) * s for s > 0, with sign(0) = 0
__device__ __forceinline__ float scaled_sign(float x, float s) { return x > 0.f ? s : (x < 0.f ? -s : 0.f); }

// The p-side product planes of a quad from the cotangent (ge, g0, g1) of (eq_0, bc_x0, bc_x1):
// A = -ge K, U0 = -ge K_0 + bc_x0 seed, U1 = -ge K_1 + bc_x1 seed.
__device__ __forceinline__ void p_products(const float ge[4], const float g0[4], const float g1[4], const float kv[4],
                                           const float k0[4], const float k1[4], int i, int j0, const DarcyGeom& g,
                                           float a[4], float u0[4], float u1[4]) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int j = j0 + k;
        a[k] = -ge[k] * kv[k];
        u0[k] = -ge[k] * k0[k] + ((i == 0) ? -g0[k] : ((i == P - 1) ? g0[k] : 0.f));
        u1[k] = -ge[k] * k1[k] + ((j == 0) ? g.bc1_sign * g1[k] : ((j == P - 1) ? -g.bc1_sign * g1[k] : 0.f));
    }
}

// d p at pixel (i, j): the transposed stencils gathered from the A, U0, U1 planes
template <bool PER>
__device__ __forceinline__ float p_adjoint(const float* sA, const float* sU0, const float* sU1, int i, int j,
                                           const DarcyGeom& g) {
    auto a_row = [&](int r) { return sA[r * P + j]; };
    auto a_col = [&](int c) { return sA[i * P + c]; };
    auto u0r = [&](int r) { return sU0[r * P + j]; };
    auto u1c = [&](int c) { return sU1[i * P + c]; };
    return adj_d2<PER>(a_row, i, g.inv_h0sq) + adj_d2<PER>(a_col, j, g.inv_h1sq) + adj_d1<PER>(u0r, i, g.inv_h0) +
           adj_d1<PER>(u1c, j, g.inv_h1);
}

// MODE 1: generic backward (cotangent tensor given).  MODE 2: fused PIDM loss (data MSE + residual NLL sums, |r| sum)
// and its gradient w.r.t. x0_hat / model_out in one pass.  MODE 3: gradient of sum|r| / n_norm (the cotangent sign(r) *
// inv_norm is formed in registers), written in the b_xy_c layout [B,P*P,2] (residual-gradient guidance).  PER: periodic
// stencils; the BC seeds still enter U0 / U1 on rows 0 / P-1 and columns 0 / P-1.
// MODE 3 declares one resident CTA per SM (what its 145 KB of shared memory allows anyway): without it ptxas squeezes
// that instantiation into 64 registers and spills.  0 leaves MODE 1 / 2 exactly as they were compiled before.
template <int MODE, bool PER>
__global__ void __launch_bounds__(DG_THREADS, MODE == 3 ? 1 : 0) darcy_grad_kernel(
    const float* __restrict__ x0hat,      // [B,2,P,P]
    const float* __restrict__ fs,         // [P*P]
    const float* __restrict__ cot,        // MODE 1: [B,P*P,3]
    float* __restrict__ grad_x0hat,       // [B,2,P,P] (may be null in MODE 2 = loss only); MODE 3: [B,P*P,2]
    const float* __restrict__ target,     // MODE 2: x0 [B,2,P,P]
    const float* __restrict__ model_out,  // MODE 2: [B,2,P,P] (data-loss operand; == x0hat in mean mode)
    float* __restrict__ grad_model_out,   // MODE 2: gradient of data term (== grad_x0hat when same tensor)
    const long long* __restrict__ t,      // MODE 2: [B]
    const float* __restrict__ p2w,        // MODE 2: p2_loss_weight table
    const float* __restrict__ pvar,       // MODE 2: posterior_variance_clipped table
    float c_data, float c_res, float* __restrict__ sums,  // MODE 2: sums[0]=data loss, [1]=residual loss, [2]=mean|r|
    int B, DarcyGeom geom,
    float inv_norm) {                     // MODE 3: 1 / n_norm
    extern __shared__ __align__(128) unsigned char smem_raw[];
    DarcyGradSmem& S = *reinterpret_cast<DarcyGradSmem*>(smem_raw);
    const int tid = threadIdx.x;
    if (tid == 0) {
        mbar_init(&S.bar[0], 1);
        mbar_init(&S.bar[1], 1);
        mbar_init_fence();
    }
    pdl_trigger();
    __syncthreads();
    pdl_wait();
    const uint32_t bytes = 2 * PP * sizeof(float);
    int n_local = 0;
    if (tid == 0 && (int)blockIdx.x < B) {
        mbar_expect_tx(&S.bar[0], bytes);
        bulk_g2s(S.planes[0], x0hat + (size_t)blockIdx.x * 2 * PP, bytes, &S.bar[0]);
    }
    float* sA = S.aux[0];
    float* sU0 = S.aux[1];
    float* sU1 = S.aux[2];
    float* sV0 = S.aux[3];
    float* sV1 = S.aux[4];
    float acc_data = 0.f, acc_res = 0.f, acc_abs = 0.f;
    for (int b = blockIdx.x; b < B; b += gridDim.x, ++n_local) {
        const int buf = n_local & 1;
        const int nb = b + gridDim.x;
        if (tid == 0 && nb < B) {
            mbar_expect_tx(&S.bar[buf ^ 1], bytes);
            bulk_g2s(S.planes[buf ^ 1], x0hat + (size_t)nb * 2 * PP, bytes, &S.bar[buf ^ 1]);
        }
        mbar_wait(&S.bar[buf], (n_local >> 1) & 1);
        const float* sp = S.planes[buf];
        const float* sk = sp + PP;
        float wr = 0.f, wd = 0.f;
        if (MODE == 2) {
            const long long tb = t[b];
            const float nres = (float)B * (float)PP * 3.f;
            wr = 0.5f * c_res / (pvar[tb] * nres);
            wd = c_data * p2w[tb] / ((float)B * 2.f * (float)PP);
        }
        float W[DG_QUADS][4];
        // ---- phase 1: residual (or given cotangent) -> the five product planes
#pragma unroll
        for (int u = 0; u < DG_QUADS; ++u) {
            const int q = tid + u * DG_THREADS;
            const int i = q / (P / 4), j0 = (q % (P / 4)) * 4;
            float req[4], rb0[4], rb1[4], kv[4], k0[4], k1[4], p0[4], p1[4], lap[4];
            residual_quad_full<PER>(sp, sk, fs, i, j0, geom, req, rb0, rb1, kv, k0, k1, p0, p1, lap);
            float ge[4], g0[4], g1[4];
            if (MODE == 1) {
                const float4* c = reinterpret_cast<const float4*>(cot + ((size_t)b * PP + i * P + j0) * 3);
                const float4 c0 = c[0], c1 = c[1], c2 = c[2];
                ge[0] = c0.x; g0[0] = c0.y; g1[0] = c0.z; ge[1] = c0.w;
                g0[1] = c1.x; g1[1] = c1.y; ge[2] = c1.z; g0[2] = c1.w;
                g1[2] = c2.x; ge[3] = c2.y; g0[3] = c2.z; g1[3] = c2.w;
            } else if (MODE == 3) {
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    ge[k] = scaled_sign(req[k], inv_norm); g0[k] = scaled_sign(rb0[k], inv_norm); g1[k] = scaled_sign(rb1[k], inv_norm);
                }
            } else {
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    acc_res += wr * (req[k] * req[k] + rb0[k] * rb0[k] + rb1[k] * rb1[k]);
                    acc_abs += fabsf(req[k]) + fabsf(rb0[k]) + fabsf(rb1[k]);
                    ge[k] = 2.f * wr * req[k]; g0[k] = 2.f * wr * rb0[k]; g1[k] = 2.f * wr * rb1[k];
                }
            }
            float a[4], u0[4], u1[4], v0[4], v1[4];
            p_products(ge, g0, g1, kv, k0, k1, i, j0, geom, a, u0, u1);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                v0[k] = -ge[k] * p0[k];
                v1[k] = -ge[k] * p1[k];
                W[u][k] = -ge[k] * lap[k];
            }
            const int o = i * P + j0;
            *reinterpret_cast<float4*>(sA + o) = make_float4(a[0], a[1], a[2], a[3]);
            *reinterpret_cast<float4*>(sU0 + o) = make_float4(u0[0], u0[1], u0[2], u0[3]);
            *reinterpret_cast<float4*>(sU1 + o) = make_float4(u1[0], u1[1], u1[2], u1[3]);
            *reinterpret_cast<float4*>(sV0 + o) = make_float4(v0[0], v0[1], v0[2], v0[3]);
            *reinterpret_cast<float4*>(sV1 + o) = make_float4(v1[0], v1[1], v1[2], v1[3]);
        }
        __syncthreads();
        // ---- phase 2: transposed stencils on the planes (+ data-term gradient in the fused mode)
        const bool want_grad = (grad_x0hat != nullptr);
        const bool same = (MODE == 2) && (model_out == x0hat);
#pragma unroll
        for (int u = 0; u < DG_QUADS; ++u) {
            const int q = tid + u * DG_THREADS;
            const int i = q / (P / 4), j0 = (q % (P / 4)) * 4;
            float dp[4] = {0, 0, 0, 0}, dk[4] = {0, 0, 0, 0};
            if (want_grad) {
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const int j = j0 + k;
                    auto v0r = [&](int r) { return sV0[r * P + j]; };
                    auto v1c = [&](int c) { return sV1[i * P + c]; };
                    dp[k] = p_adjoint<PER>(sA, sU0, sU1, i, j, geom);
                    dk[k] = W[u][k] + adj_d1<PER>(v0r, i, geom.inv_h0) + adj_d1<PER>(v1c, j, geom.inv_h1);
                }
            }
            if (MODE == 2) {
                const size_t off = (size_t)b * 2 * PP + i * P + j0;
                const float4 tp = *reinterpret_cast<const float4*>(target + off);
                const float4 tk = *reinterpret_cast<const float4*>(target + off + PP);
                float4 mp, mk;
                if (same) {
                    mp = *reinterpret_cast<const float4*>(sp + i * P + j0);
                    mk = *reinterpret_cast<const float4*>(sk + i * P + j0);
                } else {
                    mp = *reinterpret_cast<const float4*>(model_out + off);
                    mk = *reinterpret_cast<const float4*>(model_out + off + PP);
                }
                const float ep[4] = {mp.x - tp.x, mp.y - tp.y, mp.z - tp.z, mp.w - tp.w};
                const float ek[4] = {mk.x - tk.x, mk.y - tk.y, mk.z - tk.z, mk.w - tk.w};
#pragma unroll
                for (int k = 0; k < 4; ++k) acc_data += wd * (ep[k] * ep[k] + ek[k] * ek[k]);
                if (want_grad) {
                    if (same) {
#pragma unroll
                        for (int k = 0; k < 4; ++k) { dp[k] += 2.f * wd * ep[k]; dk[k] += 2.f * wd * ek[k]; }
                    } else {
                        *reinterpret_cast<float4*>(grad_model_out + off) =
                            make_float4(2.f * wd * ep[0], 2.f * wd * ep[1], 2.f * wd * ep[2], 2.f * wd * ep[3]);
                        *reinterpret_cast<float4*>(grad_model_out + off + PP) =
                            make_float4(2.f * wd * ek[0], 2.f * wd * ek[1], 2.f * wd * ek[2], 2.f * wd * ek[3]);
                    }
                }
            }
            if (MODE == 3) {                // (p, K) interleaved per pixel: 32 contiguous bytes per thread
                float4* o = reinterpret_cast<float4*>(grad_x0hat + ((size_t)b * PP + i * P + j0) * 2);
                o[0] = make_float4(dp[0], dk[0], dp[1], dk[1]);
                o[1] = make_float4(dp[2], dk[2], dp[3], dk[3]);
            } else if (want_grad) {
                const size_t off = (size_t)b * 2 * PP + i * P + j0;
                *reinterpret_cast<float4*>(grad_x0hat + off) = make_float4(dp[0], dp[1], dp[2], dp[3]);
                *reinterpret_cast<float4*>(grad_x0hat + off + PP) = make_float4(dk[0], dk[1], dk[2], dk[3]);
            }
        }
        __syncthreads();   // all readers of planes[buf] and of the product planes are done before they are rewritten
    }
    if (MODE == 2) {
        acc_data = warp_sum(acc_data);
        acc_res = warp_sum(acc_res);
        acc_abs = warp_sum(acc_abs);
        const int w = tid >> 5;
        if ((tid & 31) == 0) { S.red[0][w] = acc_data; S.red[1][w] = acc_res; S.red[2][w] = acc_abs; }
        __syncthreads();
        if (tid < 3) {
            float s = 0.f;
            for (int k = 0; k < DG_THREADS / 32; ++k) s += S.red[tid][k];
            if (tid == 2) s /= ((float)B * (float)PP * 3.f);
            atomicAdd(&sums[tid], s);
        }
    }
}

// ---- CoCoGen step size (reference residuals_darcy.py:209-240) -------------------------------------------------------
// The reference builds, per sample, the dense Jacobian d r / d p (4096 x 3 rows, 4096 columns, via vmap(jacfwd)) only to
// take its largest entry.  The residual is linear in p, so the Jacobian entries are stencil coefficients times fields of K:
//   d r_eq[i] / d p[i + (dr, 0)] = -K c00_i(dr) - K_0 c0_i(dr),   d r_eq[i] / d p[i + (0, dc)] = -K c11_j(dc) - K_1 c1_j(dc)
//   (the two centre entries add), d r_bc0 = -/+ c0_i(dr) on rows 0 / P-1, d r_bc1 = +/- s c1_j(dc) on columns 0 / P-1,
// and every other entry is zero.  One CTA per sample evaluates them from the K plane in shared memory and reduces the
// (signed, like torch.max) maximum.  Periodic: every pixel has the central entries; the neighbours wrap, and since
// P > 3 the three offsets of a row still name three distinct pixels.
template <bool PER>
__device__ __forceinline__ int stencil1(int x, int off[4], float c[4]) {           // first derivative, index x of P
    if (!PER && x == 0) { off[0] = 0; c[0] = -1.5f; off[1] = 1; c[1] = 2.f; off[2] = 2; c[2] = -0.5f; return 3; }
    if (!PER && x == P - 1) { off[0] = 0; c[0] = 1.5f; off[1] = -1; c[1] = -2.f; off[2] = -2; c[2] = 0.5f; return 3; }
    off[0] = -1; c[0] = -0.5f; off[1] = 1; c[1] = 0.5f; off[2] = 0; c[2] = 0.f;
    return 3;
}
template <bool PER>
__device__ __forceinline__ int stencil2(int x, int off[4], float c[4]) {           // second derivative
    if (PER) {
        off[0] = -1; c[0] = 1.f; off[1] = 0; c[1] = -2.f; off[2] = 1; c[2] = 1.f;
        return 3;
    }
    if (x == 0) { off[0] = 0; c[0] = 2.f; off[1] = 1; c[1] = -5.f; off[2] = 2; c[2] = 4.f; off[3] = 3; c[3] = -1.f; return 4; }
    if (x == P - 1) { off[0] = 0; c[0] = 2.f; off[1] = -1; c[1] = -5.f; off[2] = -2; c[2] = 4.f; off[3] = -3; c[3] = -1.f; return 4; }
    off[0] = -1; c[0] = 1.f; off[1] = 0; c[1] = -2.f; off[2] = 1; c[2] = 1.f;
    return 3;
}
// entries of one direction: e(d) = -K * c2(d) * inv_h2 - Kd * c1(d) * inv_h, merged over the offsets d in [-3, 3]
template <bool PER>
__device__ __forceinline__ void dir_entries(int x, float kv, float kd, float inv_h, float inv_h2, float e[7], bool has[7]) {
#pragma unroll
    for (int d = 0; d < 7; ++d) { e[d] = 0.f; has[d] = false; }
    int off[4]; float c[4];
    int n = stencil2<PER>(x, off, c);
    for (int k = 0; k < n; ++k) { e[off[k] + 3] += -kv * c[k] * inv_h2; has[off[k] + 3] = true; }
    n = stencil1<PER>(x, off, c);
    for (int k = 0; k < n; ++k) { e[off[k] + 3] += -kd * c[k] * inv_h; has[off[k] + 3] = true; }
}
// max(m, every Jacobian entry in the rows of pixel (i, j)), from the K plane sk
template <bool PER>
__device__ __forceinline__ float jacobian_max_pixel(const float* sk, int i, int j, const DarcyGeom& g, float m) {
    const float kv = sk[i * P + j];
    const float k0 = d_row<PER>(sk, i, j, g.inv_h0), k1 = d_col<PER>(sk, i, j, g.inv_h1);
    float er[7], ec[7];
    bool hr[7], hc[7];
    dir_entries<PER>(i, kv, k0, g.inv_h0, g.inv_h0sq, er, hr);
    dir_entries<PER>(j, kv, k1, g.inv_h1, g.inv_h1sq, ec, hc);
    m = fmaxf(m, er[3] + ec[3]);                         // both directions touch the pixel itself
#pragma unroll
    for (int d = 0; d < 7; ++d) {
        if (d == 3) continue;
        if (hr[d]) m = fmaxf(m, er[d]);
        if (hc[d]) m = fmaxf(m, ec[d]);
    }
    int off[4]; float c[4];
    if (i == 0 || i == P - 1) {                          // bc_x0 = -p_0 (row 0), +p_0 (row P-1)
        const int n = stencil1<PER>(i, off, c);
        const float sg = (i == 0) ? -g.inv_h0 : g.inv_h0;
        for (int k = 0; k < n; ++k) m = fmaxf(m, sg * c[k]);
    }
    if (j == 0 || j == P - 1) {                          // bc_x1 = +s p_1 (column 0), -s p_1 (column P-1)
        const int n = stencil1<PER>(j, off, c);
        const float sg = ((j == 0) ? g.bc1_sign : -g.bc1_sign) * g.inv_h1;
        for (int k = 0; k < n; ++k) m = fmaxf(m, sg * c[k]);
    }
    return m;
}

template <bool PER>
__global__ void __launch_bounds__(DARCY_THREADS) darcy_jacobian_max_kernel(const float* __restrict__ x0hat,
                                                                          float* __restrict__ out, DarcyGeom g) {
    pdl_trigger();
    pdl_wait();
    __shared__ float sk[PP];
    __shared__ float red[DARCY_THREADS / 32];
    const int b = blockIdx.x;
    const float* kp = x0hat + (size_t)b * 2 * PP + PP;
    for (int i = threadIdx.x; i < PP; i += blockDim.x) sk[i] = kp[i];
    __syncthreads();
    float m = 0.f;                                       // the Jacobian is sparse: zero entries take part in the max
    for (int q = threadIdx.x; q < PP; q += blockDim.x) {
        const int i = q / P, j = q - i * P;
        m = jacobian_max_pixel<PER>(sk, i, j, g, m);
    }
    m = warp_max(m);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
        float r = red[0];
        for (int w = 1; w < DARCY_THREADS / 32; ++w) r = fmaxf(r, red[w]);
        out[b] = r;
    }
}

// ---- CoCoGen corrections, all steps of a sample in one CTA ----------------------------------------------------------
// The corrections move p only, so K -- and with it max dr/dp and the step size -- is fixed for the whole launch, and
// the residual is affine in p: each step is a fixed-step gradient step on sum r^2 with the same operator.  One CTA owns
// one sample; p, K and the A / U0 / U1 product planes of the p adjoint stay in shared memory (80 KB) for every step:
//   forward stencil -> products of 2r -> barrier -> adjoint gather + update of p -> barrier.
// Each step computes what one multi-launch correction does (residual, cotangent 2r, pidm_darcy_residual_bwd's p
// component, p -= eps * dp with eps = 1e-6 / min(max dr/dp, 1e12)); the final residual is darcy_fwd_kernel's stencil.
struct DarcyCocogenSmem {
    float red[DG_THREADS / 32];
    float p[PP];
    float k[PP];
    float prod[3][PP];         // A, U0, U1
};

template <bool PER>
__global__ void __launch_bounds__(DG_THREADS, 1) darcy_cocogen_kernel(float* __restrict__ x /*[B,2,P,P]*/,
                                                                     const float* __restrict__ fs,
                                                                     float* __restrict__ residual /*[B,P*P,3]*/,
                                                                     const long long* __restrict__ t, int n_active,
                                                                     int steps, DarcyGeom g) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    DarcyCocogenSmem& S = *reinterpret_cast<DarcyCocogenSmem*>(smem_raw);
    const int tid = threadIdx.x, b = blockIdx.x;
    pdl_trigger();
    pdl_wait();
    if (t != nullptr && !(t[b] < n_active)) return;     // inactive sample: neither read nor written
    float* xb = x + (size_t)b * 2 * PP;
    for (int q = tid; q < PP / 4; q += DG_THREADS) {
        reinterpret_cast<float4*>(S.p)[q] = reinterpret_cast<const float4*>(xb)[q];
        reinterpret_cast<float4*>(S.k)[q] = reinterpret_cast<const float4*>(xb + PP)[q];
    }
    __syncthreads();
    float m = 0.f;                                       // max dr/dp, as darcy_jacobian_max_kernel
    for (int q = tid; q < PP; q += DG_THREADS) m = jacobian_max_pixel<PER>(S.k, q / P, q % P, g, m);
    m = warp_max(m);
    if ((tid & 31) == 0) S.red[tid >> 5] = m;
    __syncthreads();
    m = S.red[0];
    for (int w = 1; w < DG_THREADS / 32; ++w) m = fmaxf(m, S.red[w]);
    // torch: 1e-6 / clamp(m, max=1e12) is reciprocal(m) * 1e-6 (NaN propagates through the clamp)
    const float eps = __fmul_rn(1.f / (m > 1e12f ? 1e12f : m), 1e-6f);
    float* sA = S.prod[0];
    float* sU0 = S.prod[1];
    float* sU1 = S.prod[2];
#pragma unroll 1
    for (int s = 0; s < steps; ++s) {
#pragma unroll
        for (int u = 0; u < DG_QUADS; ++u) {
            const int q = tid + u * DG_THREADS;
            const int i = q / (P / 4), j0 = (q % (P / 4)) * 4;
            float req[4], rb0[4], rb1[4], kv[4], k0[4], k1[4], p0[4], p1[4], lap[4];
            residual_quad_full<PER>(S.p, S.k, fs, i, j0, g, req, rb0, rb1, kv, k0, k1, p0, p1, lap);
            float ge[4], g0[4], g1[4], a[4], u0[4], u1[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) { ge[k] = 2.f * req[k]; g0[k] = 2.f * rb0[k]; g1[k] = 2.f * rb1[k]; }
            p_products(ge, g0, g1, kv, k0, k1, i, j0, g, a, u0, u1);
            const int o = i * P + j0;
            *reinterpret_cast<float4*>(sA + o) = make_float4(a[0], a[1], a[2], a[3]);
            *reinterpret_cast<float4*>(sU0 + o) = make_float4(u0[0], u0[1], u0[2], u0[3]);
            *reinterpret_cast<float4*>(sU1 + o) = make_float4(u1[0], u1[1], u1[2], u1[3]);
        }
        __syncthreads();
        // the gather reads only the product planes, so p is updated in place
#pragma unroll
        for (int u = 0; u < DG_QUADS; ++u) {
            const int q = tid + u * DG_THREADS;
            const int i = q / (P / 4), j0 = (q % (P / 4)) * 4;
            float4* pq = reinterpret_cast<float4*>(S.p + i * P + j0);
            float4 pv = *pq;
            pv.x -= __fmul_rn(eps, p_adjoint<PER>(sA, sU0, sU1, i, j0, g));   // eps * dp rounded, then subtracted
            pv.y -= __fmul_rn(eps, p_adjoint<PER>(sA, sU0, sU1, i, j0 + 1, g));
            pv.z -= __fmul_rn(eps, p_adjoint<PER>(sA, sU0, sU1, i, j0 + 2, g));
            pv.w -= __fmul_rn(eps, p_adjoint<PER>(sA, sU0, sU1, i, j0 + 3, g));
            *pq = pv;
        }
        __syncthreads();
    }
    float* out = residual + (size_t)b * PP * 3;
#pragma unroll 1
    for (int q = tid; q < PP / 4; q += DG_THREADS) {
        const int i = q / (P / 4), j0 = (q % (P / 4)) * 4;
        float req[4], rb0[4], rb1[4];
        residual_quad<PER>(S.p, S.k, fs, i, j0, g, req, rb0, rb1);
        float4* o = reinterpret_cast<float4*>(out + (size_t)(i * P + j0) * 3);
        o[0] = make_float4(req[0], rb0[0], rb1[0], req[1]);
        o[1] = make_float4(rb0[1], rb1[1], req[2], rb0[2]);
        o[2] = make_float4(rb1[2], req[3], rb0[3], rb1[3]);
        reinterpret_cast<float4*>(xb)[q] = reinterpret_cast<const float4*>(S.p)[q];   // K is left untouched
    }
}

// single derivative field (StencilGradients.forward, grad_utils.py:161-175); global-memory version, forward only
template <bool PER>
__global__ void fd_stencil_kernel(const float* __restrict__ u, float* __restrict__ out, int planes, int mode,
                                  float inv_h0, float inv_h1) {
    pdl_trigger();
    pdl_wait();
    __shared__ float su[PP];
    __shared__ float st[PP];
    for (int pl = blockIdx.x; pl < planes; pl += gridDim.x) {
        __syncthreads();
        for (int i = threadIdx.x; i < PP; i += blockDim.x) su[i] = u[(size_t)pl * PP + i];
        __syncthreads();
        if (mode == 4) {   // d_d01 = d/dx0 (d/dx1 u): tensor product of the 1-D stencils
            for (int i = threadIdx.x; i < PP; i += blockDim.x) st[i] = d_col<PER>(su, i / P, i % P, inv_h1);
            __syncthreads();
        }
        for (int i = threadIdx.x; i < PP; i += blockDim.x) {
            int r = i / P, c = i % P;
            float v;
            if (mode == 0) v = d_row<PER>(su, r, c, inv_h0);
            else if (mode == 1) v = d_col<PER>(su, r, c, inv_h1);
            else if (mode == 2) v = d2_row<PER>(su, r, c, inv_h0 * inv_h0);
            else if (mode == 3) v = d2_col<PER>(su, r, c, inv_h1 * inv_h1);
            else v = d_row<PER>(st, r, c, inv_h0);
            out[(size_t)pl * PP + i] = v;
        }
    }
}

static DarcyGeom make_geom(float domain_length, int reverse_d1, int flags) {
    float d0 = (flags & PIDM_DARCY_PIXELS_AT_BOUNDARY) ? domain_length / (P - 1) : domain_length / P;
    float d1 = reverse_d1 ? -d0 : d0;
    DarcyGeom g;
    g.inv_h0 = 1.f / d0;
    g.inv_h1 = 1.f / d1;
    g.inv_h0sq = 1.f / (d0 * d0);
    g.inv_h1sq = 1.f / (d1 * d1);
    g.bc1_sign = reverse_d1 ? 1.f : -1.f;
    return g;
}

static int check_flags(int flags) {
    PIDM_REQUIRE((flags & ~(PIDM_DARCY_PIXELS_AT_BOUNDARY | PIDM_DARCY_PERIODIC)) == 0,
                 "darcy: unknown flag bits 0x%x (PIDM_DARCY_PIXELS_AT_BOUNDARY = 1, PIDM_DARCY_PERIODIC = 2)", flags);
    return 0;
}

template <bool PER>
static int launch_darcy_fwd(const float* x0hat, const float* fs, float* residual, int B, int pixels, float domain_length,
                            int reverse_d1, int flags, cudaStream_t stream) {
    PIDM_REQUIRE(pixels == P, "darcy kernels are built for %d x %d fields (got %d)", P, P, pixels);
    PIDM_REQUIRE(B > 0, "empty batch");
    const size_t smem = sizeof(DarcySmem);
    PIDM_CUDA(allow_smem(darcy_fwd_kernel<PER>, smem));
    const int ctas_per_sm = (int)(220 * 1024 / smem);        // smem-limited residency
    int grid = num_sms() * (ctas_per_sm > 0 ? ctas_per_sm : 1);
    if (grid > B) grid = B;
    PIDM_CUDA(launch_plain(darcy_fwd_kernel<PER>, dim3(grid), dim3(DARCY_THREADS), (size_t)(smem), stream, x0hat, fs, residual,
                           B, make_geom(domain_length, reverse_d1, flags)));
    PIDM_LAUNCH_CHECK("darcy_fwd_kernel");
    return 0;
}

template <int MODE, bool PER>
static int launch_darcy_grad(const float* x0hat, const float* fs, const float* cot, float* grad_x0hat, const float* target,
                             const float* model_out, float* grad_model_out, const long long* t, const float* p2w,
                             const float* pvar, float c_data, float c_res, float* sums, int B, int pixels,
                             float domain_length, int reverse_d1, int flags, cudaStream_t stream, float inv_norm = 0.f) {
    PIDM_REQUIRE(pixels == P, "darcy kernels are built for %d x %d fields (got %d)", P, P, pixels);
    PIDM_REQUIRE(B > 0, "empty batch");
    const size_t smem = sizeof(DarcyGradSmem);
    PIDM_CUDA(allow_smem(darcy_grad_kernel<MODE, PER>, smem));
    int grid = num_sms();                                     // 145 KB of shared memory: one CTA of 512 threads per SM
    if (grid > B) grid = B;
    PIDM_CUDA(launch_plain(darcy_grad_kernel<MODE, PER>, dim3(grid), dim3(DG_THREADS), (size_t)(smem), stream, x0hat, fs,
                           cot, grad_x0hat, target, model_out, grad_model_out, t, p2w, pvar, c_data, c_res, sums, B,
                           make_geom(domain_length, reverse_d1, flags), inv_norm));
    PIDM_LAUNCH_CHECK("darcy_grad_kernel");
    return 0;
}

template <bool PER>
static int launch_darcy_cocogen(float* x, const float* fs, float* residual, const long long* t, int n_active, int steps,
                                int B, float domain_length, int reverse_d1, int flags, cudaStream_t stream) {
    const size_t smem = sizeof(DarcyCocogenSmem);
    PIDM_CUDA(allow_smem(darcy_cocogen_kernel<PER>, smem));
    PIDM_CUDA(launch_plain(darcy_cocogen_kernel<PER>, dim3(B), dim3(DG_THREADS), smem, stream, x, fs, residual, t,
                           n_active, steps, make_geom(domain_length, reverse_d1, flags)));
    PIDM_LAUNCH_CHECK("darcy_cocogen_kernel");
    return 0;
}

template <int MODE>
static int launch_darcy_grad_any(const float* x0hat, const float* fs, const float* cot, float* grad_x0hat,
                                 const float* target, const float* model_out, float* grad_model_out, const long long* t,
                                 const float* p2w, const float* pvar, float c_data, float c_res, float* sums, int B,
                                 int pixels, float domain_length, int reverse_d1, int flags, cudaStream_t stream,
                                 float inv_norm = 0.f) {
    auto launch = (flags & PIDM_DARCY_PERIODIC) ? launch_darcy_grad<MODE, true> : launch_darcy_grad<MODE, false>;
    return launch(x0hat, fs, cot, grad_x0hat, target, model_out, grad_model_out, t, p2w, pvar, c_data, c_res, sums, B,
                  pixels, domain_length, reverse_d1, flags, stream, inv_norm);
}

}  // namespace pidm

using namespace pidm;

extern "C" int pidm_fd_stencil(const float* u, float* out, int planes, int pixels, int mode, float d0, float d1,
                               void* stream) {
    PIDM_REQUIRE(pixels == P, "fd_stencil is built for %d x %d fields (got %d)", P, P, pixels);
    const bool periodic = (mode & PIDM_FD_PERIODIC) != 0;
    mode &= ~PIDM_FD_PERIODIC;
    PIDM_REQUIRE(mode >= 0 && mode <= 4,
                 "fd_stencil: mode must be 0..4 (d_d0, d_d1, d_d00, d_d11, d_d01), optionally | PIDM_FD_PERIODIC");
    int grid = planes < num_sms() * 4 ? planes : num_sms() * 4;
    auto kernel = periodic ? fd_stencil_kernel<true> : fd_stencil_kernel<false>;
    PIDM_CUDA(launch_plain(kernel, dim3(grid), dim3(256), (size_t)(0), (cudaStream_t)stream, u, out, planes, mode, 1.f / d0,
                           1.f / d1));
    PIDM_LAUNCH_CHECK("fd_stencil");
    return 0;
}

extern "C" int pidm_darcy_residual_fwd(const float* x0hat, const float* f_s, float* residual, int B, int pixels,
                                       float domain_length, int reverse_d1, int flags, void* stream) {
    if (int e = check_flags(flags)) return e;
    auto launch = (flags & PIDM_DARCY_PERIODIC) ? launch_darcy_fwd<true> : launch_darcy_fwd<false>;
    return launch(x0hat, f_s, residual, B, pixels, domain_length, reverse_d1, flags, (cudaStream_t)stream);
}

extern "C" int pidm_darcy_residual_bwd(const float* x0hat, const float* f_s, const float* grad_residual,
                                       float* grad_x0hat, int B, int pixels, float domain_length, int reverse_d1,
                                       int flags, void* stream) {
    if (int e = check_flags(flags)) return e;
    return launch_darcy_grad_any<1>(x0hat, f_s, grad_residual, grad_x0hat, nullptr, nullptr, nullptr, nullptr, nullptr,
                                    nullptr, 0.f, 0.f, nullptr, B, pixels, domain_length, reverse_d1, flags,
                                    (cudaStream_t)stream);
}

extern "C" int pidm_darcy_pidm_loss(const float* x0hat, const float* model_out, const float* target, const float* f_s,
                                    const long long* t, const float* p2_loss_weight, const float* posterior_var_clipped,
                                    float c_data, float c_residual, float* sums3, float* grad_x0hat,
                                    float* grad_model_out, int B, int pixels, float domain_length, int reverse_d1,
                                    int flags, void* stream) {
    if (int e = check_flags(flags)) return e;
    // darcy_grad_kernel<2> writes grad_model_out only when model_out is a separate tensor, and then whenever grad_x0hat
    // is written: any other combination would store through NULL or leave a requested gradient unwritten
    PIDM_REQUIRE(x0hat != nullptr && model_out != nullptr, "darcy_pidm_loss: x0hat and model_out must not be NULL");
    PIDM_REQUIRE(model_out == x0hat ? grad_model_out == nullptr : (grad_x0hat == nullptr) == (grad_model_out == nullptr),
                 "darcy_pidm_loss: gradients must be both NULL, grad_x0hat alone (model_out == x0hat) or both "
                 "(model_out != x0hat); got grad_x0hat %s, grad_model_out %s, model_out %s x0hat",
                 grad_x0hat ? "set" : "NULL", grad_model_out ? "set" : "NULL", model_out == x0hat ? "==" : "!=");
    PIDM_CUDA(cudaMemsetAsync(sums3, 0, 3 * sizeof(float), (cudaStream_t)stream));
    return launch_darcy_grad_any<2>(x0hat, f_s, nullptr, grad_x0hat, target, model_out, grad_model_out, t, p2_loss_weight,
                                    posterior_var_clipped, c_data, c_residual, sums3, B, pixels, domain_length, reverse_d1,
                                    flags, (cudaStream_t)stream);
}

extern "C" int pidm_darcy_abs_residual_grad(const float* x_t, const float* f_s, float* cond, int B, long long n_norm,
                                            int pixels, float domain_length, int reverse_d1, int flags, void* stream) {
    if (int e = check_flags(flags)) return e;
    PIDM_REQUIRE(cond != nullptr, "darcy_abs_residual_grad: cond must not be NULL");
    PIDM_REQUIRE(n_norm >= (long long)B * pixels * pixels * 3 && (long long)(float)n_norm == n_norm,
                 "darcy_abs_residual_grad: n_norm = %lld must be at least B*P*P*3 and exact in fp32", n_norm);
    // the reference's mean backward: a float 1 / numel (exact numel), times sign(r)
    const float inv_norm = 1.f / (float)n_norm;
    return launch_darcy_grad_any<3>(x_t, f_s, nullptr, cond, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, 0.f,
                                    0.f, nullptr, B, pixels, domain_length, reverse_d1, flags, (cudaStream_t)stream,
                                    inv_norm);
}

/* max_dr_dp[b] = largest entry of the Jacobian d residual / d p of sample b (CoCoGen step size, residuals_darcy.py:218-231) */
extern "C" int pidm_darcy_jacobian_max(const float* x0hat, float* max_dr_dp, int B, int pixels, float domain_length,
                                       int reverse_d1, int flags, void* stream) {
    if (int e = check_flags(flags)) return e;
    PIDM_REQUIRE(pixels == P, "darcy kernels are built for %d x %d fields (got %d)", P, P, pixels);
    PIDM_REQUIRE(B > 0, "empty batch");
    auto kernel = (flags & PIDM_DARCY_PERIODIC) ? darcy_jacobian_max_kernel<true> : darcy_jacobian_max_kernel<false>;
    PIDM_CUDA(launch_plain(kernel, dim3(B), dim3(DARCY_THREADS), (size_t)0, (cudaStream_t)stream, x0hat, max_dr_dp,
                           make_geom(domain_length, reverse_d1, flags)));
    PIDM_LAUNCH_CHECK("darcy_jacobian_max");
    return 0;
}

/* `steps` CoCoGen corrections of every active sample in one launch (residuals_darcy.py:209-240 applied `steps` times) */
extern "C" int pidm_darcy_cocogen(float* x, const float* f_s, float* residual, const long long* t, int n_active,
                                  int steps, int B, int pixels, float domain_length, int reverse_d1, int flags,
                                  void* stream) {
    if (int e = check_flags(flags)) return e;
    PIDM_REQUIRE(pixels == P, "darcy kernels are built for %d x %d fields (got %d)", P, P, pixels);
    PIDM_REQUIRE(B > 0, "empty batch");
    PIDM_REQUIRE(steps >= 0, "darcy_cocogen: steps = %d must not be negative", steps);
    PIDM_REQUIRE(x != nullptr && f_s != nullptr && residual != nullptr, "darcy_cocogen: x, f_s and residual must not be NULL");
    auto launch = (flags & PIDM_DARCY_PERIODIC) ? launch_darcy_cocogen<true> : launch_darcy_cocogen<false>;
    return launch(x, f_s, residual, t, n_active, steps, B, domain_length, reverse_d1, flags, (cudaStream_t)stream);
}
