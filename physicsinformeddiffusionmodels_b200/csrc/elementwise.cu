// HBM-bound element-wise pieces of the PIDM step: q_sample, ancestral posterior step, layout change
// (NCHW fp32 -> NHWC activations), channel concat/split, and the tiny-N output head
// (final 1x1 conv -> NCHW fp32, optional sigmoid on the last channel).  128-bit vectorised accesses.
#include "common.cuh"
#include "pidm.h"

namespace pidm {

// ---- q_sample: x_t = sqrt(abar_t) x0 + sqrt(1-abar_t) eps   (denoising_utils.py:373-378, :633-638) -------
__global__ void qsample_kernel(const float4* __restrict__ x0, const float4* __restrict__ eps,
                               const long long* __restrict__ t, const float* __restrict__ sa,
                               const float* __restrict__ sb, float4* __restrict__ xt, int per_sample4, long long total4) {
    pdl_trigger();
    pdl_wait();
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total4;
         i += (long long)gridDim.x * blockDim.x) {
        int b = (int)(i / per_sample4);
        long long tb = t[b];
        float a = sa[tb], s = sb[tb];
        float4 x = x0[i], e = eps[i];
        xt[i] = make_float4(a * x.x + s * e.x, a * x.y + s * e.y, a * x.z + s * e.z, a * x.w + s * e.w);
    }
}

// scalar variants for per-sample sizes that are not multiples of 4 (the 65x65 fields of the mechanics branch: samples
// then start at addresses that are not 16-byte aligned)
__global__ void qsample_scalar_kernel(const float* __restrict__ x0, const float* __restrict__ eps,
                                      const long long* __restrict__ t, const float* __restrict__ sa,
                                      const float* __restrict__ sb, float* __restrict__ xt, int per_sample, long long total) {
    pdl_trigger();
    pdl_wait();
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long tb = t[i / per_sample];
        xt[i] = sa[tb] * x0[i] + sb[tb] * eps[i];
    }
}
__global__ void posterior_scalar_kernel(const float* __restrict__ xt, const float* __restrict__ x0p,
                                        const float* __restrict__ z, float* __restrict__ out, float c1, float c2, float sig,
                                        long long total) {
    pdl_trigger();
    pdl_wait();
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
        out[i] = c1 * x0p[i] + c2 * xt[i] + sig * z[i];
}
__global__ void axpby_ps_scalar_kernel(const float* __restrict__ a, const float* __restrict__ x, const float* __restrict__ b,
                                       const float* __restrict__ y, const float* __restrict__ c,
                                       const float* __restrict__ z, float* __restrict__ out, int per_sample,
                                       long long total) {
    pdl_trigger();
    pdl_wait();
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long s = i / per_sample;
        out[i] = a[s] * x[i] + b[s] * y[i] + c[s] * z[i];
    }
}

// ---- posterior step: x_{t-1} = c1 x0_pred + c2 x_t + sigma z     (denoising_utils.py:441-455) ------------
__global__ void posterior_kernel(const float4* __restrict__ xt, const float4* __restrict__ x0p,
                                 const float4* __restrict__ z, float4* __restrict__ out, float c1, float c2, float sig,
                                 long long total4) {
    pdl_trigger();
    pdl_wait();
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total4;
         i += (long long)gridDim.x * blockDim.x) {
        float4 a = xt[i], b = x0p[i], n = z[i];
        out[i] = make_float4(c1 * b.x + c2 * a.x + sig * n.x, c1 * b.y + c2 * a.y + sig * n.y,
                             c1 * b.z + c2 * a.z + sig * n.z, c1 * b.w + c2 * a.w + sig * n.w);
    }
}

// ---- NCHW fp32 -> NHWC (channel-padded) activations -----------------------------------------------------
// one thread per pixel: C coalesced plane reads, one channel-padded NHWC row written with 16-byte stores
template <typename T>
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ src, T* __restrict__ dst, int C, int HW, int Cpad,
                                    long long n_pix) {
    pdl_trigger();
    pdl_wait();  // n_pix = B*HW, Cpad % 8 == 0
    for (long long pix = blockIdx.x * (long long)blockDim.x + threadIdx.x; pix < n_pix;
         pix += (long long)gridDim.x * blockDim.x) {
        const long long b = pix / HW;
        const int hw = (int)(pix - b * HW);
        const float* sp = src + (size_t)b * C * HW + hw;
        T* dp = dst + (size_t)pix * Cpad;
        for (int c0 = 0; c0 < Cpad; c0 += 8) {
            float v[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) v[k] = (c0 + k < C) ? sp[(size_t)(c0 + k) * HW] : 0.f;
            st8(dp + c0, v);
        }
    }
}

// ---- concat, split along channels (NHWC rows) ----------------------------------------------------------
// out[m, 0:Ca] = a[m], out[m, Ca:Ca+Cb] = b[m]   (channels multiples of 8)
template <typename T>
__global__ void concat_kernel(const T* __restrict__ a, const T* __restrict__ b, T* __restrict__ o, int Ca8, int Cb8,
                              long long rows) {
    pdl_trigger();
    pdl_wait();
    const int Ct8 = Ca8 + Cb8;
    const long long total = rows * Ct8;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        long long m = i / Ct8;
        int c = (int)(i % Ct8);
        float v[8];
        if (c < Ca8) ld8(a + (m * Ca8 + c) * 8, v);
        else ld8(b + (m * Cb8 + (c - Ca8)) * 8, v);
        st8(o + i * 8, v);
    }
}
template <typename T>
__global__ void split_kernel(const T* __restrict__ g, T* __restrict__ ga, T* __restrict__ gb, int Ca8, int Cb8,
                             long long rows) {
    pdl_trigger();
    pdl_wait();
    const int Ct8 = Ca8 + Cb8;
    const long long total = rows * Ct8;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        long long m = i / Ct8;
        int c = (int)(i % Ct8);
        float v[8];
        ld8(g + i * 8, v);
        if (c < Ca8) st8(ga + (m * Ca8 + c) * 8, v);
        else st8(gb + (m * Cb8 + (c - Ca8)) * 8, v);
    }
}

// y[b, oh, ow] = x[b, (oh - halo) mod H, (ow - halo) mod W]: one 16-byte unit of a pixel row per thread iteration, copied
// as raw bits (dtype-agnostic, exact).  The output is [B, H + 2 halo, W + 2 halo, U * 16 bytes].
__global__ void wrap_pad_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, int H, int W, int halo, int U,
                                long long total) {
    pdl_trigger();
    pdl_wait();
    const int Hp = H + 2 * halo, Wp = W + 2 * halo;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int u = (int)(i % U);
        const long long pix = i / U;
        const int ow = (int)(pix % Wp);
        const long long r = pix / Wp;
        const int oh = (int)(r % Hp);
        const long long b = r / Hp;
        int ih = oh - halo, iw = ow - halo;
        ih += ih < 0 ? H : (ih >= H ? -H : 0);
        iw += iw < 0 ? W : (iw >= W ? -W : 0);
        y[i] = __ldg(x + ((b * H + ih) * W + iw) * U + u);
    }
}

// out = a_b x + b_b y + c_b z with per-sample coefficients (DDIM jump inside ddim_sample_x0, denoising_utils.py:771-785)
__global__ void axpby_ps_kernel(const float* __restrict__ a, const float4* __restrict__ x, const float* __restrict__ b,
                                const float4* __restrict__ y, const float* __restrict__ c, const float4* __restrict__ z,
                                float4* __restrict__ out, int per4, long long total4) {
    pdl_trigger();
    pdl_wait();
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total4;
         i += (long long)gridDim.x * blockDim.x) {
        int s = (int)(i / per4);
        float ca = a[s], cb = b[s], cc = c[s];
        float4 xv = x[i], yv = y[i], zv = z[i];
        out[i] = make_float4(ca * xv.x + cb * yv.x + cc * zv.x, ca * xv.y + cb * yv.y + cc * zv.y,
                             ca * xv.z + cb * yv.z + cc * zv.z, ca * xv.w + cb * yv.w + cc * zv.w);
    }
}

__global__ void scale_kernel(const float* x, const float* __restrict__ alpha, float* out, long long n) {
    pdl_trigger();
    pdl_wait();
    const float a = *alpha;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        out[i] = x[i] * a;
}

// ---- toy study (main_toy.py / src/denoising_toy_utils.py:436-511): the PIDM loss algebra on [B, D] points ----------
//   data = c_data * mean_b( w_b * mean_D (target - output)^2 ),  w_b = p2[t_b] (x0 mode) or 1 (eps mode)
//   res  = c_res  * mean_b( min(0.5 r_b^2 / var_b, 27.631) )      (Gaussian NLL, log-likelihood clamped at -27.631, :381)
//   ineq = c_ineq * mean_b( min(0.5 q_b^2 / var_b, 27.631) ),    opt = lambda * mean_b(o_b)
// one CTA; sums[0..6] = data, res, ineq, opt, mean|r|, mean q, mean o; gradients w.r.t. output, r, q, o are written.
constexpr float TOY_NLL_CLAMP = 27.6310211159f;
__global__ void toy_loss_kernel(const float* __restrict__ target, const float* __restrict__ output,
                                const float* __restrict__ r, const float* __restrict__ q, const float* __restrict__ o,
                                const long long* __restrict__ t, const float* __restrict__ p2w,
                                const float* __restrict__ pvar, float c_data, float c_res, float c_ineq, float lam,
                                float* __restrict__ sums, float* __restrict__ g_out, float* __restrict__ g_r,
                                float* __restrict__ g_q, float* __restrict__ g_o, int B, int D) {
    pdl_trigger();
    pdl_wait();
    float a[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    const float invB = 1.f / (float)B;
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
        const float w = (p2w ? p2w[t[b]] : 1.f) * c_data * invB / (float)D;
        for (int d = 0; d < D; ++d) {
            const float e = output[(size_t)b * D + d] - target[(size_t)b * D + d];
            a[0] += w * e * e;
            g_out[(size_t)b * D + d] = 2.f * w * e;
        }
        const float iv = 1.f / pvar[t[b]];
        {
            const float rv = r[b], nll = 0.5f * rv * rv * iv;
            const bool live = nll < TOY_NLL_CLAMP;
            a[1] += c_res * invB * (live ? nll : TOY_NLL_CLAMP);
            a[4] += fabsf(rv) * invB;
            g_r[b] = live ? c_res * invB * rv * iv : 0.f;
        }
        if (q) {
            const float qv = q[b], nll = 0.5f * qv * qv * iv;
            const bool live = nll < TOY_NLL_CLAMP;
            a[2] += c_ineq * invB * (live ? nll : TOY_NLL_CLAMP);
            a[5] += qv * invB;
            g_q[b] = live ? c_ineq * invB * qv * iv : 0.f;
        }
        if (o) {
            a[3] += lam * invB * o[b];
            a[6] += o[b] * invB;
            g_o[b] = lam * invB;
        }
    }
    __shared__ float red[8][7];
#pragma unroll
    for (int k = 0; k < 7; ++k) a[k] = warp_sum(a[k]);
    if ((threadIdx.x & 31) == 0)
        for (int k = 0; k < 7; ++k) red[threadIdx.x >> 5][k] = a[k];
    __syncthreads();
    if (threadIdx.x < 7) {
        float s_ = 0.f;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s_ += red[w][threadIdx.x];
        sums[threadIdx.x] = s_;
    }
}

// ---- DDIM jump coefficients (eta = 0) of ddim_sample_x0 (reference denoising_utils.py:755-781), per sample:
//   mean = c1 x0 + c2 x;  eps = (sra x - mean) / nmc;  x' = sqrt(a') x0 + sqrt(1 - a') eps,  a' = alphas_prod[t_next]
//   => x' = coef_x0 * x0 + coef_x * x   (identity where t == t_next).  One launch instead of ~20 gather / arithmetic kernels.
__global__ void ddim_coefs_kernel(const long long* __restrict__ t, const long long* __restrict__ t_next,
                                  const float* __restrict__ c1, const float* __restrict__ c2, const float* __restrict__ sra,
                                  const float* __restrict__ nmc, const float* __restrict__ aprod, float* __restrict__ coef_x0,
                                  float* __restrict__ coef_x, int B) {
    pdl_trigger();
    pdl_wait();
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const long long tt = t[b], tn = t_next[b];
    if (tt == tn) { coef_x0[b] = 0.f; coef_x[b] = 1.f; return; }
    const float an = aprod[tn < 0 ? 0 : tn];
    const float c = sqrtf(1.f - an);
    coef_x0[b] = sqrtf(an) - c * c1[tt] / nmc[tt];
    coef_x[b] = c * (sra[tt] - c2[tt]) / nmc[tt];
}

// ---- residual-gradient guidance embedding: emb_conv[0] (1x1, 2 -> C) + GELU (exact erf form, nn.GELU()) ---------------
//      (reference unet_model.py:520-524,585-603).  The 2-channel 1x1 convolution is two FMAs per output channel, so it is
//      evaluated from the fp32 cond [B,HW,2] directly instead of as a channel-padded GEMM.  Thread layout: (pixel row,
//      channel octet); a thread writes 8 channels of one pixel (16 bytes in bf16).  Samples in null_mask take cond = 0:
//      their pre-activation is b0 exactly.
__device__ __forceinline__ float2 cond_at(const float* __restrict__ cond, const unsigned char* __restrict__ null_mask,
                                          int m, int HW) {
    if (null_mask != nullptr && null_mask[m / HW]) return make_float2(0.f, 0.f);
    return reinterpret_cast<const float2*>(cond)[m];
}

template <typename T>
__global__ void __launch_bounds__(256) cond_embed_fwd_kernel(const float* __restrict__ cond,
                                                             const unsigned char* __restrict__ null_mask,
                                                             const float* __restrict__ w0, const float* __restrict__ b0,
                                                             T* __restrict__ out, int HW, int C, int M) {
    pdl_trigger();
    const int oct = C >> 3;
    const int rows = blockDim.x / oct;
    const int c0 = (threadIdx.x % oct) * 8;
    float wa[8], wb[8], bb[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) { wa[k] = w0[2 * (c0 + k)]; wb[k] = w0[2 * (c0 + k) + 1]; bb[k] = b0[c0 + k]; }
    pdl_wait();
    for (int m = blockIdx.x * rows + threadIdx.x / oct; m < M; m += gridDim.x * rows) {
        const float2 x = cond_at(cond, null_mask, m, HW);
        float v[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) v[k] = gelu_erf_f(fmaf(wb[k], x.y, fmaf(wa[k], x.x, bb[k])));
        st8(out + (size_t)m * C + c0, v);
    }
}

// dz = dg * GELU'(z) with z recomputed; per-thread sums over its pixels, lanes of the same octet reduced by shuffles, the
// warps of a block through shared memory, then one global reduction per (block, output value).
template <typename T>
__global__ void __launch_bounds__(256) cond_embed_wgrad_kernel(const float* __restrict__ cond,
                                                               const unsigned char* __restrict__ null_mask,
                                                               const float* __restrict__ w0, const float* __restrict__ b0,
                                                               const T* __restrict__ dg, float* __restrict__ dw0,
                                                               float* __restrict__ db0, int HW, int C, int M) {
    pdl_trigger();
    __shared__ float red[3 * 256];                     // [C][3]: dW0[c,0], dW0[c,1], db0[c]
    const int oct = C >> 3;
    const int rows = blockDim.x / oct;
    const int c0 = (threadIdx.x % oct) * 8;
    for (int i = threadIdx.x; i < 3 * C; i += blockDim.x) red[i] = 0.f;
    float wa[8], wb[8], bb[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) { wa[k] = w0[2 * (c0 + k)]; wb[k] = w0[2 * (c0 + k) + 1]; bb[k] = b0[c0 + k]; }
    float acc[24];
#pragma unroll
    for (int k = 0; k < 24; ++k) acc[k] = 0.f;
    pdl_wait();
    for (int m = blockIdx.x * rows + threadIdx.x / oct; m < M; m += gridDim.x * rows) {
        const float2 x = cond_at(cond, null_mask, m, HW);
        float d[8];
        ld8(dg + (size_t)m * C + c0, d);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const float dz = d[k] * gelu_erf_grad_f(fmaf(wb[k], x.y, fmaf(wa[k], x.x, bb[k])));
            acc[3 * k] += dz * x.x;
            acc[3 * k + 1] += dz * x.y;
            acc[3 * k + 2] += dz;
        }
    }
    __syncthreads();                                   // red[] is zeroed
    if (reduce_same_octet<24>(acc, oct)) {
#pragma unroll
        for (int k = 0; k < 24; ++k) atomicAdd(&red[3 * c0 + k], acc[k]);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 3 * C; i += blockDim.x) {
        const int c = i / 3, r = i - 3 * c;
        atomicAdd(r == 2 ? &db0[c] : &dw0[2 * c + r], red[i]);
    }
}

// ---- output head: y[b,o,hw] = sum_c x[b,hw,c] w[o,c] + bias[o]; sigmoid on last channel if asked --------
//      (final_conv.1 of the reference, unet_model.py:517 and :619-621).  O <= 4, C multiple of 8.
template <typename T, int O>
__global__ void head_fwd_kernel(const T* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                                float* __restrict__ y, int C, int HW, long long M, int sigmoid_last) {
    pdl_trigger();
    pdl_wait();
    extern __shared__ float sw[];  // [O][C]
    for (int i = threadIdx.x; i < O * C; i += blockDim.x) sw[i] = w[i];
    __syncthreads();
    for (long long m = blockIdx.x * (long long)blockDim.x + threadIdx.x; m < M; m += (long long)gridDim.x * blockDim.x) {
        float acc[O];
#pragma unroll
        for (int o = 0; o < O; ++o) acc[o] = bias[o];
        const T* xr = x + m * C;
        for (int c = 0; c < C; c += 8) {
            float v[8];
            ld8(xr + c, v);
#pragma unroll
            for (int o = 0; o < O; ++o)
#pragma unroll
                for (int k = 0; k < 8; ++k) acc[o] += v[k] * sw[o * C + c + k];
        }
        long long b = m / HW;
        int hw = (int)(m % HW);
#pragma unroll
        for (int o = 0; o < O; ++o) {
            float v = acc[o];
            if (sigmoid_last && o == O - 1) v = 1.f / (1.f + __expf(-v));
            y[(b * O + o) * HW + hw] = v;
        }
    }
}

// backward: dx[m,c] = sum_o dz[o,m] w[o,c];  dw[o,c] += sum_m dz[o,m] x[m,c];  db[o] += sum_m dz[o,m]
// where dz = dy * (sigmoid' on the last channel).  One warp handles 32 pixels; per-CTA smem reduction then atomics.
template <typename T, int O>
__global__ void head_bwd_kernel(const T* __restrict__ x, const float* __restrict__ w, const float* __restrict__ y,
                                const float* __restrict__ dy, T* __restrict__ dx, float* __restrict__ dw,
                                float* __restrict__ db, int C, int HW, long long M, int sigmoid_last) {
    pdl_trigger();
    pdl_wait();
    extern __shared__ float sm[];   // sw[O*C] | sdw[O*C] | sdb[O]
    float* sw = sm;
    float* sdw = sm + O * C;
    float* sdb = sdw + O * C;
    for (int i = threadIdx.x; i < O * C; i += blockDim.x) { sw[i] = w[i]; sdw[i] = 0.f; }
    if (threadIdx.x < O) sdb[threadIdx.x] = 0.f;
    __syncthreads();
    const int lane = threadIdx.x & 31;
    for (long long m0 = (blockIdx.x * (long long)blockDim.x + threadIdx.x) - lane; m0 < M;
         m0 += (long long)gridDim.x * blockDim.x) {
        long long m = m0 + lane;
        bool ok = m < M;
        float dz[O];
        long long b = ok ? m / HW : 0;
        int hw = ok ? (int)(m % HW) : 0;
#pragma unroll
        for (int o = 0; o < O; ++o) {
            float g = ok ? dy[(b * O + o) * HW + hw] : 0.f;
            if (sigmoid_last && o == O - 1 && ok) {
                float s = y[(b * O + o) * HW + hw];
                g *= s * (1.f - s);
            }
            dz[o] = g;
        }
        for (int c = 0; c < C; c += 8) {
            float v[8], d[8];
            if (ok) ld8(x + m * C + c, v);
            else {
#pragma unroll
                for (int k = 0; k < 8; ++k) v[k] = 0.f;
            }
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                float s = 0.f;
#pragma unroll
                for (int o = 0; o < O; ++o) s += dz[o] * sw[o * C + c + k];
                d[k] = s;
            }
            if (ok) st8(dx + m * C + c, d);
#pragma unroll
            for (int o = 0; o < O; ++o)
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    float s = warp_sum(dz[o] * v[k]);
                    if (lane == 0) atomicAdd(&sdw[o * C + c + k], s);
                }
        }
#pragma unroll
        for (int o = 0; o < O; ++o) {
            float s = warp_sum(dz[o]);
            if (lane == 0) atomicAdd(&sdb[o], s);
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < O * C; i += blockDim.x) atomicAdd(&dw[i], sdw[i]);
    if (threadIdx.x < O) atomicAdd(&db[threadIdx.x], sdb[threadIdx.x]);
}

// Same backward, lanes laid out over (pixel, channel octet): a warp instruction moves whole 16-byte octets of C/8-lane
// pixel rows (8 pixels x 64 B at C = 32: fully coalesced), a thread keeps the weight-gradient partials of ITS octet in
// registers over all its pixels and the lanes that share an octet are combined ONCE at the end (log2(32 / LPP) shuffles
// per value) -- the kernel above reduces every (o, c) product over the warp for every 32 pixels (320 shuffles + 64
// shared-memory atomics per warp iteration; this one is a streaming pass).
// Requires LPP = C / 8 to be a power of two <= 32.
template <typename T, int O>
__global__ void __launch_bounds__(256) head_bwd_octet_kernel(const T* __restrict__ x, const float* __restrict__ w,
                                                             const float* __restrict__ y, const float* __restrict__ dy,
                                                             T* __restrict__ dx, float* __restrict__ dw,
                                                             float* __restrict__ db, int C, int HW, long long M,
                                                             int sigmoid_last) {
    pdl_trigger();
    pdl_wait();
    extern __shared__ float sm[];   // sdw[O*C] | sdb[O]
    float* sdw = sm;
    float* sdb = sm + O * C;
    for (int i = threadIdx.x; i < O * C + O; i += blockDim.x) sm[i] = 0.f;
    __syncthreads();
    const int lpp = C >> 3;                                  // lanes per pixel
    const int q = threadIdx.x & (lpp - 1);                   // this thread's octet (blockDim % lpp == 0)
    float wq[O][8], acc[O][8], accb[O];
#pragma unroll
    for (int o = 0; o < O; ++o) {
        accb[o] = 0.f;
#pragma unroll
        for (int k = 0; k < 8; ++k) { wq[o][k] = w[o * C + q * 8 + k]; acc[o][k] = 0.f; }
    }
    const long long items = M * lpp;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < items; i += (long long)gridDim.x * blockDim.x) {
        const long long m = i / lpp;                         // lpp is a power of two: shifts
        const long long b = m / HW;
        const int hw = (int)(m - b * HW);
        float dz[O];
#pragma unroll
        for (int o = 0; o < O; ++o) {
            float g = dy[(b * O + o) * HW + hw];
            if (sigmoid_last && o == O - 1) {
                const float sgm = y[(b * O + o) * HW + hw];
                g *= sgm * (1.f - sgm);
            }
            dz[o] = g;
        }
        float v[8], d[8];
        ld8(x + m * C + q * 8, v);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            float a = 0.f;
#pragma unroll
            for (int o = 0; o < O; ++o) { a += dz[o] * wq[o][k]; acc[o][k] += dz[o] * v[k]; }
            d[k] = a;
        }
        st8(dx + m * C + q * 8, d);
        if (q == 0) {
#pragma unroll
            for (int o = 0; o < O; ++o) accb[o] += dz[o];
        }
    }
    // lanes with equal q: lane bits >= log2(lpp)
    for (int off = lpp; off < 32; off <<= 1) {
#pragma unroll
        for (int o = 0; o < O; ++o) {
            accb[o] += __shfl_xor_sync(0xffffffffu, accb[o], off);
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[o][k] += __shfl_xor_sync(0xffffffffu, acc[o][k], off);
        }
    }
    if ((threadIdx.x & 31) < lpp) {
#pragma unroll
        for (int o = 0; o < O; ++o) {
#pragma unroll
            for (int k = 0; k < 8; ++k) atomicAdd(&sdw[o * C + q * 8 + k], acc[o][k]);
            if (q == 0) atomicAdd(&sdb[o], accb[o]);
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < O * C; i += blockDim.x) atomicAdd(&dw[i], sdw[i]);
    if (threadIdx.x < O) atomicAdd(&db[threadIdx.x], sdb[threadIdx.x]);
}

static inline int grid_for(long long n, int block, int cap = 0) {    // cap 0: 16 CTAs per SM
    long long g = (n + block - 1) / block;
    if (cap <= 0) cap = num_sms() * 16;
    if (g > cap) g = cap;
    if (g < 1) g = 1;
    return (int)g;
}

}  // namespace pidm
using namespace pidm;

extern "C" int pidm_qsample(const float* x0, const float* noise, const long long* t, const float* sqrt_ab,
                            const float* sqrt_1mab, float* xt, int B, int per_sample, void* stream) {
    if (per_sample % 4 != 0) {
        const long long total = (long long)B * per_sample;
        PIDM_CUDA(launch_plain(qsample_scalar_kernel, dim3(grid_for(total, 256)), dim3(256), (size_t)0, (cudaStream_t)stream, x0,
                               noise, t, sqrt_ab, sqrt_1mab, xt, per_sample, total));
        PIDM_LAUNCH_CHECK("qsample");
        return 0;
    }
    long long total4 = (long long)B * per_sample / 4;
    PIDM_CUDA(launch_plain(qsample_kernel, dim3(grid_for(total4, 256)), dim3(256), (size_t)(0), (cudaStream_t)stream, (const float4*)x0, (const float4*)noise, t, sqrt_ab, sqrt_1mab, (float4*)xt, per_sample / 4, total4));
    PIDM_LAUNCH_CHECK("qsample");
    return 0;
}

extern "C" int pidm_posterior_step(const float* x_t, const float* x0_pred, const float* z, float* out, float coef1,
                                   float coef2, float sigma, long long n, void* stream) {
    if (n % 4 != 0) {
        PIDM_CUDA(launch_plain(posterior_scalar_kernel, dim3(grid_for(n, 256)), dim3(256), (size_t)0, (cudaStream_t)stream, x_t,
                               x0_pred, z, out, coef1, coef2, sigma, n));
        PIDM_LAUNCH_CHECK("posterior_step");
        return 0;
    }
    PIDM_CUDA(launch_plain(posterior_kernel, dim3(grid_for(n / 4, 256)), dim3(256), (size_t)(0), (cudaStream_t)stream, (const float4*)x_t, (const float4*)x0_pred, (const float4*)z, (float4*)out, coef1, coef2, sigma, n / 4));
    PIDM_LAUNCH_CHECK("posterior_step");
    return 0;
}

extern "C" int pidm_nchw_to_nhwc(const float* src, void* dst, int B, int C, int HW, int Cpad, int dtype, void* stream) {
    PIDM_REQUIRE(Cpad % 8 == 0 && Cpad >= C, "nchw_to_nhwc: padded channel count must be a multiple of 8, >= C");
    long long n_pix = (long long)B * HW;
    PIDM_DISPATCH_DTYPE(dtype, PIDM_CUDA(launch_plain(nchw_to_nhwc_kernel<T>, dim3(grid_for(n_pix, 128)), dim3(128), (size_t)(0), (cudaStream_t)stream, src, (T*)dst, C, HW, Cpad, n_pix)));
    PIDM_LAUNCH_CHECK("nchw_to_nhwc");
    return 0;
}

extern "C" int pidm_concat_channels(const void* a, const void* b, void* out, long long rows, int Ca, int Cb, int dtype,
                                    void* stream) {
    PIDM_REQUIRE(Ca % 8 == 0 && Cb % 8 == 0, "concat: channel counts must be multiples of 8");
    long long total = rows * (Ca + Cb) / 8;
    PIDM_DISPATCH_DTYPE(dtype, PIDM_CUDA(launch_plain(concat_kernel<T>, dim3(grid_for(total, 256)), dim3(256), (size_t)(0), (cudaStream_t)stream, (const T*)a, (const T*)b, (T*)out, Ca / 8, Cb / 8, rows)));
    PIDM_LAUNCH_CHECK("concat");
    return 0;
}

extern "C" int pidm_split_channels(const void* g, void* ga, void* gb, long long rows, int Ca, int Cb, int dtype,
                                   void* stream) {
    PIDM_REQUIRE(Ca % 8 == 0 && Cb % 8 == 0, "split: channel counts must be multiples of 8");
    long long total = rows * (Ca + Cb) / 8;
    PIDM_DISPATCH_DTYPE(dtype, PIDM_CUDA(launch_plain(split_kernel<T>, dim3(grid_for(total, 256)), dim3(256), (size_t)(0), (cudaStream_t)stream, (const T*)g, (T*)ga, (T*)gb, Ca / 8, Cb / 8, rows)));
    PIDM_LAUNCH_CHECK("split");
    return 0;
}

extern "C" int pidm_wrap_pad_nhwc(const void* x, void* y, int B, int H, int W, int C, int halo, int dtype,
                                  void* stream) {
    PIDM_REQUIRE(dtype == 0 || dtype == 1, "wrap_pad: unknown dtype %d", dtype);
    const int esize = dtype == 0 ? 4 : 2;
    PIDM_REQUIRE(B > 0 && H > 0 && W > 0 && C > 0 && ((long long)C * esize) % 16 == 0,
                 "wrap_pad: a pixel row must be a whole number of 16-byte units (C=%d)", C);
    PIDM_REQUIRE(halo >= 1 && halo <= 3 && halo <= H && halo <= W, "wrap_pad: halo must be 1..3 and <= H, W (got %d)",
                 halo);
    PIDM_REQUIRE(((uintptr_t)x & 15) == 0 && ((uintptr_t)y & 15) == 0, "wrap_pad: operands must be 16-byte aligned");
    const int U = C * esize / 16;
    const long long total = (long long)B * (H + 2 * halo) * (W + 2 * halo) * U;
    PIDM_CUDA(launch_plain(wrap_pad_kernel, dim3(grid_for(total, 256)), dim3(256), (size_t)0, (cudaStream_t)stream,
                           (const uint4*)x, (uint4*)y, H, W, halo, U, total));
    PIDM_LAUNCH_CHECK("wrap_pad");
    return 0;
}

extern "C" int pidm_axpby_per_sample(const float* a, const float* x, const float* b, const float* y, const float* c,
                                     const float* z, float* out, int B, int per_sample, void* stream) {
    if (per_sample % 4 != 0) {
        const long long total = (long long)B * per_sample;
        PIDM_CUDA(launch_plain(axpby_ps_scalar_kernel, dim3(grid_for(total, 256)), dim3(256), (size_t)0, (cudaStream_t)stream, a, x,
                               b, y, c, z, out, per_sample, total));
        PIDM_LAUNCH_CHECK("axpby_per_sample");
        return 0;
    }
    long long total4 = (long long)B * per_sample / 4;
    PIDM_CUDA(launch_plain(axpby_ps_kernel, dim3(grid_for(total4, 256)), dim3(256), (size_t)(0), (cudaStream_t)stream, a, (const float4*)x, b, (const float4*)y, c, (const float4*)z, (float4*)out, per_sample / 4, total4));
    PIDM_LAUNCH_CHECK("axpby_per_sample");
    return 0;
}

extern "C" int pidm_scale(const float* x, const float* alpha_dev, float* out, long long n, void* stream) {
    PIDM_CUDA(launch_plain(scale_kernel, dim3(grid_for(n, 256)), dim3(256), (size_t)(0), (cudaStream_t)stream, x, alpha_dev, out, n));
    PIDM_LAUNCH_CHECK("scale");
    return 0;
}

extern "C" int pidm_ddim_coefs(const long long* t, const long long* t_next, const float* posterior_mean_coef1,
                               const float* posterior_mean_coef2, const float* sqrt_recip_alphas, const float* noise_mean_coeff,
                               const float* alphas_prod, float* coef_x0, float* coef_x, int B, void* stream) {
    PIDM_CUDA(launch_plain(ddim_coefs_kernel, dim3(grid_for(B, 128)), dim3(128), (size_t)0, (cudaStream_t)stream, t, t_next,
                           posterior_mean_coef1, posterior_mean_coef2, sqrt_recip_alphas, noise_mean_coeff, alphas_prod, coef_x0,
                           coef_x, B));
    PIDM_LAUNCH_CHECK("ddim_coefs");
    return 0;
}

static int check_cond_embed(const float* cond, const void* act, int B, int HW, int C) {
    PIDM_REQUIRE(B > 0 && HW > 0 && (long long)B * HW < (1LL << 31), "cond_embed: B*HW out of range");
    PIDM_REQUIRE(C % 8 == 0 && C <= 256 && 32 % (C / 8) == 0, "cond_embed: C = %d must be 8, 16, 32, 64, 128 or 256", C);
    PIDM_REQUIRE(((uintptr_t)cond & 7) == 0 && ((uintptr_t)act & 15) == 0, "cond_embed: misaligned cond / activation");
    return 0;
}

extern "C" int pidm_cond_embed_fwd(const float* cond, const unsigned char* null_mask, const float* w0, const float* b0,
                                   void* out, int B, int HW, int C, int dtype, void* stream) {
    if (int e = check_cond_embed(cond, out, B, HW, C)) return e;
    const int M = B * HW, rows = 256 / (C / 8);
    PIDM_DISPATCH_DTYPE(dtype, PIDM_CUDA(launch_plain(cond_embed_fwd_kernel<T>, dim3(grid_for(M, rows)), dim3(256),
                                                      (size_t)0, (cudaStream_t)stream, cond, null_mask, w0, b0, (T*)out, HW,
                                                      C, M)));
    PIDM_LAUNCH_CHECK("cond_embed_fwd");
    return 0;
}

extern "C" int pidm_cond_embed_wgrad(const float* cond, const unsigned char* null_mask, const float* w0, const float* b0,
                                     const void* dg, float* dw0, float* db0, int B, int HW, int C, int dtype,
                                     void* stream) {
    if (int e = check_cond_embed(cond, dg, B, HW, C)) return e;
    const int M = B * HW, rows = 256 / (C / 8);
    // 4 CTAs per SM: every thread sums several pixels before the block reduction
    PIDM_DISPATCH_DTYPE(dtype, PIDM_CUDA(launch_plain(cond_embed_wgrad_kernel<T>, dim3(grid_for(M, rows, num_sms() * 4)),
                                                      dim3(256), (size_t)0, (cudaStream_t)stream, cond, null_mask, w0, b0,
                                                      (const T*)dg, dw0, db0, HW, C, M)));
    PIDM_LAUNCH_CHECK("cond_embed_wgrad");
    return 0;
}

extern "C" int pidm_toy_pidm_loss(const float* target, const float* output, const float* residual, const float* ineq,
                                  const float* opt, const long long* t, const float* p2_loss_weight,
                                  const float* posterior_var_clipped, float c_data, float c_residual, float c_ineq,
                                  float lambda_opt, float* sums7, float* grad_output, float* grad_residual, float* grad_ineq,
                                  float* grad_opt, int B, int D, void* stream) {
    PIDM_REQUIRE(B > 0 && D > 0, "toy_pidm_loss: bad sizes B=%d D=%d", B, D);
    PIDM_CUDA(launch_plain(toy_loss_kernel, dim3(1), dim3(256), (size_t)0, (cudaStream_t)stream, target, output, residual, ineq, opt,
                           t, p2_loss_weight, posterior_var_clipped, c_data, c_residual, c_ineq, lambda_opt, sums7, grad_output,
                           grad_residual, grad_ineq, grad_opt, B, D));
    PIDM_LAUNCH_CHECK("toy_pidm_loss");
    return 0;
}

extern "C" int pidm_head_fwd(const void* x, const float* w, const float* bias, float* y, int B, int HW, int C, int O,
                             int sigmoid_last, int dtype, void* stream) {
    PIDM_REQUIRE(C % 8 == 0 && O >= 1 && O <= 4, "head: C%%8==0 and 1<=O<=4 required (C=%d O=%d)", C, O);
    long long M = (long long)B * HW;
    size_t smem = (size_t)O * C * sizeof(float);
#define HEAD_F(OO)                                                                                     \
    PIDM_DISPATCH_DTYPE(dtype, PIDM_CUDA(launch_plain(head_fwd_kernel<T, OO>, dim3(grid_for(M, 256)), dim3(256), (size_t)(smem), (cudaStream_t)stream, \
                                   (const T*)x, w, bias, y, C, HW, M, sigmoid_last)))
    switch (O) { case 1: HEAD_F(1); break; case 2: HEAD_F(2); break; case 3: HEAD_F(3); break; default: HEAD_F(4); }
#undef HEAD_F
    PIDM_LAUNCH_CHECK("head_fwd");
    return 0;
}

extern "C" int pidm_head_bwd(const void* x, const float* w, const float* y, const float* dy, void* dx, float* dw,
                             float* db, int B, int HW, int C, int O, int sigmoid_last, int dtype, void* stream) {
    PIDM_REQUIRE(C % 8 == 0 && O >= 1 && O <= 4, "head: C%%8==0 and 1<=O<=4 required (C=%d O=%d)", C, O);
    long long M = (long long)B * HW;
    size_t smem = (size_t)(2 * O * C + O) * sizeof(float);
    const int lpp = C / 8;
    if (lpp <= 32 && (lpp & (lpp - 1)) == 0) {
        const long long items = M * lpp;
#define HEAD_BO(OO)                                                                                    \
    PIDM_DISPATCH_DTYPE(dtype, PIDM_CUDA(launch_plain(head_bwd_octet_kernel<T, OO>, dim3(grid_for(items, 256, num_sms() * 4)), dim3(256), (size_t)(smem), (cudaStream_t)stream, \
                                   (const T*)x, w, y, dy, (T*)dx, dw, db, C, HW, M, sigmoid_last)))
        switch (O) { case 1: HEAD_BO(1); break; case 2: HEAD_BO(2); break; case 3: HEAD_BO(3); break; default: HEAD_BO(4); }
#undef HEAD_BO
        PIDM_LAUNCH_CHECK("head_bwd");
        return 0;
    }
#define HEAD_B(OO)                                                                                     \
    PIDM_DISPATCH_DTYPE(dtype, PIDM_CUDA(launch_plain(head_bwd_kernel<T, OO>, dim3(grid_for(M, 256, num_sms() * 2)), dim3(256), (size_t)(smem), (cudaStream_t)stream, \
                                   (const T*)x, w, y, dy, (T*)dx, dw, db, C, HW, M, sigmoid_last)))
    switch (O) { case 1: HEAD_B(1); break; case 2: HEAD_B(2); break; case 3: HEAD_B(3); break; default: HEAD_B(4); }
#undef HEAD_B
    PIDM_LAUNCH_CHECK("head_bwd");
    return 0;
}
