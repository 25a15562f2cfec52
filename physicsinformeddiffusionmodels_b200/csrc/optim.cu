// Step glue on FLAT fp32 buffers (one launch each instead of ~1000 per-tensor launches of the reference loop):
//   global-norm clip (torch.nn.utils.clip_grad_norm_(params, 1.0), main.py:165)
//   Adam(lr, betas=(0.9,0.999), eps=1e-8)                          (main.py:143,166)
//   EMA shadow update mu=0.99                                       (denoising_utils.py:174-177, main.py:178-179)
// and the host plumbing (errors, SM count, shared-memory opt-in) shared by all translation units.
#include "common.cuh"
#include "pidm.h"
#include <stdarg.h>
#include <mutex>
#include <unordered_map>

namespace pidm {

thread_local char g_last_error[512] = {0};

int num_sms() {
    static int n = 0;
    if (!n) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
            n = 132;
    }
    return n;
}

cudaError_t allow_smem(const void* kernel, size_t bytes) {
    static std::mutex mu;
    static std::unordered_map<const void*, size_t> allowed;
    std::lock_guard<std::mutex> lock(mu);
    size_t& cur = allowed[kernel];
    if (bytes <= cur) return cudaSuccess;
    const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e == cudaSuccess) cur = bytes;
    return e;
}

int set_error(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_last_error, sizeof(g_last_error), fmt, ap);
    va_end(ap);
    return code;
}

// Deterministic: every CTA writes its partial sum to workspace[1 + blockIdx.x]; the CTA that arrives last (ticket counter
// in workspace[0]) adds the partials in index order.  The result does not depend on the arrival order, so every rank of a
// data-parallel job computes bit-identical clip coefficients from its (bit-identical) all-reduced gradient -- with
// atomicAdd the ranks' norms differed in the last bit and their weights drifted apart by ~1e-7 per step.
__global__ void sumsq_kernel(const float4* __restrict__ x, long long n4, const float* __restrict__ tail, int ntail,
                             float* __restrict__ out, float* __restrict__ workspace) {
    pdl_trigger();
    pdl_wait();
    float s = 0.f;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        float4 v = x[i];
        s += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
    }
    if (blockIdx.x == 0 && (int)threadIdx.x < ntail) s += tail[threadIdx.x] * tail[threadIdx.x];
    __shared__ float red[32];
    __shared__ bool last;
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x < 32) {
        float v = (threadIdx.x < (blockDim.x >> 5)) ? red[threadIdx.x] : 0.f;
        v = warp_sum(v);
        if (threadIdx.x == 0) {
            workspace[1 + blockIdx.x] = v;
            __threadfence();
            unsigned int* ticket = reinterpret_cast<unsigned int*>(workspace);
            last = atomicAdd(ticket, 1u) == gridDim.x - 1;
        }
    }
    __syncthreads();
    if (last) {
        __threadfence();
        float v = 0.f;
        for (int i = threadIdx.x; i < (int)gridDim.x; i += blockDim.x) v += __ldcg(&workspace[1 + i]);   // fixed assignment
        v = warp_sum(v);
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
        __syncthreads();
        if (threadIdx.x == 0) {
            float t = 0.f;
            for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[w];
            *out += t;
            *reinterpret_cast<unsigned int*>(workspace) = 0u;          // ready for the next launch / graph replay
        }
    }
}

// Bias corrections follow torch.optim.Adam, which evaluates 1 - beta^step in double precision on the host: with the
// step count on the device (CUDA-graph replay) one thread per CTA evaluates them in double and shares them.  In fp32
// 1 - 0.999^1 already carries a relative error of 6e-5 (cancellation), which would show up in the step size.
// ema_first_step: 0 = no EMA; k >= 1 = the shadow is updated from the k-th (1-based) optimizer step on
// (reference main.py:52,178 `if iteration > ema_start`, iteration 0-based => k = ema_start + 2).
__global__ void adam_ema_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m,
                                float* __restrict__ v, float* __restrict__ ema, long long n, float lr, double b1d,
                                double b2d, float eps, int step_host, const int* __restrict__ step_dev,
                                const float* __restrict__ gnorm_sq, float grad_scale, float max_norm, float ema_mu,
                                int ema_first_step, int zero_grad) {
    pdl_trigger();
    pdl_wait();
    __shared__ float s_step, s_rs;
    __shared__ int s_ema;
    if (threadIdx.x == 0) {
        const int st = step_dev ? *step_dev : step_host;          // 1-based count of this step
        const double bc1 = 1.0 - pow(b1d, (double)st);
        const double bc2 = 1.0 - pow(b2d, (double)st);
        s_step = (float)((double)lr / bc1);
        s_rs = (float)(1.0 / sqrt(bc2));
        s_ema = (ema_first_step > 0 && st >= ema_first_step) ? 1 : 0;
    }
    __syncthreads();
    // 1 - beta in double: 1.f - (float)0.999 is 1.3e-5 too small (the same cancellation), which biased v by that much
    // and made the step-1 update 6.4e-6 too large; torch rounds 1 - beta2 once
    const float b1 = (float)b1d, b2 = (float)b2d, omb1 = (float)(1.0 - b1d), omb2 = (float)(1.0 - b2d);
    float coef = grad_scale;
    if (gnorm_sq && max_norm > 0.f) {
        float total = sqrtf(*gnorm_sq) * grad_scale;
        coef *= fminf(max_norm / (total + 1e-6f), 1.f);
    }
    const float step = s_step, rs = s_rs;
    const bool ema_on = s_ema != 0;
    // 128-bit accesses: the pass moves 40 bytes per parameter (5 buffers read, 5 written), nothing else matters
    const long long n4 = n >> 2;
    float4* p4 = reinterpret_cast<float4*>(p);
    float4* g4 = reinterpret_cast<float4*>(g);
    float4* m4 = reinterpret_cast<float4*>(m);
    float4* v4 = reinterpret_cast<float4*>(v);
    float4* e4 = reinterpret_cast<float4*>(ema);
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        float4 gv = g4[i], mv = m4[i], vv = v4[i], pv = p4[i], ev;
        if (ema_on) ev = e4[i];
        float* gp = &gv.x; float* mp = &mv.x; float* vp = &vv.x; float* pp = &pv.x; float* ep = &ev.x;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float gi = gp[k] * coef;
            mp[k] = b1 * mp[k] + omb1 * gi;
            vp[k] = b2 * vp[k] + omb2 * gi * gi;
            pp[k] = pp[k] - step * mp[k] / (sqrtf(vp[k]) * rs + eps);
            if (ema_on) ep[k] = ema_mu * ep[k] + (1.f - ema_mu) * pp[k];
        }
        m4[i] = mv; v4[i] = vv; p4[i] = pv;
        if (ema_on) e4[i] = ev;
        if (zero_grad) g4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    for (long long i = (n4 << 2) + blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        float gi = g[i] * coef;
        float mi = b1 * m[i] + omb1 * gi;
        float vi = b2 * v[i] + omb2 * gi * gi;
        float pi = p[i] - step * mi / (sqrtf(vi) * rs + eps);
        m[i] = mi; v[i] = vi; p[i] = pi;
        if (ema_on) ema[i] = ema_mu * ema[i] + (1.f - ema_mu) * pi;
        if (zero_grad) g[i] = 0.f;
    }
}

__global__ void incr_kernel(int* c) {
    pdl_trigger();
    pdl_wait(); *c += 1; }

// a[i] <-> b[i] over n4 float4s: 16 bytes per element (each buffer read once and written once)
__global__ void swap_kernel(float4* __restrict__ a, float4* __restrict__ b, long long n4) {
    pdl_trigger();
    pdl_wait();
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        const float4 x = a[i], y = b[i];
        a[i] = y;
        b[i] = x;
    }
}

}  // namespace pidm
using namespace pidm;

extern "C" const char* pidm_last_error(void) { return g_last_error; }

extern "C" int pidm_version(void) { return 100; }

// out[0] += sum x^2   (caller zeroes out).  workspace: float[PIDM_SUMSQ_WORKSPACE_FLOATS], zero-initialised ONCE by the
// caller (element 0 is a ticket counter that every launch leaves at zero).
extern "C" int pidm_sumsq(const float* x, long long n, float* out, float* workspace, void* stream) {
    PIDM_REQUIRE(((uintptr_t)x & 15) == 0, "sumsq: buffer must be 16-byte aligned");
    PIDM_REQUIRE(workspace != nullptr, "sumsq: workspace of %d floats required", 1 + 148 * 8);
    long long n4 = n / 4;
    int grid = (int)((n4 + 255) / 256);
    if (grid > 148 * 8) grid = 148 * 8;
    if (grid < 1) grid = 1;
    PIDM_CUDA(launch_plain(sumsq_kernel, dim3(grid), dim3(256), (size_t)(0), (cudaStream_t)stream, (const float4*)x, n4, x + n4 * 4, (int)(n - n4 * 4), out, workspace));
    PIDM_LAUNCH_CHECK("sumsq");
    return 0;
}

extern "C" int pidm_adam_ema_step(float* param, float* grad, float* exp_avg, float* exp_avg_sq, float* ema_shadow,
                                  long long n, float lr, double beta1, double beta2, float eps, int step,
                                  int* step_counter_dev, const float* grad_norm_sq_dev, float grad_scale, float max_norm, float ema_mu,
                                  int ema_first_step, int zero_grad, void* stream) {
    PIDM_REQUIRE(step >= 1 || step_counter_dev, "adam: step is 1-based");
    PIDM_REQUIRE((((uintptr_t)param | (uintptr_t)grad | (uintptr_t)exp_avg | (uintptr_t)exp_avg_sq |
                   (uintptr_t)(ema_first_step > 0 ? ema_shadow : param)) & 15) == 0, "adam: buffers must be 16-byte aligned");
    if (step_counter_dev) PIDM_CUDA(launch_plain(incr_kernel, dim3(1), dim3(1), (size_t)(0), (cudaStream_t)stream, step_counter_dev));   // counter holds steps done so far
    int grid = (int)((n / 4 + 255) / 256);
    if (grid > num_sms() * 8) grid = num_sms() * 8;
    if (grid < 1) grid = 1;
    PIDM_CUDA(launch_plain(adam_ema_kernel, dim3(grid), dim3(256), (size_t)(0), (cudaStream_t)stream, param, grad, exp_avg, exp_avg_sq, ema_shadow, n, lr, beta1,
                                                             beta2, eps, step, step_counter_dev, grad_norm_sq_dev, grad_scale,
                                                             max_norm, ema_mu, ema_first_step, zero_grad));
    PIDM_LAUNCH_CHECK("adam_ema_step");
    return 0;
}

extern "C" int pidm_swap_f32(float* a, float* b, long long n, void* stream) {
    PIDM_REQUIRE(n >= 0 && n % 4 == 0, "swap_f32: n = %lld must be a non-negative multiple of 4", n);
    PIDM_REQUIRE((((uintptr_t)a | (uintptr_t)b) & 15) == 0, "swap_f32: buffers must be 16-byte aligned");
    if (n == 0) return 0;
    const long long n4 = n / 4;
    int grid = (int)std::min<long long>((n4 + 255) / 256, num_sms() * 8LL);
    PIDM_CUDA(launch_plain(swap_kernel, dim3(grid), dim3(256), (size_t)(0), (cudaStream_t)stream, (float4*)a, (float4*)b, n4));
    PIDM_LAUNCH_CHECK("swap_f32");
    return 0;
}
