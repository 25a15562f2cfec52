// Time-conditioning path of the U-Net, fp32 throughout (B x 128 activations: latency-, not throughput-bound):
//   * time_embed : SinusoidalPosEmb(dim) -> Linear(dim,4dim) -> GELU(erf) -> Linear(4dim,4dim) (+ SiLU of it)
//                  reference unet_model.py:147-159, 464-469
//   * block_mlps : every ResnetBlock's Linear(4dim, 2*C_out) on SiLU(t) (unet_model.py:246-249,258-262),
//                  ALL blocks in one launch through a device-side table (they share the same input).
#include "common.cuh"
#include "pidm.h"

namespace pidm {

// one CTA per sample, blockDim = td
__global__ void time_embed_fwd_kernel(const long long* __restrict__ t, const float* __restrict__ W1,
                                      const float* __restrict__ b1, const float* __restrict__ W2,
                                      const float* __restrict__ b2, float* __restrict__ emb /*[B,dim]*/,
                                      float* __restrict__ h1 /*[B,td]*/, float* __restrict__ temb /*[B,td]*/,
                                      float* __restrict__ silu_t /*[B,td]*/, int dim, int td) {
    pdl_trigger();
    pdl_wait();
    extern __shared__ float sm[];   // e[dim] | a1[td]
    float* e = sm;
    float* a1 = sm + dim;
    const int b = blockIdx.x, j = threadIdx.x;
    const int half = dim / 2;
    if (j < dim) {
        // frequency, argument and sinusoid in double, which --use_fast_math leaves alone: with __expf / __sinf the
        // error grew with t f and passed what fp32 PyTorch reaches (8 u (1 + |t f|)) at t = 999; B x dim evaluations
        const int k = j < half ? j : j - half;
        const double f = exp((double)k * -(log(10000.0) / (double)(half - 1)));
        const double arg = (double)t[b] * f;
        const float v = (float)(j < half ? sin(arg) : cos(arg));
        e[j] = v;
        emb[(size_t)b * dim + j] = v;
    }
    __syncthreads();
    // thread j owns output row j: its weight row is read as 16-byte vectors, 16 loads in flight (the scalar loop issued
    // td dependent-latency batches)
    float acc = b1[j];
    {
        const float4* wr = reinterpret_cast<const float4*>(W1 + (size_t)j * dim);
        float a0 = 0.f, a1_ = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll 8
        for (int k4 = 0; k4 < dim / 4; ++k4) {
            const float4 w = __ldg(wr + k4);
            a0 += w.x * e[4 * k4]; a1_ += w.y * e[4 * k4 + 1]; a2 += w.z * e[4 * k4 + 2]; a3 += w.w * e[4 * k4 + 3];
        }
        acc += (a0 + a1_) + (a2 + a3);
    }
    h1[(size_t)b * td + j] = acc;
    a1[j] = gelu_erf_f(acc);
    __syncthreads();
    float o = b2[j];
    {
        const float4* wr = reinterpret_cast<const float4*>(W2 + (size_t)j * td);
        float a0 = 0.f, a1_ = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll 16
        for (int k4 = 0; k4 < td / 4; ++k4) {
            const float4 w = __ldg(wr + k4);
            a0 += w.x * a1[4 * k4]; a1_ += w.y * a1[4 * k4 + 1]; a2 += w.z * a1[4 * k4 + 2]; a3 += w.w * a1[4 * k4 + 3];
        }
        o += (a0 + a1_) + (a2 + a3);
    }
    temb[(size_t)b * td + j] = o;
    silu_t[(size_t)b * td + j] = silu_f(o);
}

// backward, stage 1 (one CTA per sample, blockDim = td): dt = d_silu * silu'(temb), dh = (W2^T dt) * gelu'(h1); both
// are written to the workspace [2, B, td] for stage 2.
__global__ void time_embed_bwd_act_kernel(const float* __restrict__ d_silu, const float* __restrict__ h1,
                                          const float* __restrict__ temb, const float* __restrict__ W2,
                                          float* __restrict__ dt_out, float* __restrict__ dh_out, int td) {
    pdl_trigger();
    pdl_wait();
    extern __shared__ float sm[];   // dt[td]
    float* dt = sm;
    const int b = blockIdx.x, j = threadIdx.x;
    const float dtj = d_silu[(size_t)b * td + j] * silu_grad_f(temb[(size_t)b * td + j]);
    dt[j] = dtj;
    dt_out[(size_t)b * td + j] = dtj;
    __syncthreads();
    // da1[j] = sum_i dt[i] W2[i][j]  (column read: coalesced across threads j)
    float da = 0.f;
#pragma unroll 32
    for (int i = 0; i < td; ++i) da += dt[i] * __ldg(W2 + (size_t)i * td + j);
    dh_out[(size_t)b * td + j] = da * gelu_erf_grad_f(h1[(size_t)b * td + j]);
}

// backward, stage 2 (one CTA per output row j, blockDim = td = columns k): the weight gradients are small
// [td x B] x [B x td] products -- every element is owned by exactly one thread, so they are accumulated with plain
// read-modify-writes (rather than td + dim contended atomics per thread from B CTAs).
//   dW2[j,k] += sum_b dt[b,j] gelu(h1[b,k]);  db2[j] += sum_b dt[b,j];  dW1[j,k<dim] += sum_b dh[b,j] emb[b,k];  db1[j] += ...
__global__ void time_embed_bwd_wgrad_kernel(const float* __restrict__ dt, const float* __restrict__ dh,
                                            const float* __restrict__ emb, const float* __restrict__ h1,
                                            float* __restrict__ dW1, float* __restrict__ db1, float* __restrict__ dW2,
                                            float* __restrict__ db2, int B, int dim, int td) {
    pdl_trigger();
    pdl_wait();
    const int j = blockIdx.x, k = threadIdx.x;
    float w2 = 0.f, w1 = 0.f, s2 = 0.f, s1 = 0.f;
    for (int b = 0; b < B; ++b) {
        const float dtj = dt[(size_t)b * td + j], dhj = dh[(size_t)b * td + j];      // broadcast loads
        w2 += dtj * gelu_erf_f(h1[(size_t)b * td + k]);
        if (k < dim) w1 += dhj * emb[(size_t)b * dim + k];
        s2 += dtj; s1 += dhj;
    }
    dW2[(size_t)j * td + k] += w2;
    if (k < dim) dW1[(size_t)j * dim + k] += w1;
    if (k == 0) { db2[j] += s2; db1[j] += s1; }
}

struct MlpEntry {
    const float* W;      // [n, td]
    const float* b;      // [n]
    float* dW;           // accumulated
    float* db;           // accumulated
    float* out;          // [B, n]
    const float* dout;   // [B, n]
    int n, pad_;
};

constexpr int MLP_BCHUNK = 32;      // samples per pass = lanes of a warp
constexpr int MLP_ROWS = 16;        // output rows per CTA (fwd / wgrad): two per warp.  The problem is latency-bound: ~240
                                    // CTAs (one wave at two CTAs per SM) each pay one table + one tile + four weight batches
constexpr int MLP_DG_ROWS = 32;     // rows per CTA (dgrad)
constexpr int MLP_TD_MAX = 704;     // largest td: the [32][td + 1] fp32 tile of fwd / wgrad fits in 96 KB of shared memory

// out[b, j] = bias[j] + W[j,:] . s[b,:].  grid (entries, row chunks of MLP_ROWS), 256 threads.  A warp owns a row j,
// its lanes are 32 samples: W[j,k] is one broadcast load per k, s[b,k] comes from a (td+1)-padded shared tile, and
// no cross-lane reduction is needed.
__global__ void __launch_bounds__(256) block_mlps_fwd_kernel(const MlpEntry* __restrict__ table,
                                                             const float* __restrict__ s /*[B,td]*/, int B, int td) {
    pdl_trigger();
    pdl_wait();
    extern __shared__ float ss[];   // [MLP_BCHUNK][td + 1]
    const MlpEntry e = table[blockIdx.x];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    const int r0 = blockIdx.y * MLP_ROWS;
    if (r0 >= e.n) return;
    const int r1 = min(r0 + MLP_ROWS, e.n);
    const int ld = td + 1, tq = td >> 2;
    for (int b0 = 0; b0 < B; b0 += MLP_BCHUNK) {
        const int nb = min(MLP_BCHUNK, B - b0);
        __syncthreads();
        // the [32][td] input tile: 16-byte loads, four in flight per thread
        for (int i0 = threadIdx.x; i0 < MLP_BCHUNK * tq; i0 += 4 * blockDim.x) {
            float4 v[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int i = i0 + u * blockDim.x, b = i / tq, k4 = i - b * tq;
                v[u] = (i < MLP_BCHUNK * tq && b < nb) ? __ldg(reinterpret_cast<const float4*>(s + (size_t)(b0 + b) * td) + k4)
                                                       : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int i = i0 + u * blockDim.x, b = i / tq, k4 = i - b * tq;
                if (i < MLP_BCHUNK * tq) {
                    float* d = ss + b * ld + 4 * k4;
                    d[0] = v[u].x; d[1] = v[u].y; d[2] = v[u].z; d[3] = v[u].w;
                }
            }
        }
        __syncthreads();
        const float* sl = ss + lane * ld;
        for (int j = r0 + warp; j < r1; j += nw) {
            const float4* wr = reinterpret_cast<const float4*>(e.W + (size_t)j * td);
            float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
            for (int k0 = 0; k0 < tq; k0 += 16) {        // 16 weight vectors (one broadcast load each) in flight
                float4 w[16];
#pragma unroll
                for (int u = 0; u < 16; ++u) w[u] = (k0 + u < tq) ? __ldg(wr + k0 + u) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                for (int u = 0; u < 16; ++u) {
                    if (k0 + u < tq) {
                        const float* sp = sl + 4 * (k0 + u);
                        a0 += w[u].x * sp[0]; a1 += w[u].y * sp[1]; a2 += w[u].z * sp[2]; a3 += w[u].w * sp[3];
                    }
                }
            }
            if (lane < nb) e.out[(size_t)(b0 + lane) * e.n + j] = (a0 + a1) + (a2 + a3) + __ldg(e.b + j);
        }
    }
}

// dW[j,k] += sum_b d[b,j] s[b,k] ; db[j] += sum_b d[b,j]    (row j owned by exactly one warp; lane b holds d[b,j] and
// broadcasts it by shuffle, lanes run over k for the s tile)
__global__ void __launch_bounds__(256) block_mlps_wgrad_kernel(const MlpEntry* __restrict__ table,
                                                               const float* __restrict__ s, int B, int td) {
    pdl_trigger();
    pdl_wait();
    extern __shared__ float ss[];   // [MLP_BCHUNK][td]
    const MlpEntry e = table[blockIdx.x];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    const int r0 = blockIdx.y * MLP_ROWS;
    if (r0 >= e.n) return;
    const int r1 = min(r0 + MLP_ROWS, e.n);
    const int nk = td / 32;          // k values per lane (td % 32 == 0, td <= 768 -> <= 24)
    for (int b0 = 0; b0 < B; b0 += MLP_BCHUNK) {
        const int nb = min(MLP_BCHUNK, B - b0);
        __syncthreads();
        for (int i = threadIdx.x; i < MLP_BCHUNK * td; i += blockDim.x)
            ss[i] = (i / td) < nb ? s[(size_t)b0 * td + i] : 0.f;
        __syncthreads();
        for (int j = r0 + warp; j < r1; j += nw) {
            const float d = lane < nb ? e.dout[(size_t)(b0 + lane) * e.n + j] : 0.f;
            float* wr = e.dW + (size_t)j * td;
            for (int kk = 0; kk < nk; kk += 4) {
                float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
                const float* sk = ss + kk * 32 + lane;
#pragma unroll 8
                for (int b = 0; b < MLP_BCHUNK; ++b) {
                    const float db_ = __shfl_sync(0xffffffffu, d, b);
                    const float* sb = sk + b * td;
                    a0 += db_ * sb[0];
                    if (kk + 1 < nk) a1 += db_ * sb[32];
                    if (kk + 2 < nk) a2 += db_ * sb[64];
                    if (kk + 3 < nk) a3 += db_ * sb[96];
                }
                wr[kk * 32 + lane] += a0;
                if (kk + 1 < nk) wr[(kk + 1) * 32 + lane] += a1;
                if (kk + 2 < nk) wr[(kk + 2) * 32 + lane] += a2;
                if (kk + 3 < nk) wr[(kk + 3) * 32 + lane] += a3;
            }
            const float dsum = warp_sum(d);
            if (lane == 0) e.db[j] += dsum;
        }
    }
}

// d_s[b,k] += sum_e sum_j dout_e[b,j] W_e[j,k].  grid (entries, row chunks of MLP_DG_ROWS, sample chunks of 32), block td.
// Thread = k keeps 32 sample accumulators; W rows are read once (coalesced over k), dout comes from shared memory as
// broadcast float4 reads, one atomicAdd per (sample, k) and CTA at the end.  ds zeroed by the caller.  (The first version
// gave each of 37 CTAs a 128-row chunk found by scanning the table: 18 dependent table loads + 16 serial batches of
// weight loads per CTA for a 30 MFLOP problem; now ~120 CTAs with 4 batches each, addressed directly.)
// __launch_bounds__: blockDim = td goes up to MLP_TD_MAX; without the bound ptxas took 95 registers per thread and
// a 704-thread block asked for more than the SM's 64 K registers (the launch failed for td > 672)
__global__ void __launch_bounds__(MLP_TD_MAX) block_mlps_dgrad_kernel(const MlpEntry* __restrict__ table,
                                                                      float* __restrict__ ds, int B, int td) {
    pdl_trigger();
    pdl_wait();
    __shared__ __align__(16) float sd[MLP_DG_ROWS][MLP_BCHUNK];
    const MlpEntry e = table[blockIdx.x];
    const int r0 = blockIdx.y * MLP_DG_ROWS;
    if (r0 >= e.n) return;
    const int nr = min(MLP_DG_ROWS, e.n - r0);
    const int b0 = blockIdx.z * MLP_BCHUNK;
    const int nb = min(MLP_BCHUNK, B - b0);
    const int k = threadIdx.x;
    for (int i = threadIdx.x; i < nr * MLP_BCHUNK; i += blockDim.x) {
        const int b = i / nr, j = i - b * nr;      // consecutive threads walk j: coalesced reads of dout[b, r0 + j]
        sd[j][b] = b < nb ? e.dout[(size_t)(b0 + b) * e.n + r0 + j] : 0.f;
    }
    float acc[MLP_BCHUNK];
#pragma unroll
    for (int b = 0; b < MLP_BCHUNK; ++b) acc[b] = 0.f;
    const float* wp = e.W + (size_t)r0 * td + k;
    float w8[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) w8[u] = (u < nr) ? __ldg(wp + (size_t)u * td) : 0.f;      // in flight across the barrier
    __syncthreads();
    for (int j0 = 0; j0 < nr; j0 += 8) {
        float wn[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) wn[u] = (j0 + 8 + u < nr) ? __ldg(wp + (size_t)(j0 + 8 + u) * td) : 0.f;
#pragma unroll
        for (int u = 0; u < 8; ++u) {
            if (j0 + u >= nr) break;
            const float w = w8[u];
            const float4* dj = reinterpret_cast<const float4*>(sd[j0 + u]);
#pragma unroll
            for (int q = 0; q < MLP_BCHUNK / 4; ++q) {
                const float4 d = dj[q];
                acc[4 * q] += d.x * w; acc[4 * q + 1] += d.y * w; acc[4 * q + 2] += d.z * w; acc[4 * q + 3] += d.w * w;
            }
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) w8[u] = wn[u];
    }
#pragma unroll
    for (int b = 0; b < MLP_BCHUNK; ++b)
        if (b < nb) atomicAdd(&ds[(size_t)(b0 + b) * td + k], acc[b]);
}

}  // namespace pidm
using namespace pidm;

extern "C" int pidm_time_embed_fwd(const long long* t, const float* W1, const float* b1, const float* W2,
                                   const float* b2, float* emb, float* h1, float* temb, float* silu_t, int B, int dim,
                                   int td, void* stream) {
    PIDM_REQUIRE(td <= 1024 && dim <= td && dim % 4 == 0 && td % 4 == 0 && dim >= 4, "time_embed: need 4<=dim<=td<=1024, dim and td multiples of 4");
    PIDM_CUDA(launch_plain(time_embed_fwd_kernel, dim3(B), dim3(td), (size_t)((dim + td) * sizeof(float)), (cudaStream_t)stream, t, W1, b1, W2, b2, emb, h1, temb,
                                                                                        silu_t, dim, td));
    PIDM_LAUNCH_CHECK("time_embed_fwd");
    return 0;
}

// workspace: float[2 * B * td] (dt | dh), written by stage 1 and read by stage 2.
// parts: bit 1 = stage 1 (activation gradients into the workspace), bit 0 = stage 2 (weight / bias gradients from the
// workspace, ACCUMULATED).  Stage 2 only feeds the optimizer: a caller may issue it on the stream of its other
// weight-gradient kernels, ordered after stage 1.
extern "C" int pidm_time_embed_bwd(const float* d_silu_t, const float* emb, const float* h1, const float* temb,
                                   const float* W2, float* dW1, float* db1, float* dW2, float* db2, float* workspace,
                                   int B, int dim, int td, int parts, void* stream) {
    PIDM_REQUIRE(td <= 1024 && dim <= td, "time_embed_bwd: need dim<=td<=1024");
    cudaStream_t st = (cudaStream_t)stream;
    float* dt = workspace;
    float* dh = workspace + (size_t)B * td;
    if (parts & 2)
        PIDM_CUDA(launch_plain(time_embed_bwd_act_kernel, dim3(B), dim3(td), (size_t)(td * sizeof(float)), st, d_silu_t, h1, temb,
                               W2, dt, dh, td));
    if (parts & 1)
        PIDM_CUDA(launch_plain(time_embed_bwd_wgrad_kernel, dim3(td), dim3(td), (size_t)0, st, (const float*)dt,
                               (const float*)dh, emb, h1, dW1, db1, dW2, db2, B, dim, td));
    PIDM_LAUNCH_CHECK("time_embed_bwd");
    return 0;
}

extern "C" int pidm_mlp_entry_size(void) { return (int)sizeof(MlpEntry); }

extern "C" int pidm_block_mlps_fwd(const void* table_dev, int n_entries, int max_rows, const float* silu_t, int B,
                                   int td, void* stream) {
    PIDM_REQUIRE(td <= MLP_TD_MAX && td % 32 == 0, "block_mlps: td must be a multiple of 32, <= %d", MLP_TD_MAX);
    size_t smem = (size_t)MLP_BCHUNK * (td + 1) * sizeof(float);
    dim3 grid(n_entries, ceil_div(max_rows, MLP_ROWS));
    PIDM_CUDA(allow_smem(block_mlps_fwd_kernel, 96 * 1024));
    PIDM_CUDA(launch_plain(block_mlps_fwd_kernel, dim3(grid), dim3(256), (size_t)(smem), (cudaStream_t)stream, (const MlpEntry*)table_dev, silu_t, B, td));
    PIDM_LAUNCH_CHECK("block_mlps_fwd");
    return 0;
}

// weight/bias grads accumulate into the table's dW/db pointers; d_silu_t is overwritten.
// parts: bit 0 = weight / bias gradients, bit 1 = input gradient (d_silu_t) -- the two halves are independent, so a
// caller can put the weight-gradient half on the stream of its other weight-gradient kernels.
extern "C" int pidm_block_mlps_bwd(const void* table_dev, int n_entries, int max_rows, const float* silu_t,
                                   float* d_silu_t, int B, int td, int parts, void* stream) {
    PIDM_REQUIRE(td <= MLP_TD_MAX && td % 32 == 0, "block_mlps: td must be a multiple of 32, <= %d", MLP_TD_MAX);
    cudaStream_t st = (cudaStream_t)stream;
    size_t smem = (size_t)MLP_BCHUNK * (td + 1) * sizeof(float);
    if (parts & 1) {
        dim3 grid(n_entries, ceil_div(max_rows, MLP_ROWS));
        PIDM_CUDA(allow_smem(block_mlps_wgrad_kernel, 96 * 1024));
        PIDM_CUDA(launch_plain(block_mlps_wgrad_kernel, dim3(grid), dim3(256), (size_t)(smem), st, (const MlpEntry*)table_dev, silu_t, B, td));
    }
    if (parts & 2) {
        PIDM_CUDA(cudaMemsetAsync(d_silu_t, 0, (size_t)B * td * sizeof(float), st));
        dim3 dgrid(n_entries, ceil_div(max_rows, MLP_DG_ROWS), ceil_div(B, MLP_BCHUNK));
        PIDM_CUDA(launch_plain(block_mlps_dgrad_kernel, dim3(dgrid), dim3(td), (size_t)(0), st, (const MlpEntry*)table_dev, d_silu_t, B, td));
    }
    PIDM_LAUNCH_CHECK("block_mlps_bwd");
    return 0;
}
