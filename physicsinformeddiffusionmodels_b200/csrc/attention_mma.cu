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
#include "common.cuh"
#include "mma_util.cuh"
#include "pidm.h"

namespace pidm {

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
    __nv_bfloat16* ring = reinterpret_cast<__nv_bfloat16*>(raw) + (size_t)h * (LC_STAGES * 2 * LW_TILE);
    float* sM = reinterpret_cast<float*>(raw + (size_t)LM_HEADS * LC_STAGES * 2 * LW_TILE * 2) + h * 2 * LM_D;
    float* sZi = sM + LM_D;
    const int n_begin = chunk * chunk_px, n_end = min(N, n_begin + chunk_px);
    const int n_tiles = (n_end - n_begin) / 32;
    const size_t pix0 = (size_t)b * N + n_begin;
    const __nv_bfloat16* wsrc = qkv + pix0 * 3 * LM_HID + (MODE == 0 ? LM_HID : 0) + h * LM_D;
    const __nv_bfloat16* vsrc = (MODE == 0) ? qkv + pix0 * 3 * LM_HID + 2 * LM_HID + h * LM_D : dout + pix0 * LM_HID + h * LM_D;
    const size_t vstride = (MODE == 0) ? 3 * LM_HID : LM_HID;
    auto issue = [&](int it) {
        if (it < n_tiles) {
            __nv_bfloat16* buf = ring + (size_t)(it % LC_STAGES) * 2 * LW_TILE;
            lw_issue<32>(buf, wsrc + (size_t)it * 32 * 3 * LM_HID, 3 * LM_HID, lane);
            lw_issue<32>(buf + LW_TILE, vsrc + (size_t)it * 32 * vstride, vstride, lane);
        }
        cp_commit();                               // always one group per call: keeps wait_group counts uniform
    };
#pragma unroll
    for (int s = 0; s < LC_STAGES; ++s) issue(s);
    if (MODE == 0) {                               // lane = channel d of this head: combine the per-chunk statistics
        const int c = h * LM_D + lane;
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
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int k = 0; k < 4; ++k) acc[i][j][k] = 0.f;
    for (int it = 0; it < n_tiles; ++it) {
        cp_wait<LC_STAGES - 1>();
        __syncwarp();
        __nv_bfloat16* Ws = ring + (size_t)(it % LC_STAGES) * 2 * LW_TILE;
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
        __syncwarp();                              // every lane is done with this stage
        issue(it + LC_STAGES);
    }
    const int g = lane >> 2, t = lane & 3;
    float* cb = ctx + ((size_t)b * LM_HEADS + h) * LM_D * LM_D;
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const int d = mt * 16 + g + half * 8;
            const float f = (MODE == 0) ? sZi[d] / (float)N : 1.f;
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                const int e = nt * 8 + 2 * t;
                atomicAdd(cb + d * LM_D + e, acc[mt][nt][half * 2] * f);
                atomicAdd(cb + d * LM_D + e + 1, acc[mt][nt][half * 2 + 1] * f);
            }
        }
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
    __nv_bfloat16* ring = reinterpret_cast<__nv_bfloat16*>(raw) + (size_t)h * (LO_STAGES * LW_TILE);
    const int n_begin = chunk * chunk_px, n_end = min(N, n_begin + chunk_px);
    const int n_tiles = (n_end - n_begin) / 32;
    const size_t pix0 = (size_t)b * N + n_begin;
    const __nv_bfloat16* qsrc = qkv + pix0 * 3 * LM_HID + h * LM_D;
    __nv_bfloat16* odst = out + pix0 * LM_HID + h * LM_D;
    auto issue = [&](int it) {
        if (it < n_tiles) lw_issue<32>(ring + (size_t)(it % LO_STAGES) * LW_TILE, qsrc + (size_t)it * 32 * 3 * LM_HID, 3 * LM_HID, lane);
        cp_commit();
    };
#pragma unroll
    for (int s = 0; s < LO_STAGES; ++s) issue(s);
    // B[k = d][n = e] = ctx[d][e], straight from global fp32
    const float* ch = ctx + ((size_t)b * LM_HEADS + h) * LM_D * LM_D;
    uint32_t bf[2][4][2];
#pragma unroll
    for (int ks = 0; ks < 2; ++ks)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) frag_b_global<true>(bf[ks][nt], ch, ks * 16, nt * 8, lane);
    const int g = lane >> 2, t = lane & 3;
    for (int it = 0; it < n_tiles; ++it) {
        cp_wait<LO_STAGES - 1>();
        __syncwarp();
        __nv_bfloat16* Qs = ring + (size_t)(it % LO_STAGES) * LW_TILE;
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
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int k = 0; k < 4; ++k) c[i][k] = 0.f;
#pragma unroll
            for (int ks = 0; ks < 2; ++ks)
#pragma unroll
                for (int nt = 0; nt < 4; ++nt) mma_bf16(c[nt], a[mt][ks], bf[ks][nt][0], bf[ks][nt][1]);
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                __nv_bfloat16* o = Qs + (size_t)(mt * 16 + g) * LW_PITCH + nt * 8 + 2 * t;
                *reinterpret_cast<uint32_t*>(o) = pack_bf16(c[nt][0], c[nt][1]);
                *reinterpret_cast<uint32_t*>(o + 8 * LW_PITCH) = pack_bf16(c[nt][2], c[nt][3]);
            }
        }
        __syncwarp();
        lw_store<32>(odst + (size_t)it * 32 * LM_HID, LM_HID, Qs, lane);
        __syncwarp();
        issue(it + LO_STAGES);
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
    __nv_bfloat16* ring = reinterpret_cast<__nv_bfloat16*>(raw) + (size_t)h * (LB_STAGES * LB_TILE);
    float* sM = reinterpret_cast<float*>(raw + (size_t)LM_HEADS * LB_STAGES * LB_TILE * 2) + h * 3 * LM_D;
    float* sZi = sM + LM_D;
    float* scd = sZi + LM_D;
    const int n_begin = chunk * chunk_px, n_end = min(N, n_begin + chunk_px);
    const int n_tiles = (n_end - n_begin) / LB_ROWS;
    const size_t pix0 = (size_t)b * N + n_begin;
    const __nv_bfloat16* qsrc = qkv + pix0 * 3 * LM_HID + h * LM_D;
    const __nv_bfloat16* gsrc = dout + pix0 * LM_HID + h * LM_D;
    __nv_bfloat16* ddst = dqkv + pix0 * 3 * LM_HID + h * LM_D;
    auto issue = [&](int it) {
        if (it < n_tiles) {
            __nv_bfloat16* buf = ring + (size_t)(it % LB_STAGES) * LB_TILE;
            const __nv_bfloat16* q = qsrc + (size_t)it * LB_ROWS * 3 * LM_HID;
            lw_issue<LB_ROWS>(buf, gsrc + (size_t)it * LB_ROWS * LM_HID, LM_HID, lane);
            lw_issue<LB_ROWS>(buf + LB_ROWS * LW_PITCH, q, 3 * LM_HID, lane);
            lw_issue<LB_ROWS>(buf + 2 * LB_ROWS * LW_PITCH, q + LM_HID, 3 * LM_HID, lane);
            lw_issue<LB_ROWS>(buf + 3 * LB_ROWS * LW_PITCH, q + 2 * LM_HID, 3 * LM_HID, lane);
        }
        cp_commit();
    };
#pragma unroll
    for (int s = 0; s < LB_STAGES; ++s) issue(s);
    const float* cg = ctx + ((size_t)b * LM_HEADS + h) * LM_D * LM_D;
    const float* dg = dctx + ((size_t)b * LM_HEADS + h) * LM_D * LM_D;
    sM[lane] = kmax[(size_t)b * LM_HID + h * LM_D + lane];
    sZi[lane] = kzinv[(size_t)b * LM_HID + h * LM_D + lane];
    {
        float s = 0.f;                 // cd[d] = sum_e dctx[d][e] ctx[d][e]   (lane = d)
#pragma unroll
        for (int e = 0; e < LM_D; e += 4) {
            const float4 x = *reinterpret_cast<const float4*>(dg + lane * LM_D + e);
            const float4 y = *reinterpret_cast<const float4*>(cg + lane * LM_D + e);
            s += x.x * y.x + x.y * y.y + x.z * y.z + x.w * y.w;
        }
        scd[lane] = s;
    }
    uint32_t bc[2][4][2], bd[2][4][2], bt[2][4][2];
#pragma unroll
    for (int ks = 0; ks < 2; ++ks)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
            frag_b_global<false>(bc[ks][nt], cg, ks * 16, nt * 8, lane);      // B[k=e][n=d] = ctx[d][e]
            frag_b_global<false>(bd[ks][nt], dg, ks * 16, nt * 8, lane);      // B[k=e][n=d] = dctx[d][e]
            frag_b_global<true>(bt[ks][nt], dg, ks * 16, nt * 8, lane);       // B[k=d][n=e] = dctx[d][e]
        }
    __syncwarp();
    const int g = lane >> 2, t = lane & 3;
    const float invN = 1.f / (float)N;
    for (int it = 0; it < n_tiles; ++it) {
        cp_wait<LB_STAGES - 1>();
        __syncwarp();
        __nv_bfloat16* buf = ring + (size_t)(it % LB_STAGES) * LB_TILE;
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
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int k = 0; k < 4; ++k) { cq[i][k] = 0.f; ck[i][k] = 0.f; cv[i][k] = 0.f; }
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
            dot += __shfl_xor_sync(0xffffffffu, dot, 1);
            dot += __shfl_xor_sync(0xffffffffu, dot, 2);
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
        __syncwarp();
        issue(it + LB_STAGES);
    }
}

constexpr size_t LA_CTX_SMEM = (size_t)LM_HEADS * LC_STAGES * 2 * LW_TILE * 2 + (size_t)LM_HEADS * 2 * LM_D * 4;
constexpr size_t LA_OUT_SMEM = (size_t)LM_HEADS * LO_STAGES * LW_TILE * 2;
constexpr size_t LA_BWD_SMEM = (size_t)LM_HEADS * LB_STAGES * LB_TILE * 2 + (size_t)LM_HEADS * 3 * LM_D * 4;

// entry points used by attention.cu for the bf16 / 8-head case: about two CTAs per SM
int la_mma_chunk_px(int B, int N) { return chunk_px(B, N, 2); }
int la_mma_ctx(int mode, const void* qkv, const void* dout, const float* part, int n_stat_chunks, float* kmax,
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
int la_mma_out(const void* qkv, const float* ctx, void* out, int B, int N, float scale, cudaStream_t st) {
    const int cpx = chunk_px(B, N, 2);
    dim3 grid((N + cpx - 1) / cpx, B);
    PIDM_CUDA(allow_smem(la_out_mma_kernel, LA_OUT_SMEM));
    PIDM_CUDA(launch_plain(la_out_mma_kernel, dim3(grid), dim3(256), (size_t)(LA_OUT_SMEM), st, (const __nv_bfloat16*)qkv, ctx, (__nv_bfloat16*)out, N, cpx, scale));
    PIDM_LAUNCH_CHECK("la_out_mma");
    return 0;
}
int la_mma_bwd(const void* qkv, const void* dout, const float* ctx, const float* dctx, const float* kmax,
               const float* kzinv, void* dqkv, int B, int N, float scale, cudaStream_t st) {
    const int cpx = chunk_px(B, N, 2);
    dim3 grid((N + cpx - 1) / cpx, B);
    PIDM_CUDA(allow_smem(la_bwd_mma_kernel, LA_BWD_SMEM));
    PIDM_CUDA(launch_plain(la_bwd_mma_kernel, dim3(grid), dim3(256), (size_t)(LA_BWD_SMEM), st, (const __nv_bfloat16*)qkv, (const __nv_bfloat16*)dout, ctx, dctx, kmax,
                                                       kzinv, (__nv_bfloat16*)dqkv, N, cpx, scale));
    PIDM_LAUNCH_CHECK("la_bwd_mma");
    return 0;
}

}  // namespace pidm
