// The whole linear-attention block at the full-resolution levels of the U-Net (C = 32 channels, 8 heads x 32;
// reference unet_model.py:275-297 and the Residual wrapper's `+ x`):
//   y = x + b_out + to_out(attention(to_qkv(xn))),  to_qkv 1x1 32 -> 768 without bias, to_out 1x1 256 -> 32 with bias.
//
// At 64x64 the qkv tensor is 24x larger than the tensor it is projected from (768 vs 32 channels) and the attention
// output 8x (256): writing them and streaming them back through the statistics / context / output / backward kernels
// was ~1.2 GB of HBM traffic per layer.  Here every warp (one head) recomputes its q / k / v slices on the tensor cores
// from the 64-byte pixel rows of the normalised input xn -- a 32x32x32 mma.sync product per 32 pixels -- and multiplies
// its output tile by its 32 columns of W_out on chip, so that forward reads xn and x and writes y only.  Backward
// recomputes dout_h = dy W_out[:, 32h:32h+32] per head from the 32-channel dy, in two passes over (xn, dy): one
// multiplies dq | dk | dv by W and writes dxn, the other multiplies them by xn into the to_qkv weight gradient and
// accumulates the to_out weight gradient; neither the [B, N, 768] dqkv nor the [B, N, 256] dout is written.
// All intermediate tiles stay in registers: accumulator fragments are converted to A fragments directly and to
// transposed (K-major) fragments with movmatrix; only xn / dy tiles, the W_out slices and the cross-head partial sums
// touch shared memory.  The unfused path differs by the bf16 rounding of the q, k, v and attention output it
// materialises.
#include "common.cuh"
#include "mma_util.cuh"
#include "pidm.h"

namespace pidm {

constexpr int LF_C = 32;                       // channels of xn

// B fragments of a 32-row block of the K-major projection weights W[n][c] (bf16): B[k = c][n] = W[n][c]
__device__ __forceinline__ void load_w_frags(uint32_t (&w)[2][4][2], const __nv_bfloat16* __restrict__ Wrows, int lane) {
    const int g = lane >> 2, t = lane & 3;
#pragma unroll
    for (int ks = 0; ks < 2; ++ks)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
            const uint32_t* row = reinterpret_cast<const uint32_t*>(Wrows + (size_t)(nt * 8 + g) * LF_C + ks * 16 + 2 * t);
            w[ks][nt][0] = __ldg(row);
            w[ks][nt][1] = __ldg(row + 4);
        }
}
// A fragments of MT 16-pixel row blocks of an xn tile [rows][LW_PITCH]
template <int MT>
__device__ __forceinline__ void load_x_frags(uint32_t (&a)[MT][2][4], const __nv_bfloat16* Xs, int lane) {
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) frag_a_rowmajor(a[mt][ks], Xs, LW_PITCH, mt * 16, ks * 16, lane);
}
// c[mt][nt] = xn_tile(mt) * W^T in fp32.  (The unfused path rounds q, k, v to bf16 when it materialises them; the
// fused path keeps the fp32 products -- closer to the fp32 reference, and conversions share the XU pipe with exp.)
template <int MT>
__device__ __forceinline__ void project(float (&c)[MT][4][4], const uint32_t (&a)[MT][2][4], const uint32_t (&w)[2][4][2]) {
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
            zero(c[mt][nt]);
#pragma unroll
            for (int ks = 0; ks < 2; ++ks) mma_bf16(c[mt][nt], a[mt][ks], w[ks][nt][0], w[ks][nt][1]);
        }
}
// per-thread column constants: column (nt, j) = nt*8 + 2*(lane&3) + j
__device__ __forceinline__ void load_cols(float (&v)[8], const float* __restrict__ src, int lane) {
    const int t = lane & 3;
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) { v[nt * 2] = src[nt * 8 + 2 * t]; v[nt * 2 + 1] = src[nt * 8 + 2 * t + 1]; }
}

// ---- pass 1: per-chunk column maxima of k = xn Wk^T (the exp-sums are accumulated by the context kernel) -------------
constexpr int LFS_STAGES = 2;      // a tile is consumed into registers at once: one tile of look-ahead is enough,
                                   // and 41 KB per CTA lets five CTAs share an SM
__global__ void __launch_bounds__(256) laf_kmax_kernel(const __nv_bfloat16* __restrict__ xn,
                                                       const __nv_bfloat16* __restrict__ W, float* __restrict__ part,
                                                       int N, int rows_per_chunk) {
    pdl_trigger();
    pdl_wait();
    extern __shared__ __align__(16) unsigned char raw[];
    const int b = blockIdx.y, chunk = blockIdx.x, lane = threadIdx.x & 31, h = threadIdx.x >> 5;
    const int n_begin = chunk * rows_per_chunk, n_end = min(N, n_begin + rows_per_chunk);
    const int n_tiles = (n_end - n_begin) / 32;
    const __nv_bfloat16* xsrc = xn + ((size_t)b * N + n_begin) * LF_C;
    const CpRing<LFS_STAGES, LW_TILE> ring{reinterpret_cast<__nv_bfloat16*>(raw) + (size_t)h * (LFS_STAGES * LW_TILE),
                                           n_tiles};
    auto load = [&](__nv_bfloat16* buf, int it) {
        lw_issue<32>(buf, xsrc + (size_t)it * 32 * LF_C, LF_C, lane);
    };
    ring.prime(load);
    uint32_t wk[2][4][2];
    load_w_frags(wk, W + (size_t)(LM_HID + h * DH) * LF_C, lane);
    float m[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) m[i] = -INFINITY;
    for (int it = 0; it < n_tiles; ++it) {
        uint32_t ax[2][2][4];
        load_x_frags<2>(ax, ring.wait(it, load), lane);
        ring.release(it, load);
        float ck[2][4][4];
        project<2>(ck, ax, wk);
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
            for (int j = 0; j < 2; ++j)
                m[nt * 2 + j] = fmaxf(fmaxf(m[nt * 2 + j], fmaxf(ck[0][nt][j], ck[0][nt][2 + j])),
                                      fmaxf(ck[1][nt][j], ck[1][nt][2 + j]));
    }
#pragma unroll
    for (int off = 4; off < 32; off <<= 1)
#pragma unroll
        for (int i = 0; i < 8; ++i) m[i] = fmaxf(m[i], __shfl_xor_sync(0xffffffffu, m[i], off));
    if (lane < 4) {
        float* o = part + ((size_t)b * gridDim.x + chunk) * LM_HID + h * DH;
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
            for (int j = 0; j < 2; ++j) o[nt * 8 + 2 * lane + j] = m[nt * 2 + j];
    }
}

// ctx[b][h][d][:] *= 1 / Z[b][h][d]  and  kzinv = 1 / Z, after the context kernel has accumulated both
__global__ void laf_finalize_kernel(float* __restrict__ ctx, float* __restrict__ kzinv, int n_rows) {
    pdl_trigger();
    pdl_wait();
    const int row = blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= n_rows) return;
    const float zi = 1.f / kzinv[row];
    ctx[(size_t)row * DH + lane] *= zi;
    __syncwarp();
    if (lane == 0) kzinv[row] = zi;
}

// ---- to_out projection: the block output y = x + b + sum_h out_h W_out[:, 32h:32h+32]^T -------------------------------
// The kernels below never see `out` or `dout` [B, N, 256]: the forward multiplies each head's out tile by its 32-column
// slice of W_out and sums the eight partials, and backward recomputes dout_h = dy W_out[:, 32h:32h+32] from the
// 32-channel dy tile.  Every warp keeps its slice Wo_h[c][e] = W_out[c][32h + e] (packed forward to_out weights
// [32][256]) in shared memory; ldmatrix reads it in both orientations.
constexpr int LFP_WO_TILE = LF_C * LW_PITCH;                        // one head's W_out slice [32 c][LW_PITCH]

// c[16 px][32 e] = dy[16 px][32 c] Wo_h[c][e]   (dy as A fragments)
__device__ __forceinline__ void lfp_dout_acc(float (&c)[4][4], const uint32_t (&ady)[2][4], const __nv_bfloat16* Wo, int lane) {
    zero(c);
#pragma unroll
    for (int kc = 0; kc < 2; ++kc)
#pragma unroll
        for (int np = 0; np < 2; ++np) {
            uint32_t bw[4];
            frag_b_krows(bw, Wo, LW_PITCH, kc * 16, np * 16, lane);
            mma_bf16(c[2 * np], ady[kc], bw[0], bw[1]);
            mma_bf16(c[2 * np + 1], ady[kc], bw[2], bw[3]);
        }
}
// dout_h of the 16-pixel dy tile dyt [16][LW_PITCH], as the bf16 A fragments a materialised bf16 dout would give
__device__ __forceinline__ void lfp_dout(uint32_t (&ag)[2][4], const __nv_bfloat16* dyt, const __nv_bfloat16* Wo, int lane) {
    uint32_t ady[2][4];
    frag_a_rowmajor(ady[0], dyt, LW_PITCH, 0, 0, lane);
    frag_a_rowmajor(ady[1], dyt, LW_PITCH, 0, 16, lane);
    float c[4][4];
    lfp_dout_acc(c, ady, Wo, lane);
    c_to_a(ag, c);
}

// ---- context (MODE 0) / dcontext (MODE 1) --------------------------------------------------------------------------
//   MODE 0: ctx[h][d][e]  += sum_n exp(k[n,d] - M_d) v[n,e]          k, v projected from xn
//   MODE 1: dctx[h][d][e] += sum_n softmax_d(q[n,:])[d] s dout[n,e]  q projected from xn, dout recomputed from the
//           streamed dy
template <int MODE>
struct LfcCfg {
    static constexpr int STAGES = MODE == 0 ? 4 : 2;                       // tiles are consumed into registers at once
    static constexpr int STAGE_ELEMS = MODE == 0 ? LW_TILE : 2 * LW_TILE;  // xn tile (| dy tile)
    static constexpr size_t SMEM_BASE = (size_t)LM_HEADS * STAGES * STAGE_ELEMS * 2 + (size_t)LM_HEADS * 2 * DH * 4;
    static constexpr size_t SMEM = SMEM_BASE + (MODE == 1 ? (size_t)LM_HEADS * LFP_WO_TILE * 2 : 0);
};
template <int MODE>
__global__ void __launch_bounds__(256, 2) laf_ctx_kernel(const __nv_bfloat16* __restrict__ xn, const __nv_bfloat16* __restrict__ W,
                                                      const __nv_bfloat16* __restrict__ dy, const float* __restrict__ part,
                                                      int n_stat_chunks, float* __restrict__ kmax, float* __restrict__ kzinv,
                                                      float* __restrict__ ctx, int N, int chunk_px, float scale,
                                                      const __nv_bfloat16* __restrict__ w_out) {
    pdl_trigger();
    pdl_wait();
    extern __shared__ __align__(16) unsigned char raw[];
    constexpr int LFC_STAGES = LfcCfg<MODE>::STAGES, LFC_STAGE_ELEMS = LfcCfg<MODE>::STAGE_ELEMS;
    const int b = blockIdx.y, chunk = blockIdx.x, lane = threadIdx.x & 31, h = threadIdx.x >> 5;
    float* sM = reinterpret_cast<float*>(raw + (size_t)LM_HEADS * LFC_STAGES * LFC_STAGE_ELEMS * 2) + h * 2 * DH;
    __nv_bfloat16* Wo = reinterpret_cast<__nv_bfloat16*>(raw + LfcCfg<MODE>::SMEM_BASE) + h * LFP_WO_TILE;   // MODE 1
    const int n_begin = chunk * chunk_px, n_end = min(N, n_begin + chunk_px);
    const int n_tiles = (n_end - n_begin) / 32;
    const size_t pix0 = (size_t)b * N + n_begin;
    const __nv_bfloat16* xsrc = xn + pix0 * LF_C;
    const __nv_bfloat16* gsrc = (MODE == 1) ? dy + pix0 * LF_C : nullptr;
    const CpRing<LFC_STAGES, LFC_STAGE_ELEMS> ring{reinterpret_cast<__nv_bfloat16*>(raw) +
                                                       (size_t)h * (LFC_STAGES * LFC_STAGE_ELEMS),
                                                   n_tiles};
    auto load = [&](__nv_bfloat16* buf, int it) {
        lw_issue<32>(buf, xsrc + (size_t)it * 32 * LF_C, LF_C, lane);
        if (MODE == 1) lw_issue<32>(buf + LW_TILE, gsrc + (size_t)it * 32 * LF_C, LF_C, lane);
    };
    if (MODE == 1) ring.prologue([&] { lw_issue<32>(Wo, w_out + h * DH, LM_HID, lane); });    // this head's W_out slice
    ring.prime(load);
    uint32_t w0[2][4][2], w1[2][4][2];               // MODE 0: Wk, Wv   MODE 1: Wq, (unused)
    load_w_frags(w0, W + (size_t)((MODE == 0 ? LM_HID : 0) + h * DH) * LF_C, lane);
    if (MODE == 0) load_w_frags(w1, W + (size_t)(2 * LM_HID + h * DH) * LF_C, lane);
    float Mc[8];
    float zacc[8];
    zero(zacc);
    if (MODE == 0) {                               // lane = channel d of this head: combine the per-chunk maxima
        const int c = h * DH + lane;
        float M = -INFINITY;
        for (int i = 0; i < n_stat_chunks; ++i) M = fmaxf(M, part[((size_t)b * n_stat_chunks + i) * LM_HID + c]);
        sM[lane] = M;
        if (chunk == 0) kmax[(size_t)b * LM_HID + c] = M;
        __syncwarp();
        load_cols(Mc, sM, lane);
    }
    float acc[2][4][4];
    zero(acc);
    for (int it = 0; it < n_tiles; ++it) {
        const __nv_bfloat16* buf = ring.wait(it, load);
        uint32_t ax[2][2][4];
        load_x_frags<2>(ax, buf, lane);
        uint32_t bv[2][4][2];                         // B fragments [k = px][n = e] per 16-pixel step
        if (MODE == 1) {                              // dout accumulator [px][e] -> transposed 8x8 blocks, as v in MODE 0
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) {
                uint32_t ady[2][4];
                frag_a_rowmajor(ady[0], buf + LW_TILE, LW_PITCH, mt * 16, 0, lane);
                frag_a_rowmajor(ady[1], buf + LW_TILE, LW_PITCH, mt * 16, 16, lane);
                float cd[4][4];
                lfp_dout_acc(cd, ady, Wo, lane);
                c_to_bt(bv[mt], cd);
            }
        }
        ring.release(it, load);                    // the tile is in registers
        float cw[2][4][4];
        project<2>(cw, ax, w0);
        if (MODE == 0) {
#pragma unroll
            for (int mt = 0; mt < 2; ++mt)
#pragma unroll
                for (int nt = 0; nt < 4; ++nt)
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        cw[mt][nt][i] = __expf(cw[mt][nt][i] - Mc[nt * 2 + (i & 1)]);
                        zacc[nt * 2 + (i & 1)] += cw[mt][nt][i];
                    }
            float cv[2][4][4];
            project<2>(cv, ax, w1);
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) c_to_bt(bv[mt], cv[mt]);
        } else {
            frag_softmax(cw[0], scale);
            frag_softmax(cw[1], scale);
        }
        // A[d][px] = w~[px][d]^T: transposed 8x8 blocks of the accumulator fragments
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {           // 16-pixel k step
#pragma unroll
            for (int md = 0; md < 2; ++md) {       // 16-channel m tile
                uint32_t a[4];
                c_to_at(a, cw[mt], md);
#pragma unroll
                for (int ne = 0; ne < 4; ++ne) mma_bf16(acc[md][ne], a, bv[mt][ne][0], bv[mt][ne][1]);
            }
        }
    }
    if (MODE == 0) {                               // Z_d = sum_n exp(k[n,d] - M_d): column sums over the 8 row-lanes
#pragma unroll
        for (int off = 4; off < 32; off <<= 1)
#pragma unroll
            for (int i = 0; i < 8; ++i) zacc[i] += __shfl_xor_sync(0xffffffffu, zacc[i], off);
        if (lane < 4) {
#pragma unroll
            for (int nt = 0; nt < 4; ++nt)
#pragma unroll
                for (int j = 0; j < 2; ++j)
                    atomicAdd(kzinv + (size_t)b * LM_HID + h * DH + nt * 8 + 2 * lane + j, zacc[nt * 2 + j]);
        }
    }
    // MODE 0: 1 / Z_d is applied by laf_finalize_kernel
    ctx_atomic_add(ctx + ((size_t)b * LM_HEADS + h) * DH * DH, acc,
                   [&](int) { return (MODE == 0) ? 1.f / (float)N : 1.f; }, lane);
}

// ---- y = x + b + sum_h out_h Wo_h^T,  out[n,h,e] = sum_d softmax_d(q[n,:])[d] * s * ctx[h][d][e],  q projected from xn
// The warps share one xn ring and step through the tiles together; each leaves its fp32 [32 px][32] partial in shared
// memory, and after a CTA barrier every thread sums two columns of two rows over the eight heads, adds the bias and the
// residual and writes y once.
constexpr int LFO_STAGES = 3;      // 68 KB per CTA; 112 registers: two CTAs per SM
constexpr int LFO_R_PITCH = LF_C + 8;                              // fp32 partial rows: conflict-free float2 stores
constexpr size_t LAF_OUT_SMEM = (size_t)LFO_STAGES * LW_TILE * 2 + (size_t)LM_HEADS * LFP_WO_TILE * 2 +
                                (size_t)LM_HEADS * 32 * LFO_R_PITCH * 4;
__global__ void __launch_bounds__(256) laf_out_kernel(const __nv_bfloat16* __restrict__ xn, const __nv_bfloat16* __restrict__ W,
                                                      const float* __restrict__ ctx, __nv_bfloat16* __restrict__ y, int N,
                                                      int chunk_px, float scale, const __nv_bfloat16* __restrict__ w_out,
                                                      const float* __restrict__ b_out,
                                                      const __nv_bfloat16* __restrict__ residual) {
    pdl_trigger();
    pdl_wait();
    extern __shared__ __align__(16) unsigned char raw[];
    const int b = blockIdx.y, chunk = blockIdx.x, lane = threadIdx.x & 31, h = threadIdx.x >> 5;
    __nv_bfloat16* tiles = reinterpret_cast<__nv_bfloat16*>(raw);
    __nv_bfloat16* Wo = tiles + LFO_STAGES * LW_TILE + h * LFP_WO_TILE;
    float* R = reinterpret_cast<float*>(tiles + LFO_STAGES * LW_TILE + LM_HEADS * LFP_WO_TILE);
    const int n_begin = chunk * chunk_px, n_end = min(N, n_begin + chunk_px);
    const int n_tiles = (n_end - n_begin) / 32;
    const size_t pix0 = (size_t)b * N + n_begin;
    const __nv_bfloat16* xsrc = xn + pix0 * LF_C;
    const CpRing<LFO_STAGES, LW_TILE, true> ring{tiles, n_tiles};
    auto load = [&](__nv_bfloat16* buf, int it) {
        if (h == 0) lw_issue<32>(buf, xsrc + (size_t)it * 32 * LF_C, LF_C, lane);
    };
    ring.prologue([&] { lw_issue<32>(Wo, w_out + h * DH, LM_HID, lane); });   // this head's W_out slice
    ring.prime(load);
    uint32_t wq[2][4][2];
    load_w_frags(wq, W + (size_t)(h * DH) * LF_C, lane);
    uint32_t bf[2][4][2];
    frags_b_global<true>(bf, ctx + ((size_t)b * LM_HEADS + h) * DH * DH, lane);
    const int g = lane >> 2, t = lane & 3;
    const int rrow = threadIdx.x >> 4, rcol = (threadIdx.x & 15) * 2;     // the y elements this thread sums
    const float2 bias = make_float2(b_out[rcol], b_out[rcol + 1]);
    float* Rw = R + h * 32 * LFO_R_PITCH;
    for (int it = 0; it < n_tiles; ++it) {
        uint32_t ax[2][2][4];
        load_x_frags<2>(ax, ring.wait(it, load), lane);  // its CTA barrier also frees R
        __nv_bfloat162 res[2];                     // the residual elements this thread adds, loaded early
#pragma unroll
        for (int rh = 0; rh < 2; ++rh)
            res[rh] = *reinterpret_cast<const __nv_bfloat162*>(residual + (pix0 + (size_t)it * 32 + rrow + rh * 16) * LF_C + rcol);
        float cq[2][4][4];
        project<2>(cq, ax, wq);
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
            frag_softmax(cq[mt], scale);
            uint32_t a[2][4];
            c_to_a(a, cq[mt]);
            float c[4][4];
            zero(c);
#pragma unroll
            for (int ks = 0; ks < 2; ++ks)
#pragma unroll
                for (int nt = 0; nt < 4; ++nt) mma_bf16(c[nt], a[ks], bf[ks][nt][0], bf[ks][nt][1]);
            c_to_a(a, c);                          // yh[16 px][32 c] = out_h Wo_h^T: B[k = e][n = c] = Wo_h[c][e]
            float yh[4][4];
            zero(yh);
#pragma unroll
            for (int ke = 0; ke < 2; ++ke)
#pragma unroll
                for (int np = 0; np < 2; ++np) {
                    uint32_t bw[4];
                    frag_b_nrows(bw, Wo, LW_PITCH, np * 16, ke * 16, lane);
                    mma_bf16(yh[2 * np], a[ke], bw[0], bw[1]);
                    mma_bf16(yh[2 * np + 1], a[ke], bw[2], bw[3]);
                }
#pragma unroll
            for (int nt = 0; nt < 4; ++nt)
#pragma unroll
                for (int half = 0; half < 2; ++half)
                    *reinterpret_cast<float2*>(Rw + (mt * 16 + g + half * 8) * LFO_R_PITCH + nt * 8 + 2 * t) =
                        make_float2(yh[nt][half * 2], yh[nt][half * 2 + 1]);
        }
        __syncthreads();                           // the eight head partials of this tile are in R
#pragma unroll
        for (int rh = 0; rh < 2; ++rh) {
            const int row = rrow + rh * 16;
            const size_t pix = pix0 + (size_t)it * 32 + row;
            const float2 x = __bfloat1622float2(res[rh]);
            float sx = x.x + bias.x, sy = x.y + bias.y;
#pragma unroll
            for (int w = 0; w < LM_HEADS; ++w) {
                const float2 v = *reinterpret_cast<const float2*>(R + (w * 32 + row) * LFO_R_PITCH + rcol);
                sx += v.x;
                sy += v.y;
            }
            *reinterpret_cast<uint32_t*>(y + pix * LF_C + rcol) = pack_bf16(sx, sy);
        }
    }
}

// ---- backward: dq | dk | dv per 16-pixel tile from xn, dout, ctx, dctx and the saved column statistics ----------------
//   dq = s p (dp - sum_d p dp),  dp = dout ctx^T,  p = softmax_d(q)
//   dk = k~ (dk~ - cd),          dk~ = (v / N) dctx^T,  k~ = exp(k - M) Zinv,  cd[d] = sum_e dctx[d][e] ctx[d][e]
//   dv = (k~ dctx) / N
// Neither pass below writes dq, dk or dv: the input-gradient pass multiplies them by W on the spot, the weight-gradient
// pass multiplies them by xn.  They enter those products as bf16 tensor-core operands, like every other mma operand.
constexpr int LFB_ROWS = 16;
constexpr int LFB_STAGES = 4;
constexpr int LFB_TILE = LFB_ROWS * LW_PITCH;                       // one [16 px][32] bf16 tile

struct LfbTile {                     // what every head needs from one 16-pixel tile (A fragments of xn and of dout)
    uint32_t ax[1][2][4], ag[2][4];
};
// dq (fp32 accumulator fragment [16 px][32 d])
__device__ __forceinline__ void lfb_dq(float (&dq)[4][4], const LfbTile& tl, const uint32_t (&wq)[2][4][2],
                                       const uint32_t (&bc)[2][4][2], float scale) {
    float c1[1][4][4], c2[4][4];
    project<1>(c1, tl.ax, wq);
    frag_softmax(c1[0], 1.f);
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
        zero(c2[nt]);
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) mma_bf16(c2[nt], tl.ag[ks], bc[ks][nt][0], bc[ks][nt][1]);
    }
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        float dot = 0.f;
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
            dot += c1[0][nt][half * 2] * c2[nt][half * 2] + c1[0][nt][half * 2 + 1] * c2[nt][half * 2 + 1];
        dot = quad_sum(dot);
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
            for (int j = 0; j < 2; ++j) dq[nt][half * 2 + j] = scale * c1[0][nt][half * 2 + j] * (c2[nt][half * 2 + j] - dot);
    }
}
// dk and dv (fp32 accumulator fragments [16 px][32 d])
__device__ __forceinline__ void lfb_dkdv(float (&dk)[4][4], float (&dv)[4][4], const uint32_t (&ax)[1][2][4],
                                         const uint32_t (&wk)[2][4][2], const uint32_t (&wv)[2][4][2],
                                         const uint32_t (&bd)[2][4][2], const uint32_t (&bt)[2][4][2],
                                         const float (&Mc)[8], const float (&Zc)[8], const float (&cdc)[8], float invN) {
    float c1[1][4][4];
    uint32_t a[2][4];
    project<1>(c1, ax, wv);
    c_to_a(a, c1[0]);
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {               // dk~ N = v dctx^T
        zero(dk[nt]);
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) mma_bf16(dk[nt], a[ks], bd[ks][nt][0], bd[ks][nt][1]);
    }
    project<1>(c1, ax, wk);
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            c1[0][nt][i] = __expf(c1[0][nt][i] - Mc[nt * 2 + (i & 1)]) * Zc[nt * 2 + (i & 1)];
            dk[nt][i] = c1[0][nt][i] * (dk[nt][i] * invN - cdc[nt * 2 + (i & 1)]);
        }
    c_to_a(a, c1[0]);
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
        zero(dv[nt]);
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) mma_bf16(dv[nt], a[ks], bt[ks][nt][0], bt[ks][nt][1]);
#pragma unroll
        for (int i = 0; i < 4; ++i) dv[nt][i] *= invN;
    }
}
// cd as per-thread column constants, through a 32-float shared scratch
__device__ __forceinline__ void lfb_cd(float (&cdc)[8], float* scd, const float* __restrict__ cg, const float* __restrict__ dg,
                                       int lane) {
    scd[lane] = ctx_dot_row(cg, dg, lane);
    __syncwarp();
    load_cols(cdc, scd, lane);
}

// ---- pass A (input gradient): dxn = sum_h dq_h Wq_h + dk_h Wk_h + dv_h Wv_h -----------------------------------------
// The eight warps (= heads) of a CTA step through the same 16-pixel tiles, sharing one xn tile.  A warp multiplies its
// head's dq | dk | dv by its 32-row slices of W at once (B fragments [k = d][n = c] by ldmatrix.trans from a shared
// copy of W), leaving a [16 px][32] fp32 partial; the eight partials are summed through shared memory and dxn is
// written once, in bf16.  The nine loop-invariant 32x32 B-operand fragment sets stay in registers: one CTA per SM.
// A stage holds the xn tile and the one dy tile all heads share; each warp recomputes its dout tile from dy.
constexpr int LFB_W_PITCH = LF_C + 8;                              // W copy [768][40] bf16: conflict-free ldmatrix
constexpr int LFB_R_PITCH = LF_C + 8;                              // fp32 partial rows: conflict-free float2 stores
struct LfbCfg {
    static constexpr int STAGE_ELEMS = 2 * LFB_TILE;                            // xn tile | dy tile
    static constexpr size_t SMEM_BASE = (size_t)LFB_STAGES * STAGE_ELEMS * 2 + (size_t)3 * LM_HID * LFB_W_PITCH * 2 +
                                        (size_t)LM_HEADS * LFB_ROWS * LFB_R_PITCH * 4 + (size_t)LM_HEADS * DH * 4;
    static constexpr size_t SMEM = SMEM_BASE + (size_t)LM_HEADS * LFP_WO_TILE * 2;
};

// c[16 px][32 c] += g[16 px][32 d] Wh[d][c]   (g as A fragments; Wh = one head's 32 rows of the shared W copy)
__device__ __forceinline__ void mma_w(float (&c)[4][4], const uint32_t (&g)[2][4], const __nv_bfloat16* Wh, int lane) {
#pragma unroll
    for (int kd = 0; kd < 2; ++kd)
#pragma unroll
        for (int np = 0; np < 2; ++np) {
            uint32_t bw[4];
            frag_b_krows(bw, Wh, LFB_W_PITCH, kd * 16, np * 16, lane);
            mma_bf16(c[2 * np], g[kd], bw[0], bw[1]);
            mma_bf16(c[2 * np + 1], g[kd], bw[2], bw[3]);
        }
}

__global__ void __launch_bounds__(256) laf_bwd_kernel(const __nv_bfloat16* __restrict__ xn, const __nv_bfloat16* __restrict__ W,
                                                      const __nv_bfloat16* __restrict__ dy, const float* __restrict__ ctx,
                                                      const float* __restrict__ dctx, const float* __restrict__ kmax,
                                                      const float* __restrict__ kzinv, __nv_bfloat16* __restrict__ dxn,
                                                      int N, int chunk_px, float scale, const __nv_bfloat16* __restrict__ w_out) {
    pdl_trigger();
    pdl_wait();
    extern __shared__ __align__(16) unsigned char raw[];
    constexpr int LFB_STAGE_ELEMS = LfbCfg::STAGE_ELEMS;
    const int b = blockIdx.y, chunk = blockIdx.x, lane = threadIdx.x & 31, h = threadIdx.x >> 5;
    __nv_bfloat16* tiles = reinterpret_cast<__nv_bfloat16*>(raw);
    __nv_bfloat16* Ws = tiles + LFB_STAGES * LFB_STAGE_ELEMS;
    __nv_bfloat16* Wo = reinterpret_cast<__nv_bfloat16*>(raw + LfbCfg::SMEM_BASE) + h * LFP_WO_TILE;
    float* R = reinterpret_cast<float*>(Ws + 3 * LM_HID * LFB_W_PITCH);
    float* scd = R + LM_HEADS * LFB_ROWS * LFB_R_PITCH + h * DH;
    const int n_begin = chunk * chunk_px, n_end = min(N, n_begin + chunk_px);
    const int n_tiles = (n_end - n_begin) / LFB_ROWS;
    const size_t pix0 = (size_t)b * N + n_begin;
    const __nv_bfloat16* xsrc = xn + pix0 * LF_C;
    const __nv_bfloat16* gsrc = dy + pix0 * LF_C;
    const CpRing<LFB_STAGES, LFB_STAGE_ELEMS, true> ring{tiles, n_tiles};
    auto load = [&](__nv_bfloat16* buf, int it) {
        if (h == 0) lw_issue<LFB_ROWS>(buf, xsrc + (size_t)it * LFB_ROWS * LF_C, LF_C, lane);
        if (h == 1) lw_issue<LFB_ROWS>(buf + LFB_TILE, gsrc + (size_t)it * LFB_ROWS * LF_C, LF_C, lane);
    };
    ring.prologue([&] {                            // W and this head's W_out slice
        for (int i = threadIdx.x; i < 3 * LM_HID * (LF_C / 8); i += blockDim.x)
            cp_async16(Ws + (i >> 2) * LFB_W_PITCH + (i & 3) * 8, W + (size_t)(i >> 2) * LF_C + (i & 3) * 8);
        lw_issue<32>(Wo, w_out + h * DH, LM_HID, lane);
    });
    ring.prime(load);
    const float* cg = ctx + ((size_t)b * LM_HEADS + h) * DH * DH;
    const float* dg = dctx + ((size_t)b * LM_HEADS + h) * DH * DH;
    float Mc[8], Zc[8], cdc[8];
    lfb_cd(cdc, scd, cg, dg, lane);
    load_cols(Mc, kmax + (size_t)b * LM_HID + h * DH, lane);
    load_cols(Zc, kzinv + (size_t)b * LM_HID + h * DH, lane);
    uint32_t wq[2][4][2], wk[2][4][2], wv[2][4][2];
    load_w_frags(wq, W + (size_t)(h * DH) * LF_C, lane);
    load_w_frags(wk, W + (size_t)(LM_HID + h * DH) * LF_C, lane);
    load_w_frags(wv, W + (size_t)(2 * LM_HID + h * DH) * LF_C, lane);
    uint32_t bc[2][4][2], bd[2][4][2], bt[2][4][2];
    frags_b_global<false>(bc, cg, lane);           // B[k=e][n=d] = ctx[d][e]
    frags_b_global<false>(bd, dg, lane);           // B[k=e][n=d] = dctx[d][e]
    frags_b_global<true>(bt, dg, lane);            // B[k=d][n=e] = dctx[d][e]
    const int g = lane >> 2, t = lane & 3;
    const float invN = 1.f / (float)N;
    const __nv_bfloat16* Wq = Ws + (size_t)(h * DH) * LFB_W_PITCH;
    const __nv_bfloat16* Wk = Wq + (size_t)LM_HID * LFB_W_PITCH;
    const __nv_bfloat16* Wv = Wk + (size_t)LM_HID * LFB_W_PITCH;
    float* Rw = R + h * LFB_ROWS * LFB_R_PITCH;
    const int rrow = threadIdx.x >> 4, rcol = (threadIdx.x & 15) * 2;     // the two dxn elements this thread sums
    for (int it = 0; it < n_tiles; ++it) {
        const __nv_bfloat16* buf = ring.wait(it, load);  // its CTA barrier also frees R
        LfbTile tl;
        load_x_frags<1>(tl.ax, buf, lane);
        lfp_dout(tl.ag, buf + LFB_TILE, Wo, lane);
        float dx[4][4];
        zero(dx);
        uint32_t a[2][4];
        {
            float dq[4][4];
            lfb_dq(dq, tl, wq, bc, scale);
            c_to_a(a, dq);
            mma_w(dx, a, Wq, lane);
        }
        {
            float dk[4][4], dv[4][4];
            lfb_dkdv(dk, dv, tl.ax, wk, wv, bd, bt, Mc, Zc, cdc, invN);
            c_to_a(a, dk);
            mma_w(dx, a, Wk, lane);
            c_to_a(a, dv);
            mma_w(dx, a, Wv, lane);
        }
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
            for (int half = 0; half < 2; ++half)
                *reinterpret_cast<float2*>(Rw + (g + half * 8) * LFB_R_PITCH + nt * 8 + 2 * t) =
                    make_float2(dx[nt][half * 2], dx[nt][half * 2 + 1]);
        __syncthreads();                           // the eight head partials of this tile are in R
        float sx = 0.f, sy = 0.f;
#pragma unroll
        for (int w = 0; w < LM_HEADS; ++w) {
            const float2 v = *reinterpret_cast<const float2*>(R + (w * LFB_ROWS + rrow) * LFB_R_PITCH + rcol);
            sx += v.x;
            sy += v.y;
        }
        *reinterpret_cast<uint32_t*>(dxn + (pix0 + (size_t)it * LFB_ROWS + rrow) * LF_C + rcol) = pack_bf16(sx, sy);
    }
}

// ---- pass B (weight gradient): dW_h = [dq | dk | dv]_h^T xn over the CTA's pixels, one reduction per CTA ---------------
// PART 0 streams xn and dy, recomputes dout_h from dy and accumulates dWq and the to_out weight gradient
// dW_out[c][32h + e] = sum_n dy[n][c] out_h[n][e], with out_h recomputed exactly as the forward forms it; PART 1
// accumulates dWk and dWv (reads xn only): split so that neither instantiation holds more than 64 accumulators next to
// its operand fragments.  Warps are independent (one head each, own tiles).  The [32][32] sums leave through shared
// memory as coalesced 128-byte red.global.add rows of the fp32 gradient.
template <int PART>
struct LfwCfg {
    static constexpr int STAGE_ELEMS = (PART == 0 ? 2 : 1) * LFB_TILE;     // xn tile (| dy tile)
    static constexpr int S_PITCH = DH + 1;                                 // epilogue staging [32 d][33] fp32
    static_assert(LFB_STAGES * STAGE_ELEMS * 2 >= DH * S_PITCH * 4, "the epilogue staging reuses the tile ring");
    static constexpr size_t SMEM_BASE = (size_t)LM_HEADS * (LFB_STAGES * STAGE_ELEMS * 2 + DH * 4);
    static constexpr size_t SMEM = SMEM_BASE + (PART == 0 ? (size_t)LM_HEADS * LFP_WO_TILE * 2 : 0);
};

// acc[32 d][32 c] += gf^T x over one 16-pixel tile: gf = accumulator fragment [16 px][32 d], bx = B fragments
// [k = px][n = c] of the xn tile (two n-tile pairs)
__device__ __forceinline__ void acc_gtx(float (&acc)[2][4][4], const float (&gf)[4][4], const uint32_t (&bx)[2][4]) {
#pragma unroll
    for (int md = 0; md < 2; ++md) {               // A[d][px]: transposed 8x8 blocks of the accumulator fragment
        uint32_t a[4];
        c_to_at(a, gf, md);
#pragma unroll
        for (int np = 0; np < 2; ++np) {
            mma_bf16(acc[md][2 * np], a, bx[np][0], bx[np][1]);
            mma_bf16(acc[md][2 * np + 1], a, bx[np][2], bx[np][3]);
        }
    }
}

template <int PART>
__global__ void __launch_bounds__(256) laf_wgrad_kernel(const __nv_bfloat16* __restrict__ xn, const __nv_bfloat16* __restrict__ W,
                                                        const __nv_bfloat16* __restrict__ dy, const float* __restrict__ ctx,
                                                        const float* __restrict__ dctx, const float* __restrict__ kmax,
                                                        const float* __restrict__ kzinv, float* __restrict__ grad_w, int N,
                                                        int chunk_px, long long w_stride_n, long long w_stride_c, float scale,
                                                        const __nv_bfloat16* __restrict__ w_out, float* __restrict__ grad_wo,
                                                        long long wo_stride_n, long long wo_stride_c) {
    pdl_trigger();
    pdl_wait();
    extern __shared__ __align__(16) unsigned char raw[];
    using Cfg = LfwCfg<PART>;
    constexpr int STAGE_ELEMS = Cfg::STAGE_ELEMS, S_PITCH = Cfg::S_PITCH;
    const int b = blockIdx.y, chunk = blockIdx.x, lane = threadIdx.x & 31, h = threadIdx.x >> 5;
    float* scd = reinterpret_cast<float*>(raw + (size_t)LM_HEADS * LFB_STAGES * STAGE_ELEMS * 2) + h * DH;
    __nv_bfloat16* Wo = reinterpret_cast<__nv_bfloat16*>(raw + Cfg::SMEM_BASE) + h * LFP_WO_TILE;        // PART 0
    const int n_begin = chunk * chunk_px, n_end = min(N, n_begin + chunk_px);
    const int n_tiles = (n_end - n_begin) / LFB_ROWS;
    const size_t pix0 = (size_t)b * N + n_begin;
    const __nv_bfloat16* xsrc = xn + pix0 * LF_C;
    const __nv_bfloat16* gsrc = dy + pix0 * LF_C;
    const CpRing<LFB_STAGES, STAGE_ELEMS> ring{reinterpret_cast<__nv_bfloat16*>(raw) +
                                                   (size_t)h * (LFB_STAGES * STAGE_ELEMS),
                                               n_tiles};
    auto load = [&](__nv_bfloat16* buf, int it) {
        lw_issue<LFB_ROWS>(buf, xsrc + (size_t)it * LFB_ROWS * LF_C, LF_C, lane);
        if (PART == 0) lw_issue<LFB_ROWS>(buf + LFB_TILE, gsrc + (size_t)it * LFB_ROWS * LF_C, LF_C, lane);
    };
    if (PART == 0) ring.prologue([&] { lw_issue<32>(Wo, w_out + h * DH, LM_HID, lane); });   // this head's W_out slice
    ring.prime(load);
    const float* cg = ctx + ((size_t)b * LM_HEADS + h) * DH * DH;
    const float* dg = dctx + ((size_t)b * LM_HEADS + h) * DH * DH;
    float Mc[8], Zc[8], cdc[8];
    uint32_t w0[2][4][2], w1[2][4][2];             // PART 0: Wq, (unused)   PART 1: Wk, Wv
    uint32_t b0[2][4][2], b1[2][4][2];             // PART 0: ctx^T, ctx   PART 1: dctx^T, dctx
    if (PART == 0) {
        load_w_frags(w0, W + (size_t)(h * DH) * LF_C, lane);
    } else {
        lfb_cd(cdc, scd, cg, dg, lane);
        load_cols(Mc, kmax + (size_t)b * LM_HID + h * DH, lane);
        load_cols(Zc, kzinv + (size_t)b * LM_HID + h * DH, lane);
        load_w_frags(w0, W + (size_t)(LM_HID + h * DH) * LF_C, lane);
        load_w_frags(w1, W + (size_t)(2 * LM_HID + h * DH) * LF_C, lane);
    }
    frags_b_global<false>(b0, PART == 0 ? cg : dg, lane);
    frags_b_global<true>(b1, PART == 1 ? dg : cg, lane);
    const float invN = 1.f / (float)N;
    float acc[2][2][4][4];
    zero(acc);
    for (int it = 0; it < n_tiles; ++it) {
        const __nv_bfloat16* buf = ring.wait(it, load);
        LfbTile tl;
        load_x_frags<1>(tl.ax, buf, lane);
        uint32_t bx[2][4];
        frag_b_krows(bx[0], buf, LW_PITCH, 0, 0, lane);        // B[k = px][n = c] = xn[px][c]
        frag_b_krows(bx[1], buf, LW_PITCH, 0, 16, lane);
        uint32_t ady[2][4], bdy[2][4];             // PART 0: A fragments [px][c] and B fragments [k = px][n = c] of dy
        if (PART == 0) {
            frag_a_rowmajor(ady[0], buf + LFB_TILE, LW_PITCH, 0, 0, lane);
            frag_a_rowmajor(ady[1], buf + LFB_TILE, LW_PITCH, 0, 16, lane);
            frag_b_krows(bdy[0], buf + LFB_TILE, LW_PITCH, 0, 0, lane);
            frag_b_krows(bdy[1], buf + LFB_TILE, LW_PITCH, 0, 16, lane);
        }
        ring.release(it, load);                    // the tile is in registers
        if (PART == 0) {
            {
                float c[4][4];
                lfp_dout_acc(c, ady, Wo, lane);
                c_to_a(tl.ag, c);
            }
            float dq[4][4];
            lfb_dq(dq, tl, w0, b0, scale);
            acc_gtx(acc[0], dq, bx);
            // out_h as laf_out_kernel forms it, then dW_out^T += out_h^T dy
            float cq[1][4][4], o[4][4];
            project<1>(cq, tl.ax, w0);
            frag_softmax(cq[0], scale);
            uint32_t a[2][4];
            c_to_a(a, cq[0]);
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                zero(o[nt]);
#pragma unroll
                for (int ks = 0; ks < 2; ++ks) mma_bf16(o[nt], a[ks], b1[ks][nt][0], b1[ks][nt][1]);
            }
            acc_gtx(acc[1], o, bdy);
        } else {
            float dk[4][4], dv[4][4];
            lfb_dkdv(dk, dv, tl.ax, w0, w1, b0, b1, Mc, Zc, cdc, invN);
            acc_gtx(acc[0], dk, bx);
            acc_gtx(acc[1], dv, bx);
        }
    }
    float* S = reinterpret_cast<float*>(ring.drain());     // the ring is free: stage the sums there
    const int g = lane >> 2, t = lane & 3;
#pragma unroll
    for (int m = 0; m < 2; ++m) {
#pragma unroll
        for (int md = 0; md < 2; ++md)
#pragma unroll
            for (int nc = 0; nc < 4; ++nc)
#pragma unroll
                for (int i = 0; i < 4; ++i) S[(md * 16 + g + 8 * (i >> 1)) * S_PITCH + nc * 8 + 2 * t + (i & 1)] = acc[m][md][nc][i];
        __syncwarp();
        if (PART == 0 && m == 1) {                    // S[e][c] = dW_out[c][32h + e]: lane = e, one row c at a time
            float* dst = grad_wo + (long long)(h * DH + lane) * wo_stride_c;
#pragma unroll 4
            for (int c = 0; c < LF_C; ++c) atomicAdd(dst + c * wo_stride_n, S[lane * S_PITCH + c]);
        } else {
            // rows of dW: to_qkv output channel (q | k | v block) * 256 + h * 32 + d;  lane = input channel c
            float* dst = grad_w + (long long)((PART + m) * LM_HID + h * DH) * w_stride_n + lane * w_stride_c;
#pragma unroll 4
            for (int d = 0; d < DH; ++d) atomicAdd(dst + d * w_stride_n, S[d * S_PITCH + lane]);
        }
        __syncwarp();
    }
}

constexpr size_t LAF_STATS_SMEM = (size_t)LM_HEADS * LFS_STAGES * LW_TILE * 2;

static int laf_stat_chunks(int N) {
    int c = N / 128;
    if (c < 1) c = 1;
    if (c > 16) c = 16;                 // B * chunks CTAs: one wave at batch 32
    return c;
}

}  // namespace pidm
using namespace pidm;

extern "C" int pidm_linattn_block_supported(int C, int heads, int N, int dtype) {
    return (C == LF_C && heads == LM_HEADS && dtype == PIDM_BF16 && N % 128 == 0) ? 1 : 0;
}

extern "C" int pidm_linattn_block_workspace_floats(int B, int N) { return B * laf_stat_chunks(N) * LM_HID; }

// pixel chunking of the block's kernels: out[5] = {statistics chunks (kmax), ctx px, fwd (y) px, bwd px, wgrad px}
extern "C" int pidm_linattn_block_plan(int B, int N, int* out) {
    PIDM_REQUIRE(N % 128 == 0 && B > 0, "linattn_block_plan: N must be a multiple of 128 (got %d)", N);
    const int v[5] = {laf_stat_chunks(N), chunk_px(B, N, 2), chunk_px(B, N, 2), chunk_px(B, N, 1), chunk_px(B, N, 1)};
    for (int i = 0; i < 5; ++i) out[i] = v[i];
    return 0;
}

// The whole linear-attention block: y = residual + b_out + to_out(attention(to_qkv(xn))), see pidm.h.
extern "C" int pidm_linattn_block_fwd(const void* xn, const void* w_qkv, const void* w_out, const float* b_out,
                                      const void* residual, void* y, float* ctx, float* kmax, float* kzinv,
                                      float* workspace, int B, int N, void* stream) {
    PIDM_REQUIRE(w_out && b_out && residual, "linattn_block_fwd: w_out, b_out and residual are required");
    PIDM_REQUIRE(N % 128 == 0, "linattn_block: N must be a multiple of 128 (got %d)", N);
    cudaStream_t st = (cudaStream_t)stream;
    const __nv_bfloat16* x = (const __nv_bfloat16*)xn;
    const __nv_bfloat16* w = (const __nv_bfloat16*)w_qkv;
    PIDM_CUDA(cudaMemsetAsync(ctx, 0, (size_t)B * LM_HEADS * DH * DH * sizeof(float), st));
    PIDM_CUDA(cudaMemsetAsync(kzinv, 0, (size_t)B * LM_HID * sizeof(float), st));
    const int chunks = laf_stat_chunks(N);
    const int rpc = N / chunks;
    PIDM_REQUIRE(rpc % 32 == 0 && rpc * chunks == N, "linattn_block: bad statistics chunking for N=%d", N);
    PIDM_CUDA(allow_smem(laf_kmax_kernel, LAF_STATS_SMEM));
    PIDM_CUDA(launch_plain(laf_kmax_kernel, dim3(dim3(chunks, B)), dim3(256), (size_t)(LAF_STATS_SMEM), st, x, w, workspace, N, rpc));
    const int px = chunk_px(B, N, 2);             // the context and output kernels: two CTAs per SM
    const dim3 grid((N + px - 1) / px, B);
    PIDM_CUDA(allow_smem(laf_ctx_kernel<0>, LfcCfg<0>::SMEM));
    PIDM_CUDA(launch_plain(laf_ctx_kernel<0>, grid, dim3(256), LfcCfg<0>::SMEM, st, x, w, nullptr, workspace, chunks, kmax, kzinv,
                           ctx, N, px, ATTN_SCALE, nullptr));
    PIDM_CUDA(launch_plain(laf_finalize_kernel, dim3((B * LM_HID + 7) / 8), dim3(256), (size_t)(0), st, ctx, kzinv, B * LM_HID));
    PIDM_CUDA(allow_smem(laf_out_kernel, LAF_OUT_SMEM));
    PIDM_CUDA(launch_plain(laf_out_kernel, grid, dim3(256), LAF_OUT_SMEM, st, x, w, ctx, (__nv_bfloat16*)y, N, px,
                           ATTN_SCALE, (const __nv_bfloat16*)w_out, b_out, (const __nv_bfloat16*)residual));
    PIDM_LAUNCH_CHECK("linattn_block_fwd");
    return 0;
}

extern "C" int pidm_linattn_block_bwd(const void* xn, const void* w_qkv, const void* w_out, const void* dy, const float* ctx,
                                      const float* kmax, const float* kzinv, void* dxn, float* dctx, int B, int N,
                                      void* stream) {
    PIDM_REQUIRE(N % 128 == 0, "linattn_block: N must be a multiple of 128 (got %d)", N);
    cudaStream_t st = (cudaStream_t)stream;
    const __nv_bfloat16* x = (const __nv_bfloat16*)xn;
    const __nv_bfloat16* w = (const __nv_bfloat16*)w_qkv;
    const __nv_bfloat16* wo = (const __nv_bfloat16*)w_out;
    const __nv_bfloat16* g = (const __nv_bfloat16*)dy;
    PIDM_CUDA(cudaMemsetAsync(dctx, 0, (size_t)B * LM_HEADS * DH * DH * sizeof(float), st));
    const int cpx = chunk_px(B, N, 2);
    PIDM_CUDA(allow_smem(laf_ctx_kernel<1>, LfcCfg<1>::SMEM));
    PIDM_CUDA(launch_plain(laf_ctx_kernel<1>, dim3(dim3((N + cpx - 1) / cpx, B)), dim3(256), LfcCfg<1>::SMEM, st, x, w, g,
                           nullptr, 0, nullptr, nullptr, dctx, N, cpx, ATTN_SCALE, wo));
    const int bpx = chunk_px(B, N, 1);
    PIDM_CUDA(allow_smem(laf_bwd_kernel, LfbCfg::SMEM));
    PIDM_CUDA(launch_plain(laf_bwd_kernel, dim3(dim3((N + bpx - 1) / bpx, B)), dim3(256), LfbCfg::SMEM, st, x, w, g, ctx, dctx,
                           kmax, kzinv, (__nv_bfloat16*)dxn, N, bpx, ATTN_SCALE, wo));
    PIDM_LAUNCH_CHECK("linattn_block_bwd");
    return 0;
}

extern "C" int pidm_linattn_block_wgrad(const void* xn, const void* w_qkv, const void* w_out, const void* dy,
                                        const float* ctx, const float* dctx, const float* kmax, const float* kzinv,
                                        float* grad_w_qkv, long long qkv_stride_n, long long qkv_stride_c,
                                        float* grad_w_out, long long out_stride_n, long long out_stride_c, int B, int N,
                                        void* stream) {
    PIDM_REQUIRE(N % 128 == 0, "linattn_block: N must be a multiple of 128 (got %d)", N);
    cudaStream_t st = (cudaStream_t)stream;
    const __nv_bfloat16* x = (const __nv_bfloat16*)xn;
    const __nv_bfloat16* w = (const __nv_bfloat16*)w_qkv;
    const __nv_bfloat16* wo = (const __nv_bfloat16*)w_out;
    const __nv_bfloat16* g = (const __nv_bfloat16*)dy;
    const int px = chunk_px(B, N, 1);
    const dim3 grid((N + px - 1) / px, B);
    PIDM_CUDA(allow_smem(laf_wgrad_kernel<0>, LfwCfg<0>::SMEM));
    PIDM_CUDA(launch_plain(laf_wgrad_kernel<0>, grid, dim3(256), LfwCfg<0>::SMEM, st, x, w, g, ctx, dctx, kmax, kzinv, grad_w_qkv,
                           N, px, qkv_stride_n, qkv_stride_c, ATTN_SCALE, wo, grad_w_out, out_stride_n, out_stride_c));
    PIDM_CUDA(allow_smem(laf_wgrad_kernel<1>, LfwCfg<1>::SMEM));
    PIDM_CUDA(launch_plain(laf_wgrad_kernel<1>, grid, dim3(256), LfwCfg<1>::SMEM, st, x, w, g, ctx, dctx, kmax, kzinv, grad_w_qkv,
                           N, px, qkv_stride_n, qkv_stride_c, ATTN_SCALE, nullptr, nullptr, 0LL, 0LL));
    PIDM_LAUNCH_CHECK("linattn_block_wgrad");
    return 0;
}
