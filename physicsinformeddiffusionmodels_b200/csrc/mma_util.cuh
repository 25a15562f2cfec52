// Warp-level tensor-core helpers of the attention kernels (attention.cu, attention_mid.cu, attention_fused.cu):
// mma.sync m16n8k16 bf16, ldmatrix fragment loaders, accumulator-fragment steps (softmax, conversion to A and to
// transposed fragments, bf16 row stores, the context epilogue), the cp.async ring every tile pipeline runs on, and
// the pixel chunking.
#pragma once
#include "common.cuh"

namespace pidm {

constexpr int DH = 32;                                  // dim_head of every attention in the U-Net
constexpr float ATTN_SCALE = 0.17677669529663687f;      // DH^-1/2
constexpr int LM_HEADS = 8, LM_HID = LM_HEADS * DH;     // the tensor-core linear attention: 8 heads

// pixels per CTA: about ctas_per_sm CTAs per SM over the whole batch, a multiple of 32, never more than the image.
// Chunks are per sample: k chunks per sample with B * k <= resident CTA slots (one wave), 32-pixel granularity.
static inline int chunk_px(int B, int N, int ctas_per_sm) {
    int k = (num_sms() * ctas_per_sm) / B;
    if (k < 1) k = 1;
    int px = ((N + k - 1) / k + 31) / 32 * 32;
    if (px < 64) px = 64;
    if (px > N) px = N;
    return px;
}

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void mma_bf16(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
    __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ uint32_t movm_t(uint32_t x) {
    uint32_t y;
    asm volatile("movmatrix.sync.aligned.m8n8.trans.b16 %0, %1;" : "=r"(y) : "r"(x));
    return y;
}
__device__ __forceinline__ void st8_smem(__nv_bfloat16* p, const float v[8]) {
    uint4 t = make_uint4(pack_bf16(v[0], v[1]), pack_bf16(v[2], v[3]), pack_bf16(v[4], v[5]), pack_bf16(v[6], v[7]));
    *reinterpret_cast<uint4*>(p) = t;
}

// A fragment (16 rows x 16 k) from a row-major smem tile S[row][col]: rows = M index, cols = K index
__device__ __forceinline__ void frag_a_rowmajor(uint32_t (&a)[4], const __nv_bfloat16* S, int pitch, int m0, int k0, int lane) {
    const int mi = lane >> 3, r = lane & 7;
    ldsm_x4(a, smem_u32(S + (size_t)(m0 + r + 8 * (mi & 1)) * pitch + k0 + 8 * (mi >> 1)));
}
// A fragment when smem holds the transpose: S[k][m] (rows = K index, cols = M index)
__device__ __forceinline__ void frag_a_kmajor(uint32_t (&a)[4], const __nv_bfloat16* S, int pitch, int k0, int m0, int lane) {
    const int mi = lane >> 3, r = lane & 7;
    ldsm_x4_t(a, smem_u32(S + (size_t)(k0 + r + 8 * (mi >> 1)) * pitch + m0 + 8 * (mi & 1)));
}
// B fragments of TWO adjacent n-tiles (n0..n0+15) for one k16 step, from S[k][n] (rows = K index): b[0..1] tile 0, b[2..3] tile 1
__device__ __forceinline__ void frag_b_krows(uint32_t (&b)[4], const __nv_bfloat16* S, int pitch, int k0, int n0, int lane) {
    const int mi = lane >> 3, r = lane & 7;
    ldsm_x4_t(b, smem_u32(S + (size_t)(k0 + r + 8 * (mi & 1)) * pitch + n0 + 8 * (mi >> 1)));
}
// same from S[n][k] (rows = N index, cols = K index)
__device__ __forceinline__ void frag_b_nrows(uint32_t (&b)[4], const __nv_bfloat16* S, int pitch, int n0, int k0, int lane) {
    const int mi = lane >> 3, r = lane & 7;
    ldsm_x4(b, smem_u32(S + (size_t)(n0 + r + 8 * (mi >> 1)) * pitch + k0 + 8 * (mi & 1)));
}

constexpr int LW_PITCH = DH + 8;        // bf16 per smem row of a head tile: 80 B -> conflict-free ldmatrix / row access
constexpr int LW_TILE = 32 * LW_PITCH;   // one [32 px][32 ch] tile

__device__ __forceinline__ void cp_async16(void* dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int PENDING>
__device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(PENDING) : "memory"); }

// ---- the cp.async tile ring of every attention pipeline ------------------------------------------------------------
// STAGES slots of STAGE_ELEMS bf16 from `base`.  The kernel supplies only `load(slot, it)`, which issues the copies of
// tile `it` into `slot`; the ring decides where each tile lands and when it is issued, waited for and refilled.
//   * Every issue commits exactly one cp.async group, also past the last tile (an empty group then), so a tile always
//     has the same number of younger groups and one compile-time wait_group count fits every iteration.
//   * A group committed before prime() (prologue(): a W_out slice, the W copy) is older than every ring group, so the
//     first wait() covers it too.
//   * Warp-private discipline (SHARED = false): a warp streams its own head through its own ring, STAGES tiles ahead.
//     wait(it) leaves STAGES - 1 groups in flight and syncs the warp; release(it) syncs the warp again and refills the
//     slot with tile it + STAGES, so between the two the kernel may transform the slot in place or stage its output
//     there; drain() ends the copies so the ring can be reused.  la_ctx_mma, la_out_mma, la_bwd_mma, laf_kmax, laf_ctx
//     and laf_wgrad.
//   * CTA-shared discipline (SHARED = true): one or two warps issue, every warp reads, STAGES - 1 tiles ahead with one
//     slot of slack.  wait(it) leaves STAGES - 2 groups in flight; its __syncthreads both publishes tile `it` and shows
//     every warp done with tile it - 1, whose slot it refills at once with tile it + STAGES - 1.  laf_out and laf_bwd.
template <int STAGES, int STAGE_ELEMS, bool SHARED = false>
struct CpRing {
    static constexpr int AHEAD = SHARED ? STAGES - 1 : STAGES;
    __nv_bfloat16* base;
    int n_tiles;

    __device__ __forceinline__ __nv_bfloat16* slot(int it) const { return base + (size_t)(it % STAGES) * STAGE_ELEMS; }
    template <class Load>
    __device__ __forceinline__ void issue(int it, Load& load) const {
        if (it < n_tiles) load(slot(it), it);
        cp_commit();
    }
    template <class Copies>
    __device__ __forceinline__ void prologue(Copies&& copies) const { copies(); cp_commit(); }
    template <class Load>
    __device__ __forceinline__ void prime(Load& load) const {
#pragma unroll
        for (int s = 0; s < AHEAD; ++s) issue(s, load);
    }
    template <class Load>
    __device__ __forceinline__ __nv_bfloat16* wait(int it, Load& load) const {
        cp_wait<AHEAD - 1>();
        if (SHARED) {
            __syncthreads();
            issue(it + AHEAD, load);
        } else {
            __syncwarp();
        }
        return slot(it);
    }
    template <class Load>
    __device__ __forceinline__ void release(int it, Load& load) const {
        static_assert(!SHARED, "a CTA-shared ring refills in wait()");
        __syncwarp();
        issue(it + STAGES, load);
    }
    __device__ __forceinline__ __nv_bfloat16* drain() const {
        static_assert(!SHARED, "only warp-private rings are reused");
        cp_wait<0>();
        __syncwarp();
        return base;
    }
};

// one head's 64-byte slice of ROWS consecutive pixel rows -> smem [ROWS][LW_PITCH]; a warp instruction moves 8 rows
template <int ROWS>
__device__ __forceinline__ void lw_issue(__nv_bfloat16* dst, const __nv_bfloat16* __restrict__ src, size_t row_stride, int lane) {
    const int r = lane >> 2, c = (lane & 3) * 8;
#pragma unroll
    for (int i = 0; i < ROWS / 8; ++i)
        cp_async16(dst + (r + 8 * i) * LW_PITCH + c, src + (size_t)(r + 8 * i) * row_stride + c);
}
// the same mapping for writing a staged tile back: 16-byte vectors, 64-byte row segments
template <int ROWS>
__device__ __forceinline__ void lw_store(__nv_bfloat16* __restrict__ dst, size_t row_stride, const __nv_bfloat16* src, int lane) {
    const int r = lane >> 2, c = (lane & 3) * 8;
#pragma unroll
    for (int i = 0; i < ROWS / 8; ++i)
        *reinterpret_cast<uint4*>(dst + (size_t)(r + 8 * i) * row_stride + c) =
            *reinterpret_cast<const uint4*>(src + (r + 8 * i) * LW_PITCH + c);
}
__device__ __forceinline__ void row_load32(const __nv_bfloat16* p, float (&v)[32]) {
#pragma unroll
    for (int j = 0; j < 4; ++j) ld8(p + 8 * j, &v[8 * j]);
}
__device__ __forceinline__ void row_store32(__nv_bfloat16* p, const float (&v)[32]) {
#pragma unroll
    for (int j = 0; j < 4; ++j) st8_smem(p + 8 * j, &v[8 * j]);
}
// softmax over the 32 channels of one pixel row (held by one lane), times mul
__device__ __forceinline__ void row_softmax32(float (&v)[32], float mul) {
    float mx = v[0];
#pragma unroll
    for (int j = 1; j < 32; ++j) mx = fmaxf(mx, v[j]);
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < 32; ++j) { v[j] = __expf(v[j] - mx); s += v[j]; }
    const float inv = mul / s;
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] *= inv;
}
// B fragment (k16 x n8) built straight from a row-major fp32 matrix G[32][32] in global memory.
//   KROWS = true : B[k][n] = G[k][n]      KROWS = false: B[k][n] = G[n][k]
template <bool KROWS>
__device__ __forceinline__ void frag_b_global(uint32_t (&b)[2], const float* __restrict__ G, int k0, int n0, int lane) {
    const int g = lane >> 2, t = lane & 3;
    if (KROWS) {
        b[0] = pack_bf16(G[(k0 + 2 * t) * DH + n0 + g], G[(k0 + 2 * t + 1) * DH + n0 + g]);
        b[1] = pack_bf16(G[(k0 + 2 * t + 8) * DH + n0 + g], G[(k0 + 2 * t + 9) * DH + n0 + g]);
    } else {
        const float2 lo = *reinterpret_cast<const float2*>(G + (n0 + g) * DH + k0 + 2 * t);
        const float2 hi = *reinterpret_cast<const float2*>(G + (n0 + g) * DH + k0 + 2 * t + 8);
        b[0] = pack_bf16(lo.x, lo.y);
        b[1] = pack_bf16(hi.x, hi.y);
    }
}
// all eight B fragments (2 k16 steps x 4 n-tiles) of a 32x32 matrix G, see frag_b_global
template <bool KROWS>
__device__ __forceinline__ void frags_b_global(uint32_t (&b)[2][4][2], const float* __restrict__ G, int lane) {
#pragma unroll
    for (int ks = 0; ks < 2; ++ks)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) frag_b_global<KROWS>(b[ks][nt], G, ks * 16, nt * 8, lane);
}

// ---- steps on accumulator fragments (lane = 4 g + t holds rows g, g + 8 and columns 8 nt + 2 t, + 1 of each n-tile nt)
__device__ __forceinline__ void zero(float& x) { x = 0.f; }
template <class T, int N>
__device__ __forceinline__ void zero(T (&a)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) zero(a[i]);
}
// sum over the quad of lanes that share a row
__device__ __forceinline__ float quad_sum(float x) {
    x += __shfl_xor_sync(0xffffffffu, x, 1);
    x += __shfl_xor_sync(0xffffffffu, x, 2);
    return x;
}
// softmax over the NT * 8 columns of rows g and g + 8, times mul
template <int NT>
__device__ __forceinline__ void frag_softmax(float (&c)[NT][4], float mul) {
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        float mx = -INFINITY;
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) mx = fmaxf(mx, fmaxf(c[nt][half * 2], c[nt][half * 2 + 1]));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        float s = 0.f;
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
            c[nt][half * 2] = __expf(c[nt][half * 2] - mx);
            c[nt][half * 2 + 1] = __expf(c[nt][half * 2 + 1] - mx);
            s += c[nt][half * 2] + c[nt][half * 2 + 1];
        }
        const float inv = mul / quad_sum(s);
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) { c[nt][half * 2] *= inv; c[nt][half * 2 + 1] *= inv; }
    }
}
// accumulator fragments [16][16 KS] -> the KS A fragments (k16 steps over the columns) of the same matrix, bf16
template <int KS>
__device__ __forceinline__ void c_to_a(uint32_t (&a)[KS][4], const float (&c)[2 * KS][4]) {
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
        a[ks][0] = pack_bf16(c[2 * ks][0], c[2 * ks][1]);
        a[ks][1] = pack_bf16(c[2 * ks][2], c[2 * ks][3]);
        a[ks][2] = pack_bf16(c[2 * ks + 1][0], c[2 * ks + 1][1]);
        a[ks][3] = pack_bf16(c[2 * ks + 1][2], c[2 * ks + 1][3]);
    }
}
// the transpose of an accumulator tile c [16 rows][32 cols] as bf16 operands, each 8x8 block moved by movmatrix:
// c_to_at gives the A fragment of columns 16 md .. 16 md + 15 (rows of the transpose; k = the 16 rows of c),
// c_to_bt the B fragments [k = row][n = col] of the four column n-tiles
__device__ __forceinline__ void c_to_at(uint32_t (&a)[4], const float (&c)[4][4], int md) {
    a[0] = movm_t(pack_bf16(c[2 * md][0], c[2 * md][1]));
    a[1] = movm_t(pack_bf16(c[2 * md + 1][0], c[2 * md + 1][1]));
    a[2] = movm_t(pack_bf16(c[2 * md][2], c[2 * md][3]));
    a[3] = movm_t(pack_bf16(c[2 * md + 1][2], c[2 * md + 1][3]));
}
__device__ __forceinline__ void c_to_bt(uint32_t (&b)[4][2], const float (&c)[4][4]) {
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
        b[nt][0] = movm_t(pack_bf16(c[nt][0], c[nt][1]));
        b[nt][1] = movm_t(pack_bf16(c[nt][2], c[nt][3]));
    }
}
// rows g and g + 8 of an accumulator tile [16][NT * 8], times mul -> bf16 rows of dst (`stride` elements apart)
template <int NT>
__device__ __forceinline__ void store_rows_bf16(__nv_bfloat16* dst, size_t stride, const float (&c)[NT][4], int lane,
                                                float mul = 1.f) {
    const int g = lane >> 2, t = lane & 3;
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
        *reinterpret_cast<uint32_t*>(dst + (size_t)g * stride + nt * 8 + 2 * t) = pack_bf16(c[nt][0] * mul, c[nt][1] * mul);
        *reinterpret_cast<uint32_t*>(dst + (size_t)(g + 8) * stride + nt * 8 + 2 * t) =
            pack_bf16(c[nt][2] * mul, c[nt][3] * mul);
    }
}

// ---- per-head steps of the linear attention ------------------------------------------------------------------------
// cd[d] = sum_e dctx[d][e] ctx[d][e] for d = lane: the k-softmax term of the backward
__device__ __forceinline__ float ctx_dot_row(const float* __restrict__ cg, const float* __restrict__ dg, int lane) {
    float s = 0.f;
#pragma unroll
    for (int e = 0; e < DH; e += 4) {
        const float4 x = *reinterpret_cast<const float4*>(dg + lane * DH + e);
        const float4 y = *reinterpret_cast<const float4*>(cg + lane * DH + e);
        s += x.x * y.x + x.y * y.y + x.z * y.z + x.w * y.w;
    }
    return s;
}
// ctx[d][e] += acc[d][e] * row_scale(d): a warp's [32 d][32 e] context accumulator, added into one head's block
template <class RowScale>
__device__ __forceinline__ void ctx_atomic_add(float* cb, const float (&acc)[2][4][4], RowScale row_scale, int lane) {
    const int g = lane >> 2, t = lane & 3;
#pragma unroll
    for (int md = 0; md < 2; ++md)
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const int d = md * 16 + g + half * 8;
            const float f = row_scale(d);
#pragma unroll
            for (int ne = 0; ne < 4; ++ne) {
                const int e = ne * 8 + 2 * t;
                atomicAdd(cb + d * DH + e, acc[md][ne][half * 2] * f);
                atomicAdd(cb + d * DH + e + 1, acc[md][ne][half * 2 + 1] * f);
            }
        }
}

}  // namespace pidm
