// Warp-level tensor-core helpers shared by the linear-attention kernels (attention_mma.cu, attention_fused.cu):
// mma.sync m16n8k16 bf16, ldmatrix fragment loaders, per-warp cp.async tile movers, and their pixel chunking.
#pragma once
#include "common.cuh"

namespace pidm {


constexpr int LM_HEADS = 8, LM_D = 32, LM_HID = 256;
constexpr int LM_PITCH = LM_HID + 8;          // bf16 elements per smem row (528 B: 16-byte aligned, conflict-free ldmatrix)
constexpr int LM_CPITCH = LM_D + 8;           // ctx rows [d][e] in bf16
constexpr int LM_CHUNK = 256;                 // pixels per CTA

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

constexpr int LW_PITCH = LM_D + 8;            // bf16 per smem row of a head tile: 80 B -> conflict-free ldmatrix / row access
constexpr int LW_TILE = 32 * LW_PITCH;        // one [32 px][32 ch] tile

__device__ __forceinline__ void cp_async16(void* dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int PENDING>
__device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(PENDING) : "memory"); }

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
        b[0] = pack_bf16(G[(k0 + 2 * t) * LM_D + n0 + g], G[(k0 + 2 * t + 1) * LM_D + n0 + g]);
        b[1] = pack_bf16(G[(k0 + 2 * t + 8) * LM_D + n0 + g], G[(k0 + 2 * t + 9) * LM_D + n0 + g]);
    } else {
        const float2 lo = *reinterpret_cast<const float2*>(G + (n0 + g) * LM_D + k0 + 2 * t);
        const float2 hi = *reinterpret_cast<const float2*>(G + (n0 + g) * LM_D + k0 + 2 * t + 8);
        b[0] = pack_bf16(lo.x, lo.y);
        b[1] = pack_bf16(hi.x, hi.y);
    }
}


}  // namespace pidm
