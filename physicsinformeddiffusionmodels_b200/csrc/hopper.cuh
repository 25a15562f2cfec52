// Hopper (sm_90a) building blocks of the tensor-core convolution kernels (conv_tc.cu, wgrad_tc.cu): the TMA ring,
// TMA tensor loads, wgmma shared-memory descriptors and the warpgroup MMA itself; on the host, the activation tensor
// maps and the pixel tiling those kernels share.
#pragma once
#include "common.cuh"
#include <cuda.h>

namespace pidm {

__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(
            smem_u32(dst)),
        "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
            smem_u32(dst)),
        "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "elect.sync _|p, 0xffffffff;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(pred));
    return pred != 0;
}
// named barrier over `threads` threads (a multiple of 32), id 1..15 (0 is __syncthreads)
__device__ __forceinline__ void named_bar(int id, int threads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// Swizzled wgmma shared-memory descriptor (sm_90 layout): [0,14) start >> 4, [16,30) LBO >> 4, [32,46) SBO >> 4,
// [62,64) swizzle mode (1 = 128B, 2 = 64B).  SBO = byte stride between 8-row groups along K (8 * swizzle span).
// K-major operands ignore LBO; MN-major operands use it as the byte stride between swizzle atoms along M / N.
// The start address advances by integer adds to the low word (16-byte units): descriptors are built once per kernel.
template <int SWIZZLE_BYTES>
__host__ __device__ constexpr uint32_t gmma_desc_hi() {
    return (uint32_t)((8 * SWIZZLE_BYTES) >> 4) | ((SWIZZLE_BYTES == 128 ? 1u : 2u) << 30);
}
__device__ __forceinline__ uint32_t gmma_desc_lo(uint32_t smem_addr, uint32_t lbo_bytes) {
    return ((smem_addr & 0x3FFFF) >> 4) | (((lbo_bytes >> 4) & 0x3FFF) << 16);
}
__device__ __forceinline__ uint64_t gmma_desc(uint32_t hi, uint32_t lo) { return ((uint64_t)hi << 32) | lo; }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int PENDING>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(PENDING) : "memory"); }

// ---- TMA ring ---------------------------------------------------------------------------------------------------
// Operand stages in shared memory between a TMA producer and two consumer warpgroups, each stage with two mbarriers:
// full[s] takes one arrival (the producer's expect_tx) plus the bytes of its TMA loads; empty[s] one arrival per
// consumer warp (8) once the wgmmas that read the stage have retired.  Both sides walk the stages in the same order,
// each with its own TmaRing.  A barrier completes once per pass through the ring: consumers wait for `full` with the
// parity of the current pass, the producer for `empty` with that of the previous pass (complete on a fresh barrier,
// so the first pass finds every stage free).  Consumers keep one wgmma group in flight (consumed()).
// The weight-gradient kernels run one pass of split-K steps per CTA and end there, so their consumers never release
// the last stage.  The convolution's ring runs across tile boundaries: its consumers release the last stage of every
// tile (release_held()), and its four producer warps each walk every stage but take turns loading them.

// bytes from the start of the dynamic shared memory to the first 1024-byte boundary, where the ring starts (the 128B
// swizzle atoms of TMA and wgmma need that alignment)
__device__ __forceinline__ uint32_t smem_pad_1024(const unsigned char* smem_raw) {
    return (1024 - (smem_u32(smem_raw) & 1023)) & 1023;
}
__device__ __forceinline__ void prefetch_tensormap(const CUtensorMap* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}

struct TmaRing {
    uint64_t* full;
    uint64_t* empty;
    uint32_t stage = 0, phase = 0;
    uint32_t held = 0;       // consumer side only: the stage read by the wgmma group still in flight

    // the first `stages` barrier pairs (one thread; mbar_init_fence() and a CTA barrier must follow)
    __device__ __forceinline__ void init(int stages) const {
        for (int s = 0; s < stages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }
    }
    // producer: wait until the current stage is free and arm its `full` barrier with the bytes the loads will bring;
    // returns that barrier for the loads to complete on
    __device__ __forceinline__ uint64_t* acquire(uint32_t tx_bytes) const {
        mbar_wait(&empty[stage], phase ^ 1);
        mbar_expect_tx(&full[stage], tx_bytes);
        return &full[stage];
    }
    // consumer: wait until the current stage's operands have landed
    __device__ __forceinline__ void wait_full() const { mbar_wait(&full[stage], phase); }
    // consumer, after issuing the wgmmas that read the current stage: commit them, wait for the previous group and,
    // unless this stage is the first of the run, release that group's stage (lane 0 of each warp arrives)
    __device__ __forceinline__ void consumed(bool first, int lane) {
        wgmma_commit();
        wgmma_wait<1>();
        if (!first && lane == 0) mbar_arrive(&empty[held]);
        held = stage;
    }
    // consumer, once the last group has retired: release its stage too (a ring that runs on past the consumer's run)
    __device__ __forceinline__ void release_held(int lane) const {
        if (lane == 0) mbar_arrive(&empty[held]);
    }
    // next stage; true when the ring wrapped back to stage 0 (the caller rewinds its stage address)
    __device__ __forceinline__ bool advance(uint32_t stages) {
        if (++stage == stages) { stage = 0; phase ^= 1; return true; }
        return false;
    }
};

// Pixel tiles [begin, begin + count) of this CTA's split-K range (blockIdx.z) when n_pix_tiles are cut into ranges
// of per_split (one_wave_split); count <= 0 for a CTA past the last range
struct SplitRange { int begin, count; };
__device__ __forceinline__ SplitRange split_k_range(int per_split, int n_pix_tiles) {
    const int begin = blockIdx.z * per_split;
    int end = begin + per_split;
    if (end > n_pix_tiles) end = n_pix_tiles;
    return {begin, end - begin};
}

// D[64 x N] (+)= A[64 x 16] * B[16 x N], bf16 operands in shared memory, fp32 accumulator fragment in registers
// (thread t of warp w of the warpgroup holds rows 16w + t/4 (+8), columns 8j + 2(t%4) (+1): d[4j + {0,1,2,3}]).
// TRANS = 0: both operands K-major; TRANS = 1: both MN-major.  scale_d = 0 overwrites D.
template <int TRANS>
__device__ __forceinline__ void wgmma_bf16(float (&d)[16], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
        "%16, %17, p, 1, 1, %19, %19;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(da), "l"(db), "r"(scale_d), "n"(TRANS)
        : "memory");
}

template <int TRANS>
__device__ __forceinline__ void wgmma_bf16(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "%32, %33, p, 1, 1, %35, %35;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(scale_d), "n"(TRANS)
        : "memory");
}

template <int TRANS>
__device__ __forceinline__ void wgmma_bf16(float (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, %67, %67;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(scale_d), "n"(TRANS)
        : "memory");
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
// cuTensorMapEncodeTiled through the runtime's driver entry point (no link against libcuda).  It is a driver-API call:
// the primary context is bound to the calling thread first, since that thread (e.g. the autograd worker) may not have
// run a runtime call yet.  Returns 0, or an error code through set_error naming `who`.
int tensor_map_encoder(const char* who, EncodeTiledFn* enc);

// Tensor map of a bf16 NHWC activation [B, H, W, C], box {atom, box_w, box_h, box_n} with element stride
// `elem_stride` on W and H (a strided box spans box_w x box_h elements and loads every elem_stride-th).  128-byte
// swizzle for a 64-channel atom, 64-byte for a 32-channel one.
int encode_nhwc_map(CUtensorMap* map, const char* who, const void* ptr, int B, int H, int W, int C, int atom, int box_w,
                    int box_h, int box_n, int elem_stride);

// Cut a GH x GW pixel grid into tiles of px pixels: TW = GW (whole rows), TH = min(px / GW, GH) rows, and TN samples
// when one tile holds whole images.  False when such tiles do not cover the grid exactly or a tile side spans more
// than the 256-element TMA box limit at element stride elem_stride.
static inline bool box_tiling(int GH, int GW, int px, int elem_stride, int& TW, int& TH, int& TN) {
    if (GW > px || GW < 1 || px % GW != 0) return false;
    TW = GW;
    TH = px / GW < GH ? px / GW : GH;
    if (GH % TH != 0) return false;
    TN = px / (TW * TH);
    if (TW * TH * TN != px) return false;
    return TW * elem_stride <= 256 && TH * elem_stride <= 256;
}

// Split n_pix_tiles pixel tiles into contiguous ranges so that `ctas` CTAs per range make one wave (one CTA per SM:
// the ring takes the shared memory); fewer, longer CTAs also mean fewer reductions of partial tiles.  Returns the
// tiles per range and sets `splits` to the number of ranges.
static inline int one_wave_split(int n_pix_tiles, int ctas, int& splits) {
    int s = num_sms() / ctas;
    if (s > n_pix_tiles) s = n_pix_tiles;
    if (s < 1) s = 1;
    const int per = (n_pix_tiles + s - 1) / s;
    splits = (n_pix_tiles + per - 1) / per;
    return per;
}

}  // namespace pidm
