// Convolutions of the U-Net on NHWC bf16 activations as implicit GEMMs on the Hopper tensor cores (wgmma), operands
// staged by TMA through an mbarrier ring, fp32 accumulators in registers.
//
//   y[b,h,w,n] = sum_{r,q,c} x[b, s*h+r-pad, s*w+q-pad, c] * Wp[n][(r*KW+q)*Cin + c] (+ bias[n]) (+ residual[b,h,w,n])
//
// One kernel covers every layer of the network and its dgrad: 3x3 / 1x1 / 7x7 stride-1 layers (ResnetBlock convs,
// res_conv, to_qkv, to_out, stem: reference unet_model.py:227,253,275,279,453), the 4x4/stride-2 down-sampling conv
// (:197, TMA elementStrides) and the 4x4/stride-2 transposed conv (:163, four output-parity classes).
//
// Tiling.  GEMM M = 128 output pixels, N = BN output channels, K = taps * Cin walked in K-steps.
//   plain mode     : the pixel tile is a TN x TH x TW box (TW = W); one K-step = one tap x BK channels; the A operand
//                    is ONE 4-D TMA box {BK, TW, TH, TN} at spatial offset (r-pad, q-pad) -- the im2col gather, the zero
//                    padding (TMA out-of-bounds fill) and the 128B/64B swizzle all happen in the copy engine.
//   row-group mode : (stride-1 KxK layers whose image splits into 16x8 tiles) one K-step = one kernel COLUMN q x BK
//                    channels; its A box holds (16 + KH - 1) x 8 pixels and the KH kernel rows are row-shifted views of
//                    that one shared-memory tile (a shift of 8 pixels = one swizzle period), so L2 -> SM operand
//                    traffic drops from KH*KW to KW*(16+KH-1)/16 tiles per output tile.
//   The B operand (K-major packed weights) is a 2-D TMA box per tap, or resident in shared memory for the whole kernel
//   when the layer has a single n-tile.  Both land in the canonical K-major swizzled layout that the wgmma descriptors
//   expect: no thread ever touches the operands.
//
// Persistent, warp-specialised (512 threads, one CTA per SM, tiles walked with stride gridDim.x):
//   warps 0-3    TMA producers (one elected lane each, K-step i belongs to producer i % 4), <= 12-stage mbarrier ring
//                that runs across tile boundaries
//   warps 4-11   two consumer warpgroups, wgmma.m64nBNk16 on rows 0-63 / 64-127 of the tile, descriptors advanced by
//                integer adds; each warp releases a ring stage once the wgmma group that read it has retired
//   warps 12-15  epilogue: parked fp32 tile -> +bias +residual -> GroupNorm sum / sum-of-squares (optional) -> bf16 ->
//                XOR-swizzled smem transpose -> 64/128-byte coalesced row-segment stores; it overlaps the main loop of
//                the next tile
#include "hopper.cuh"
#include "pidm.h"

namespace pidm {

constexpr int TC_BM = 128;
constexpr int TC_THREADS = 512;

struct TcClass {             // one output-parity class of a transposed (stride-2) gather: <= 16 taps
    int n_taps, off_h, off_w;
    signed char dh[16], dw[16];
    short ktap[16];          // tap index into the packed weights (k offset = ktap * Cin)
};

struct TcParams {
    int B, GH, GW;           // pixel grid that forms the GEMM M dimension (TW == GW)
    int Cin, Cout;
    int mode;                // 0: regular conv, taps by formula (KH, KW, pad), input sampled with in_stride
                             // 1: transposed gather, per-class tap tables, output scattered with out_scale / offsets
    int KH, KW, pad;
    int in_stride, out_scale;
    int Ho, Wo;              // spatial size of the output tensor
    int TW, TH, TN;          // pixel box; TW*TH*TN == 128
    int tiles_h, tiles_w;    // GH / TH, GW / TW
    // operand staging plan (see tc_plan):
    //   rg = 1  "row-group" mode for stride-1 KxK convs on 16x8 (rows x cols) pixel tiles: one A box of
    //           (TH + KH - 1) x TW pixels per kernel COLUMN q serves the KH vertical taps as row-shifted views of the
    //           same shared-memory tile (a shift of r rows = r * TW * row_bytes, a whole swizzle period), so the
    //           L2 -> SM operand traffic drops from KH*KW to KW * (TH + KH - 1) / TH tiles per output tile
    //   nb      B (weight) tiles consumed per K-step (KH in row-group mode, else 1)
    //   resident = 1: all weights of the CTA's (single) n-tile are loaded once into shared memory
    int rg, nb, a_bytes, stage_bytes, stages, resident, res_bytes;
    int operand_bytes;       // resident weights + ring, rounded up to 1 KB: the barriers / epilogue staging follow it
    int m_tiles, n_tiles, n_classes;   // persistent tile walk: tile = (cls * n_tiles + nt) * m_tiles + mt
    const float* bias;
    const __nv_bfloat16* residual;
    __nv_bfloat16* y;
    float* gn_sums;          // optional [B, G, 2]: GroupNorm sum / sum-of-squares of the output, fused into the epilogue
    int gn_cpg, gn_groups;   // channels per group, groups
    TcClass cls[4];
};

// GroupNorm statistics of one 32-channel chunk held by a warp (one pixel row per lane).  Per group the channels
// are summed in registers; the 2*NG partial sums of the 32 lanes are then reduced with a butterfly that halves the
// number of live values at every step (NV + log2-many shuffles instead of 5 per value), leaving value i on lanes
// {i*32/NV ...}; those lanes issue one atomic each.
template <int NV>
__device__ __forceinline__ float butterfly_reduce(float (&v)[NV], int lane) {
    // after the step with offset `off`, a lane keeps the half of its values selected by bit `off` of its lane id
    int n = NV;
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {
        if (n > 1) {
            const int half = n >> 1;
            const bool upper = (lane & off) != 0;
#pragma unroll
            for (int i = 0; i < NV / 2; ++i) {
                if (i < half) {
                    const float keep = upper ? v[i + half] : v[i];
                    const float send = upper ? v[i] : v[i + half];
                    v[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
                }
            }
            n = half;
        } else {
            v[0] += __shfl_xor_sync(0xffffffffu, v[0], off);
        }
    }
    return v[0];
}

template <int CPG>
__device__ __forceinline__ void gn_stats_chunk(const float* f, float* sums_b, int first_group, int lane) {
    constexpr int NG = (CPG >= 32) ? 1 : 32 / CPG;
    constexpr int W = (CPG >= 32) ? 32 : CPG;
    constexpr int NV = 2 * NG;                      // (sum, sumsq) per group: 2, 4, 8 or 16 values
    float v[NV];
#pragma unroll
    for (int gi = 0; gi < NG; ++gi) {
        float s = 0.f, ss = 0.f;
#pragma unroll
        for (int j = 0; j < W; ++j) { float x = f[gi * W + j]; s += x; ss += x * x; }
        v[2 * gi] = s; v[2 * gi + 1] = ss;
    }
    const float total = butterfly_reduce<NV>(v, lane);
    // value index held by this lane: built from the lane bits consumed while n > 1 (bit 16 first = most significant)
    int idx = 0, n = NV;
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {
        if (n > 1) { n >>= 1; if (lane & off) idx += n; }
    }
    // lanes that differ only in the bits consumed after n reached 1 hold the same total: the lowest one publishes
    constexpr int DUP = 32 / NV;
    if ((lane & (DUP - 1)) == 0) atomicAdd(sums_b + first_group * 2 + idx, total);
}

template <int BN, int BK>
struct TcCfg {
    static constexpr int SW = BK * 2;                                     // swizzle span in bytes (128 or 64)
    static constexpr int B_BYTES = BN * BK * 2;
    static constexpr int ACC_PITCH = BN + 4;                              // fp32 staging row: conflict-free float4 rows
    static constexpr int ACC_BYTES = TC_BM * ACC_PITCH * 4;
    static constexpr int SMEM_BYTES = 227 * 1024;                         // the per-block maximum of sm_90
};
// persistent kernel, one CTA per SM: the operand ring takes most of the shared memory so that the TMA producers run
// many K-steps (and tiles) ahead of the tensor cores; latency is hidden by the ring, not by co-resident CTAs
constexpr int TC_MAX_STAGES = 12;

// Persistent, warp-specialised implicit-GEMM convolution.  Tiles (m_tile, n_tile, class) are walked with a static
// stride of gridDim.x by all three roles in lock step:
//   warps 0-3   TMA producers: keep the smem ring full across tile boundaries
//   warps 4-11  two consumer warpgroups: wgmma of output rows 0-63 / 64-127 of the tile into register accumulators,
//               then the fp32 tile is parked in shared memory (acc_full) and the next tile's main loop starts
//   warps 12-15 epilogue: drain the parked tile while the tensor cores already work on the next one
template <int BN, int BK>
__global__ void __launch_bounds__(TC_THREADS, 1) conv_tc_kernel(const __grid_constant__ CUtensorMap map_x,
                                                                const __grid_constant__ CUtensorMap map_w, TcParams p) {
    using Cfg = TcCfg<BN, BK>;
    extern __shared__ unsigned char smem_raw[];
    const uint32_t pad_bytes = smem_pad_1024(smem_raw);
    unsigned char* wres = smem_raw + pad_bytes;              // resident weights (res_bytes, may be 0)
    unsigned char* ring = wres + p.res_bytes;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw + pad_bytes + p.operand_bytes);
    TmaRing tma{bars, bars + TC_MAX_STAGES};                 // full / empty barriers: [TC_MAX_STAGES] each
    uint64_t* acc_full = bars + 2 * TC_MAX_STAGES;           // the accumulator tile is parked in shared memory
    uint64_t* acc_empty = acc_full + 1;                      // ... and has been read back by the epilogue
    uint64_t* wfull = acc_empty + 1;                         // resident weights have landed
    unsigned char* stage_base = smem_raw + pad_bytes + p.operand_bytes + 512;   // 4 warps x 4 KB epilogue staging
    float* acc_tile = reinterpret_cast<float*>(stage_base + 4 * 4096);          // [TC_BM][ACC_PITCH] fp32
    const int n_stages = p.stages;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int kc_per_tap = p.Cin / BK;
    const int total_tiles = p.m_tiles * p.n_tiles * p.n_classes;
    pdl_trigger();

    if (warp == 0 && lane == 0) {
        prefetch_tensormap(&map_x);
        prefetch_tensormap(&map_w);
    }
    if (warp == 1 && lane == 0) {
        tma.init(n_stages);
        mbar_init(acc_full, 256);
        mbar_init(acc_empty, 128);
        mbar_init(wfull, 1);
        mbar_init_fence();
    }
    __syncthreads();
    pdl_wait();                 // prologue done; everything below reads what the previous kernel wrote

    if (warp < 4) {
        // ===== TMA producers: four warps, one elected lane each, K-step i belongs to producer i % 4 ================
        // (a single thread can only issue a K-step every ~600 cycles -- wait + expect_tx + 2 TMA -- which starves the
        //  tensor cores on the small-channel layers; the issue streams are independent)
        const uint32_t pidx = (uint32_t)warp;
        if (elect_one()) {
            if (p.resident && pidx == 0) {
                // all K tiles of the (single) n-tile: [tap][kc] boxes of BN x BK
                const int n_k = p.KH * p.KW * kc_per_tap;
                mbar_expect_tx(wfull, (uint32_t)(n_k * Cfg::B_BYTES));
                for (int i = 0; i < n_k; ++i) tma_load_2d(wres + (size_t)i * Cfg::B_BYTES, &map_w, wfull, i * BK, 0);
            }
            // ring position and whose turn it is are carried incrementally: no integer divisions in the loop.  Every
            // producer walks every stage; only the one whose turn it is loads it.
            uint32_t turn = 0;
            unsigned char* a_dst = ring;
            const int groups_m0 = p.rg ? p.KW : p.KH * p.KW;
            int tile_m = blockIdx.x % p.m_tiles, rest = blockIdx.x / p.m_tiles;      // tile = rest * m_tiles + tile_m
            const int step_m = gridDim.x % p.m_tiles, step_r = gridDim.x / p.m_tiles;
            for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
                const int n0 = (rest % p.n_tiles) * BN;
                const TcClass& cl = p.cls[rest / p.n_tiles];
                const int tw_idx = tile_m % p.tiles_w;
                const int t2 = tile_m / p.tiles_w;
                const int tb = t2 / p.tiles_h, th_idx = t2 - tb * p.tiles_h;
                const int b0 = tb * p.TN, hh0 = p.in_stride * th_idx * p.TH, ww0 = p.in_stride * tw_idx * p.TW;
                const int n_groups = (p.mode == 0) ? groups_m0 : cl.n_taps;
                int r = 0, q = 0;                              // mode 0, plain: tap (r, q) walked incrementally
                for (int g = 0; g < n_groups; ++g) {
                    int dh, dw, ktap;
                    if (p.mode == 0) {
                        if (p.rg) { dh = -p.pad; dw = g - p.pad; }
                        else { dh = r - p.pad; dw = q - p.pad; if (++q == p.KW) { q = 0; ++r; } }
                        ktap = g;
                    } else {
                        dh = cl.dh[g]; dw = cl.dw[g]; ktap = cl.ktap[g];
                    }
                    int kcol = ktap * p.Cin;
                    for (int kc = 0; kc < kc_per_tap; ++kc, kcol += BK) {
                        if (turn == pidx) {
                            uint64_t* full = tma.acquire((uint32_t)p.stage_bytes);
                            tma_load_4d(a_dst, &map_x, full, kc * BK, ww0 + dw, hh0 + dh, b0);
                            if (!p.resident) {
                                unsigned char* b_dst = a_dst + p.a_bytes;
                                int kj = kcol;
                                for (int j = 0; j < p.nb; ++j, kj += p.KW * p.Cin, b_dst += Cfg::B_BYTES)
                                    tma_load_2d(b_dst, &map_w, full, kj, n0);   // row-group mode: tap (r = j, q = g)
                            }
                        }
                        if (++turn == 4u) turn = 0;
                        if (tma.advance((uint32_t)n_stages)) a_dst = ring; else a_dst += p.stage_bytes;
                    }
                }
                tile_m += step_m; rest += step_r;
                if (tile_m >= p.m_tiles) { tile_m -= p.m_tiles; ++rest; }
            }
        }
    } else if (warp < 12) {
        // ===== consumers: warpgroup cg computes output rows [64 cg, 64 cg + 64) of every tile =====
        // The loop body is kept free of integer divisions and descriptor re-encoding: descriptors are advanced by adds
        // to their low word (16-byte units).  One wgmma group is kept in flight: the stage of K-step i - 1 is released
        // once the group of K-step i has been issued and the older one has retired.
        const int cg = (warp - 4) >> 2;
        constexpr uint32_t desc_hi = gmma_desc_hi<Cfg::SW>();
        const uint32_t row_half_lo = (uint32_t)(64 * BK * 2) >> 4;           // 64 pixel rows of the A tile
        const uint32_t ring_lo = gmma_desc_lo(smem_u32(ring), 16) + (uint32_t)cg * row_half_lo;
        const uint32_t wres_lo = gmma_desc_lo(smem_u32(wres), 16);
        const uint32_t stage_lo = (uint32_t)p.stage_bytes >> 4;
        const uint32_t a_shift_lo = (uint32_t)(p.TW * BK * 2) >> 4;      // one tile row of pixels
        const uint32_t b_off_lo = ((uint32_t)p.a_bytes >> 4) - (uint32_t)cg * row_half_lo;
        constexpr uint32_t b_tile_lo = (uint32_t)Cfg::B_BYTES >> 4;
        const uint32_t res_j_lo = (uint32_t)(p.KW * kc_per_tap) * b_tile_lo;   // resident: next kernel row
        const int groups_m0 = p.rg ? p.KW : p.KH * p.KW;
        const int nb = p.nb;
        const bool resident = p.resident != 0;
        // fragment -> staging tile: this thread's rows 64 cg + 16 (warp % 4) + lane / 4 (+ 8), columns 8 j + 2 (lane % 4)
        float* acc_row = acc_tile + (size_t)(64 * cg + 16 * (warp & 3) + (lane >> 2)) * Cfg::ACC_PITCH + 2 * (lane & 3);
        uint32_t a_lo = ring_lo;
        int rest = blockIdx.x / p.m_tiles, tile_m = blockIdx.x % p.m_tiles;
        const int step_m = gridDim.x % p.m_tiles, step_r = gridDim.x / p.m_tiles;
        int lt = 0;
        float acc[BN / 2];
        for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x, ++lt) {
            const int n_iters = ((p.mode == 0) ? groups_m0 : p.cls[rest / p.n_tiles].n_taps) * kc_per_tap;
            if (lt == 0 && resident) mbar_wait(wfull, 0);
            uint32_t accum = 0;
            uint32_t res_lo = wres_lo;                           // resident weights: tile (it) of kernel row 0
            for (int it = 0; it < n_iters; ++it, res_lo += b_tile_lo) {
                tma.wait_full();
                uint32_t aj = a_lo;
                uint32_t bj = resident ? res_lo : a_lo + b_off_lo;
                const uint32_t bj_step = resident ? res_j_lo : b_tile_lo;
                wgmma_fence();
                for (int j = 0; j < nb; ++j, aj += a_shift_lo, bj += bj_step) {
#pragma unroll
                    for (int k = 0; k < BK / 16; ++k) {
                        wgmma_bf16<0>(acc, gmma_desc(desc_hi, aj + 2 * k), gmma_desc(desc_hi, bj + 2 * k), accum);
                        accum = 1;
                    }
                }
                tma.consumed(it == 0, lane);
                if (tma.advance((uint32_t)n_stages)) a_lo = ring_lo; else a_lo += stage_lo;
            }
            wgmma_wait<0>();
            if (n_iters > 0) tma.release_held(lane);            // the ring runs on into the next tile
            mbar_wait(acc_empty, (lt & 1) ^ 1);                 // the epilogue has read the previous tile back
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
                *reinterpret_cast<float2*>(acc_row + 8 * j) = make_float2(acc[4 * j], acc[4 * j + 1]);
                *reinterpret_cast<float2*>(acc_row + 8 * Cfg::ACC_PITCH + 8 * j) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
            }
            mbar_arrive(acc_full);
            tile_m += step_m; rest += step_r;
            if (tile_m >= p.m_tiles) { tile_m -= p.m_tiles; ++rest; }
        }
    } else {
        // ===== epilogue: parked fp32 tile -> registers (+bias, +residual, GroupNorm statistics) -> bf16 -> global
        // A lane owns one accumulator row (pixel).  Writing its row straight to global memory would make every store
        // instruction touch 32 different lines (16 bytes each): the LSU, not HBM, bounds the wide-N layers that way.
        // Instead each warp stages its 32 rows x CH columns in a private, XOR-swizzled shared-memory tile and writes it
        // back with LPR lanes per row, i.e. whole 64/128-byte row segments per quarter-warp.  The residual is read the
        // same way (coalesced -> staged -> own row) so that it is still added in fp32 before the single rounding.
        constexpr int CH = BN >= 64 ? 64 : 32;        // columns per pass
        constexpr int LPR = CH / 8;                   // 16-byte units per staged row = lanes per row when storing
        constexpr int RPI = 32 / LPR;                 // rows per store instruction
        const int quarter = warp & 3;                 // rows [32 quarter, 32 quarter + 32) of the tile
        uint4* stage = reinterpret_cast<uint4*>(stage_base) + quarter * (32 * 8);
        const int m = quarter * 32 + lane;            // accumulator row = pixel within the tile
        const float* acc_src = acc_tile + (size_t)m * Cfg::ACC_PITCH;
        const int tn = m / (p.TH * p.TW);
        const int rem = m - tn * p.TH * p.TW;
        const int th = rem / p.TW, tw = rem - th * p.TW;
        const int my_sw = (LPR == 8) ? (lane & 7) : ((lane >> 1) & 3);
        const int sr = lane / LPR, su = lane % LPR;   // store phase: row within the group of RPI rows, 16-byte unit
        int tile_m = blockIdx.x % p.m_tiles, rest = blockIdx.x / p.m_tiles;
        const int step_m = gridDim.x % p.m_tiles, step_r = gridDim.x / p.m_tiles;
        int lt = 0;
        for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x, ++lt) {
            const int n0 = (rest % p.n_tiles) * BN;
            const TcClass& cl = p.cls[rest / p.n_tiles];
            const int tw_idx = tile_m % p.tiles_w;
            const int t2 = tile_m / p.tiles_w;
            const int tb = t2 / p.tiles_h, th_idx = t2 - tb * p.tiles_h;
            const int b = tb * p.TN + tn, h = th_idx * p.TH + th, w = tw_idx * p.TW + tw;
            const bool row_ok = (b < p.B) && (h < p.GH);
            const int oh = p.out_scale * h + cl.off_h, ow = p.out_scale * w + cl.off_w;
            const long long row_off = row_ok ? (long long)((((size_t)b * p.Ho + oh) * p.Wo + ow) * p.Cout + n0) : -1ll;
            // offsets of the rows this lane stores (row it * RPI + sr), -1 = masked
            long long st_off[LPR];
#pragma unroll
            for (int it = 0; it < LPR; ++it) st_off[it] = __shfl_sync(0xffffffffu, row_off, it * RPI + sr);
            mbar_wait(acc_full, lt & 1);
#pragma unroll 1
            for (int c = 0; c < BN; c += CH) {
                float f[CH];
#pragma unroll
                for (int j = 0; j < CH; j += 4) {
                    const float4 v = *reinterpret_cast<const float4*>(acc_src + c + j);
                    f[j] = row_ok ? v.x : 0.f; f[j + 1] = row_ok ? v.y : 0.f;
                    f[j + 2] = row_ok ? v.z : 0.f; f[j + 3] = row_ok ? v.w : 0.f;
                }
                // the last columns of the parked tile are in registers: hand the staging tile back to the consumers
                if (c + CH >= BN) mbar_arrive(acc_empty);
                if (p.bias && row_ok) {
#pragma unroll
                    for (int j = 0; j < CH; j += 4) {
                        const float4 bv = __ldg(reinterpret_cast<const float4*>(p.bias + n0 + c + j));
                        f[j] += bv.x; f[j + 1] += bv.y; f[j + 2] += bv.z; f[j + 3] += bv.w;
                    }
                }
                if (p.residual) {
#pragma unroll
                    for (int it = 0; it < LPR; ++it) {
                        const int r = it * RPI + sr;
                        const int sw = (LPR == 8) ? (r & 7) : ((r >> 1) & 3);
                        uint4 rv = make_uint4(0u, 0u, 0u, 0u);
                        if (st_off[it] >= 0) rv = *reinterpret_cast<const uint4*>(p.residual + st_off[it] + c + su * 8);
                        stage[r * LPR + (su ^ sw)] = rv;
                    }
                    __syncwarp();
#pragma unroll
                    for (int u = 0; u < LPR; ++u) {
                        const uint4 rv = stage[lane * LPR + (u ^ my_sw)];
                        const __nv_bfloat162* hp = reinterpret_cast<const __nv_bfloat162*>(&rv);
#pragma unroll
                        for (int k = 0; k < 4; ++k) {
                            f[u * 8 + 2 * k] += __low2float(hp[k]);
                            f[u * 8 + 2 * k + 1] += __high2float(hp[k]);
                        }
                    }
                    __syncwarp();
                }
                // bf16 rows -> swizzled staging tile
#pragma unroll
                for (int u = 0; u < LPR; ++u) {
                    uint4 pk;
                    __nv_bfloat162* hp = reinterpret_cast<__nv_bfloat162*>(&pk);
#pragma unroll
                    for (int k = 0; k < 4; ++k) hp[k] = __floats2bfloat162_rn(f[u * 8 + 2 * k], f[u * 8 + 2 * k + 1]);
                    stage[lane * LPR + (u ^ my_sw)] = pk;
                }
                __syncwarp();
#pragma unroll
                for (int it = 0; it < LPR; ++it) {
                    const int r = it * RPI + sr;
                    const int sw = (LPR == 8) ? (r & 7) : ((r >> 1) & 3);
                    if (st_off[it] >= 0)
                        *reinterpret_cast<uint4*>(p.y + st_off[it] + c + su * 8) = stage[r * LPR + (su ^ sw)];
                }
                if (p.gn_sums != nullptr && b < p.B) {        // warp-uniform: the 32 rows of a warp lie in one sample
                    float* sums_b = p.gn_sums + (size_t)b * p.gn_groups * 2;
#pragma unroll
                    for (int hh = 0; hh < CH / 32; ++hh) {
                        const int fg = (n0 + c + hh * 32) / p.gn_cpg;
                        const float* fh = f + hh * 32;
                        if (p.gn_cpg == 4) gn_stats_chunk<4>(fh, sums_b, fg, lane);
                        else if (p.gn_cpg == 8) gn_stats_chunk<8>(fh, sums_b, fg, lane);
                        else if (p.gn_cpg == 16) gn_stats_chunk<16>(fh, sums_b, fg, lane);
                        else gn_stats_chunk<32>(fh, sums_b, fg, lane);     // cpg >= 32 (multiple of 32): one group
                    }
                }
                __syncwarp();                                   // staging tile is reused by the next pass
            }
            tile_m += step_m; rest += step_r;
            if (tile_m >= p.m_tiles) { tile_m -= p.m_tiles; ++rest; }
        }
    }
}

// ---- host side ------------------------------------------------------------------------------------------
int tensor_map_encoder(const char* who, EncodeTiledFn* enc) {
    static thread_local bool ctx_bound = false;
    if (!ctx_bound) {
        PIDM_CUDA(cudaFree(0));
        ctx_bound = true;
    }
    static const EncodeTiledFn fn = [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        const bool ok = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
                        qres == cudaDriverEntryPointSuccess;
        return ok ? (EncodeTiledFn)p : nullptr;
    }();
    PIDM_REQUIRE(fn != nullptr, "%s: cuTensorMapEncodeTiled is not available from the driver", who);
    *enc = fn;
    return 0;
}

int encode_nhwc_map(CUtensorMap* map, const char* who, const void* ptr, int B, int H, int W, int C, int atom, int box_w,
                    int box_h, int box_n, int elem_stride) {
    EncodeTiledFn enc;
    if (int e = tensor_map_encoder(who, &enc)) return e;
    cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
    cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
    cuuint32_t box[4] = {(cuuint32_t)atom, (cuuint32_t)box_w, (cuuint32_t)box_h, (cuuint32_t)box_n};
    cuuint32_t es[4] = {1, (cuuint32_t)elem_stride, (cuuint32_t)elem_stride, 1};
    CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(ptr), dims, strides, box, es,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, atom == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    PIDM_REQUIRE(r == CUDA_SUCCESS, "%s: cuTensorMapEncodeTiled failed with %d", who, (int)r);
    return 0;
}

// resident weights + operand ring of an n-tile width (TcCfg<BN, *>::OPERAND_BYTES)
static int tc_operand_bytes(int bn) { return (227 * 1024 - 1024 - 512 - 4 * 4096 - TC_BM * (bn + 4) * 4) / 1024 * 1024; }

struct TcPlan {
    int TW, TH, TN, BN, BK;
    int rg, nb, a_bytes, stage_bytes, stages, resident, res_bytes, operand_bytes;
};

// GH x GW = pixel grid of the GEMM (output grid for regular convs, input grid for the transposed gather)
static bool tc_plan(int B, int GH, int GW, int Cin, int Cout, int KH, int KW, int mode, int in_stride, int classes,
                    TcPlan& pl) {
    if (Cin % 32 != 0 || Cout % 32 != 0) return false;
    pl.BK = (Cin % 64 == 0) ? 64 : 32;
    // row-group mode: stride-1 KxK (K > 1) convs whose image splits into 16-row x 8-column tiles
    pl.rg = (mode == 0 && in_stride == 1 && KH > 1 && KH <= 7 && GW % 8 == 0 && GH % 16 == 0) ? 1 : 0;
    if (pl.rg) {
        pl.TW = 8; pl.TH = 16; pl.TN = 1;
    } else if (!box_tiling(GH, GW, 128, in_stride, pl.TW, pl.TH, pl.TN)) {
        return false;
    }
    pl.nb = pl.rg ? KH : 1;
    pl.a_bytes = (pl.TH + (pl.rg ? KH - 1 : 0)) * pl.TW * pl.TN * pl.BK * 2;
    const long long K = (long long)KH * KW * Cin;
    const long long m_tiles = (long long)((B + pl.TN - 1) / pl.TN) * (GH / pl.TH) * (GW / pl.TW) * classes;
    // n-tile widths: a consumer warpgroup holds 64 x BN fp32 accumulators in registers, BN / 2 per thread
    const int cands[3] = {128, 64, 32};
    pl.BN = 0;
    for (int i = 0; i < 3; ++i) {
        const int bn = cands[i];
        if (Cout % bn != 0) continue;
        // weights resident in shared memory when the CTA only ever sees one n-tile and they leave room for the ring
        const long long wbytes = (long long)bn * K * 2;
        int resident = (mode == 0 && Cout == bn && wbytes <= 100 * 1024) ? 1 : 0;
        int stage = pl.a_bytes + (resident ? 0 : pl.nb * bn * pl.BK * 2);
        int stages = (int)((tc_operand_bytes(bn) - (resident ? wbytes : 0)) / stage);
        if (stages > TC_MAX_STAGES) stages = TC_MAX_STAGES;
        if (stages < 3) continue;
        pl.BN = bn; pl.resident = resident; pl.res_bytes = resident ? (int)wbytes : 0;
        pl.stage_bytes = stage; pl.stages = stages;
        pl.operand_bytes = (int)(((resident ? wbytes : 0) + (long long)stages * stage + 1023) / 1024 * 1024);
        // widest tile that still (nearly) fills the machine (one persistent CTA per SM): fewer, wider tiles re-read
        // the A operand less often, but a grid well short of one wave leaves SMs idle
        if (m_tiles * (Cout / bn) >= 128) break;
    }
    return pl.BN != 0;
}

template <int BN, int BK>
static int launch_tc(const CUtensorMap& mx, const CUtensorMap& mw, const TcParams& p, dim3 grid, cudaStream_t st) {
    PIDM_CUDA(allow_smem(conv_tc_kernel<BN, BK>, TcCfg<BN, BK>::SMEM_BYTES));
    const size_t smem = (size_t)p.operand_bytes + 1024 /*align slack*/ + 512 /*barriers*/ + 4 * 4096 /*epilogue staging*/ +
                        TcCfg<BN, BK>::ACC_BYTES;
    PIDM_CUDA(launch_pdl(conv_tc_kernel<BN, BK>, grid, dim3(TC_THREADS), smem, st, mx, mw, p));
    PIDM_LAUNCH_CHECK("conv2d_tc");
    return 0;
}

// geometry of one call -> (pixel grid, classes).  Returns false when the tensor-core kernel does not cover it.
static bool tc_geometry(int B, int H, int W, int Cin, int Ho, int Wo, int Cout, int KH, int KW, int stride, int pad,
                        int transposed, TcParams& p, TcPlan& pl, int& classes) {
    if (KH != KW) return false;
    p.B = B; p.Cin = Cin; p.Cout = Cout; p.KH = KH; p.KW = KW; p.pad = pad; p.Ho = Ho; p.Wo = Wo;
    for (int c = 0; c < 4; ++c) { p.cls[c].n_taps = 0; p.cls[c].off_h = 0; p.cls[c].off_w = 0; }
    if (!transposed) {
        if (stride != 1 && stride != 2) return false;
        if ((H + 2 * pad - KH) / stride + 1 != Ho || (W + 2 * pad - KW) / stride + 1 != Wo) return false;
        p.mode = 0; p.GH = Ho; p.GW = Wo; p.in_stride = stride; p.out_scale = 1; classes = 1;
    } else {
        // 4x4/s2/p1 style up-sampling: GEMM grid = output / 2 (= the input grid when pad = KH/2 - 1).  An input that
        // carries a wrapped 1-pixel halo (circular padding) is the same gather with pad + 2: the grid stays the
        // unpadded one and every class offset dh shifts by +1
        if (stride != 2 || (KH & 1) || (KW & 1) || (Ho & 1) || (Wo & 1)) return false;
        if (Ho != 2 * (H - 1) - 2 * pad + KH || Wo != 2 * (W - 1) - 2 * pad + KW) return false;
        p.mode = 1; p.GH = Ho / 2; p.GW = Wo / 2; p.in_stride = 1; p.out_scale = 2; classes = 4;
        for (int pa = 0; pa < 2; ++pa)
            for (int pb = 0; pb < 2; ++pb) {
                TcClass& c = p.cls[pa * 2 + pb];
                c.off_h = pa; c.off_w = pb;
                for (int r = 0; r < KH; ++r) {
                    if ((pa + pad - r) & 1) continue;
                    for (int q = 0; q < KW; ++q) {
                        if ((pb + pad - q) & 1) continue;
                        if (c.n_taps >= 16) return false;
                        c.dh[c.n_taps] = (signed char)((pa + pad - r) / 2);
                        c.dw[c.n_taps] = (signed char)((pb + pad - q) / 2);
                        c.ktap[c.n_taps] = (short)(r * KW + q);
                        ++c.n_taps;
                    }
                }
            }
    }
    if (!tc_plan(B, p.GH, p.GW, Cin, Cout, KH, KW, p.mode, p.in_stride, classes, pl)) return false;
    p.TW = pl.TW; p.TH = pl.TH; p.TN = pl.TN; p.tiles_h = p.GH / pl.TH; p.tiles_w = p.GW / pl.TW;
    p.rg = pl.rg; p.nb = pl.nb; p.a_bytes = pl.a_bytes; p.stage_bytes = pl.stage_bytes; p.stages = pl.stages;
    p.resident = pl.resident; p.res_bytes = pl.res_bytes; p.operand_bytes = pl.operand_bytes;
    p.m_tiles = ((B + pl.TN - 1) / pl.TN) * p.tiles_h * p.tiles_w;
    p.n_tiles = Cout / pl.BN;
    p.n_classes = classes;
    return true;
}

// persistent grid: one CTA per SM, or one per tile when there are fewer tiles than SMs
static int tc_grid(const TcParams& p) {
    const int total_tiles = p.m_tiles * p.n_tiles * p.n_classes;
    const int slots = num_sms();
    return total_tiles < slots ? total_tiles : slots;
}

static int tc_run(const void* x, const void* w_packed, const float* bias, const void* residual, void* y, int B, int H,
                  int W, int Cin, int Ho, int Wo, int Cout, int KH, int KW, int stride, int pad, int transposed,
                  float* gn_sums, int gn_groups, int gn_sums_zeroed, cudaStream_t st) {
    TcParams p;
    TcPlan pl;
    int classes = 1;
    PIDM_REQUIRE(tc_geometry(B, H, W, Cin, Ho, Wo, Cout, KH, KW, stride, pad, transposed, p, pl, classes),
                 "conv2d_tc: unsupported geometry");
    PIDM_REQUIRE(((uintptr_t)x & 15) == 0 && ((uintptr_t)w_packed & 15) == 0, "conv2d_tc: operands must be 16-byte aligned");
    CUtensorMap mx, mw;
    const int s = p.in_stride;
    const int box_h = pl.rg ? pl.TH + KH - 1 : pl.TH * s;
    if (int e = encode_nhwc_map(&mx, "conv2d_tc", x, B, H, W, Cin, pl.BK, pl.TW * s, box_h, pl.TN, s)) return e;
    {
        EncodeTiledFn enc;
        if (int e = tensor_map_encoder("conv2d_tc", &enc)) return e;
        const int K = KH * KW * Cin;
        cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)Cout};
        cuuint64_t strides[1] = {(cuuint64_t)K * 2};
        cuuint32_t box[2] = {(cuuint32_t)pl.BK, (cuuint32_t)pl.BN};
        cuuint32_t es[2] = {1, 1};
        CUresult r = enc(&mw, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(w_packed), dims, strides, box, es,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, pl.BK == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        PIDM_REQUIRE(r == CUDA_SUCCESS, "conv2d_tc: cuTensorMapEncodeTiled(w) failed with %d", (int)r);
    }
    p.bias = bias; p.residual = (const __nv_bfloat16*)residual; p.y = (__nv_bfloat16*)y;
    p.gn_sums = gn_sums; p.gn_groups = gn_groups; p.gn_cpg = gn_groups > 0 ? Cout / gn_groups : 0;
    if (gn_sums) {
        PIDM_REQUIRE(gn_groups > 0 && Cout % gn_groups == 0, "conv2d_tc: bad GroupNorm group count %d", gn_groups);
        const int cpg = p.gn_cpg;
        PIDM_REQUIRE(cpg == 4 || cpg == 8 || cpg == 16 || cpg % 32 == 0, "conv2d_tc: fused GroupNorm statistics need "
                     "4, 8, 16 or a multiple of 32 channels per group (got %d)", cpg);
        if (!gn_sums_zeroed) PIDM_CUDA(cudaMemsetAsync(gn_sums, 0, (size_t)B * gn_groups * 2 * sizeof(float), st));
    }
    dim3 grid(tc_grid(p));
#define TC_CASE(bn, bk) if (pl.BN == bn && pl.BK == bk) return launch_tc<bn, bk>(mx, mw, p, grid, st)
    TC_CASE(128, 64); TC_CASE(64, 64); TC_CASE(32, 64);
    TC_CASE(128, 32); TC_CASE(64, 32); TC_CASE(32, 32);
#undef TC_CASE
    return set_error(2, "conv2d_tc: no kernel for BN=%d BK=%d", pl.BN, pl.BK);
}

}  // namespace pidm
using namespace pidm;

extern "C" int pidm_conv2d_tc_general_supported(int B, int H, int W, int Cin, int Ho, int Wo, int Cout, int KH, int KW,
                                                int stride, int pad, int transposed) {
    TcParams p; TcPlan pl; int classes;
    return tc_geometry(B, H, W, Cin, Ho, Wo, Cout, KH, KW, stride, pad, transposed, p, pl, classes) ? 1 : 0;
}

extern "C" int pidm_conv2d_tc_plan(int B, int H, int W, int Cin, int Ho, int Wo, int Cout, int KH, int KW, int stride,
                                   int pad, int transposed, int* out) {
    TcParams p; TcPlan pl; int classes;
    PIDM_REQUIRE(tc_geometry(B, H, W, Cin, Ho, Wo, Cout, KH, KW, stride, pad, transposed, p, pl, classes),
                 "conv2d_tc_plan: unsupported geometry");
    const int v[10] = {pl.BN, pl.BK, pl.rg, pl.resident, pl.stages, p.m_tiles * p.n_tiles * p.n_classes, tc_grid(p),
                       pl.TN, pl.TH, pl.TW};
    for (int i = 0; i < 10; ++i) out[i] = v[i];
    return 0;
}

extern "C" int pidm_conv2d_tc_general(const void* x, const void* w_packed, const float* bias, const void* residual,
                                      void* y, int B, int H, int W, int Cin, int Ho, int Wo, int Cout, int KH, int KW,
                                      int stride, int pad, int transposed, float* gn_sums, int gn_groups,
                                      int gn_sums_zeroed, void* stream) {
    return tc_run(x, w_packed, bias, residual, y, B, H, W, Cin, Ho, Wo, Cout, KH, KW, stride, pad, transposed, gn_sums,
                  gn_groups, gn_sums_zeroed, (cudaStream_t)stream);
}
