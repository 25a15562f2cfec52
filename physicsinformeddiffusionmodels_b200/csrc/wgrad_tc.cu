// Weight gradient of a stride-1 "same" KxK convolution on the Hopper tensor cores (wgmma): a generic kernel and a
// tap-complete one for 3x3 layers (below), which pidm_conv2d_wgrad_tc runs wherever it applies.
//
//   dW[co][ci][tap] += sum_{pixels m} dy[m][co] * x[m shifted by tap][ci]
//
// GEMM view: D[M' = (tap, ci)][N' = co] = A^T B with the reduction dimension K' = pixels.  Both operands live in
// HBM pixel-major (NHWC), i.e. the M'/N' dimension (channels) is contiguous and K' (pixels) is strided: they are
// "MN-major" wgmma operands.  One K' step = one 128-pixel box (TN x TH x TW) fetched by TMA:
//   A: 128/ATOM_A shifted boxes of x  {ATOM_A channels, TW, TH, TN}, one per (tap, channel-chunk) pair of this M' tile
//   B: NP/ATOM_B boxes of dy          {ATOM_B channels, TW, TH, TN}
// Each box lands as [128 pixel rows][ATOM channels] with the 128B/64B swizzle = one column of MN-major swizzle atoms
// (8 pixel rows x ATOM channels); atoms along M'/N' are LBO = one box apart, along K' SBO = 8 rows apart.
// Warp 0 produces the ring; two consumer warpgroups each own 64 rows of M' and issue the 8 wgmmas (K' = 16 pixels
// each) of a stage into register accumulators.  CTAs split the pixel range (split-K) and add their partial D into the
// fp32 gradient with red.global.add (framework layout through strides), straight from the accumulator fragments.
#include "hopper.cuh"
#include "pidm.h"

namespace pidm {

constexpr int WG_THREADS = 384;

struct WgParams {
    int B, Cin, Cout;            // Cin = channels of the A-side (gathered) tensor, Cout = channels of the B-side tensor
    int c_real;                  // A-side channels >= c_real are padding (their rows are not written)
    int KH, KW, pad, a_stride;   // A-side pixel = a_stride * g - pad + tap for grid pixel g
    int TW, TH, TN, tiles_h;
    int n_pix_tiles, tiles_per_split;
    float* dw;
    long long s_row, s_col;      // dw index = cA*s_row + cB*s_col + tap
};

template <int NP, int ATOM_A, int ATOM_B>
struct WgCfg {
    static constexpr int NA = 128 / ATOM_A, NB = NP / ATOM_B;
    static constexpr int A_TILE = 128 * ATOM_A * 2, B_TILE = 128 * ATOM_B * 2;
    static constexpr int STAGE_BYTES = NA * A_TILE + NB * B_TILE;
    static constexpr int STAGES_RAW = (192 * 1024) / STAGE_BYTES;
    static constexpr int STAGES = STAGES_RAW > 4 ? 4 : STAGES_RAW;
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 + 256;
};

template <int NP, int ATOM_A, int ATOM_B>
__global__ void __launch_bounds__(WG_THREADS, 1) wgrad_tc_kernel(const __grid_constant__ CUtensorMap map_x,
                                                                 const __grid_constant__ CUtensorMap map_dy, WgParams p) {
    using Cfg = WgCfg<NP, ATOM_A, ATOM_B>;
    extern __shared__ unsigned char smem_raw[];
    unsigned char* ring = smem_raw + smem_pad_1024(smem_raw);
    uint64_t* bars = reinterpret_cast<uint64_t*>(ring + Cfg::STAGES * Cfg::STAGE_BYTES);
    TmaRing tma{bars, bars + Cfg::STAGES};

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    pdl_trigger();
    const int mt = blockIdx.x, n0 = blockIdx.y * NP;
    const int chunks = p.Cin / ATOM_A;                 // channel chunks per tap
    const int n_pairs = p.KH * p.KW * chunks;          // (tap, chunk) pairs = M' extent / ATOM_A
    const auto [pt_begin, n_iters] = split_k_range(p.tiles_per_split, p.n_pix_tiles);

    if (warp == 0 && lane == 0) {
        prefetch_tensormap(&map_x);
        prefetch_tensormap(&map_dy);
    }
    if (warp == 1 && lane == 0) {
        tma.init(Cfg::STAGES);
        mbar_init_fence();
    }
    __syncthreads();
    pdl_wait();

    if (n_iters <= 0) return;
    if (warp == 0) {
        if (elect_one()) {
            // per-box coordinates of this M' tile are loop invariant: resolve (tap, chunk) -> (c0, dw, dh) once
            int ac[Cfg::NA], aw[Cfg::NA], ah[Cfg::NA];
#pragma unroll
            for (int j = 0; j < Cfg::NA; ++j) {
                int pr = mt * Cfg::NA + j;
                if (pr >= n_pairs) pr = n_pairs - 1;          // padding rows of the last M' tile (discarded later)
                const int tap = pr / chunks, ch = pr - tap * chunks;
                const int r = tap / p.KW, q = tap - r * p.KW;
                ac[j] = ch * ATOM_A; aw[j] = q - p.pad; ah[j] = r - p.pad;
            }
            int tb = pt_begin / p.tiles_h, th_idx = pt_begin - tb * p.tiles_h;
            unsigned char* a_dst = ring;
            for (int it = 0; it < n_iters; ++it) {
                const int b0 = tb * p.TN, h0 = th_idx * p.TH;
                unsigned char* b_dst = a_dst + Cfg::NA * Cfg::A_TILE;
                uint64_t* full = tma.acquire(Cfg::STAGE_BYTES);
#pragma unroll
                for (int j = 0; j < Cfg::NA; ++j)
                    tma_load_4d(a_dst + j * Cfg::A_TILE, &map_x, full, ac[j], aw[j], p.a_stride * h0 + ah[j], b0);
#pragma unroll
                for (int j = 0; j < Cfg::NB; ++j)
                    tma_load_4d(b_dst + j * Cfg::B_TILE, &map_dy, full, n0 + j * ATOM_B, 0, h0, b0);
                if (++th_idx == p.tiles_h) { th_idx = 0; ++tb; }
                if (tma.advance(Cfg::STAGES)) a_dst = ring; else a_dst += Cfg::STAGE_BYTES;
            }
        }
    } else if (warp >= 4) {
        // ===== consumer warpgroup cg: M' rows [64 cg, 64 cg + 64) =====
        const int cg = (warp - 4) >> 2;
        // rows 64 cg.. start (64 / ATOM_A) * cg atoms into the A boxes
        const uint32_t a_lo0 = gmma_desc_lo(smem_u32(ring) + cg * (64 / ATOM_A) * Cfg::A_TILE, Cfg::A_TILE);
        const uint32_t b_lo0 = gmma_desc_lo(smem_u32(ring) + Cfg::NA * Cfg::A_TILE, Cfg::B_TILE);
        constexpr uint32_t a_hi = gmma_desc_hi<ATOM_A * 2>(), b_hi = gmma_desc_hi<ATOM_B * 2>();
        constexpr uint32_t stage_lo = Cfg::STAGE_BYTES >> 4;
        constexpr uint32_t ka_lo = (16 * ATOM_A * 2) >> 4, kb_lo = (16 * ATOM_B * 2) >> 4;
        float acc[NP / 2];
        uint32_t off_lo = 0;
        for (int it = 0; it < n_iters; ++it) {
            tma.wait_full();
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 8; ++k)        // 8 x 16 pixels
                wgmma_bf16<1>(acc, gmma_desc(a_hi, a_lo0 + off_lo + k * ka_lo), gmma_desc(b_hi, b_lo0 + off_lo + k * kb_lo),
                              (it | k) != 0);
            tma.consumed(it == 0, lane);
            if (tma.advance(Cfg::STAGES)) off_lo = 0; else off_lo += stage_lo;
        }
        wgmma_wait<0>();             // the kernel ends here: the last stage is never released
        // fragment rows: 64 cg + 16 (warp % 4) + lane / 4 + 8 i; columns 8 j + 2 (lane % 4) + e
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int mrow = 64 * cg + 16 * (warp & 3) + (lane >> 2) + 8 * i;    // = (pair j, channel within atom)
            const int j = mrow / ATOM_A, cl = mrow - j * ATOM_A;
            const int pr = mt * Cfg::NA + j;
            const int tap = (pr < n_pairs) ? pr / chunks : 0;
            const int ci = (pr < n_pairs) ? (pr - tap * chunks) * ATOM_A + cl : 0;
            if (pr >= n_pairs || ci >= p.c_real) continue;
            float* dst = p.dw + (long long)ci * p.s_row + tap + (long long)(n0 + 2 * (lane & 3)) * p.s_col;
#pragma unroll
            for (int jj = 0; jj < NP / 8; ++jj) {
                atomicAdd(dst + (long long)(8 * jj) * p.s_col, acc[4 * jj + 2 * i]);
                atomicAdd(dst + (long long)(8 * jj + 1) * p.s_col, acc[4 * jj + 2 * i + 1]);
            }
        }
    }
}

// ---- tap-complete 3x3 kernel ----------------------------------------------------------------------------------
// wgrad_tc_kernel gives every CTA 128 rows of the (tap, ci) dimension; the rows of one CTA then belong to a few taps of
// MANY input channels, their addresses in the framework layout [co][ci][tap] are 9 floats apart, and the split-K
// epilogue degenerates into scattered 4-byte red.global.add (16 K transactions per CTA; it dominated every layer
// with few pixels).  Here a CTA owns ALL nine taps of a 32-channel chunk of ci and an NP-wide tile of co:
//   * three accumulators (M = 128 rows each = 4 atoms of 32 channels; each of the two consumer warpgroups holds
//     rows 0-63 or 64-127 of all three in registers, so NP <= 64),
//   * for a fixed co its 9 x 32 results are 288 CONTIGUOUS floats of dW: the epilogue transposes through shared
//     memory and issues fully coalesced 128-byte reductions,
//   * the dy tile (B operand) is fetched once per K' step for all nine taps (it was fetched by three CTAs before).
// Two operand-staging modes:
//   RG = true  (image splits into 16x8 pixel tiles): per kernel COLUMN q one halo box of (16 + 3) x 8 pixels; the
//              three kernel rows r are row-shifted views of it -- atom j of accumulator q starts j * 8 pixel rows
//              further down, which the MN-major descriptor expresses as LBO = 8 rows (the 4th atom is discarded).
//   RG = false (small images, e.g. 8x8): nine separate boxes of 64 pixels, 12 atom slots (3 unused).
struct W3Params {
    int B, pad;
    int TW, TH, TN, tiles_h, tiles_w;    // pixel tile of one K' step and the tile grid per TN samples
    int n_pix_tiles, tiles_per_split;
    float* dw;
    long long s_col;                     // dw index = cB * s_col + cA * 9 + tap
};

template <int NP, int AB, bool RG>
struct W3Cfg {
    static constexpr int PX = RG ? 128 : 64;                      // pixels per K' step
    static constexpr int A_ATOM = PX * 64;                        // [PX][32 ch] bf16 (RG = false)
    static constexpr int A_BOX_RG = 19 * 8 * 64;                  // (16 + 3) rows x 8 pixels x 32 ch
    static constexpr int A_RG_ALLOC = 10240;
    static constexpr int A_BYTES = RG ? 3 * A_RG_ALLOC : 12 * A_ATOM;
    static constexpr int NBOX = NP / AB;
    static constexpr int B_TILE = PX * AB * 2;
    static constexpr int B_BYTES = NBOX * B_TILE;
    static constexpr int STAGE_BYTES = B_BYTES + A_BYTES;         // B tiles first (they need the stricter alignment)
    static constexpr int TX_BYTES = B_BYTES + (RG ? 3 * A_BOX_RG : 9 * A_ATOM);
    static constexpr int STAGES_RAW = (184 * 1024) / STAGE_BYTES;
    static constexpr int STAGES = STAGES_RAW > 4 ? 4 : STAGES_RAW;
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 + 256;
    static_assert(STAGES * STAGE_BYTES >= 32 * 288 * 4, "epilogue staging must fit in the ring");
};

template <int NP, int AB, bool RG>
__global__ void __launch_bounds__(WG_THREADS, 1) wgrad3_kernel(const __grid_constant__ CUtensorMap map_x,
                                                               const __grid_constant__ CUtensorMap map_dy, W3Params p) {
    using Cfg = W3Cfg<NP, AB, RG>;
    extern __shared__ unsigned char smem_raw[];
    unsigned char* ring = smem_raw + smem_pad_1024(smem_raw);
    uint64_t* bars = reinterpret_cast<uint64_t*>(ring + Cfg::STAGES * Cfg::STAGE_BYTES);
    TmaRing tma{bars, bars + Cfg::STAGES};

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    pdl_trigger();
    const int c0 = blockIdx.x * 32, n0 = blockIdx.y * NP;
    const auto [pt_begin, n_iters] = split_k_range(p.tiles_per_split, p.n_pix_tiles);

    if (warp == 0 && lane == 0) {
        prefetch_tensormap(&map_x);
        prefetch_tensormap(&map_dy);
    }
    if (warp == 1 && lane == 0) {
        tma.init(Cfg::STAGES);
        mbar_init_fence();
    }
    __syncthreads();
    pdl_wait();

    if (n_iters <= 0) return;
    if (warp == 0) {
        if (elect_one()) {
            // pixel tile index -> (sample group, tile row, tile column), walked incrementally
            int tw_idx = pt_begin % p.tiles_w;
            int t2 = pt_begin / p.tiles_w;
            int th_idx = t2 % p.tiles_h, tb = t2 / p.tiles_h;
            unsigned char* stage = ring;
            for (int it = 0; it < n_iters; ++it) {
                uint64_t* full = tma.acquire(Cfg::TX_BYTES);
                const int b0 = tb * p.TN, h0 = th_idx * p.TH, w0 = tw_idx * p.TW;
                unsigned char* a_dst = stage + Cfg::B_BYTES;
#pragma unroll
                for (int j = 0; j < Cfg::NBOX; ++j)
                    tma_load_4d(stage + j * Cfg::B_TILE, &map_dy, full, n0 + j * AB, w0, h0, b0);
                if (RG) {
#pragma unroll
                    for (int q = 0; q < 3; ++q)
                        tma_load_4d(a_dst + q * Cfg::A_RG_ALLOC, &map_x, full, c0, w0 + q - p.pad, h0 - p.pad, b0);
                } else {
#pragma unroll
                    for (int tap = 0; tap < 9; ++tap)
                        tma_load_4d(a_dst + tap * Cfg::A_ATOM, &map_x, full, c0, w0 + tap % 3 - p.pad,
                                    h0 + tap / 3 - p.pad, b0);
                }
                if (++tw_idx == p.tiles_w) { tw_idx = 0; if (++th_idx == p.tiles_h) { th_idx = 0; ++tb; } }
                if (tma.advance(Cfg::STAGES)) stage = ring; else stage += Cfg::STAGE_BYTES;
            }
        }
    } else if (warp >= 4) {
        // ===== consumer warpgroup cg: rows [64 cg, 64 cg + 64) = atoms 2 cg, 2 cg + 1 of each accumulator =====
        const int cg = (warp - 4) >> 2;
        const uint32_t ring_addr = smem_u32(ring);
        // accumulator t: RG -> halo box of kernel column t, atoms (kernel rows) 8 pixel rows = 512 B apart;
        //                else -> atom slots 4t .. 4t+3, one atom apart
        constexpr uint32_t a_lbo = RG ? 8 * 64 : Cfg::A_ATOM;
        constexpr uint32_t a_acc_stride = RG ? Cfg::A_RG_ALLOC : 4 * Cfg::A_ATOM;
        const uint32_t a_lo0 = gmma_desc_lo(ring_addr + Cfg::B_BYTES + 2 * cg * a_lbo, a_lbo);
        const uint32_t b_lo0 = gmma_desc_lo(ring_addr, Cfg::B_TILE);
        constexpr uint32_t a_hi = gmma_desc_hi<64>(), b_hi = gmma_desc_hi<AB * 2>();
        constexpr uint32_t stage_lo = Cfg::STAGE_BYTES >> 4;
        constexpr uint32_t ka_lo = (16 * 64) >> 4, kb_lo = (16 * AB * 2) >> 4, acc_lo = a_acc_stride >> 4;
        float acc[3][NP / 2];
        uint32_t off_lo = 0;
        for (int it = 0; it < n_iters; ++it) {
            tma.wait_full();
            wgmma_fence();
#pragma unroll
            for (int t = 0; t < 3; ++t) {
#pragma unroll
                for (int k = 0; k < Cfg::PX / 16; ++k)
                    wgmma_bf16<1>(acc[t], gmma_desc(a_hi, a_lo0 + off_lo + t * acc_lo + k * ka_lo),
                                  gmma_desc(b_hi, b_lo0 + off_lo + k * kb_lo), (it | k) != 0);
            }
            tma.consumed(it == 0, lane);
            if (tma.advance(Cfg::STAGES)) off_lo = 0; else off_lo += stage_lo;
        }
        wgmma_wait<0>();             // the kernel ends here: the last stage is never released
        // ===== epilogue: both warpgroups are done with the ring, which now stages S[32 co][ci * 9 + tap]
        named_bar(1, 256);
        float* S = reinterpret_cast<float*>(ring);
        const int cw = warp - 4;                                   // consumer warp 0..7
#pragma unroll
        for (int c = 0; c < NP; c += 32) {
            // fragment rows 64 cg + 16 (warp % 4) + lane / 4 + 8 i = (atom quarter, channel ci); columns 8 j + 2 (lane % 4)
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int row = 64 * cg + 16 * (warp & 3) + (lane >> 2) + 8 * i;
                const int quarter = row >> 5, ci = row & 31;
#pragma unroll
                for (int t = 0; t < 3; ++t) {
                    const int tap = RG ? quarter * 3 + t : t * 4 + quarter;        // RG: (r = quarter, q = t)
                    const bool valid = RG ? quarter < 3 : tap < 9;
                    if (!valid) continue;
#pragma unroll
                    for (int j = c / 8; j < c / 8 + 4; ++j) {
                        const int col = 8 * j + 2 * (lane & 3) - c;
                        S[col * 288 + ci * 9 + tap] = acc[t][4 * j + 2 * i];
                        S[(col + 1) * 288 + ci * 9 + tap] = acc[t][4 * j + 2 * i + 1];
                    }
                }
            }
            named_bar(1, 256);
            // 288 contiguous floats of dW per co: coalesced reductions, 4 output channels per warp
#pragma unroll 1
            for (int j = cw; j < 32; j += 8) {
                float* dst = p.dw + (long long)(n0 + c + j) * p.s_col + (long long)c0 * 9;
#pragma unroll
                for (int i = 0; i < 9; ++i) atomicAdd(dst + i * 32 + lane, S[j * 288 + i * 32 + lane]);
            }
            named_bar(1, 256);
        }
    }
}

// bias gradient: db[c] += sum_m dy[m][c]   (column sums of an NHWC tensor)
template <typename T>
__global__ void colsum_kernel(const T* __restrict__ dy, float* __restrict__ out, long long M, int C) {
    extern __shared__ float sacc[];   // [C]
    pdl_trigger();
    pdl_wait();
    const int oct = C / 8;
    const int o = threadIdx.x % oct, r0 = threadIdx.x / oct, rows = blockDim.x / oct;
    for (int i = threadIdx.x; i < C; i += blockDim.x) sacc[i] = 0.f;
    __syncthreads();
    float a[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    // four independent row loads in flight per thread (one load per iteration left the kernel waiting on one memory
    // round trip per ~38 k rows)
    const long long stride = (long long)gridDim.x * rows;
    for (long long m = (long long)blockIdx.x * rows + r0; m < M; m += 4 * stride) {
        float v[4][8];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            if (m + u * stride < M) ld8(dy + (m + u * stride) * C + o * 8, v[u]);
            else {
#pragma unroll
                for (int k = 0; k < 8; ++k) v[u][k] = 0.f;
            }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u)
#pragma unroll
            for (int k = 0; k < 8; ++k) a[k] += v[u][k];
    }
    if (reduce_same_octet(a, oct)) {
#pragma unroll
        for (int k = 0; k < 8; ++k) atomicAdd(&sacc[o * 8 + k], a[k]);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < C; i += blockDim.x) atomicAdd(&out[i], sacc[i]);
}

struct WgPlan { int TW, TH, TN, NP, AA, AB; };

// GH x GW: pixel grid of the reduction (the B-side tensor's spatial size); the A side is sampled at a_stride*g-pad+tap
static bool wg_plan(int B, int GH, int GW, int CA, int CB, int a_stride, WgPlan& pl) {
    if (CA % 32 != 0 || CB % 32 != 0) return false;
    if (a_stride != 1 && a_stride != 2) return false;
    if (!box_tiling(GH, GW, 128, a_stride, pl.TW, pl.TH, pl.TN)) return false;
    pl.AA = (CA % 64 == 0) ? 64 : 32;
    pl.AB = (CB % 64 == 0) ? 64 : 32;
    pl.NP = (CB % 128 == 0) ? 128 : ((CB % 64 == 0) ? 64 : 32);
    return true;
}

template <int NP, int AA, int AB>
static int wg_launch(const CUtensorMap& mx, const CUtensorMap& my, const WgParams& p, dim3 grid, cudaStream_t st) {
    using Cfg = WgCfg<NP, AA, AB>;
    PIDM_CUDA(allow_smem(wgrad_tc_kernel<NP, AA, AB>, Cfg::SMEM_BYTES));
    PIDM_CUDA(launch_pdl(wgrad_tc_kernel<NP, AA, AB>, grid, dim3(WG_THREADS), Cfg::SMEM_BYTES, st, mx, my, p));
    PIDM_LAUNCH_CHECK("conv2d_wgrad_tc");
    return 0;
}

// launch geometry of the generic kernel: M' tiles x n-tiles x pixel splits
static bool wg_geometry(int B, int GH, int GW, int CA, int CB, int KH, int KW, int a_stride, WgPlan& pl, WgParams& p,
                        dim3& grid) {
    if (KH != KW || !wg_plan(B, GH, GW, CA, CB, a_stride, pl)) return false;
    p.TW = pl.TW; p.TH = pl.TH; p.TN = pl.TN; p.tiles_h = GH / pl.TH;
    p.n_pix_tiles = ((B + pl.TN - 1) / pl.TN) * p.tiles_h;
    const int na = 128 / pl.AA;
    const int n_pairs = KH * KW * (CA / pl.AA);
    const int m_tiles = (n_pairs + na - 1) / na;
    const int n_tiles = CB / pl.NP;
    int splits;
    p.tiles_per_split = one_wave_split(p.n_pix_tiles, m_tiles * n_tiles, splits);
    grid = dim3(m_tiles, n_tiles, splits);
    return true;
}

template <int NP, int AB, bool RG>
static int w3_launch(const CUtensorMap& mx, const CUtensorMap& my, const W3Params& p, dim3 grid, cudaStream_t st) {
    using Cfg = W3Cfg<NP, AB, RG>;
    PIDM_CUDA(allow_smem(wgrad3_kernel<NP, AB, RG>, Cfg::SMEM_BYTES));
    PIDM_CUDA(launch_pdl(wgrad3_kernel<NP, AB, RG>, grid, dim3(WG_THREADS), Cfg::SMEM_BYTES, st, mx, my, p));
    PIDM_LAUNCH_CHECK("conv2d_wgrad_tc(3x3)");
    return 0;
}

// Is this call covered?  a = x [B,HA,WA,CA], b = dy [B,GH,GW,CB], stride 1, 3x3, framework layout dw[cB][cA][tap]
// (s_row == 9), no channel padding.  a is either the unpadded input ("same" padding, pad 1, TMA zero fill) or a copy
// that already carries a 1-pixel halo (circular padding: HA = GH + 2, pad 0).
static bool wgrad3_supported(int B, int HA, int WA, int CA, int CA_real, int GH, int GW, int CB, int KH, int KW, int a_stride,
                             int pad, long long s_row) {
    if (KH != 3 || KW != 3 || a_stride != 1 || s_row != 9) return false;
    const bool same = pad == 1 && HA == GH && WA == GW;
    const bool halo = pad == 0 && HA == GH + 2 && WA == GW + 2;
    if (CA % 32 != 0 || CA_real != CA || CB % 32 != 0 || !(same || halo)) return false;
    if (GW % 8 == 0 && GH % 16 == 0) return true;                       // RG
    int TW, TH, TN;
    return box_tiling(GH, GW, 64, 1, TW, TH, TN) && B % TN == 0;
}

// tile plan and launch grid of a supported call
static void w3_geometry(int B, int GH, int GW, int CA, int CB, W3Params& p, bool& rg, int& NP, int& AB, dim3& grid) {
    rg = (GW % 8 == 0 && GH % 16 == 0);
    p.B = B;
    if (rg) { p.TW = 8; p.TH = 16; p.TN = 1; }
    else box_tiling(GH, GW, 64, 1, p.TW, p.TH, p.TN);      // true: wgrad3_supported
    p.tiles_h = GH / p.TH; p.tiles_w = GW / p.TW;
    p.n_pix_tiles = (B / p.TN) * p.tiles_h * p.tiles_w;
    NP = (CB % 64 == 0) ? 64 : 32;          // 3 x NP / 2 accumulator registers per consumer thread
    AB = (CB % 64 == 0) ? 64 : 32;
    const int chunks = CA / 32, n_tiles = CB / NP;
    int splits;
    p.tiles_per_split = one_wave_split(p.n_pix_tiles, chunks * n_tiles, splits);
    grid = dim3(chunks, n_tiles, splits);
}

static int wgrad3_run(const void* a, const void* b, float* dw, int B, int HA, int WA, int CA, int GH, int GW, int CB,
                      int pad, long long s_col, cudaStream_t st) {
    W3Params p;
    bool rg;
    int NP, AB;
    dim3 grid;
    w3_geometry(B, GH, GW, CA, CB, p, rg, NP, AB, grid);
    p.pad = pad;
    p.dw = dw; p.s_col = s_col;
    CUtensorMap mx, my;
    if (int e = encode_nhwc_map(&mx, "wgrad3", a, B, HA, WA, CA, 32, p.TW, rg ? p.TH + 3 : p.TH, p.TN, 1)) return e;
    if (int e = encode_nhwc_map(&my, "wgrad3", b, B, GH, GW, CB, AB, p.TW, p.TH, p.TN, 1)) return e;
#define W3_CASE(np, ab) \
    if (NP == np && AB == ab) return rg ? w3_launch<np, ab, true>(mx, my, p, grid, st) : w3_launch<np, ab, false>(mx, my, p, grid, st)
    W3_CASE(64, 64); W3_CASE(32, 32);
#undef W3_CASE
    return set_error(2, "wgrad3: no kernel for NP=%d AB=%d", NP, AB);
}

}  // namespace pidm
using namespace pidm;

extern "C" int pidm_conv2d_wgrad_tc_supported(int B, int GH, int GW, int CA, int CB, int KH, int KW, int a_stride) {
    WgPlan pl;
    return (KH == KW && wg_plan(B, GH, GW, CA, CB, a_stride, pl)) ? 1 : 0;
}

// plan of one pidm_conv2d_wgrad_tc call: out[12] = {wgrad3, NP, AA, AB, splits, tiles_per_split, n_pix_tiles,
// CTAs per split, row-group staging (wgrad3 only), TN, TH, TW}
extern "C" int pidm_conv2d_wgrad_tc_plan(int B, int HA, int WA, int CA, int CA_real, int GH, int GW, int CB, int KH,
                                         int KW, int a_stride, int pad, long long s_row, long long s_col, int* out) {
    (void)s_col;
    if (wgrad3_supported(B, HA, WA, CA, CA_real, GH, GW, CB, KH, KW, a_stride, pad, s_row)) {
        W3Params p; bool rg; int NP, AB; dim3 grid;
        w3_geometry(B, GH, GW, CA, CB, p, rg, NP, AB, grid);
        const int v[12] = {1, NP, 32, AB, (int)grid.z, p.tiles_per_split, p.n_pix_tiles, (int)(grid.x * grid.y), rg ? 1 : 0,
                           p.TN, p.TH, p.TW};
        for (int i = 0; i < 12; ++i) out[i] = v[i];
        return 0;
    }
    WgPlan pl; WgParams p; dim3 grid;
    PIDM_REQUIRE(wg_geometry(B, GH, GW, CA, CB, KH, KW, a_stride, pl, p, grid), "conv2d_wgrad_tc_plan: unsupported geometry");
    const int v[12] = {0, pl.NP, pl.AA, pl.AB, (int)grid.z, p.tiles_per_split, p.n_pix_tiles, (int)(grid.x * grid.y), 0,
                       pl.TN, pl.TH, pl.TW};
    for (int i = 0; i < 12; ++i) out[i] = v[i];
    return 0;
}

// D[(tap, cA)][cB] = sum over grid pixels g of a[a_stride*g - pad + tap][cA] * b[g][cB], ACCUMULATED into
// dw[cA*s_row + cB*s_col + tap] (fp32).  a: [B,HA,WA,CA] bf16 (CA may be channel-padded: rows >= CA_real are dropped),
// b: [B,GH,GW,CB] bf16.
extern "C" int pidm_conv2d_wgrad_tc(const void* a, const void* b, float* dw, int B, int HA, int WA, int CA, int CA_real,
                                    int GH, int GW, int CB, int KH, int KW, int a_stride, int pad, long long s_row,
                                    long long s_col, void* stream) {
    if (wgrad3_supported(B, HA, WA, CA, CA_real, GH, GW, CB, KH, KW, a_stride, pad, s_row))
        return wgrad3_run(a, b, dw, B, HA, WA, CA, GH, GW, CB, pad, s_col, (cudaStream_t)stream);
    WgPlan pl;
    WgParams p;
    dim3 grid;
    PIDM_REQUIRE(wg_geometry(B, GH, GW, CA, CB, KH, KW, a_stride, pl, p, grid), "conv2d_wgrad_tc: unsupported geometry");
    cudaStream_t st = (cudaStream_t)stream;
    CUtensorMap mx, my;
    if (int e = encode_nhwc_map(&mx, "wgrad_tc", a, B, HA, WA, CA, pl.AA, pl.TW * a_stride, pl.TH * a_stride, pl.TN,
                                a_stride))
        return e;
    if (int e = encode_nhwc_map(&my, "wgrad_tc", b, B, GH, GW, CB, pl.AB, pl.TW, pl.TH, pl.TN, 1)) return e;
    p.B = B; p.Cin = CA; p.Cout = CB; p.c_real = CA_real; p.KH = KH; p.KW = KW; p.pad = pad; p.a_stride = a_stride;
    p.dw = dw; p.s_row = s_row; p.s_col = s_col;
#define WG_CASE(np, aa, ab) if (pl.NP == np && pl.AA == aa && pl.AB == ab) return wg_launch<np, aa, ab>(mx, my, p, grid, st)
    WG_CASE(128, 64, 64); WG_CASE(128, 32, 64); WG_CASE(64, 64, 64); WG_CASE(64, 32, 64);
    WG_CASE(32, 64, 32); WG_CASE(32, 32, 32);
#undef WG_CASE
    return set_error(2, "conv2d_wgrad_tc: no kernel for NP=%d AA=%d AB=%d", pl.NP, pl.AA, pl.AB);
}

// out[c] += sum_m x[m][c]   (bias gradient: column sums of an NHWC tensor)
extern "C" int pidm_colsum(const void* x, float* out, long long M, int C, int dtype, void* stream) {
    PIDM_REQUIRE(C % 8 == 0 && C / 8 <= 1024, "colsum: C must be a multiple of 8");
    int oct = C / 8, rows = 256 / oct;
    if (rows < 1) rows = 1;
    int grid1 = (int)((M + rows * 8 - 1) / (rows * 8));
    if (grid1 > num_sms() * 4) grid1 = num_sms() * 4;
    if (grid1 < 1) grid1 = 1;
    PIDM_DISPATCH_DTYPE(dtype, PIDM_CUDA(launch_pdl(colsum_kernel<T>, dim3(grid1), dim3(oct * rows), C * sizeof(float),
                                                    (cudaStream_t)stream, (const T*)x, out, M, C)));
    PIDM_LAUNCH_CHECK("colsum");
    return 0;
}
