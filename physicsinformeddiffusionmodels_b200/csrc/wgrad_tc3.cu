// Weight gradient of a stride-1 3x3 convolution on the Hopper tensor cores (wgmma), "tap-complete" tiling.
//
//   dW[co][ci][tap] += sum_{pixels m} dy[m][co] * x[m shifted by tap][ci]
//
// wgrad_tc.cu gives every CTA 128 rows of the (tap, ci) dimension; the rows of one CTA then belong to a few taps of
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
#include "hopper.cuh"
#include "pidm.h"

namespace pidm {

constexpr int W3_THREADS = 384;

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
__global__ void __launch_bounds__(W3_THREADS, 1) wgrad3_kernel(const __grid_constant__ CUtensorMap map_x,
                                                               const __grid_constant__ CUtensorMap map_dy, W3Params p) {
    using Cfg = W3Cfg<NP, AB, RG>;
    extern __shared__ unsigned char smem_raw[];
    const uint32_t raw_addr = smem_u32(smem_raw);
    unsigned char* ring = smem_raw + ((1024 - (raw_addr & 1023)) & 1023);
    uint64_t* bars = reinterpret_cast<uint64_t*>(ring + Cfg::STAGES * Cfg::STAGE_BYTES);
    uint64_t* full = bars;
    uint64_t* empty = bars + Cfg::STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    pdl_trigger();
    const int c0 = blockIdx.x * 32, n0 = blockIdx.y * NP;
    const int pt_begin = blockIdx.z * p.tiles_per_split;
    int pt_end = pt_begin + p.tiles_per_split;
    if (pt_end > p.n_pix_tiles) pt_end = p.n_pix_tiles;
    const int n_iters = pt_end - pt_begin;

    if (warp == 0 && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_x) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_dy) : "memory");
    }
    if (warp == 1 && lane == 0) {
        // a stage is free once all 8 consumer warps have retired the wgmmas that read it
        for (int s = 0; s < Cfg::STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
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
            uint32_t st = 0, ph = 0;
            unsigned char* stage = ring;
            for (int it = 0; it < n_iters; ++it) {
                mbar_wait(&empty[st], ph ^ 1);
                const int b0 = tb * p.TN, h0 = th_idx * p.TH, w0 = tw_idx * p.TW;
                unsigned char* a_dst = stage + Cfg::B_BYTES;
                mbar_expect_tx(&full[st], Cfg::TX_BYTES);
#pragma unroll
                for (int j = 0; j < Cfg::NBOX; ++j)
                    tma_load_4d(stage + j * Cfg::B_TILE, &map_dy, &full[st], n0 + j * AB, w0, h0, b0);
                if (RG) {
#pragma unroll
                    for (int q = 0; q < 3; ++q)
                        tma_load_4d(a_dst + q * Cfg::A_RG_ALLOC, &map_x, &full[st], c0, w0 + q - p.pad, h0 - p.pad, b0);
                } else {
#pragma unroll
                    for (int tap = 0; tap < 9; ++tap)
                        tma_load_4d(a_dst + tap * Cfg::A_ATOM, &map_x, &full[st], c0, w0 + tap % 3 - p.pad,
                                    h0 + tap / 3 - p.pad, b0);
                }
                if (++tw_idx == p.tiles_w) { tw_idx = 0; if (++th_idx == p.tiles_h) { th_idx = 0; ++tb; } }
                if (++st == (uint32_t)Cfg::STAGES) { st = 0; ph ^= 1; stage = ring; } else stage += Cfg::STAGE_BYTES;
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
        uint32_t st = 0, ph = 0, off_lo = 0, prev_st = 0;
        for (int it = 0; it < n_iters; ++it) {
            mbar_wait(&full[st], ph);
            wgmma_fence();
#pragma unroll
            for (int t = 0; t < 3; ++t) {
#pragma unroll
                for (int k = 0; k < Cfg::PX / 16; ++k)
                    wgmma_bf16<1>(acc[t], gmma_desc(a_hi, a_lo0 + off_lo + t * acc_lo + k * ka_lo),
                                  gmma_desc(b_hi, b_lo0 + off_lo + k * kb_lo), (it | k) != 0);
            }
            wgmma_commit();
            wgmma_wait<1>();
            if (it > 0 && lane == 0) mbar_arrive(&empty[prev_st]);
            prev_st = st;
            if (++st == (uint32_t)Cfg::STAGES) { st = 0; ph ^= 1; off_lo = 0; } else off_lo += stage_lo;
        }
        wgmma_wait<0>();
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

template <int NP, int AB, bool RG>
static int w3_launch(const CUtensorMap& mx, const CUtensorMap& my, const W3Params& p, dim3 grid, cudaStream_t st) {
    using Cfg = W3Cfg<NP, AB, RG>;
    PIDM_CUDA(allow_smem(wgrad3_kernel<NP, AB, RG>, Cfg::SMEM_BYTES));
    PIDM_CUDA(launch_pdl(wgrad3_kernel<NP, AB, RG>, grid, dim3(W3_THREADS), Cfg::SMEM_BYTES, st, mx, my, p));
    PIDM_LAUNCH_CHECK("conv2d_wgrad_tc(3x3)");
    return 0;
}

// Is this call covered?  a = x [B,HA,WA,CA], b = dy [B,GH,GW,CB], stride 1, 3x3, framework layout dw[cB][cA][tap]
// (s_row == 9), no channel padding.  a is either the unpadded input ("same" padding, pad 1, TMA zero fill) or a copy
// that already carries a 1-pixel halo (circular padding: HA = GH + 2, pad 0).
bool wgrad3_supported(int B, int HA, int WA, int CA, int CA_real, int GH, int GW, int CB, int KH, int KW, int a_stride,
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

// plan[11] = {NP, AA (= 32), AB, splits, tiles_per_split, n_pix_tiles, CTAs per split, row-group staging, TN, TH, TW}
void wgrad3_geometry(int B, int GH, int GW, int CA, int CB, int* plan) {
    W3Params p; bool rg; int NP, AB; dim3 grid;
    w3_geometry(B, GH, GW, CA, CB, p, rg, NP, AB, grid);
    const int v[11] = {NP, 32, AB, (int)grid.z, p.tiles_per_split, p.n_pix_tiles, (int)(grid.x * grid.y), rg ? 1 : 0,
                       p.TN, p.TH, p.TW};
    for (int i = 0; i < 11; ++i) plan[i] = v[i];
}

int wgrad3_run(const void* a, const void* b, float* dw, int B, int HA, int WA, int CA, int GH, int GW, int CB, int pad,
               long long s_col, cudaStream_t st) {
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
