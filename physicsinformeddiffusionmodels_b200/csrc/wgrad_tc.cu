// Weight gradient of a stride-1 "same" KxK convolution on the Hopper tensor cores (wgmma).
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
    const uint32_t raw_addr = smem_u32(smem_raw);
    unsigned char* ring = smem_raw + ((1024 - (raw_addr & 1023)) & 1023);
    uint64_t* bars = reinterpret_cast<uint64_t*>(ring + Cfg::STAGES * Cfg::STAGE_BYTES);
    uint64_t* full = bars;
    uint64_t* empty = bars + Cfg::STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    pdl_trigger();
    const int mt = blockIdx.x, n0 = blockIdx.y * NP;
    const int chunks = p.Cin / ATOM_A;                 // channel chunks per tap
    const int n_pairs = p.KH * p.KW * chunks;          // (tap, chunk) pairs = M' extent / ATOM_A
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
            uint32_t st = 0, ph = 0;
            unsigned char* a_dst = ring;
            for (int it = 0; it < n_iters; ++it) {
                mbar_wait(&empty[st], ph ^ 1);
                const int b0 = tb * p.TN, h0 = th_idx * p.TH;
                unsigned char* b_dst = a_dst + Cfg::NA * Cfg::A_TILE;
                mbar_expect_tx(&full[st], Cfg::STAGE_BYTES);
#pragma unroll
                for (int j = 0; j < Cfg::NA; ++j)
                    tma_load_4d(a_dst + j * Cfg::A_TILE, &map_x, &full[st], ac[j], aw[j], p.a_stride * h0 + ah[j], b0);
#pragma unroll
                for (int j = 0; j < Cfg::NB; ++j)
                    tma_load_4d(b_dst + j * Cfg::B_TILE, &map_dy, &full[st], n0 + j * ATOM_B, 0, h0, b0);
                if (++th_idx == p.tiles_h) { th_idx = 0; ++tb; }
                if (++st == (uint32_t)Cfg::STAGES) { st = 0; ph ^= 1; a_dst = ring; } else a_dst += Cfg::STAGE_BYTES;
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
        uint32_t st = 0, ph = 0, off_lo = 0, prev_st = 0;
        for (int it = 0; it < n_iters; ++it) {
            mbar_wait(&full[st], ph);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 8; ++k)        // 8 x 16 pixels
                wgmma_bf16<1>(acc, gmma_desc(a_hi, a_lo0 + off_lo + k * ka_lo), gmma_desc(b_hi, b_lo0 + off_lo + k * kb_lo),
                              (it | k) != 0);
            wgmma_commit();
            wgmma_wait<1>();
            if (it > 0 && lane == 0) mbar_arrive(&empty[prev_st]);
            prev_st = st;
            if (++st == (uint32_t)Cfg::STAGES) { st = 0; ph ^= 1; off_lo = 0; } else off_lo += stage_lo;
        }
        wgmma_wait<0>();
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

// tap-complete 3x3 kernel (wgrad_tc3.cu)
bool wgrad3_supported(int B, int HA, int WA, int CA, int CA_real, int GH, int GW, int CB, int KH, int KW, int a_stride,
                      int pad, long long s_row);
void wgrad3_geometry(int B, int GH, int GW, int CA, int CB, int* plan);
int wgrad3_run(const void* a, const void* b, float* dw, int B, int HA, int WA, int CA, int GH, int GW, int CB, int pad,
               long long s_col, cudaStream_t st);

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
        out[0] = 1;
        wgrad3_geometry(B, GH, GW, CA, CB, out + 1);
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
