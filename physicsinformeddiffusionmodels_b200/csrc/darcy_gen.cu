// Darcy training-data generation (reference src/darcy_data_generation.py), fp64 throughout, P = 64.
//
//   KLE        K[b] = exp(Phi_s z[b]),  Phi_s = [sqrt(lambda_k) phi_k]  [q, P*P]              (:63-78, :131-133)
//   operator   M = [A; BC] with A = -K D00 - K_0 D0 - K D11 - K_1 D1 (K_0, K_1 the FD derivatives of K, second order,
//              one-sided at the ends) and the 4P Neumann rows -D0 | +D0 | +-D1 | -+D1          (:135-153)
//   solve      p = lstsq([M; w^T], [f_s; 0; 0]) with w the trapezoid (or mean) weights        (:99-121, :157-161)
//
// Constants span the null space of M, so the least-squares optimum meets the integral row exactly: it is the solution
// of the normal equations N p = A^T f_s, N = M^T M with one node pinned (N_00 doubled), shifted by -(w^T p / w^T 1).
// N is banded with half-bandwidth BW = 3P + 3 = 195 (point index i*P + j, i = axis 0).  Its condition number is ~1e14,
// so every stage is fp64.  One CTA per sample in every kernel: a sample's result never depends on its batch.
//
//   assemble   N in row-band storage band[r][d] = N[r][r-d], d in [0, 195] (zeros included), rhs = A^T f_s.  One thread
//              per row r of N: the 25 lower stencil offsets of N are accumulated in registers over the <= 14 A rows and
//              <= 2 BC rows that touch point r, in a fixed order (deterministic, no atomics).
//   factor     blocked right-looking Cholesky, 16 x 16 blocks.  The trailing window (block rows J..J+13, lower triangle,
//              105 blocks = 210 KB) stays in shared memory; a slot table maps block (I, K) to one of the 105 slots, and
//              the 14 slots freed by the finished block column J take the entering block row J+14, which is prefetched
//              into registers at the start of the step.  The trailing update runs on the fp64 tensor cores
//              (mma.sync.m8n8k4.f64).  The right-hand side rides along as an extra row of the matrix, so the forward
//              substitution y = L^-1 rhs falls out of the factorisation sweep.  L overwrites N in place, y overwrites rhs.
//   post       blocked back substitution L^T p = y, the constant shift, res = mean |M p - b| over all P*P + 4P + 1 rows
//              (the reference's res_data), and optionally the fp32 [B, 2, P, P] (p, K) batch the training engine takes.
#include "common.cuh"
#include "pidm.h"
#include <math.h>

namespace pidm {
namespace dgen {

constexpr int P = 64;
constexpr int N = P * P;
constexpr int BW = 3 * P + 3;                 // half-bandwidth of N
constexpr int LD = BW + 1;                    // row-band leading dimension
constexpr int NB = 16;                        // Cholesky block
constexpr int NBLK = N / NB;                  // 256 block columns
constexpr int KB = (BW + NB - 1) / NB;        // 13 sub-diagonal blocks
constexpr int WIN = KB + 1;                   // 14 block rows in the window
constexpr int NSLOT = WIN * (WIN + 1) / 2;    // 105 resident blocks
constexpr int FT = 256;                       // factor threads
constexpr int ROWQ = WIN * NB * NB / FT;      // 14 prefetched doubles per thread (one block row of the window)
constexpr size_t FACTOR_SMEM = (size_t)NSLOT * NB * NB * 8 + WIN * NB * 8 + 2 * NB * 8 + 2 * WIN * WIN * 4;
constexpr int ASM_THREADS = 128;              // two x-lines per CTA
constexpr int POST_THREADS = 256;
constexpr size_t POST_SMEM = (2 * N + POST_THREADS / 32) * 8;

// offsets (dx, dy) of N with |dx|, |dy| <= 3 in the lower triangle (dx * P + dy <= 0) -> accumulator index 0..24;
// two entries of one row of M are never more than 3 points apart along an axis
__host__ __device__ constexpr bool lower(int dx, int dy) {
    return dx >= -3 && dx <= 3 && dy >= -3 && dy <= 3 && (dx < 0 || (dx == 0 && dy <= 0));
}
__host__ __device__ constexpr int lidx(int dx, int dy) { return dx < 0 ? (dx + 3) * 7 + (dy + 3) : 21 + (dy + 3); }

// ---- second-order FD tables (findiff acc=2; reference grad_utils / oracle/ref_shims/findiff.py), coefficient of
// u[i + o] at index o + 3; entries that fall outside the grid are zero ------------------------------------------------
__device__ __forceinline__ void d1_tab(int i, double h, double c[7]) {
#pragma unroll
    for (int o = 0; o < 7; ++o) c[o] = 0.0;
    if (i == 0) { c[3] = -1.5 / h; c[4] = 2.0 / h; c[5] = -0.5 / h; }
    else if (i == P - 1) { c[3] = 1.5 / h; c[2] = -2.0 / h; c[1] = 0.5 / h; }
    else { c[2] = -0.5 / h; c[4] = 0.5 / h; }
}
__device__ __forceinline__ void d2_tab(int i, double h, double c[7]) {
    const double h2 = h * h;
#pragma unroll
    for (int o = 0; o < 7; ++o) c[o] = 0.0;
    if (i == 0) { c[3] = 2.0 / h2; c[4] = -5.0 / h2; c[5] = 4.0 / h2; c[6] = -1.0 / h2; }
    else if (i == P - 1) { c[3] = 2.0 / h2; c[2] = -5.0 / h2; c[1] = 4.0 / h2; c[0] = -1.0 / h2; }
    else { c[2] = 1.0 / h2; c[3] = -2.0 / h2; c[4] = 1.0 / h2; }
}

// Coefficients of the A row at point (x, y): cx[o] multiplies p(x + o - 3, y) (the diagonal of both axes is folded
// into cx[3]), cy[o] multiplies p(x, y + o - 3), cy[3] = 0.  Kat(x', y') reads K.
template <class KAt>
__device__ __forceinline__ void a_row(int x, int y, double h0, double h1, const KAt& Kat, double cx[7], double cy[7]) {
    double t1x[7], t2x[7], t1y[7], t2y[7];
    d1_tab(x, h0, t1x); d2_tab(x, h0, t2x);
    d1_tab(y, h1, t1y); d2_tab(y, h1, t2y);
    const double k = Kat(x, y);
    double k0 = 0.0, k1 = 0.0;
#pragma unroll
    for (int o = 0; o < 7; ++o) {
        if (t1x[o] != 0.0) k0 += t1x[o] * Kat(x + o - 3, y);
        if (t1y[o] != 0.0) k1 += t1y[o] * Kat(x, y + o - 3);
    }
#pragma unroll
    for (int o = 0; o < 7; ++o) {
        cx[o] = -k * t2x[o] - k0 * t1x[o];
        cy[o] = -k * t2y[o] - k1 * t1y[o];
    }
    cx[3] += cy[3];
    cy[3] = 0.0;
}

// ==== KLE: K[b, i] = exp(sum_k phi_s[k, i] z[b, k]), k in ascending order ==========================================
__global__ void __launch_bounds__(256) kle_kernel(const double* __restrict__ phi, const double* __restrict__ z,
                                                  double* __restrict__ K, int q) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (i >= N) return;
    const double* zb = z + (size_t)b * q;
    double g = 0.0;
    for (int k = 0; k < q; ++k) g = fma(phi[(size_t)k * N + i], zb[k], g);
    K[(size_t)b * N + i] = exp(g);
}

// ==== assembly ===================================================================================================
__global__ void __launch_bounds__(ASM_THREADS) assemble_kernel(const double* __restrict__ K,
                                                               const double* __restrict__ f_s,
                                                               double* __restrict__ band, double* __restrict__ rhs,
                                                               double h0, double h1, double bc1_sign) {
    constexpr int XL = 12;                                   // K lines x0-5 .. x0+6
    __shared__ double Kw[XL][P];
    __shared__ double stage[ASM_THREADS / 32][25][32];
    const int b = blockIdx.y;
    const int x0 = blockIdx.x * 2;
    const double* Kb = K + (size_t)b * N;
    for (int e = threadIdx.x; e < XL * P; e += ASM_THREADS) {
        const int xl = x0 - 5 + e / P;
        Kw[e / P][e % P] = (xl >= 0 && xl < P) ? Kb[xl * P + e % P] : 0.0;
    }
    __syncthreads();
    const int x = x0 + threadIdx.x / P, y = threadIdx.x % P;
    const int r = x * P + y;
    auto Kat = [&](int xx, int yy) { return Kw[xx - (x0 - 5)][yy]; };

    double acc[25];
#pragma unroll
    for (int a = 0; a < 25; ++a) acc[a] = 0.0;
    double rh = 0.0;

    // rows centred on (x - a, y): r is their x-offset a
#pragma unroll
    for (int a = -3; a <= 3; ++a) {
        const int rx = x - a;
        if (rx < 0 || rx >= P) continue;
        double cx[7], cy[7];
        a_row(rx, y, h0, h1, Kat, cx, cy);
        const double m = cx[a + 3];
        if (m != 0.0) {
#pragma unroll
            for (int a2 = -3; a2 <= 3; ++a2)
                if (lower(a2 - a, 0)) acc[lidx(a2 - a, 0)] = fma(m, cx[a2 + 3], acc[lidx(a2 - a, 0)]);
#pragma unroll
            for (int b2 = -3; b2 <= 3; ++b2)
                if (b2 != 0 && lower(-a, b2)) acc[lidx(-a, b2)] = fma(m, cy[b2 + 3], acc[lidx(-a, b2)]);
            rh = fma(m, f_s[rx * P + y], rh);
        }
        if (rx == 0 || rx == P - 1) {                        // BC row -D0 (x = 0) / +D0 (x = P-1)
            double t[7];
            d1_tab(rx, h0, t);
            const double s = rx == 0 ? -1.0 : 1.0;
            const double mb = s * t[a + 3];
            if (mb != 0.0) {
#pragma unroll
                for (int a2 = -3; a2 <= 3; ++a2)
                    if (lower(a2 - a, 0)) acc[lidx(a2 - a, 0)] = fma(mb, s * t[a2 + 3], acc[lidx(a2 - a, 0)]);
            }
        }
    }
    // rows centred on (x, y - c): r is their y-offset c
#pragma unroll
    for (int c = -3; c <= 3; ++c) {
        const int ry = y - c;
        if (ry < 0 || ry >= P) continue;
        if (c != 0) {
            double cx[7], cy[7];
            a_row(x, ry, h0, h1, Kat, cx, cy);
            const double m = cy[c + 3];
            if (m != 0.0) {
#pragma unroll
                for (int a2 = -3; a2 <= 3; ++a2)
                    if (lower(a2, -c)) acc[lidx(a2, -c)] = fma(m, cx[a2 + 3], acc[lidx(a2, -c)]);
#pragma unroll
                for (int b2 = -3; b2 <= 3; ++b2)
                    if (b2 != 0 && lower(0, b2 - c)) acc[lidx(0, b2 - c)] = fma(m, cy[b2 + 3], acc[lidx(0, b2 - c)]);
                rh = fma(m, f_s[x * P + ry], rh);
            }
        }
        if (ry == 0 || ry == P - 1) {                        // BC row s*D1 (y = 0) / -s*D1 (y = P-1)
            double t[7];
            d1_tab(ry, h1, t);
            const double s = ry == 0 ? bc1_sign : -bc1_sign;
            const double mb = s * t[c + 3];
            if (mb != 0.0) {
#pragma unroll
                for (int b2 = -3; b2 <= 3; ++b2)
                    if (lower(0, b2 - c)) acc[lidx(0, b2 - c)] = fma(mb, s * t[b2 + 3], acc[lidx(0, b2 - c)]);
            }
        }
    }
    if (r == 0) acc[lidx(0, 0)] *= 2.0;                      // pin node 0: the constant mode is fixed afterwards

    // stage the 25 values per row, then each warp writes its 32 band rows with coalesced stores
    const int w = threadIdx.x / 32, lane = threadIdx.x % 32;
#pragma unroll
    for (int a = 0; a < 25; ++a) stage[w][a][lane] = acc[a];
    rhs[(size_t)b * N + r] = rh;
    __syncwarp();
    double* bb = band + ((size_t)b * N + (r - lane)) * LD;
    for (int j = 0; j < 32; ++j) {
        for (int d = lane; d < LD; d += 32) {
            // d = -(dx * P + dy): dx = 0 -> d in [0, 3]; dx = -1, -2, -3 -> d in [P*|dx| - 3, P*|dx| + 3]
            const int adx = (d + 3) / P, dy = adx * P - d;
            double v = 0.0;
            if (dy >= -3 && dy <= 3 && (adx > 0 || dy <= 0)) v = stage[w][adx > 0 ? (3 - adx) * 7 + (dy + 3) : 21 + (dy + 3)][j];
            bb[(size_t)j * LD + d] = v;
        }
    }
}

// ==== factorisation ===============================================================================================
// element (i, k) of a 16 x 16 block: rows 16 doubles apart, columns XOR-swizzled so that the fragment loads of
// mma.m8n8k4 (8 rows x 4 columns per instruction) are free of bank conflicts
__device__ __forceinline__ int sw(int i, int k) { return i * NB + (k ^ ((i & 3) << 2)); }

__device__ __forceinline__ void dmma(double& c0, double& c1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
                 : "+d"(c0), "+d"(c1)
                 : "d"(a), "d"(b));
}

// value of N at (r, c) (c <= r) from row-band storage, 0 outside the band
__device__ __forceinline__ double band_at(const double* __restrict__ Ab, int r, int c) {
    const int d = r - c;
    return (d >= 0 && d <= BW) ? Ab[(size_t)r * LD + d] : 0.0;
}

__global__ void __launch_bounds__(FT, 1) factor_kernel(double* __restrict__ band, double* __restrict__ rhs) {
    extern __shared__ __align__(16) double fsm[];
    double* slots = fsm;                                  // NSLOT blocks of 256
    double* rw = slots + NSLOT * NB * NB;                 // WIN right-hand-side row blocks, block I at I % WIN
    double* colbuf = rw + WIN * NB;                       // 2 x 16
    int* tab = reinterpret_cast<int*>(colbuf + 2 * NB);   // 2 slot tables [WIN][WIN], block (I, K) at [I % WIN][K % WIN]
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    double* Ab = band + (size_t)blockIdx.x * N * LD;
    double* yb = rhs + (size_t)blockIdx.x * N;

    // initial window: block rows 0..13
    if (tid < WIN * WIN) tab[tid] = -1;
    __syncthreads();
    if (tid == 0) {
        int s = 0;
        for (int I = 0; I < WIN; ++I)
            for (int K = 0; K <= I; ++K) tab[I * WIN + K] = s++;
    }
    for (int q = tid; q < NSLOT * NB * NB; q += FT) {
        // q enumerates (block row I, row i, column c in [0, 16 (I+1)))
        int I = 0, base = 0;
        while (q >= base + NB * NB * (I + 1)) { base += NB * NB * (I + 1); ++I; }
        const int rem = q - base, i = rem / (NB * (I + 1)), c = rem % (NB * (I + 1));
        const int K = c / NB, e = c % NB;
        const int s = I * (I + 1) / 2 + K;
        slots[s * NB * NB + sw(i, e)] = band_at(Ab, I * NB + i, c);
    }
    for (int q = tid; q < WIN * NB; q += FT) rw[q] = yb[q];
    __syncthreads();

    for (int J = 0; J < NBLK; ++J) {
        const int* T = tab + (J & 1) * WIN * WIN;
        const int jm = J % WIN;
        // ---- prefetch the entering block row J + 14 (columns of blocks J+1 .. J+14) ----
        double pre[ROWQ];
        const int Inew = J + WIN;
#pragma unroll
        for (int u = 0; u < ROWQ; ++u) {
            const int q = tid + u * FT, i = q / (WIN * NB), c = q % (WIN * NB);
            pre[u] = Inew < NBLK ? band_at(Ab, Inew * NB + i, (J + 1) * NB + c) : 0.0;
        }

        // ---- panel: block column J (rows 16J .. 16J+223) and the right-hand-side row, unblocked ----
        const int tI = tid / NB, ti = tid % NB;
        const bool mrow = tid < WIN * NB && J + tI < NBLK;
        const bool rrow = tid == WIN * NB;
        double v[NB];
        double* prow = mrow ? slots + T[((J + tI) % WIN) * WIN + jm] * NB * NB : nullptr;
        if (mrow) {
#pragma unroll
            for (int k = 0; k < NB; ++k) v[k] = prow[sw(ti, k)];
        } else if (rrow) {
#pragma unroll
            for (int k = 0; k < NB; ++k) v[k] = rw[jm * NB + k];
        }
#pragma unroll
        for (int k = 0; k < NB; ++k) {
            double* cb = colbuf + (k & 1) * NB;
            if (tid < NB) cb[tid] = v[k];
            __syncthreads();
            if ((mrow && tid >= k) || rrow) {
                const double lkk = sqrt(cb[k]), rinv = 1.0 / lkk;
                if (tid == k) {
                    v[k] = lkk;
                } else {
                    const double l = v[k] * rinv;
                    v[k] = l;
#pragma unroll
                    for (int c = k + 1; c < NB; ++c) v[c] = fma(-l, cb[c] * rinv, v[c]);
                }
            }
        }
        if (mrow) {
#pragma unroll
            for (int k = 0; k < NB; ++k) prow[sw(ti, k)] = v[k];
        } else if (rrow) {
#pragma unroll
            for (int k = 0; k < NB; ++k) rw[jm * NB + k] = v[k];
        }
        __syncthreads();

        // ---- trailing update A_IK -= L_IJ L_KJ^T, J < K <= I <= J+13, on the fp64 tensor cores ----
        if (tid == 0) {      // next step's slot table: block (J+14, J+1+t) takes the slot of (J+t, J)
            int* Tn = tab + ((J + 1) & 1) * WIN * WIN;
            for (int e = 0; e < WIN * WIN; ++e) Tn[e] = T[e];
            for (int t = 0; t < WIN; ++t) Tn[jm * WIN + (J + 1 + t) % WIN] = T[((J + t) % WIN) * WIN + jm];
        }
        {
            const int g = lane >> 2, qd = lane & 3;
            int cnt = 0;
            for (int dI = 1; dI <= KB; ++dI) {
                if (J + dI >= NBLK) break;
                for (int dK = 1; dK <= dI; ++dK, ++cnt) {
                    if (cnt % (FT / 32) != warp) continue;
                    const double* sA = slots + T[((J + dI) % WIN) * WIN + jm] * NB * NB;
                    const double* sB = slots + T[((J + dK) % WIN) * WIN + jm] * NB * NB;
                    double* sC = slots + T[((J + dI) % WIN) * WIN + (J + dK) % WIN] * NB * NB;
                    double fa[2][4], fb[2][4];
#pragma unroll
                    for (int m = 0; m < 2; ++m)
#pragma unroll
                        for (int kt = 0; kt < 4; ++kt) {
                            fa[m][kt] = -sA[sw(8 * m + g, 4 * kt + qd)];
                            fb[m][kt] = sB[sw(8 * m + g, 4 * kt + qd)];
                        }
#pragma unroll
                    for (int m = 0; m < 2; ++m)
#pragma unroll
                        for (int n = 0; n < 2; ++n) {
                            double2* cp = reinterpret_cast<double2*>(sC + sw(8 * m + g, 8 * n + 2 * qd));
                            double2 c = *cp;
#pragma unroll
                            for (int kt = 0; kt < 4; ++kt) dmma(c.x, c.y, fa[m][kt], fb[n][kt]);
                            *cp = c;
                        }
                }
            }
        }
        // right-hand-side rows: rhs_K -= y_J L_KJ^T
        if (tid < KB * NB) {
            const int dK = 1 + tid / NB, e = tid % NB;
            if (J + dK < NBLK) {
                const double* sB = slots + T[((J + dK) % WIN) * WIN + jm] * NB * NB;
                double s = rw[((J + dK) % WIN) * NB + e];
#pragma unroll
                for (int k = 0; k < NB; ++k) s = fma(-rw[jm * NB + k], sB[sw(e, k)], s);
                rw[((J + dK) % WIN) * NB + e] = s;
            }
        }
        __syncthreads();

        // ---- write L's block column J over N (row-band storage) and y_J over rhs ----
        for (int q = tid; q < WIN * NB * NB; q += FT) {
            const int rho = q / NB, e = q % NB, d = rho - e;
            const int r = J * NB + rho;
            if (d >= 0 && d <= BW && r < N)
                Ab[(size_t)r * LD + d] = slots[T[((J + rho / NB) % WIN) * WIN + jm] * NB * NB + sw(rho % NB, e)];
        }
        if (tid < NB) yb[J * NB + tid] = rw[jm * NB + tid];
        __syncthreads();

        // ---- the entering block row takes the freed slots ----
        if (Inew < NBLK) {
#pragma unroll
            for (int u = 0; u < ROWQ; ++u) {
                const int q = tid + u * FT, i = q / (WIN * NB), c = q % (WIN * NB), t = c / NB;
                slots[T[((J + t) % WIN) * WIN + jm] * NB * NB + sw(i, c % NB)] = pre[u];
            }
            if (tid < NB) rw[jm * NB + tid] = yb[Inew * NB + tid];
        }
        __syncthreads();
    }
}

// ==== back substitution, shift, residual, outputs =====================================================================
__device__ __forceinline__ double block_sum(double v, double* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double s = 0.0;
    for (int w = 0; w < POST_THREADS / 32; ++w) s += red[w];
    return s;
}

__global__ void __launch_bounds__(POST_THREADS) post_kernel(const double* __restrict__ band,
                                                            const double* __restrict__ y, const double* __restrict__ K,
                                                            const double* __restrict__ f_s, double* __restrict__ p_out,
                                                            double* __restrict__ res, float* __restrict__ batch,
                                                            double h0, double h1, int trapezoid) {
    extern __shared__ __align__(16) double psm[];
    double* ps = psm;                 // y, then p
    double* Ks = psm + N;
    double* red = psm + 2 * N;        // POST_THREADS / 32
    const int b = blockIdx.x, tid = threadIdx.x;
    const double* Lb = band + (size_t)b * N * LD;
    for (int i = tid; i < N; i += POST_THREADS) {
        ps[i] = y[(size_t)b * N + i];
        Ks[i] = K[(size_t)b * N + i];
    }
    __syncthreads();

    // L^T p = y, block rows of 16 from the bottom: the diagonal block by warp 0, then the rows of block J update the
    // 195 unknowns above it (row r of L is contiguous in the band, so each update reads 16 contiguous rows)
    for (int J = NBLK - 1; J >= 0; --J) {
        const int r0 = J * NB;
        if (tid < 32) {
            const int e = tid & (NB - 1);
            double x = ps[r0 + e];
            double Lrow[NB];                           // Lrow[i] = L[r0 + i][r0 + e] for i >= e
#pragma unroll
            for (int i = 0; i < NB; ++i) Lrow[i] = i >= e ? Lb[(size_t)(r0 + i) * LD + (i - e)] : 0.0;
#pragma unroll
            for (int i = NB - 1; i >= 0; --i) {
                const double pi = __shfl_sync(0xffffffffu, x / Lrow[i], i);
                if (e < i) x = fma(-Lrow[i], pi, x);
                if (e == i) x = pi;
            }
            if (tid < NB) ps[r0 + e] = x;
        }
        __syncthreads();
        if (tid < BW) {
            const int c = r0 - 1 - tid;
            if (c >= 0) {
                double s = ps[c];
#pragma unroll
                for (int a = 0; a < NB; ++a) {
                    const int d = r0 + a - c;
                    if (d <= BW) s = fma(-Lb[(size_t)(r0 + a) * LD + d], ps[r0 + a], s);
                }
                ps[c] = s;
            }
        }
        __syncthreads();
    }

    // integral condition: p -= (w^T p) / (w^T 1); trapezoid weights {1, 2, 4} h0^2 / 4 or the plain mean
    auto weight = [&](int i) {
        if (!trapezoid) return 1.0 / (double)N;
        const int x = i / P, yy = i % P;
        const double c = ((x == 0 || x == P - 1) ? 1.0 : 2.0) * ((yy == 0 || yy == P - 1) ? 1.0 : 2.0);
        return c * (h0 * h0 / 4.0);
    };
    double wp = 0.0, w1 = 0.0;
    for (int i = tid; i < N; i += POST_THREADS) {
        const double w = weight(i);
        wp = fma(w, ps[i], wp);
        w1 += w;
    }
    wp = block_sum(wp, red);
    w1 = block_sum(w1, red);
    const double shift = wp / w1;
    __syncthreads();
    for (int i = tid; i < N; i += POST_THREADS) ps[i] -= shift;
    __syncthreads();

    // res = mean |M p - b| over the P*P operator rows, the 4P BC rows and the integral row
    auto Kat = [&](int xx, int yy) { return Ks[xx * P + yy]; };
    double sabs = 0.0, wq = 0.0;
    for (int i = tid; i < N; i += POST_THREADS) {
        const int x = i / P, yy = i % P;
        double cx[7], cy[7];
        a_row(x, yy, h0, h1, Kat, cx, cy);
        double r = -f_s[i];
#pragma unroll
        for (int o = 0; o < 7; ++o) {
            if (cx[o] != 0.0) r = fma(cx[o], ps[(x + o - 3) * P + yy], r);
            if (cy[o] != 0.0) r = fma(cy[o], ps[x * P + yy + o - 3], r);
        }
        sabs += fabs(r);
        if (x == 0 || x == P - 1) {
            double t[7], g = 0.0;
            d1_tab(x, h0, t);
#pragma unroll
            for (int o = 0; o < 7; ++o)
                if (t[o] != 0.0) g = fma(t[o], ps[(x + o - 3) * P + yy], g);
            sabs += fabs(g);
        }
        if (yy == 0 || yy == P - 1) {
            double t[7], g = 0.0;
            d1_tab(yy, h1, t);
#pragma unroll
            for (int o = 0; o < 7; ++o)
                if (t[o] != 0.0) g = fma(t[o], ps[x * P + yy + o - 3], g);
            sabs += fabs(g);
        }
        wq = fma(weight(i), ps[i], wq);
        if (p_out) p_out[(size_t)b * N + i] = ps[i];
        if (batch) {
            batch[(size_t)b * 2 * N + i] = (float)ps[i];
            batch[(size_t)b * 2 * N + N + i] = (float)Ks[i];
        }
    }
    sabs = block_sum(sabs, red);
    wq = block_sum(wq, red);
    if (tid == 0 && res) res[b] = (sabs + fabs(wq)) / (double)(N + 4 * P + 1);
}

}  // namespace dgen
}  // namespace pidm

using namespace pidm;

extern "C" int pidm_darcy_gen_kle(const double* phi, const double* z, double* K, int B, int q, int pixels,
                                  void* stream) {
    PIDM_REQUIRE(pixels == dgen::P, "pidm_darcy_gen_kle: pixels must be %d, got %d", dgen::P, pixels);
    PIDM_REQUIRE(B >= 0 && B <= 65535, "pidm_darcy_gen_kle: B = %d out of range [0, 65535]", B);
    PIDM_REQUIRE(q >= 1 && q <= dgen::N, "pidm_darcy_gen_kle: q = %d out of range [1, %d]", q, dgen::N);
    if (B == 0) return 0;
    dgen::kle_kernel<<<dim3(dgen::N / 256, B), 256, 0, (cudaStream_t)stream>>>(phi, z, K, q);
    PIDM_LAUNCH_CHECK("pidm_darcy_gen_kle");
    return 0;
}

extern "C" long long pidm_darcy_gen_workspace_bytes(int B, int pixels) {
    if (pixels != dgen::P || B < 0) {
        set_error(2, "pidm_darcy_gen_workspace_bytes: pixels must be %d (got %d), B >= 0 (got %d)", dgen::P, pixels, B);
        return -1;
    }
    return (long long)B * ((long long)dgen::N * dgen::LD + dgen::N) * (long long)sizeof(double);
}

extern "C" int pidm_darcy_gen_solve(const double* K, const double* f_s, double* p, double* res, float* batch,
                                    void* workspace, long long workspace_bytes, int B, int pixels,
                                    double domain_length, int reverse_dy, int flags, int stages, void* stream) {
    PIDM_REQUIRE(pixels == dgen::P, "pidm_darcy_gen_solve: pixels must be %d, got %d", dgen::P, pixels);
    PIDM_REQUIRE((flags & ~PIDM_DARCY_PIXELS_AT_BOUNDARY) == 0,
                 "pidm_darcy_gen_solve: unknown flags 0x%x (only PIDM_DARCY_PIXELS_AT_BOUNDARY)", flags);
    PIDM_REQUIRE(stages != 0 && (stages & ~PIDM_DARCY_GEN_ALL) == 0, "pidm_darcy_gen_solve: bad stages mask 0x%x",
                 stages);
    PIDM_REQUIRE(B >= 0 && B <= 65535, "pidm_darcy_gen_solve: B = %d out of range [0, 65535]", B);
    PIDM_REQUIRE(domain_length > 0.0, "pidm_darcy_gen_solve: domain_length must be positive");
    const long long need = pidm_darcy_gen_workspace_bytes(B, pixels);
    PIDM_REQUIRE(workspace_bytes >= need, "pidm_darcy_gen_solve: workspace of %lld bytes, need %lld",
                 workspace_bytes, need);
    if (B == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    const bool pab = flags & PIDM_DARCY_PIXELS_AT_BOUNDARY;
    const double h0 = pab ? domain_length / (dgen::P - 1) : domain_length / dgen::P;
    const double h1 = reverse_dy ? -h0 : h0;
    const double bc1_sign = reverse_dy ? 1.0 : -1.0;
    double* band = static_cast<double*>(workspace);
    double* rhs = band + (size_t)B * dgen::N * dgen::LD;
    if (stages & PIDM_DARCY_GEN_ASSEMBLE) {
        dgen::assemble_kernel<<<dim3(dgen::P / 2, B), dgen::ASM_THREADS, 0, st>>>(K, f_s, band, rhs, h0, h1, bc1_sign);
        PIDM_LAUNCH_CHECK("pidm_darcy_gen_solve (assemble)");
    }
    if (stages & PIDM_DARCY_GEN_FACTOR) {
        PIDM_CUDA(allow_smem(dgen::factor_kernel, dgen::FACTOR_SMEM));
        dgen::factor_kernel<<<B, dgen::FT, dgen::FACTOR_SMEM, st>>>(band, rhs);
        PIDM_LAUNCH_CHECK("pidm_darcy_gen_solve (factor)");
    }
    if (stages & PIDM_DARCY_GEN_POST) {
        PIDM_CUDA(allow_smem(dgen::post_kernel, dgen::POST_SMEM));
        dgen::post_kernel<<<B, dgen::POST_THREADS, dgen::POST_SMEM, st>>>(band, rhs, K, f_s, p, res, batch, h0, h1,
                                                                         pab ? 1 : 0);
        PIDM_LAUNCH_CHECK("pidm_darcy_gen_solve (post)");
    }
    return 0;
}
