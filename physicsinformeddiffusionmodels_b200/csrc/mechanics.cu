// Linear-elasticity (topology-optimisation) residual, MATRIX-FREE.
// Reference src/residuals_mechanics_K.py:198-274 assembles a dense B x 8450 x 8450 stiffness matrix
// (285.6 MB per sample) by index_put, replaces Dirichlet rows by identity rows and multiplies by u.
// Here K(rho) u is evaluated by gathering, for every node, the <= 4 adjacent Q4 elements:
//     (K u)_i = sum_{e ni i} rho_e sum_j KE[loc_e(i)][j] u_{dof_e(j)}
// which touches ~150 KB per sample instead of >1 GB.  Node id = row*(nel+1)+col, dof = 2*node+d, element
// (er,ec) has nodes n1=(er+1,ec), n2=(er+1,ec+1), n3=(er,ec+1), n4=(er,ec) (counter-clockwise, y up).
//   residual_i = mask_i ? u_i : (K u)_i - f_i ;   compliance = sum_i u_i * (mask_i ? u_i : (K u)_i)
// Also: bilinear resize (torchvision Resize(antialias=False) == align_corners=False), reference :10-21.
#include "common.cuh"
#include "pidm.h"

#include <algorithm>

namespace pidm {

__constant__ float c_KE[64];
__constant__ double c_KEd[64];
__device__ double g_KEd[64];     // staging copy of KE in fp64 (a kernel writes it, c_KEd is copied from it)

// Row-band tiling: a CTA owns MECH_BAND consecutive node rows of one sample and stages the nodal field it applies K to
// (both dof planes, rows r0-1 .. r0+MECH_BAND) and the element densities (rows r0-1 .. r0+MECH_BAND-1) in shared memory
// with coalesced row loads; the 9-node / 4-element gather of every node then runs on shared memory.  (The first
// version gathered straight from global memory: 18 + 4 scattered loads per node.)
constexpr int MECH_BAND = 8;
constexpr int MECH_THREADS = 256;

// KE entry i in the precision of the field K is applied to (the fp64 copy feeds the PCG solve)
template <typename T> __device__ __forceinline__ T ke(int i);
template <> __device__ __forceinline__ float ke<float>(int i) { return c_KE[i]; }
template <> __device__ __forceinline__ double ke<double>(int i) { return c_KEd[i]; }

template <typename T>
struct MechTile {
    const T* v0;          // dof-0 plane of the staged rows: v0[(r - rlo) * nn + c]
    const T* v1;
    const float* rho;     // rho[(er - elo) * nel + ec]
    int rlo, elo;
};

// stage rows of field v [2][nn][nn] and rho [nel][nel] of one sample for the band starting at node row r0
__device__ __forceinline__ MechTile<float> mech_stage(float* sm, const float* __restrict__ v, const float* __restrict__ rho,
                                                      int nel, int r0) {
    const int nn = nel + 1;
    const int rlo = max(r0 - 1, 0), rhi = min(r0 + MECH_BAND, nn - 1);            // node rows [rlo, rhi]
    const int elo = max(r0 - 1, 0), ehi = min(r0 + MECH_BAND - 1, nel - 1);       // element rows [elo, ehi]
    float* s0 = sm;
    float* s1 = s0 + (MECH_BAND + 2) * nn;
    float* sr = s1 + (MECH_BAND + 2) * nn;
    const int nv = (rhi - rlo + 1) * nn, ne = (ehi - elo + 1) * nel;
    for (int i = threadIdx.x; i < nv; i += blockDim.x) {
        s0[i] = v[rlo * nn + i];
        s1[i] = v[nn * nn + rlo * nn + i];
    }
    for (int i = threadIdx.x; i < ne; i += blockDim.x) sr[i] = rho[elo * nel + i];
    __syncthreads();
    MechTile<float> t;
    t.v0 = s0; t.v1 = s1; t.rho = sr; t.rlo = rlo; t.elo = elo;
    return t;
}

// (K v)_{node (r,c), both dofs} from the staged tile (a band of rows, or a whole sample with rlo = elo = 0)
template <typename T>
__device__ __forceinline__ void kv_node(const MechTile<T>& t, int nel, int r, int c, T& o0, T& o1) {
    const int nn = nel + 1;
    o0 = 0.f; o1 = 0.f;
    // adjacent elements and the local index of this node inside them
    const int der[4] = {-1, -1, 0, 0}, dec[4] = {-1, 0, -1, 0}, loc[4] = {1, 0, 2, 3};
#pragma unroll
    for (int a = 0; a < 4; ++a) {
        int er = r + der[a], ec = c + dec[a];
        if (er < 0 || er >= nel || ec < 0 || ec >= nel) continue;
        T re = t.rho[(er - t.elo) * nel + ec];
        const int nr[4] = {er + 1, er + 1, er, er}, nc[4] = {ec, ec + 1, ec + 1, ec};
        T ue[8];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            ue[2 * k] = t.v0[(nr[k] - t.rlo) * nn + nc[k]];
            ue[2 * k + 1] = t.v1[(nr[k] - t.rlo) * nn + nc[k]];
        }
        T s0 = 0.f, s1 = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) { s0 += ke<T>((2 * loc[a]) * 8 + j) * ue[j]; s1 += ke<T>((2 * loc[a] + 1) * 8 + j) * ue[j]; }
        o0 += re * s0; o1 += re * s1;
    }
}

// MODE 0: forward.  MODE 1: backward stage A (z and the direct terms).  MODE 2: backward stage B (du += K z).
// grid (row bands, B)
template <int MODE>
__global__ void __launch_bounds__(MECH_THREADS) mech_node_kernel(
        const float* __restrict__ u, const float* __restrict__ rho, const float* __restrict__ bcs,
        float* __restrict__ residual, float* __restrict__ compliance, const float* __restrict__ g_r,
        const float* __restrict__ g_c, float* __restrict__ z, float* __restrict__ du, int nel) {
    extern __shared__ float msm[];
    const int nn = nel + 1, b = blockIdx.y, r0 = blockIdx.x * MECH_BAND;
    const float* ub = u + (size_t)b * 2 * nn * nn;
    const float* rb = rho + (size_t)b * nel * nel;
    const float* bb = bcs + (size_t)b * 4 * nn * nn;
    const MechTile<float> t = mech_stage(msm, MODE == 2 ? z + (size_t)b * 2 * nn * nn : ub, rb, nel, r0);
    const int n_band = min(MECH_BAND, nn - r0) * nn;
    float csum = 0.f;
    for (int i = threadIdx.x; i < n_band; i += blockDim.x) {
        const int node = r0 * nn + i;
        const int r = node / nn, c = node - r * nn;
        float k0, k1;
        kv_node(t, nel, r, c, k0, k1);
        if (MODE == 2) {
            du[(size_t)b * 2 * nn * nn + node] += k0;
            du[(size_t)b * 2 * nn * nn + nn * nn + node] += k1;
            continue;
        }
        const bool m0 = bb[node] != 0.f, m1 = bb[nn * nn + node] != 0.f;
        const float u0 = t.v0[(r - t.rlo) * nn + c], u1 = t.v1[(r - t.rlo) * nn + c];
        const float w0 = m0 ? u0 : k0, w1 = m1 ? u1 : k1;
        if (MODE == 0) {
            const float f0 = m0 ? 0.f : bb[2 * nn * nn + node], f1 = m1 ? 0.f : bb[3 * nn * nn + node];
            *reinterpret_cast<float2*>(residual + (size_t)b * 2 * nn * nn + 2 * node) = make_float2(w0 - f0, w1 - f1);
            csum += u0 * w0 + u1 * w1;
        } else {
            const float gc = g_c ? g_c[b] : 0.f;
            float2 gr = make_float2(0.f, 0.f);
            if (g_r) gr = *reinterpret_cast<const float2*>(g_r + (size_t)b * 2 * nn * nn + 2 * node);
            const float wb0 = gr.x + gc * u0, wb1 = gr.y + gc * u1;
            z[(size_t)b * 2 * nn * nn + node] = m0 ? 0.f : wb0;
            z[(size_t)b * 2 * nn * nn + nn * nn + node] = m1 ? 0.f : wb1;
            du[(size_t)b * 2 * nn * nn + node] = gc * w0 + (m0 ? wb0 : 0.f);
            du[(size_t)b * 2 * nn * nn + nn * nn + node] = gc * w1 + (m1 ? wb1 : 0.f);
        }
    }
    if (MODE == 0 && compliance) {
        __shared__ float red[MECH_THREADS / 32];
        csum = warp_sum(csum);
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = csum;
        __syncthreads();
        if (threadIdx.x == 0) {
            float s = 0.f;
            for (int w = 0; w < MECH_THREADS / 32; ++w) s += red[w];
            atomicAdd(&compliance[b], s);
        }
    }
}

// d rho_e = z_e^T KE u_e
__global__ void mech_drho_kernel(const float* __restrict__ u, const float* __restrict__ z, float* __restrict__ drho,
                                 int nel) {
    const int nn = nel + 1, b = blockIdx.y;
    const float* ub = u + (size_t)b * 2 * nn * nn;
    const float* zb = z + (size_t)b * 2 * nn * nn;
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < nel * nel; e += gridDim.x * blockDim.x) {
        int er = e / nel, ec = e - er * nel;
        const int nr[4] = {er + 1, er + 1, er, er}, nc[4] = {ec, ec + 1, ec + 1, ec};
        float ue[8], ze[8];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            ue[2 * k] = ub[nr[k] * nn + nc[k]]; ue[2 * k + 1] = ub[nn * nn + nr[k] * nn + nc[k]];
            ze[2 * k] = zb[nr[k] * nn + nc[k]]; ze[2 * k + 1] = zb[nn * nn + nr[k] * nn + nc[k]];
        }
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            float t = 0.f;
#pragma unroll
            for (int j = 0; j < 8; ++j) t += c_KE[i * 8 + j] * ue[j];
            s += ze[i] * t;
        }
        drho[(size_t)b * nel * nel + e] = s;
    }
}

// bilinear resize, align_corners=False, no antialias (matches F.interpolate / torchvision Resize(antialias=False))
__device__ __forceinline__ void bil_src(int o, float scale, int in, int& i0, int& i1, float& w1) {
    float s = ((float)o + 0.5f) * scale - 0.5f;
    if (s < 0.f) s = 0.f;
    i0 = (int)s;
    if (i0 > in - 1) i0 = in - 1;
    i1 = i0 + ((i0 < in - 1) ? 1 : 0);
    w1 = s - (float)i0;
}
// one output pixel (oh, ow) of the bilinear resize of the in x in plane p
__device__ __forceinline__ float bil_sample(const float* p, int in, float scale, int oh, int ow) {
    int h0, h1, w0, w1; float lh, lw;
    bil_src(oh, scale, in, h0, h1, lh);
    bil_src(ow, scale, in, w0, w1, lw);
    return (1.f - lh) * ((1.f - lw) * p[h0 * in + w0] + lw * p[h0 * in + w1]) +
           lh * ((1.f - lw) * p[h1 * in + w0] + lw * p[h1 * in + w1]);
}
__global__ void bilinear_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, int planes, int in, int out) {
    const float scale = (float)in / (float)out;
    long long total = (long long)planes * out * out;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        int ow = (int)(i % out), oh = (int)((i / out) % out);
        long long pl = i / ((long long)out * out);
        y[i] = bil_sample(x + pl * in * in, in, scale, oh, ow);
    }
}
__global__ void bilinear_bwd_kernel(const float* __restrict__ dy, float* __restrict__ dx, int planes, int in, int out) {
    const float scale = (float)in / (float)out;
    long long total = (long long)planes * out * out;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        int ow = (int)(i % out), oh = (int)((i / out) % out);
        long long pl = i / ((long long)out * out);
        int h0, h1, w0, w1; float lh, lw;
        bil_src(oh, scale, in, h0, h1, lh);
        bil_src(ow, scale, in, w0, w1, lw);
        float g = dy[i];
        float* p = dx + pl * in * in;
        atomicAdd(&p[h0 * in + w0], g * (1.f - lh) * (1.f - lw));
        atomicAdd(&p[h0 * in + w1], g * (1.f - lh) * lw);
        atomicAdd(&p[h1 * in + w0], g * lh * (1.f - lw));
        atomicAdd(&p[h1 * in + w1], g * lh * lw);
    }
}

// Fused PIDM loss of the mechanics branch (reference denoising_utils.py:669-710) and its gradients, one CTA per
// sample.  With n = (nel+1)^2 nodes, the data target x0 [B,3,n] = (disp_x, disp_y, E field) and the model output
// (u [B,2,n] = displacements resampled to the node grid, rho [B,nel,nel] zero-padded to the node grid by the reference):
//   data = c_data * mean_b( p2[t_b] * mean_{3n}( (x0 - out)^2 ) )            -> g_u, g_rho (data part)
//   res  = mean_{B x 2n}( c_res * 0.5 r^2 / var_b )                           -> g_r
//   ineq = c_ineq * 0.5 * mean_i(1/var_i) * mean_j(q_j^2), q_j = mean(rho_j) - vf_j   (the reference's [B,1] x [B]
//          broadcast, :679,:694)                                             -> g_rho (+= dq_j / nel^2)
//   opt  = lambda * mean_b(compliance_b)                                      -> g_c
// sums[0..5] += data, res, ineq, opt, sum|r| / (B 2n), mean_b q_b   (caller zeroes; tracked scalars of the reference)
// Loss only: g_u == NULL (the entry point admits all four gradients NULL or none); the sums are computed alike.
__global__ void __launch_bounds__(256) mech_loss_kernel(
        const float* __restrict__ u, const float* __restrict__ rho, const float* __restrict__ x0,
        const float* __restrict__ r, const float* __restrict__ comp, const float* __restrict__ vf,
        const long long* __restrict__ t, const float* __restrict__ p2w, const float* __restrict__ pvar, float c_data,
        float c_res, float c_ineq, float lam, float* __restrict__ sums, float* __restrict__ g_u, float* __restrict__ g_rho,
        float* __restrict__ g_r, float* __restrict__ g_c, int B, int nel) {
    const int nn = nel + 1, n = nn * nn, ne = nel * nel, b = blockIdx.x, tid = threadIdx.x;
    __shared__ float red[8][4];
    __shared__ float s_q;
    const long long tb = t[b];
    const float wd = c_data * p2w[tb] / ((float)B * 3.f * (float)n);
    const float wr = 0.5f * c_res / (pvar[tb] * (float)B * 2.f * (float)n);
    const float* ub = u + (size_t)b * 2 * n;
    const float* xb = x0 + (size_t)b * 3 * n;
    const float* rb = rho + (size_t)b * ne;
    float a_data = 0.f, a_res = 0.f, a_abs = 0.f, a_rho = 0.f;
    for (int i = tid; i < 2 * n; i += blockDim.x) {                 // displacement channels + residual (both 2n long)
        const float e = ub[i] - xb[i];
        a_data += wd * e * e;
        const float rv = r[(size_t)b * 2 * n + i];
        a_res += wr * rv * rv;
        a_abs += fabsf(rv);
        if (g_u) {
            g_u[(size_t)b * 2 * n + i] = 2.f * wd * e;
            g_r[(size_t)b * 2 * n + i] = 2.f * wr * rv;
        }
    }
    for (int i = tid; i < n; i += blockDim.x) {                     // density channel on the node grid (zero outside nel x nel)
        const int row = i / nn, col = i - row * nn;
        const bool inside = row < nel && col < nel;
        const float o = inside ? rb[row * nel + col] : 0.f;
        const float e = o - xb[2 * n + i];
        a_data += wd * e * e;
        if (inside) a_rho += o;
    }
    a_data = warp_sum(a_data); a_res = warp_sum(a_res); a_abs = warp_sum(a_abs); a_rho = warp_sum(a_rho);
    if ((tid & 31) == 0) { red[tid >> 5][0] = a_data; red[tid >> 5][1] = a_res; red[tid >> 5][2] = a_abs; red[tid >> 5][3] = a_rho; }
    __syncthreads();
    if (tid == 0) {
        float sd = 0.f, sr = 0.f, sa = 0.f, srho = 0.f;
        for (int w = 0; w < 8; ++w) { sd += red[w][0]; sr += red[w][1]; sa += red[w][2]; srho += red[w][3]; }
        const float q = srho / (float)ne - vf[b];
        float mvar = 0.f;                                           // mean_i 1 / var_i  (B is a batch size: tiny loop)
        if (c_ineq > 0.f) {
            for (int i = 0; i < B; ++i) mvar += 1.f / pvar[t[i]];
            mvar /= (float)B;
        }
        s_q = c_ineq * mvar * q / (float)B;                         // d loss / d q_b
        atomicAdd(&sums[0], sd);
        atomicAdd(&sums[1], sr);
        atomicAdd(&sums[2], 0.5f * c_ineq * mvar * q * q / (float)B);
        atomicAdd(&sums[3], lam * comp[b] / (float)B);
        atomicAdd(&sums[4], sa / ((float)B * 2.f * (float)n));
        atomicAdd(&sums[5], q / (float)B);
        if (g_c) g_c[b] = lam / (float)B;
    }
    if (!g_u) return;
    __syncthreads();
    const float dq = s_q / (float)ne;
    for (int i = tid; i < ne; i += blockDim.x) {
        const int row = i / nel, col = i - row * nel;
        g_rho[(size_t)b * ne + i] = 2.f * wd * (rb[i] - xb[2 * n + row * nn + col]) + dq;
    }
}


// ---- conditional sampling of the topology-optimisation model (reference denoising_utils.py:388-455 with
// residuals_mechanics_K.py:176-205): the two per-step pieces around the network call -------------------------------

// U-Net input [B, 3 + NC, P, P]: channels 0..2 = bilinear resize of the sample x [B,3,P+1,P+1] to P x P, channels
// 3.. = the NC constant planes [B,NC,P,P] (the resized conditioning and boundary conditions, resized once per loop).
// Resizing acts on each plane alone, so this equals resize(cat(x, cond)) bit for bit.
__global__ void mech_sample_input_kernel(const float* __restrict__ x, const float* __restrict__ planes,
                                         float* __restrict__ out, int B, int nc, int P) {
    const int in = P + 1, C = 3 + nc;
    const float scale = (float)in / (float)P;
    const long long total = (long long)B * C * P * P;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int pix = (int)(i % (P * P)), ch = (int)((i / (P * P)) % C), b = (int)(i / ((long long)C * P * P));
        out[i] = ch < 3 ? bil_sample(x + ((long long)b * 3 + ch) * in * in, in, scale, pix / P, pix % P)
                        : planes[((long long)b * nc + ch - 3) * P * P + pix];
    }
}

// Posterior step from the network output y [B,3,P,P]: model_out = (bilinear P -> P+1 of u_x, u_y ; rho zero-padded to
// (P+1)^2), x' = c1[t_b] model_out + c2[t_b] x + sigma[t_b] z with the per-sample step index read on the device.
// Same arithmetic as pidm_axpby_per_sample.  x' may alias x.
__global__ void mech_posterior_kernel(const float* __restrict__ y, const float* x, const float* __restrict__ z,
                                      const long long* __restrict__ t, const float* __restrict__ c1,
                                      const float* __restrict__ c2, const float* __restrict__ sigma, float* xo,
                                      int B, int P) {
    const int nn = P + 1;
    const float scale = (float)P / (float)nn;
    const long long total = (long long)B * 3 * nn * nn;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int pix = (int)(i % (nn * nn)), ch = (int)((i / (nn * nn)) % 3), b = (int)(i / (3LL * nn * nn));
        const int r = pix / nn, c = pix % nn;
        const float* yp = y + ((long long)b * 3 + ch) * P * P;
        float mo;
        if (ch < 2) mo = bil_sample(yp, P, scale, r, c);
        else mo = (r < P && c < P) ? yp[r * P + c] : 0.f;
        const long long tb = t[b];
        xo[i] = c1[tb] * mo + c2[tb] * x[i] + sigma[tb] * z[i];
    }
}

// ---- batched Jacobi-PCG of the compliance check (ResidualsMechanics.fem_solve, reference :296-325) -----------------
// K(rho) u = f on the free dofs, u = 0 on the Dirichlet dofs, Jacobi preconditioner diag = KE[0,0] * sum of the
// adjacent element densities, stop when ||r|| / ||f|| < tol (fp64 norms) or after max_iter iterations.  One CTA owns
// one sample for the whole solve, so the batch needs one launch and no host round trip, and every sample stops on its
// own.  Shared memory holds p and u (fp64, both dof planes) and rho; r and A p live in registers, owned by node.
// Everything is fp64 except rho and KE, which are the fp32 values the residual kernels use.
constexpr int PCG_THREADS = 512;
constexpr int PCG_NPT = 9;               // nodes per thread: (nel+1)^2 <= 4608

// fp64 sums of a and b over the CTA, returned to every thread (same order everywhere, so decisions are uniform).
// Two callers alternate `red` buffers, which lets one barrier per call suffice.
__device__ __forceinline__ double2 pcg_block_sum2(double a, double b, double* red) {
    constexpr int NW = PCG_THREADS / 32;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, o);
        b += __shfl_xor_sync(0xffffffffu, b, o);
    }
    if ((threadIdx.x & 31) == 0) { red[threadIdx.x >> 5] = a; red[NW + (threadIdx.x >> 5)] = b; }
    __syncthreads();
    a = 0.0; b = 0.0;
#pragma unroll
    for (int w = 0; w < NW; ++w) { a += red[w]; b += red[NW + w]; }
    return make_double2(a, b);
}

__global__ void mech_ke_to_double_kernel(const float* __restrict__ KE) {
    if (threadIdx.x < 64) g_KEd[threadIdx.x] = (double)KE[threadIdx.x];
}

__global__ void __launch_bounds__(PCG_THREADS, 1) mech_pcg_kernel(
        const float* __restrict__ rho, const float* __restrict__ bcs, float* __restrict__ u_out, int* __restrict__ iters,
        double* __restrict__ relres, double tol, int max_iter, int nel) {
    extern __shared__ double pcg_sm[];
    const int nn = nel + 1, NN = nn * nn, ne = nel * nel, b = blockIdx.x, tid = threadIdx.x;
    double* p = pcg_sm;                                  // [2][NN]
    double* u = p + 2 * NN;                              // [2][NN]
    double* red = u + 2 * NN;                            // [2][2 * warps]
    float* rho_s = reinterpret_cast<float*>(red + 4 * (PCG_THREADS / 32));
    const float* rb = rho + (size_t)b * ne;
    const float* bb = bcs + (size_t)b * 4 * NN;
    for (int i = tid; i < ne; i += PCG_THREADS) rho_s[i] = rb[i];
    __syncthreads();
    MechTile<double> tile;
    tile.v0 = p; tile.v1 = p + NN; tile.rho = rho_s; tile.rlo = 0; tile.elo = 0;

    double r0[PCG_NPT], r1[PCG_NPT], a0[PCG_NPT], a1[PCG_NPT];
    float dinv[PCG_NPT];
    unsigned fixed0 = 0u, fixed1 = 0u;                   // bit k: dof d of node k is a Dirichlet dof
    double rz = 0.0, ff = 0.0;
    const double ke00 = ke<double>(0);
#pragma unroll
    for (int k = 0; k < PCG_NPT; ++k) {
        const int node = tid + k * PCG_THREADS;
        r0[k] = 0.0; r1[k] = 0.0; dinv[k] = 0.f;
        if (node >= NN) continue;
        const int r = node / nn, c = node - r * nn;
        const bool m0 = bb[node] != 0.f, m1 = bb[NN + node] != 0.f;
        fixed0 |= (unsigned)m0 << k; fixed1 |= (unsigned)m1 << k;
        double nr = 0.0;
        for (int er = max(r - 1, 0); er <= min(r, nel - 1); ++er)
            for (int ec = max(c - 1, 0); ec <= min(c, nel - 1); ++ec) nr += (double)rho_s[er * nel + ec];
        dinv[k] = (float)(1.0 / fmax(ke00 * nr, 1e-12));
        r0[k] = m0 ? 0.0 : (double)bb[2 * NN + node];
        r1[k] = m1 ? 0.0 : (double)bb[3 * NN + node];
        const double z0 = dinv[k] * r0[k], z1 = dinv[k] * r1[k];
        p[node] = z0; p[NN + node] = z1;
        u[node] = 0.0; u[NN + node] = 0.0;
        rz += r0[k] * z0 + r1[k] * z1;
        ff += r0[k] * r0[k] + r1[k] * r1[k];
    }
    double2 s = pcg_block_sum2(rz, ff, red + 2 * (PCG_THREADS / 32));
    rz = s.x;
    const double f2 = fmax(s.y, 1e-300);
    double rel = sqrt(s.y / f2);
    int it = 0;
    while (it < max_iter) {
        double pap = 0.0;
#pragma unroll
        for (int k = 0; k < PCG_NPT; ++k) {
            const int node = tid + k * PCG_THREADS;
            a0[k] = 0.0; a1[k] = 0.0;
            if (node >= NN) continue;
            const int r = node / nn, c = node - r * nn;
            double k0, k1;
            kv_node(tile, nel, r, c, k0, k1);
            a0[k] = (fixed0 >> k) & 1u ? 0.0 : k0;
            a1[k] = (fixed1 >> k) & 1u ? 0.0 : k1;
            pap += p[node] * a0[k] + p[NN + node] * a1[k];
        }
        const double alpha = rz / fmax(pcg_block_sum2(pap, 0.0, red).x, 1e-300);
        double rr = 0.0, rzn = 0.0;
#pragma unroll
        for (int k = 0; k < PCG_NPT; ++k) {
            const int node = tid + k * PCG_THREADS;
            if (node >= NN) continue;
            u[node] += alpha * p[node];
            u[NN + node] += alpha * p[NN + node];
            r0[k] -= alpha * a0[k];
            r1[k] -= alpha * a1[k];
            rr += r0[k] * r0[k] + r1[k] * r1[k];
            rzn += dinv[k] * (r0[k] * r0[k] + r1[k] * r1[k]);
        }
        s = pcg_block_sum2(rr, rzn, red + 2 * (PCG_THREADS / 32));    // its barrier also ends every read of p above
        ++it;
        rel = sqrt(s.x / f2);
        if (rel < tol) break;
        const double beta = s.y / fmax(rz, 1e-300);
        rz = s.y;
#pragma unroll
        for (int k = 0; k < PCG_NPT; ++k) {
            const int node = tid + k * PCG_THREADS;
            if (node >= NN) continue;
            p[node] = dinv[k] * r0[k] + beta * p[node];
            p[NN + node] = dinv[k] * r1[k] + beta * p[NN + node];
        }
        __syncthreads();
    }
    __syncthreads();
    float* ub = u_out + (size_t)b * 2 * NN;
    for (int i = tid; i < 2 * NN; i += PCG_THREADS) ub[i] = (float)u[i];
    if (tid == 0) { iters[b] = it; relres[b] = rel; }
}

// Floating-material flag of a density field (reference :369-380: cv2 threshold at 0.5 and connectedComponents with
// 8-connectivity; flag = the solid pixels do not form exactly one component).  One CTA per sample: every solid pixel
// starts with its own index as label, labels are lowered to the smallest label among the 8 neighbours (plus one pointer
// jump) until nothing changes; a label only ever names a pixel of the same component, so at the fixed point each
// component carries the index of its first pixel and the roots count the components.
__global__ void __launch_bounds__(1024) mech_fm_kernel(const float* __restrict__ rho, long long* __restrict__ fm, int nel) {
    extern __shared__ int lab[];
    __shared__ int roots;
    const int ne = nel * nel, b = blockIdx.x;
    const float* rb = rho + (size_t)b * ne;
    for (int i = threadIdx.x; i < ne; i += blockDim.x) lab[i] = rb[i] > 0.5f ? i : -1;
    if (threadIdx.x == 0) roots = 0;
    int changed = 1;
    while (__syncthreads_or(changed)) {
        changed = 0;
        for (int i = threadIdx.x; i < ne; i += blockDim.x) {
            const int l = lab[i];
            if (l < 0) continue;
            const int r = i / nel, c = i - r * nel;
            int m = l;
            for (int rr = max(r - 1, 0); rr <= min(r + 1, nel - 1); ++rr)
                for (int cc = max(c - 1, 0); cc <= min(c + 1, nel - 1); ++cc) {
                    const int q = lab[rr * nel + cc];
                    if (q >= 0 && q < m) m = q;
                }
            m = min(m, lab[m]);
            if (m < l) { lab[i] = m; changed = 1; }
        }
    }
    int mine = 0;
    for (int i = threadIdx.x; i < ne; i += blockDim.x) mine += lab[i] == i;
    if (mine) atomicAdd(&roots, mine);
    __syncthreads();
    if (threadIdx.x == 0) fm[b] = roots != 1;
}

static int upload_ke(const float* KE_dev, cudaStream_t st) {
    PIDM_CUDA(cudaMemcpyToSymbolAsync(c_KE, KE_dev, 64 * sizeof(float), 0, cudaMemcpyDeviceToDevice, st));
    return 0;
}

}  // namespace pidm
using namespace pidm;

extern "C" int pidm_mechanics_residual_fwd(const float* u, const float* rho, const float* bcs, const float* KE,
                                           float* residual, float* compliance, int B, int nel, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if (int e = upload_ke(KE, st)) return e;
    if (compliance) PIDM_CUDA(cudaMemsetAsync(compliance, 0, B * sizeof(float), st));
    const int nn = nel + 1;
    PIDM_REQUIRE((2 * nn * nn) % 2 == 0 && nel >= 2 && nel <= 256, "mechanics: 2 <= nel <= 256 required (got %d)", nel);
    dim3 grid(ceil_div(nn, MECH_BAND), B);
    const size_t smem = (size_t)(2 * (MECH_BAND + 2) * nn + (MECH_BAND + 1) * nel) * sizeof(float);
    mech_node_kernel<0><<<grid, MECH_THREADS, smem, st>>>(u, rho, bcs, residual, compliance, nullptr, nullptr, nullptr, nullptr, nel);
    PIDM_LAUNCH_CHECK("mechanics_residual_fwd");
    return 0;
}

// workspace: float[B * 2 * (nel+1)^2].  grad_residual / grad_compliance may be NULL.  grad_u, grad_rho overwritten.
extern "C" int pidm_mechanics_residual_bwd(const float* u, const float* rho, const float* bcs, const float* KE,
                                           const float* grad_residual, const float* grad_compliance, float* grad_u,
                                           float* grad_rho, float* workspace, int B, int nel, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if (int e = upload_ke(KE, st)) return e;
    const int nn = nel + 1;
    PIDM_REQUIRE(nel >= 2 && nel <= 256, "mechanics: 2 <= nel <= 256 required (got %d)", nel);
    dim3 grid(ceil_div(nn, MECH_BAND), B);
    const size_t smem = (size_t)(2 * (MECH_BAND + 2) * nn + (MECH_BAND + 1) * nel) * sizeof(float);
    mech_node_kernel<1><<<grid, MECH_THREADS, smem, st>>>(u, rho, bcs, nullptr, nullptr, grad_residual, grad_compliance,
                                                        workspace, grad_u, nel);
    mech_node_kernel<2><<<grid, MECH_THREADS, smem, st>>>(u, rho, bcs, nullptr, nullptr, nullptr, nullptr, workspace, grad_u, nel);
    mech_drho_kernel<<<dim3(ceil_div(nel * nel, 128), B), 128, 0, st>>>(u, workspace, grad_rho, nel);
    PIDM_LAUNCH_CHECK("mechanics_residual_bwd");
    return 0;
}

extern "C" int pidm_bilinear_resize_fwd(const float* x, float* y, int planes, int in, int out, void* stream) {
    long long total = (long long)planes * out * out;
    int grid = (int)((total + 255) / 256);
    if (grid > num_sms() * 8) grid = num_sms() * 8;
    bilinear_fwd_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, y, planes, in, out);
    PIDM_LAUNCH_CHECK("bilinear_resize_fwd");
    return 0;
}

// dx [planes,in,in] is zeroed here, then accumulated.
extern "C" int pidm_bilinear_resize_bwd(const float* dy, float* dx, int planes, int in, int out, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    PIDM_CUDA(cudaMemsetAsync(dx, 0, (size_t)planes * in * in * sizeof(float), st));
    long long total = (long long)planes * out * out;
    int grid = (int)((total + 255) / 256);
    if (grid > num_sms() * 8) grid = num_sms() * 8;
    bilinear_bwd_kernel<<<grid, 256, 0, st>>>(dy, dx, planes, in, out);
    PIDM_LAUNCH_CHECK("bilinear_resize_bwd");
    return 0;
}

/* fused mechanics PIDM loss + gradients, see mech_loss_kernel.  sums6 is zeroed here; NULL gradients = loss only. */
extern "C" int pidm_mech_pidm_loss(const float* u, const float* rho, const float* x0, const float* residual,
                                   const float* compliance, const float* vf, const long long* t,
                                   const float* p2_loss_weight, const float* posterior_var_clipped, float c_data,
                                   float c_residual, float c_ineq, float lambda_opt, float* sums6, float* grad_u,
                                   float* grad_rho, float* grad_residual, float* grad_compliance, int B, int nel,
                                   void* stream) {
    PIDM_REQUIRE(B > 0 && nel >= 2, "mech_pidm_loss: bad sizes B=%d nel=%d", B, nel);
    const int n_grads = (grad_u != nullptr) + (grad_rho != nullptr) + (grad_residual != nullptr) + (grad_compliance != nullptr);
    PIDM_REQUIRE(n_grads == 0 || n_grads == 4, "mech_pidm_loss: the four gradient pointers must be all set or all NULL "
                 "(%d of 4 set)", n_grads);
    cudaStream_t st = (cudaStream_t)stream;
    PIDM_CUDA(cudaMemsetAsync(sums6, 0, 6 * sizeof(float), st));
    mech_loss_kernel<<<B, 256, 0, st>>>(u, rho, x0, residual, compliance, vf, t, p2_loss_weight, posterior_var_clipped, c_data,
                                       c_residual, c_ineq, lambda_opt, sums6, grad_u, grad_rho, grad_residual,
                                       grad_compliance, B, nel);
    PIDM_LAUNCH_CHECK("mech_pidm_loss");
    return 0;
}

extern "C" int pidm_mech_sample_input(const float* x, const float* planes, float* out, int B, int nc, int P, void* stream) {
    PIDM_REQUIRE(B > 0 && nc >= 0 && P >= 2, "mech_sample_input: bad sizes B=%d nc=%d P=%d", B, nc, P);
    const long long total = (long long)B * (3 + nc) * P * P;
    mech_sample_input_kernel<<<(int)std::min<long long>((total + 255) / 256, num_sms() * 8LL), 256, 0,
                               (cudaStream_t)stream>>>(x, planes, out, B, nc, P);
    PIDM_LAUNCH_CHECK("mech_sample_input");
    return 0;
}

extern "C" int pidm_mech_posterior_step(const float* y, const float* x, const float* z, const long long* t,
                                        const float* coef1, const float* coef2, const float* sigma, float* x_out, int B,
                                        int P, void* stream) {
    PIDM_REQUIRE(B > 0 && P >= 2, "mech_posterior_step: bad sizes B=%d P=%d", B, P);
    const long long total = (long long)B * 3 * (P + 1) * (P + 1);
    mech_posterior_kernel<<<(int)std::min<long long>((total + 255) / 256, num_sms() * 8LL), 256, 0,
                            (cudaStream_t)stream>>>(y, x, z, t, coef1, coef2, sigma, x_out, B, P);
    PIDM_LAUNCH_CHECK("mech_posterior_step");
    return 0;
}

extern "C" int pidm_mech_fem_pcg(const float* rho, const float* bcs, const float* KE, float* u, int* iters,
                                 double* relres, double tol, int max_iter, int B, int nel, void* stream) {
    const int nn = nel + 1;
    PIDM_REQUIRE(B > 0 && nel >= 2 && nn * nn <= PCG_THREADS * PCG_NPT,
                 "mech_fem_pcg: 2 <= nel and (nel+1)^2 <= %d required (B=%d nel=%d)", PCG_THREADS * PCG_NPT, B, nel);
    PIDM_REQUIRE(max_iter >= 0 && tol >= 0.0, "mech_fem_pcg: max_iter=%d tol=%g", max_iter, tol);
    cudaStream_t st = (cudaStream_t)stream;
    if (int e = upload_ke(KE, st)) return e;
    mech_ke_to_double_kernel<<<1, 64, 0, st>>>(KE);
    PIDM_LAUNCH_CHECK("mech_fem_pcg (KE)");
    void* kd = nullptr;
    PIDM_CUDA(cudaGetSymbolAddress(&kd, g_KEd));
    PIDM_CUDA(cudaMemcpyToSymbolAsync(c_KEd, kd, 64 * sizeof(double), 0, cudaMemcpyDeviceToDevice, st));
    const size_t smem = (size_t)(4 * nn * nn + 4 * (PCG_THREADS / 32)) * sizeof(double) + (size_t)nel * nel * sizeof(float);
    PIDM_CUDA(allow_smem(mech_pcg_kernel, smem));
    mech_pcg_kernel<<<B, PCG_THREADS, smem, st>>>(rho, bcs, u, iters, relres, tol, max_iter, nel);
    PIDM_LAUNCH_CHECK("mech_fem_pcg");
    return 0;
}

extern "C" int pidm_mech_floating_material(const float* rho, long long* fm, int B, int nel, void* stream) {
    PIDM_REQUIRE(B > 0 && nel >= 1 && nel <= 128, "mech_floating_material: 1 <= nel <= 128 required (B=%d nel=%d)", B, nel);
    const size_t smem = (size_t)nel * nel * sizeof(int);
    PIDM_CUDA(allow_smem(mech_fm_kernel, smem));
    mech_fm_kernel<<<B, 1024, smem, (cudaStream_t)stream>>>(rho, fm, nel);
    PIDM_LAUNCH_CHECK("mech_floating_material");
    return 0;
}
