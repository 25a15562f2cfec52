"""Host fp64 oracle of the Darcy data generator (reference src/darcy_data_generation.py:123-165), numpy / scipy.

Every function takes the reference's geometry as keywords: pixels_at_boundary (grid points on the boundary, h = L/(P-1)
and trapezoid weights, else pixel centres, h = L/P and the plain mean), reverse_dy (h1 = -h, BC rows +D1 | -D1) and
domain_length L.  `system(K)` assembles M = [A; BC rows; integral row] sparsely from the closed-form second-order tables (the findiff acc=2
tables: central in the interior, one-sided 3- / 4-point stencils at the ends of each axis) and the right-hand side b.
Two solvers:
  * `solve_lstsq`   dense scipy lstsq of M p = b: the reference algorithm (about 10 s per sample on 8 cores);
  * `solve_banded`  the normal equations of [A; BC] with node 0 pinned (N_00 doubled), banded fp64 Cholesky
                    (scipy solveh_banded, half-bandwidth 3P + 3), then p -= (w^T p) / (w^T 1).
`normal_band(K, f_s)` is the pinned normal equations in the generator's row-band layout, the per-stage reference of its
assembly.  `residual(M, b, p)` is the reference's res = mean |M p - b|."""
import numpy as np
import scipy.linalg
import scipy.sparse as sp

P = 64


def _d1(n, h):
    D = sp.lil_matrix((n, n))
    for i in range(n):
        if i == 0:
            D[0, 0:3] = np.array([-1.5, 2., -0.5]) / h
        elif i == n - 1:
            D[i, n - 3:n] = np.array([0.5, -2., 1.5]) / h
        else:
            D[i, i - 1], D[i, i + 1] = -0.5 / h, 0.5 / h
    return D.tocsr()


def _d2(n, h):
    D = sp.lil_matrix((n, n))
    for i in range(n):
        if i == 0:
            D[0, 0:4] = np.array([2., -5., 4., -1.]) / h ** 2
        elif i == n - 1:
            D[i, n - 4:n] = np.array([-1., 4., -5., 2.]) / h ** 2
        else:
            D[i, i - 1:i + 2] = np.array([1., -2., 1.]) / h ** 2
    return D.tocsr()


def geometry(pixels_at_boundary=True, reverse_dy=True, domain_length=1.):
    h0 = domain_length / (P - 1) if pixels_at_boundary else domain_length / P
    return h0, (-h0 if reverse_dy else h0)


BW = 3 * P + 3                                 # half-bandwidth of the normal equations


def source(pixels_at_boundary=True, domain_length=1.):
    """f_s on the reference's grid (uniform_points_pixelwise, create_f_s): +10 on the lower-left 0.125 x 0.125 corner,
    -10 on the one at (1, 1), whatever the domain length"""
    h = domain_length / P
    x = np.linspace(0., domain_length, P) if pixels_at_boundary else np.linspace(h / 2, domain_length - h / 2, P)
    X, Y = np.meshgrid(x, x, indexing='ij')
    f = np.zeros((P, P))
    f[(np.abs(X - 0.0625) <= 0.0625) & (np.abs(Y - 0.0625) <= 0.0625)] = 10.
    f[(np.abs(X - 1 + 0.0625) <= 0.0625) & (np.abs(Y - 1 + 0.0625) <= 0.0625)] = -10.
    return f.reshape(-1)


def weights(pixels_at_boundary=True, domain_length=1.):
    h0, _ = geometry(pixels_at_boundary, True, domain_length)
    if not pixels_at_boundary:
        return np.full(P * P, 1. / P ** 2)
    c = np.full(P, 2.)
    c[0] = c[-1] = 1.
    return (np.outer(c, c) * (h0 ** 2 / 4.)).reshape(-1)


def operators(K, pixels_at_boundary=True, reverse_dy=True, domain_length=1., absolute=False):
    """(A, BC) sparse for K [P*P]; BC stacks -D0 on row 0, +D0 on row P-1, then +-D1 on column 0 and -+D1 on column P-1.
    absolute=True: every stencil, field and sign by its magnitude (A(|p|, |K|) bounds the rounding of A p, and the
    chain of absolute values bounds the rounding of A's coefficients themselves)."""
    h0, h1 = geometry(pixels_at_boundary, reverse_dy, domain_length)
    I = sp.identity(P, format='csr')
    D0, D00 = sp.kron(_d1(P, h0), I).tocsr(), sp.kron(_d2(P, h0), I).tocsr()
    D1, D11 = sp.kron(I, _d1(P, h1)).tocsr(), sp.kron(I, _d2(P, h1)).tocsr()
    K = np.asarray(K, dtype=np.float64).reshape(-1)
    if absolute:
        D0, D00, D1, D11, K = abs(D0), abs(D00), abs(D1), abs(D11), np.abs(K)
        K0, K1 = D0 @ K, D1 @ K
        A = (sp.diags(K) @ D00 + sp.diags(K0) @ D0 + sp.diags(K) @ D11 + sp.diags(K1) @ D1).tocsr()
    else:
        K0, K1 = D0 @ K, D1 @ K
        A = (-sp.diags(K) @ D00 - sp.diags(K0) @ D0 - sp.diags(K) @ D11 - sp.diags(K1) @ D1).tocsr()
    idx = np.arange(P * P).reshape(P, P)
    s = 1. if reverse_dy or absolute else -1.
    sb = 1. if absolute else -1.
    BC = sp.vstack([sb * D0[idx[0, :]], D0[idx[-1, :]], s * D1[idx[:, 0]], sb * s * D1[idx[:, -1]]]).tocsr()
    return A, BC


def _f_s(f_s, geo):
    if f_s is None:
        return source(geo.get('pixels_at_boundary', True), geo.get('domain_length', 1.))
    return np.asarray(f_s, dtype=np.float64).reshape(-1)


def system(K, f_s=None, **geo):
    """(M, b): the reference's A_bc_int and b_bc_int (P*P + 4P + 1 rows); f_s defaults to the geometry's source"""
    A, BC = operators(K, **geo)
    w = weights(geo.get('pixels_at_boundary', True), geo.get('domain_length', 1.))
    M = sp.vstack([A, BC, sp.csr_matrix(w.reshape(1, -1))]).tocsr()
    b = np.concatenate([_f_s(f_s, geo), np.zeros(4 * P + 1)])
    return M, b


def pinned_normal(A, BC):
    """N = [A; BC]^T [A; BC] with N_00 doubled (the pin), sparse"""
    MA = sp.vstack([A, BC]).tocsr()
    Nm = (MA.T @ MA).tocsr()
    Nm[0, 0] *= 2.
    return Nm


def to_band(Nm):
    """row-band layout [P*P, BW + 1] of the lower triangle of sparse Nm: band[r, d] = N[r, r - d], 0 where r - d < 0"""
    n = P * P
    band = np.zeros((n, BW + 1))
    Nd = sp.tril(Nm).todia()
    for off, data in zip(Nd.offsets, Nd.data):
        d = -off
        assert 0 <= d <= BW, d
        band[d:, d] = data[:n - d]              # dia data[j] sits at column j, row j + d
    return band


def normal_band(K, f_s=None, **geo):
    """(band [P*P, BW + 1], rhs [P*P]): the pinned normal equations and A^T f_s, laid out as the generator's
    workspace holds them after its assembly stage"""
    A, BC = operators(K, **geo)
    return to_band(pinned_normal(A, BC)), A.T @ _f_s(f_s, geo)


def solve_lstsq(K, f_s=None, **geo):
    M, b = system(K, f_s, **geo)
    p = scipy.linalg.lstsq(M.toarray(), b)[0]
    return p, residual(M, b, p)


def solve_banded(K, f_s=None, **geo):
    A, BC = operators(K, **geo)
    w = weights(geo.get('pixels_at_boundary', True), geo.get('domain_length', 1.))
    band = to_band(pinned_normal(A, BC))
    ab = np.zeros((BW + 1, P * P))             # LAPACK lower band: ab[d, c] = N[c + d, c]
    for d in range(BW + 1):
        ab[d, :P * P - d] = band[d:, d]
    p = scipy.linalg.solveh_banded(ab, A.T @ _f_s(f_s, geo), lower=True)
    p = p - (w @ p) / w.sum()
    M, b = system(K, f_s, **geo)
    return p, residual(M, b, p)


def residual(M, b, p):
    return float(np.abs(M @ p - b).mean())
