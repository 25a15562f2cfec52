"""Host fp64 oracle of the Darcy data generator (reference src/darcy_data_generation.py:123-165), numpy / scipy.

`system(K)` assembles M = [A; BC rows; integral row] sparsely from the closed-form second-order tables (the findiff acc=2
tables: central in the interior, one-sided 3- / 4-point stencils at the ends of each axis) and the right-hand side b.
Two solvers:
  * `solve_lstsq`   dense scipy lstsq of M p = b: the reference algorithm (about 10 s per sample on 8 cores);
  * `solve_banded`  the normal equations of [A; BC] with node 0 pinned (N_00 doubled), banded fp64 Cholesky
                    (scipy solveh_banded, half-bandwidth 3P + 3), then p -= (w^T p) / (w^T 1).
`residual(M, b, p)` is the reference's res = mean |M p - b|."""
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


def source():
    """f_s on the grid x_i = i / (P-1) (reference create_f_s)"""
    x = np.arange(P) / (P - 1)
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
    absolute=True: every stencil, field and sign by its magnitude (A(|p|, |K|) bounds the rounding of A p)."""
    h0, h1 = geometry(pixels_at_boundary, reverse_dy, domain_length)
    I = sp.identity(P, format='csr')
    D0, D00 = sp.kron(_d1(P, h0), I).tocsr(), sp.kron(_d2(P, h0), I).tocsr()
    D1, D11 = sp.kron(I, _d1(P, h1)).tocsr(), sp.kron(I, _d2(P, h1)).tocsr()
    K = np.asarray(K, dtype=np.float64).reshape(-1)
    if absolute:
        D0, D00, D1, D11, K = abs(D0), abs(D00), abs(D1), abs(D11), np.abs(K)
        K0, K1 = D0 @ K, D1 @ K
        A = (sp.diags(K) @ D00 + sp.diags(K0) @ D0 + sp.diags(K) @ D11 + sp.diags(K1) @ D1).tocsr()
        return A, None
    K0, K1 = D0 @ K, D1 @ K
    A = (-sp.diags(K) @ D00 - sp.diags(K0) @ D0 - sp.diags(K) @ D11 - sp.diags(K1) @ D1).tocsr()
    idx = np.arange(P * P).reshape(P, P)
    s = 1. if reverse_dy else -1.
    BC = sp.vstack([-D0[idx[0, :]], D0[idx[-1, :]], s * D1[idx[:, 0]], -s * D1[idx[:, -1]]]).tocsr()
    return A, BC


def system(K, **geo):
    """(M, b): the reference's A_bc_int and b_bc_int (P*P + 4P + 1 rows)"""
    A, BC = operators(K, **geo)
    w = weights(geo.get('pixels_at_boundary', True), geo.get('domain_length', 1.))
    M = sp.vstack([A, BC, sp.csr_matrix(w.reshape(1, -1))]).tocsr()
    b = np.concatenate([source(), np.zeros(4 * P + 1)])
    return M, b


def solve_lstsq(K, **geo):
    M, b = system(K, **geo)
    p = scipy.linalg.lstsq(M.toarray(), b)[0]
    return p, residual(M, b, p)


def solve_banded(K, **geo):
    A, BC = operators(K, **geo)
    w = weights(geo.get('pixels_at_boundary', True), geo.get('domain_length', 1.))
    MA = sp.vstack([A, BC]).tocsr()
    Nm = (MA.T @ MA).tocsr()
    Nm[0, 0] *= 2.
    rhs = A.T @ source()
    u = 3 * P + 3
    ab = np.zeros((u + 1, P * P))
    Nd = Nm.todia()
    for off, data in zip(Nd.offsets, Nd.data):
        if 0 <= -off <= u:                     # lower diagonal -off: ab[d, c] = N[c + d, c]
            d = -off
            ab[d, :P * P - d] = data[:P * P - d]
    p = scipy.linalg.solveh_banded(ab, rhs, lower=True)
    p = p - (w @ p) / w.sum()
    M, b = system(K, **geo)
    return p, residual(M, b, p)


def residual(M, b, p):
    return float(np.abs(M @ p - b).mean())
