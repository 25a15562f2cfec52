"""Host checks of the Darcy data generator's spec (no GPU): oracle/darcy_gen_oracle.py against the unmodified
reference's output (tests/golden/darcy_gen.pt, its geometry_* keys at a second geometry; oracle/make_golden.py
darcy_gen), the pinned banded solve against the reference's lstsq, the set-up the generator computes on the host, its
constructor and C-ABI validation, and the exactness of the known-answer operands the GPU replays rely on."""
import numpy as np
import pytest
import scipy.linalg
import scipy.sparse as sp
import torch

import checks
from oracle import darcy_gen_oracle as DO

P = 64


@pytest.fixture(scope='module')
def fx(golden):
    return golden('darcy_gen.pt')


@pytest.fixture(scope='module')
def lstsq_solutions(fx):
    return [DO.solve_lstsq(K.numpy()) for K in fx['K']]


def test_lstsq_reproduces_reference(fx, lstsq_solutions):
    # same entries as the reference's findiff matrices, summed in another order; cond(M) ~ 1e7
    for (p, res), p_ref, res_ref in zip(lstsq_solutions, fx['p'].numpy(), fx['res'].numpy()):
        assert np.abs(p - p_ref).max() <= 1e-8 * np.abs(p_ref).max()
        assert abs(res - res_ref) <= 1e-8 * res_ref


def test_banded_solve_matches_lstsq(fx, lstsq_solutions):
    for K, (p_ls, res_ls) in zip(fx['K'].numpy(), lstsq_solutions):
        p, res = DO.solve_banded(K)
        assert np.abs(p - p_ls).max() <= 1e-5 * np.abs(p_ls).max()
        assert abs(res - res_ls) <= 1e-4 * res_ls
        assert abs(DO.weights() @ p) <= 1e-15 * np.abs(p).max()


def test_setup_matches_reference(fx):
    from physicsinformeddiffusionmodels_b200 import darcy_data_generation as G
    grid = G.uniform_points_pixelwise(P, 1., True)
    lam, _ = G.compute_eigenpairs(G.complete_covariance_matrix(grid, 0.1), 64)
    ref = fx['eigenvalues'].numpy()
    assert np.abs(lam - ref).max() <= 1e-10 * np.abs(ref).max()
    assert np.array_equal(G.create_f_s(grid[:, 0], grid[:, 1]), fx['f_s'].numpy())
    assert np.array_equal(G.create_int_cond(True, (P, P), 1. / (P - 1)).reshape(-1), fx['int_cond'].numpy())
    assert np.array_equal(DO.weights(), fx['int_cond'].numpy())
    for s, z in zip(fx['seed'].tolist(), fx['z'].numpy()):
        assert np.array_equal(G.z_from_seed(s, 64), z)


def test_source_equals_training_residual_source(fx):
    from physicsinformeddiffusionmodels_b200.residuals_darcy import ResidualsDarcy
    res = ResidualsDarcy(model=None, fd_acc=2, pixels_per_dim=P, pixels_at_boundary=True, reverse_d1=True, device='cpu')
    assert np.array_equal(res.f_s.reshape(-1).double().numpy(), fx['f_s'].numpy())
    assert np.array_equal(DO.source(), fx['f_s'].numpy())


def test_constructor_validation():
    from physicsinformeddiffusionmodels_b200.darcy_data_generation import DarcyDataGenerator
    with pytest.raises(NotImplementedError):
        DarcyDataGenerator(acc=4)
    with pytest.raises(ValueError):
        DarcyDataGenerator(pixels_per_dim=32)
    with pytest.raises(ValueError):
        DarcyDataGenerator(device='cpu')
    with pytest.raises(ValueError):
        DarcyDataGenerator(q=0)


def test_c_entry_points_reject_bad_arguments():
    from physicsinformeddiffusionmodels_b200._lib import call
    per_sample = (P * P * (3 * P + 4) + P * P) * 8
    assert call('pidm_darcy_gen_workspace_bytes', 3, P) == 3 * per_sample
    assert call('pidm_darcy_gen_workspace_bytes', 3, 32) == -1
    ws = 1 << 40
    args = dict(B=1, pixels=P, flags=1, stages=7, wsb=ws)

    def solve(**kw):
        a = {**args, **kw}
        call('pidm_darcy_gen_solve', None, None, None, None, None, None, a['wsb'], a['B'], a['pixels'], 1.0, 1,
             a['flags'], a['stages'], None)
    for kw, msg in ((dict(pixels=32), 'pixels'), (dict(flags=2), 'flags'), (dict(flags=4), 'flags'),
                    (dict(stages=8), 'stages'), (dict(stages=0), 'stages'), (dict(wsb=per_sample - 1), 'workspace')):
        with pytest.raises(RuntimeError, match=msg):
            solve(**kw)
    with pytest.raises(RuntimeError, match='pixels'):
        call('pidm_darcy_gen_kle', None, None, None, 1, 64, 32, None)
    for B in (65536, -1):
        with pytest.raises(RuntimeError, match='B = '):
            call('pidm_darcy_gen_kle', None, None, None, B, 64, P, None)
        with pytest.raises(RuntimeError, match='B = '):
            solve(B=B)
    for q in (0, P * P + 1):
        with pytest.raises(RuntimeError, match='q'):
            call('pidm_darcy_gen_kle', None, None, None, 1, q, P, None)


# ---- a second geometry of the reference: pixel centres, h = L / P, the plain mean, reverse_dy = False ----------------
@pytest.fixture(scope='module')
def fxg(golden):
    return {k[len('geometry_'):]: v for k, v in golden('darcy_gen.pt').items() if k.startswith('geometry_')}


def _geo(fxg):
    return dict(pixels_at_boundary=bool(fxg['pixels_at_boundary']), reverse_dy=bool(fxg['reverse_dy']),
                domain_length=float(fxg['domain_length']))


def test_oracle_reproduces_reference_at_another_geometry(fxg):
    geo = _geo(fxg)
    assert geo == dict(pixels_at_boundary=False, reverse_dy=False, domain_length=2.)
    assert np.array_equal(DO.source(geo['pixels_at_boundary'], geo['domain_length']), fxg['f_s'].numpy())
    assert np.array_equal(DO.weights(geo['pixels_at_boundary'], geo['domain_length']), fxg['int_cond'].numpy())
    for K, p_ref, res_ref in zip(fxg['K'].numpy(), fxg['p'].numpy(), fxg['res'].numpy()):
        p, res = DO.solve_lstsq(K, **geo)
        assert np.abs(p - p_ref).max() <= 1e-8 * np.abs(p_ref).max()
        assert abs(res - res_ref) <= 1e-8 * res_ref
        p, res = DO.solve_banded(K, **geo)
        assert np.abs(p - p_ref).max() <= 1e-5 * np.abs(p_ref).max()
        assert abs(res - res_ref) <= 1e-4 * res_ref


def test_setup_matches_reference_at_another_geometry(fxg):
    from physicsinformeddiffusionmodels_b200 import darcy_data_generation as G
    geo = _geo(fxg)
    grid = G.uniform_points_pixelwise(P, geo['domain_length'], geo['pixels_at_boundary'])
    assert np.array_equal(G.create_f_s(grid[:, 0], grid[:, 1]), fxg['f_s'].numpy())
    int_cond = G.create_int_cond(False, (P, P), geo['domain_length'] / P)
    assert int_cond.shape == (P * P, 1) and np.array_equal(int_cond.reshape(-1), fxg['int_cond'].numpy())


def test_reverse_dy_leaves_the_normal_equations_unchanged():
    """h1 and the sign of the y BC rows enter N, A^T f_s and |M p - b| squared or under | |: A and BC^T BC are identical"""
    K = np.exp(0.5 * np.random.default_rng(3).standard_normal(P * P))
    for pab, dl in ((True, 1.), (False, 0.3)):
        A1, B1 = DO.operators(K, pixels_at_boundary=pab, reverse_dy=True, domain_length=dl)
        A0, B0 = DO.operators(K, pixels_at_boundary=pab, reverse_dy=False, domain_length=dl)
        assert (A1 != A0).nnz == 0
        assert ((B1.T @ B1) != (B0.T @ B0)).nnz == 0


# ---- the known-answer operands of tests/test_gpu_darcy_gen_replay.py are exact in fp64 -------------------------------
def _int_stencils():
    """2h D1 and h^2 D2 of one axis as int64 sparse matrices"""
    E, F = DO._d1(P, 0.5), DO._d2(P, 1.)
    assert np.array_equal(E.data, np.round(E.data)) and np.array_equal(F.data, np.round(F.data))
    return E.astype(np.int64), F.astype(np.int64)


@pytest.mark.parametrize('geo', checks.DGEN_EXACT_GEOMETRIES, ids=lambda g: f"pab{int(g['pixels_at_boundary'])}"
                         f"_L{g['domain_length']:g}")
def test_dyadic_assembly_is_exact(geo):
    """integer evaluation of N and A^T f_s for K = k / 16, h = 2^-s:  64 h^2 A = -4 k (F0 + F1) - (E0 k) E0 - (E1 k) E1
    and 2 h BC = +-E rows are integer matrices, so N = X / (4096 h^4) + Y / (4 h^2) with X = Aint^T Aint, Y = Bint^T Bint;
    the oracle's fp64 band must equal that bit for bit (and hence so must every order of summation)"""
    h, _ = DO.geometry(**geo)
    s = -int(np.log2(h))
    assert h == 2.0 ** -s
    g = torch.Generator().manual_seed(11)
    K, f = checks.dgen_dyadic_K(1, g, 'cpu')[0].numpy(), checks.dgen_dyadic_source(g, 'cpu').numpy()
    k = np.round(K * 16).astype(np.int64)
    E, F = _int_stencils()
    I = sp.identity(P, dtype=np.int64, format='csr')
    E0, F0, E1, F1 = (sp.kron(a, b).tocsr() for a, b in ((E, I), (F, I), (I, E), (I, F)))
    diag = lambda v: sp.diags(v, dtype=np.int64)  # noqa: E731
    Aint = (-4 * diag(k) @ (F0 + F1) - diag(E0 @ k) @ E0 - diag(E1 @ k) @ E1).tocsr()
    idx = np.arange(P * P).reshape(P, P)
    Bint = sp.vstack([E0[idx[0, :]], E0[idx[-1, :]], E1[idx[:, 0]], E1[idx[:, -1]]]).tocsr()
    X, Y = (Aint.T @ Aint).tocsr(), (Bint.T @ Bint).tocsr()
    # N = 2^(4s - 12) X + 2^(2s - 2) Y = 2^e Z with Z integer
    if 2 * s <= 10:
        Z, e = X + (2 ** (10 - 2 * s)) * Y, 4 * s - 12
    else:
        Z, e = (2 ** (2 * s - 10)) * X + Y, 2 * s - 2
    Z = Z.tolil()
    Z[0, 0] *= 2
    Z = Z.tocsr()
    assert abs(Z).max() < 2 ** 53 and abs(Aint).max() < 2 ** 53
    band, rhs = DO.normal_band(K, f, **geo)
    Zb = DO.to_band(Z.astype(np.float64))
    assert np.array_equal(band, Zb * 2.0 ** e)
    rhs_int = Aint.T @ np.round(f).astype(np.int64)            # A^T f = Aint^T f / (64 h^2)
    assert np.abs(rhs_int).max() < 2 ** 53
    assert np.array_equal(rhs, rhs_int.astype(np.float64) * 2.0 ** (2 * s - 6))


def test_dyadic_factor_is_exact():
    """L0 L0^T and L0 y0 of the factor stage's known answer are exact (integer products of 256 L0 and 16 y0), and a
    Cholesky factorisation in another order (LAPACK's) returns L0 bit for bit"""
    g = torch.Generator().manual_seed(12)
    Lb = checks.dgen_dyadic_factor(1, g, 'cpu', fill=0.)[0]
    L = checks.dgen_band_to_dense(Lb).numpy()
    y0 = (torch.randint(-8, 9, (P * P,), generator=g).double() / 16).numpy()
    Li = np.round(L * 256).astype(np.int64)
    assert np.array_equal(Li, L * 256)
    Nint = Li @ Li.T                                             # 2^16 N, |.| < 2^20
    Nf = L @ L.T
    assert np.abs(Nint).max() < 2 ** 53 and np.array_equal(Nf, Nint * 2.0 ** -16)
    rhs_int = Li @ np.round(y0 * 16).astype(np.int64)            # 2^12 L0 y0
    assert np.array_equal(L @ y0, rhs_int * 2.0 ** -12)
    assert np.array_equal(np.linalg.cholesky(Nf), L)
    assert np.array_equal(scipy.linalg.solve_triangular(L, L @ y0, lower=True), y0)
    # the post stage's known answer: y = L0^T x0, back substitution returns x0
    x0 = y0[::-1].copy()
    assert np.array_equal(L.T @ x0, (Li.T @ np.round(x0 * 16).astype(np.int64)) * 2.0 ** -12)
    assert np.array_equal(scipy.linalg.solve_triangular(L.T, L.T @ x0, lower=False), x0)
