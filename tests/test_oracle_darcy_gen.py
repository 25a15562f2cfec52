"""Host checks of the Darcy data generator's spec (no GPU): oracle/darcy_gen_oracle.py against the unmodified
reference's output (tests/golden/darcy_gen.pt, oracle/make_golden.py darcy_gen), the pinned banded solve against the
reference's lstsq, the set-up the generator computes on the host, and its constructor validation."""
import numpy as np
import pytest
import torch

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
    with pytest.raises(RuntimeError, match='q'):
        call('pidm_darcy_gen_kle', None, None, None, 1, 0, P, None)
