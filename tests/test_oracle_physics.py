"""The fp64 physics references the per-element GPU tests compare against (test_gpu_physics_census.py), checked on the
CPU: the Darcy stencil-matrix form against the restatement of the reference at every geometry, and the matrix-free
mechanics operator against the resize-based restatement and against the assembled scipy stiffness matrix."""
import numpy as np
import pytest
import torch

from oracle import pidm_oracle as O

P = 64
GEOMETRIES = [dict(domain_length=L, reverse_d1=rev, pixels_at_boundary=pab)
              for L in (1.0, 2.5) for rev in (False, True) for pab in (False, True)]


def _geom_id(g):
    return f'L{g["domain_length"]}-rev{int(g["reverse_d1"])}-pab{int(g["pixels_at_boundary"])}'


@pytest.mark.parametrize('periodic', [False, True], ids=['none', 'periodic'])
@pytest.mark.parametrize('geom', GEOMETRIES, ids=_geom_id)
def test_darcy_residual_matrix_equals_restatement(geom, periodic):
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 2, P, P, generator=g, dtype=torch.float64)
    x[:, 1] = torch.exp(0.5 * x[:, 1])
    r = O.darcy_residual_matrix(x, periodic, **geom)
    ref = O.darcy_residual(x, periodic=periodic, **geom)
    for c in range(3):
        assert ((r[..., c] - ref[..., c]).norm() / ref[..., c].norm()).item() < 1e-12, c
    # the absolute form bounds the signed one, and the VJP is the transpose of the same linear map in p
    assert (r.abs() <= O.darcy_residual_matrix(x, periodic, absolute=True, **geom) * (1 + 1e-12)).all()
    cot = torch.randn(2, P * P, 3, generator=g, dtype=torch.float64)
    xg = x.clone().requires_grad_(True)
    want = torch.autograd.grad((O.darcy_residual(xg, periodic=periodic, **geom) * cot).sum(), xg)[0]
    got = O.darcy_residual_vjp(x, cot, periodic, **geom)
    assert ((got - want).norm() / want.norm()).item() < 1e-12


def _mech_operands(B, nel, seed):
    """fp64 u, rho (with exact zeros), bcs with Dirichlet values 1, 0.5 and -1, loads on fixed dofs and at corners"""
    g = torch.Generator().manual_seed(seed)
    nn = nel + 1
    u = torch.randn(B, 2, nn, nn, generator=g, dtype=torch.float64)
    rho = torch.rand(B, nel, nel, generator=g, dtype=torch.float64)
    rho[rho < 0.1] = 0
    bcs = torch.zeros(B, 4, nn, nn, dtype=torch.float64)
    bcs[:, 0, :, 0] = 1.
    bcs[:, 1, :, 0] = 0.5
    bcs[:, 1, -1, :] = -1.
    bcs[:, 2:] = torch.randn(B, 2, nn, nn, generator=g, dtype=torch.float64) * (torch.rand(B, 2, nn, nn, generator=g) < 0.2)
    bcs[:, 2, 0, 0], bcs[:, 3, -1, -1], bcs[:, 3, 0, -1] = 2., -3., 1.5
    return u, rho, bcs


def test_mechanics_matfree_equals_resized_restatement():
    g = torch.Generator().manual_seed(8)
    B = 2
    x = torch.randn(B, 3, 64, 64, generator=g, dtype=torch.float64) * 0.1
    x[:, 2] = torch.rand(B, 64, 64, generator=g, dtype=torch.float64)
    _, _, bcs = _mech_operands(B, 64, 9)
    vf = torch.tensor([0.4, 0.5], dtype=torch.float64)
    r_ref, c_ref, _ = O.mechanics_residual(x, bcs, vf)
    r, c = O.mechanics_matfree(O.bilinear_resize(x[:, :2], 65), x[:, 2], bcs)
    assert ((r - r_ref).norm() / r_ref.norm()).item() < 1e-12
    assert ((c - c_ref).abs() / c_ref.abs()).max().item() < 1e-12


@pytest.mark.parametrize('nel', [2, 7, 64])
def test_mechanics_matfree_equals_assembled_matrix(nel):
    B = 2
    u, rho, bcs = _mech_operands(B, nel, nel)
    r, comp = O.mechanics_matfree(u, rho, bcs)
    ra, ca = O.mechanics_matfree(u, rho, bcs, absolute=True)
    ug = u.clone().requires_grad_(True)
    rg, cg = O.mechanics_matfree(ug, rho, bcs)
    cot = torch.randn(B, r.shape[1], generator=torch.Generator().manual_seed(nel), dtype=torch.float64)
    du = torch.autograd.grad((rg * cot).sum() + cg.sum(), ug)[0]
    for b in range(B):
        K, f = O.reduced_system(rho[b].numpy(), bcs[b].numpy())
        ub = u[b].permute(1, 2, 0).reshape(-1).numpy()
        want = K @ ub - f
        assert np.abs(r[b].numpy() - want).max() <= 1e-12 * np.abs(want).max()
        assert abs(comp[b].item() - ub @ (K @ ub)) <= 1e-12 * abs(ub) @ np.abs(K @ ub)
        assert (r[b].abs() <= ra[b] * (1 + 1e-12)).all() and abs(comp[b]) <= ca[b] * (1 + 1e-12)
        # VJP of r . cot + compliance: K^T cot + (K + K^T) u with the modified (non-symmetric) K
        want_du = K.T @ cot[b].numpy() + (K + K.T) @ ub
        got_du = du[b].permute(1, 2, 0).reshape(-1).numpy()
        assert np.abs(got_du - want_du).max() <= 1e-12 * np.abs(want_du).max()
