"""bcs='periodic' on the CPU: the oracle's periodic residual, its VJP and stencils (oracle/pidm_oracle.py) against
fixtures produced by the UNMODIFIED reference with ResidualsDarcy(bcs='periodic') (oracle/make_golden.py periodic), an
fp64 known answer, and the host logic of the flag.  The periodic loss, sampling loop and CoCoGen correction are rows of
test_oracle_golden.py."""
import math

import pytest
import torch

from checks import rel
from oracle import pidm_oracle as O


def test_periodic_residual_and_vjp_match_reference(golden):
    gd = golden('darcy_residual_periodic.pt')
    assert torch.equal(gd['x0_pred'], golden('darcy_residual.pt')['x0_pred'])
    assert rel(O.darcy_residual(gd['x0_pred'], periodic=True), gd['residual']) < 1e-5
    # periodic differs from 'none' (else this file would test nothing new)
    assert rel(O.darcy_residual(gd['x0_pred']), gd['residual']) > 1e-2
    x = gd['x0_pred'].clone().requires_grad_(True)
    (O.darcy_residual(x, periodic=True) * gd['cotangent']).sum().backward()
    assert rel(x.grad, gd['grad_x0_pred']) < 1e-5


@pytest.mark.parametrize('mode', ['d_d0', 'd_d1', 'd_d00', 'd_d11', 'd_d01'])
def test_periodic_stencil_modes_match_reference(golden, mode):
    gd = golden('darcy_residual_periodic.pt')
    d0, d1 = O.spacing(64)
    assert rel(O.stencil_gradients(gd['x0_pred'][:, 0], mode, d0, d1, periodic=True), gd['stencil_' + mode]) < 1e-5


def test_periodic_residual_known_answer_fourier_modes():
    """p = sin(a i) cos(b j), K = 2 + cos(c i) + sin(e j) with a, b, c, e multiples of 2 pi / 64.  On the periodic grid
    the wrapped central differences of such modes are exact: D1 sin(t x) = cos(t x) sin t / h and
    D2 sin(t x) = -4 sin^2(t/2) sin(t x) / h^2 (likewise for cos), so eq_0 and both BC channels are known in closed form."""
    P = 64
    h0 = 1.0 / 63
    h1 = -h0                                                   # reverse_d1
    a, b, c, e = (2 * math.pi * k / P for k in (1, 2, 3, 1))
    idx = torch.arange(P, dtype=torch.float64)
    I, J = torch.meshgrid(idx, idx, indexing='ij')
    p = torch.sin(a * I) * torch.cos(b * J)
    K = 2 + torch.cos(c * I) + torch.sin(e * J)
    r = O.darcy_residual(torch.stack([p, K])[None], periodic=True).reshape(P, P, 3)
    p0 = math.sin(a) / h0 * torch.cos(a * I) * torch.cos(b * J)
    p1 = torch.sin(a * I) * (-math.sin(b) / h1 * torch.sin(b * J))
    p00 = -4 * math.sin(a / 2) ** 2 / h0 ** 2 * p
    p11 = -4 * math.sin(b / 2) ** 2 / h1 ** 2 * p
    K0 = -math.sin(c) / h0 * torch.sin(c * I)
    K1 = math.sin(e) / h1 * torch.cos(e * J)
    fs = O.darcy_source(P, dtype=torch.float64)
    exact = -(K * p00 + K0 * p0) - (K * p11 + K1 * p1) - fs
    assert (r[..., 0] - exact).abs().max() < 1e-9
    assert (r[0, :, 1] + p0[0]).abs().max() < 1e-9 and (r[-1, :, 1] - p0[-1]).abs().max() < 1e-9
    assert (r[:, 0, 2] - p1[:, 0]).abs().max() < 1e-9 and (r[:, -1, 2] + p1[:, -1]).abs().max() < 1e-9
    assert r[1:-1, :, 1].abs().max() == 0 and r[:, 1:-1, 2].abs().max() == 0


def test_periodic_flag_is_accepted_by_the_host_classes():
    from physicsinformeddiffusionmodels_b200.grad_utils import StencilGradients
    from physicsinformeddiffusionmodels_b200.residuals_darcy import ResidualsDarcy
    from physicsinformeddiffusionmodels_b200.residuals_mechanics_K import ResidualsMechanics
    res = ResidualsDarcy(model=None, fd_acc=2, pixels_per_dim=64, pixels_at_boundary=True, reverse_d1=True,
                         device='cpu', bcs='periodic')
    assert res.periodic and res.geometry == (1.0, True, True, True)
    assert res.grads.stencil_gradients.periodic
    none = ResidualsDarcy(model=None, fd_acc=2, pixels_per_dim=64, pixels_at_boundary=True, reverse_d1=True,
                          device='cpu', bcs='none')
    assert none.geometry == (1.0, True, True, False)
    assert torch.equal(res.f_s, none.f_s) and torch.equal(res.trapezoidal_weights, none.trapezoidal_weights)
    assert StencilGradients(d0=1.0, d1=1.0, periodic=True).periodic
    with pytest.raises(NotImplementedError):
        StencilGradients(d0=1.0, d1=1.0, fd_acc=4, periodic=True)
    assert ResidualsMechanics(model=None, pixels_per_dim=64, pixels_at_boundary=True, no_BC_folder='',
                              bcs='periodic').periodic


def test_darcy_flags_word():
    from physicsinformeddiffusionmodels_b200 import ops
    assert ops.darcy_flags(False) == 0 and ops.darcy_flags(True) == 1        # the values callers passed before
    assert ops.darcy_flags(False, True) == 2 and ops.darcy_flags(True, True) == 3


@pytest.mark.parametrize('name', ['pidm_darcy_residual_fwd', 'pidm_darcy_residual_bwd', 'pidm_darcy_pidm_loss',
                                  'pidm_darcy_jacobian_max', 'pidm_fd_stencil'])
def test_unknown_flag_bits_are_rejected_by_the_library(name):
    """The flag check runs before any CUDA call, so it needs no device (null pointers, no stream)."""
    from physicsinformeddiffusionmodels_b200._lib import call
    args = {'pidm_darcy_residual_fwd': (None, None, None, 1, 64, 1.0, 1, 4, None),
            'pidm_darcy_residual_bwd': (None, None, None, None, 1, 64, 1.0, 1, 1 | 8, None),
            'pidm_darcy_pidm_loss': (None,) * 7 + (1.0, 1e-3) + (None,) * 3 + (1, 64, 1.0, 1, 16, None),
            'pidm_darcy_jacobian_max': (None, None, 1, 64, 1.0, 1, -1, None),
            'pidm_fd_stencil': (None, None, 1, 64, 4 | 16, 1.0, 1.0, None)}[name]
    with pytest.raises(RuntimeError, match='flag|mode'):
        call(name, *args)
