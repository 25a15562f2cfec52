"""bcs='periodic' on the GPU: the guidance branch with the periodic residual against the oracle, and the mechanics
residual's 'periodic' option.  Every periodic Darcy kernel is checked per element against the fp64 oracle in
test_gpu_physics_census.py (bcs = none and periodic); the engine against the periodic fixtures of the unmodified reference
(oracle/make_golden.py periodic) runs as the 'periodic' rows of test_gpu_e2e.py, test_gpu_parity_bench_path.py,
test_gpu_cocogen.py and test_gpu_dropin.py."""
import pytest
import torch

from checks import rel
from oracle import pidm_oracle as O
from study import build_darcy, config, state_dict

pytestmark = pytest.mark.gpu
DEV = 'cuda'


# ---- end to end ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def ops():
    from physicsinformeddiffusionmodels_b200 import ops
    yield ops
    ops.set_precision('bf16')


def test_periodic_residual_gradient_guidance_matches_oracle(ops):
    """guidance branch (cond = d mean|r(x_t)| / d x_t with the periodic residual) through the engine vs the periodic
    oracle, fp32, with a classifier-free mask that drops one sample"""
    ops.set_precision('fp32')
    g = torch.Generator().manual_seed(77)
    B = 4
    x0 = torch.randn(B, 2, 64, 64, generator=g)
    t = torch.randint(0, 100, (B,), generator=g)
    e = torch.randn(B, 2, 64, 64, generator=g)
    mask = torch.tensor([False, True, False, False])
    sdr = {k: v.clone().requires_grad_('freqs' not in k) for k, v in state_dict().items()}
    loss_ref, _ = O.darcy_training_loss(sdr, config(), x0, t, e, O.diffusion_tables(100), guidance_null_mask=mask,
                                        periodic=True)
    loss_ref.backward()
    model, diff, res = build_darcy('periodic', residual_grad_guidance=True)
    model._null_mask_override = mask.to(DEV)
    loss, _, _, _, _ = diff.darcy_loss_from_draws(x0.to(DEV), t.to(DEV), e.to(DEV), res, 1.0, 1e-3)
    model._null_mask_override = None
    assert abs(loss.item() / loss_ref.item() - 1) < 5e-5, (loss.item(), loss_ref.item())
    loss.backward()
    named = dict(model.named_parameters())
    for k in ('emb_conv.0.weight', 'combine_conv.weight', 'final_conv.1.weight'):
        assert rel(named[k].grad, sdr[k].grad) < 2e-3, (k, rel(named[k].grad, sdr[k].grad))


def test_mechanics_periodic_equals_none():
    """ResidualsMechanics only stores the flag in the reference: 'periodic' computes exactly what 'none' computes"""
    from physicsinformeddiffusionmodels_b200.residuals_mechanics_K import ResidualsMechanics
    g = torch.Generator().manual_seed(4)
    x = torch.randn(2, 3, 64, 64, generator=g) * 0.1
    x[:, 2] = torch.sigmoid(torch.randn(2, 64, 64, generator=g))
    bcs = torch.zeros(2, 4, 65, 65)
    bcs[:, 0, :, 0] = 1.
    bcs[:, 1, :, 0] = 1.
    bcs[:, 3, 20:24, 64] = -1.
    vf = torch.tensor([0.4, 0.5])
    outs = {}
    for b in ('none', 'periodic'):
        res = ResidualsMechanics(model=None, pixels_per_dim=64, pixels_at_boundary=True, no_BC_folder='', device=DEV,
                                 bcs=b)
        assert res.periodic == (b == 'periodic')
        outs[b] = res.compute_residual((x.to(DEV), bcs.to(DEV), vf.to(DEV), None), reduce='per-batch',
                                       return_optimizer=True, return_inequality=True, pass_through=True)
    assert torch.equal(outs['none']['residual'], outs['periodic']['residual'])
    assert torch.equal(outs['none']['inequality'], outs['periodic']['inequality'])
    # compliance is a sum of fp32 atomics: equal up to their ordering
    assert rel(outs['periodic']['optimizer'], outs['none']['optimizer']) < 1e-6
