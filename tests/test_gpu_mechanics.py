"""configs[2] (topology optimisation / linear elasticity): the mechanics branch of the training loss through the
engine against the UNMODIFIED reference (tests/golden/mechanics_loss.pt, dense 8450 x 8450 assembly) and against the CPU
oracle at the reference's model size (Unet3D dim=128, channels=10, out_dim=3; main.py:102-109,126), and the
topology-optimisation evaluation metrics.  The TrainEngine (flat buffers, fused Adam/EMA, CUDA graph) on that branch is
the 'mechanics' row of test_gpu_parity_bench_path.py, which builds it with `build` and `synthetic_batch`."""
import pytest
import torch

from checks import rel

pytestmark = pytest.mark.gpu
DEV = 'cuda'


@pytest.fixture(scope='module')
def env():
    from oracle import pidm_oracle as O
    from physicsinformeddiffusionmodels_b200 import ops
    yield dict(O=O, ops=ops)
    ops.set_precision('bf16')


def build(O, dim, seed):
    from physicsinformeddiffusionmodels_b200.denoising_utils import DenoisingDiffusion
    from physicsinformeddiffusionmodels_b200.residuals_mechanics_K import ResidualsMechanics
    from physicsinformeddiffusionmodels_b200.unet_model import Unet3D
    cfg = O.unet_config(dim=dim, channels=10, out_dim=3, sigmoid_last_channel=True)
    sd = O.make_test_state_dict(cfg, seed)
    model = Unet3D(dim=dim, channels=10, out_dim=3, sigmoid_last_channel=True).to(DEV)
    model.load_state_dict(sd)
    diff = DenoisingDiffusion(100, DEV)
    res = ResidualsMechanics(model=model, pixels_per_dim=64, pixels_at_boundary=True, no_BC_folder='', device=DEV)
    return cfg, sd, model, diff, res


def synthetic_batch(B, seed):
    g = torch.Generator().manual_seed(seed)
    cond = torch.rand(B, 3, 65, 65, generator=g)
    cond[:, 0] = (0.3 + 0.4 * torch.rand(B, generator=g))[:, None, None]          # volume-fraction plane (constant)
    x0 = torch.cat((0.2 * torch.randn(B, 2, 65, 65, generator=g), torch.rand(B, 1, 65, 65, generator=g)), dim=1)
    bcs = torch.zeros(B, 4, 65, 65)
    bcs[:, 0, :, 0] = 1.; bcs[:, 1, :, 0] = 1.                                    # clamped left edge
    bcs[:, 3, 32, 64] = -1.                                                       # point load
    t = torch.randint(0, 100, (B,), generator=g)
    noise = torch.randn(B, 3, 65, 65, generator=g)
    return torch.cat((cond, x0, bcs), dim=1), t, noise


@pytest.mark.parametrize('mode,tol_loss,tol_grad', [('fp32', 1e-4, 3e-3), ('bf16', 3e-2, 1e-1)])
def test_mechanics_loss_matches_reference_golden(env, golden, monkeypatch, mode, tol_loss, tol_grad):
    """All four terms of the reference loss (data, residual NLL, inequality with its [B,1] x [B] broadcast, compliance)
    and three weight gradients vs the unmodified reference, B = 2, Unet3D(dim=32)."""
    O, ops = env['O'], env['ops']
    ops.set_precision(mode)
    gd = golden('mechanics_loss.pt')
    _, _, model, diff, res = build(O, 32, 3)
    c_data, c_res, c_ineq, lam = gd['coefs'].tolist()
    monkeypatch.setattr(torch, 'randint', lambda *a, **k: gd['t'].to(DEV))
    monkeypatch.setattr(torch, 'randn_like', lambda *a, **k: gd['noise'].to(DEV))
    loss, data_l, rabs, ineq, opt = diff.model_estimation_loss(gd['input'].to(DEV), residual_func=res, c_data=c_data,
                                                               c_residual=c_res, c_ineq=c_ineq, lambda_opt=lam)
    monkeypatch.undo()
    assert abs(loss.item() / gd['loss'].item() - 1) < tol_loss, (loss.item(), gd['loss'].item())
    assert abs(data_l / gd['data_loss'].item() - 1) < tol_loss
    assert abs(rabs / gd['residual_abs'].item() - 1) < tol_loss
    assert abs(ineq - gd['inequality'].item()) < (1e-5 if mode == 'fp32' else 2e-3)
    assert abs(opt / gd['compliance'].item() - 1) < tol_loss
    loss.backward()
    named = dict(model.named_parameters())
    for k, g in (('final_conv.1.weight', 'grad_final_w'), ('init_conv.weight', 'grad_init_w'),
                 ('downs.1.0.block1.proj.weight', 'grad_mid_w')):
        assert rel(named[k].grad, gd[g]) < tol_grad, (k, rel(named[k].grad, gd[g]))


def test_mechanics_reference_model_size_matches_oracle(env, monkeypatch):
    """The model the reference trains for this study: Unet3D(dim=128, channels=10, out_dim=3, sigmoid_last_channel)
    (136 M parameters; channel widths 128..1024 exercise other tile plans than the Darcy model).  bf16 production
    path vs the CPU oracle, B = 2."""
    O, ops = env['O'], env['ops']
    ops.set_precision('bf16')
    cfg, sd, model, diff, res = build(O, 128, 5)
    inp, t, noise = synthetic_batch(2, 11)
    sdr = {k: v.clone().requires_grad_(v.is_floating_point() and 'freqs' not in k) for k, v in sd.items()}
    loss_o, aux = O.mechanics_training_loss(sdr, cfg, inp, t, noise, O.diffusion_tables(100), 1.0, 1e-2, 0.0, 1e-3)
    loss_o.backward()
    monkeypatch.setattr(torch, 'randint', lambda *a, **k: t.to(DEV))
    monkeypatch.setattr(torch, 'randn_like', lambda *a, **k: noise.to(DEV))
    loss, data_l, rabs, _, opt = diff.model_estimation_loss(inp.to(DEV), residual_func=res, c_data=1.0, c_residual=1e-2,
                                                            c_ineq=0., lambda_opt=1e-3)
    monkeypatch.undo()
    assert abs(loss.item() / loss_o.item() - 1) < 3e-2, (loss.item(), loss_o.item())
    assert abs(data_l / aux['data'].item() - 1) < 3e-2
    loss.backward()
    named = dict(model.named_parameters())
    for k in ('final_conv.1.weight', 'init_conv.weight', 'downs.3.0.block1.proj.weight', 'ups.0.2.fn.fn.to_qkv.weight'):
        assert rel(named[k].grad, sdr[k].grad) < 1e-1, (k, rel(named[k].grad, sdr[k].grad))


def test_topopt_evaluation_metrics_match_reference(env, golden):
    """SURVEY 8f.4 (residuals_mechanics_K.py:276-354): compliance error of the binarised design (matrix-free PCG solve
    here, dense 8450 x 8450 LU in the reference), volume-fraction error and the floating-material flag, vs the unmodified
    reference (tests/golden/mechanics_eval.pt).  The design has 1e-3-stiffness voids: the system is ill-conditioned and
    both solvers work in fp32, hence 5e-2 on the compliance ratio."""
    from physicsinformeddiffusionmodels_b200.residuals_mechanics_K import ResidualsMechanics
    gd = golden('mechanics_eval.pt')
    res = ResidualsMechanics(model=None, pixels_per_dim=64, pixels_at_boundary=True, no_BC_folder='', device=DEV,
                             topopt_eval=True)
    out = res.compute_residual((gd['x0_pred'].to(DEV), gd['bcs'].to(DEV), gd['vf'].to(DEV), gd['solution'].to(DEV)),
                               reduce='per-batch', return_optimizer=True, return_inequality=True, sample=True,
                               pass_through=True)
    ce, ce_ref = out['rel_CE_error_full_batch'].cpu(), gd['rel_CE_error']
    assert torch.allclose(ce, ce_ref, rtol=5e-2), (ce, ce_ref)
    assert torch.allclose(out['vf_error_full_batch'].cpu(), gd['vf_error'], atol=1e-6)
    assert torch.equal(out['fm_error_full_batch'].cpu().long(), gd['fm_error'].long())
    # the solver itself: K(rho) u = f to 1e-5 relative residual on a well-conditioned design
    rho = gd['solution'][:, 2, :-1, :-1].contiguous().to(DEV)
    u = res.fem_solve(rho, gd['bcs'].to(DEV))
    assert rel(u, gd['solution'][:, :2]) < 2e-3, rel(u, gd['solution'][:, :2])
