"""Golden vectors for bcs='periodic'.  TEST INFRASTRUCTURE ONLY; runs on CPU, not on the GPU box.

Runs the UNMODIFIED reference modules (checkout in PIDM_REFERENCE, imported through oracle/ref_shims/ exactly as
oracle/make_golden.py does) with ResidualsDarcy(bcs='periodic') and writes four NEW fixtures to tests/golden/.  Every
existing fixture is left as it is; the recipes mirror the 'none' fixtures of oracle/make_golden.py:

    darcy_residual_periodic.pt   residual, VJP and the five stencil_gradients modes on the fields of darcy_residual.pt
    cocogen_periodic.pt          residual_correction (vmap(jacfwd) Jacobian) on two of those fields
    darcy_loss_periodic.pt       mean-mode model_estimation_loss, loss terms and the gradients of darcy_loss_mean.pt
    sample_loop_periodic.pt      the sample_loop_6 recipe

    PIDM_REFERENCE=<checkout of the original project> python scripts/make_golden_periodic.py
"""
import importlib.util
import os

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
# make_golden sets up the import path (reference first, shims, repository root removed) and provides the helpers
_spec = importlib.util.spec_from_file_location('make_golden', os.path.join(ROOT, 'oracle', 'make_golden.py'))
MG = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(MG)
O = MG.O


def main():
    torch.set_num_threads(8)
    import src.unet_model as _ref_mod
    assert os.path.abspath(_ref_mod.__file__).startswith(os.path.abspath(MG.REF)), _ref_mod.__file__
    from src.denoising_utils import DenoisingDiffusion
    from src.residuals_darcy import ResidualsDarcy
    from src.unet_model import Unet3D

    cfg = O.unet_config(dim=32, channels=2)
    model = Unet3D(dim=32, channels=2)
    model.load_state_dict(O.make_test_state_dict(cfg, seed=0), strict=True)

    def darcy(**kw):
        return ResidualsDarcy(model=model, fd_acc=2, pixels_per_dim=64, pixels_at_boundary=True, reverse_d1=True,
                              device='cpu', bcs='periodic', domain_length=1., **kw)

    res = darcy()
    assert res.periodic

    # ---- residual, VJP and the stencil modes on the smooth + rough fields of darcy_residual.pt --------------------
    x0p = torch.load(os.path.join(MG.OUT, 'darcy_residual.pt'), weights_only=True)['x0_pred']
    g = torch.Generator().manual_seed(31)
    r = res.compute_residual(x0p, pass_through=True)['residual']
    xg = x0p.clone().requires_grad_(True)
    rg = res.compute_residual(xg, pass_through=True)['residual']
    wgt = torch.randn(rg.shape, generator=g)
    (rg * wgt).sum().backward()
    modes = ('d_d0', 'd_d1', 'd_d00', 'd_d11', 'd_d01')
    with torch.no_grad():
        sg = {'stencil_' + m: res.grads.stencil_gradients(x0p[:, 0].clone(), mode=m).clone() for m in modes}
    MG.save('darcy_residual_periodic.pt', dict(x0_pred=x0p, residual=r.detach(), cotangent=wgt,
                                               grad_x0_pred=xg.grad.clone(), **sg))

    # ---- CoCoGen correction through the reference's vmap(jacfwd) Jacobian ---------------------------------------------
    xc = x0p[:2].clone()
    xin = xc.permute(0, 2, 3, 1).reshape(2, 4096, 2).clone()
    x_corr, r_corr = res.residual_correction(xin)
    MG.save('cocogen_periodic.pt', dict(x0_pred=xc,
                                        corrected=x_corr.reshape(2, 64, 64, 2).permute(0, 3, 1, 2).contiguous().clone(),
                                        residual_corrected=r_corr.detach().clone()))

    # ---- training loss + gradients, mean mode (the darcy_loss_mean.pt recipe) -----------------------------------------
    diff = DenoisingDiffusion(100, 'cpu')
    model.train()
    x0 = MG.smooth_fields(2, seed=9)
    torch.manual_seed(123)
    loss, data_l, res_l, _, _ = diff.model_estimation_loss(x0, residual_func=res, c_data=1., c_residual=1e-3,
                                                           c_ineq=0., lambda_opt=0.)
    model.zero_grad()
    loss.backward()
    torch.manual_seed(123)
    t_l = torch.randint(0, 100, size=(2,))
    e_l = torch.randn_like(x0)
    keys = ['init_conv.weight', 'time_mlp.1.weight', 'downs.0.0.block1.proj.weight', 'downs.0.0.mlp.1.weight',
            'downs.0.2.fn.fn.to_qkv.weight', 'downs.1.3.weight', 'mid_spatial_attn.fn.fn.fn.to_qkv.weight',
            'ups.0.3.weight', 'ups.3.2.fn.norm.gamma', 'final_conv.1.weight', 'final_conv.1.bias',
            'downs.3.1.block2.norm.weight', 'ups.1.0.res_conv.weight']
    named = dict(model.named_parameters())
    grads = {'grad_' + k: O.golden_sample(named[k].grad) for k in keys}
    gn = torch.sqrt(sum((p.grad.double() ** 2).sum() for p in model.parameters() if p.grad is not None)).float()
    MG.save('darcy_loss_periodic.pt', dict(x0=x0, t=t_l, noise=e_l, loss=loss.detach(), data_loss=torch.tensor(data_l),
                                           residual_abs=torch.tensor(res_l), grad_norm=gn, **grads))

    # ---- ancestral sampling loop, 6 diffusion steps, B=1 (the sample_loop_6.pt recipe) --------------------------------
    model.eval()
    d6 = DenoisingDiffusion(6, 'cpu')
    torch.manual_seed(77)
    (x_seq, interm), aux = d6.p_sample_loop(None, (1, 2, 64, 64), save_output=True, surpress_noise=True,
                                            residual_func=res, eval_residuals=True)
    torch.manual_seed(77)
    x_T = torch.randn(1, 2, 64, 64)
    zs = [torch.randn(1, 2, 64, 64) for _ in range(6)]
    MG.save('sample_loop_periodic.pt', dict(x_T=x_T, noises=torch.stack(zs), x_final=x_seq[-1], x_after_first=x_seq[1],
                                            x0_pred_last=interm[-1], residual=aux['residual'].detach()))


if __name__ == '__main__':
    main()
