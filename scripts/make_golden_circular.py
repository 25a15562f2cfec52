"""Golden vectors for Unet3D(padding_mode='circular').  TEST INFRASTRUCTURE ONLY; runs on CPU, not on the GPU box.

Runs the UNMODIFIED reference modules (checkout in PIDM_REFERENCE, imported through oracle/ref_shims/ exactly as
oracle/make_golden.py does) with a circular U-Net and writes NEW fixtures to tests/golden/.  Every existing fixture is
left as it is; the recipes mirror the zero-padded fixtures of oracle/make_golden.py and scripts/make_golden_periodic.py.
The circular model loads the state_dict of oracle.make_test_state_dict(seed=0) with the six up-sampling keys renamed
(`ups.{i}.3.*` -> `ups.{i}.3.conv_transpose.*`).

    unet_circular_fwd.pt         forward output + taps on the unet_darcy_fwd.pt inputs
    darcy_loss_circular.pt       mean-mode loss, loss terms, grad-norm and gradients with ResidualsDarcy(bcs='periodic')
    sample_loop_circular.pt      the sample_loop_6 recipe with bcs='periodic'
    darcy_guidance_circular.pt   residual-gradient guidance loss + gradients (emb_conv[2] stays zero-padded)
    unet_circular_keys.pt        the circular state_dict key list, in order

    PIDM_REFERENCE=<checkout of the original project> python scripts/make_golden_circular.py
"""
import importlib.util
import os

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
_spec = importlib.util.spec_from_file_location('make_golden', os.path.join(ROOT, 'oracle', 'make_golden.py'))
MG = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(MG)
O = MG.O


def circular_state_dict(sd):
    """zeros-mode state_dict -> the circular model's keys (the up-sampling layers move under `conv_transpose`)"""
    out = {}
    for k, v in sd.items():
        parts = k.split('.')
        if parts[0] == 'ups' and parts[2] == '3':
            k = '.'.join(parts[:3] + ['conv_transpose'] + parts[3:])
        out[k] = v
    return out


def main():
    torch.set_num_threads(8)
    import src.unet_model as _um
    assert os.path.abspath(_um.__file__).startswith(os.path.abspath(MG.REF)), _um.__file__
    from src.denoising_utils import DenoisingDiffusion
    from src.residuals_darcy import ResidualsDarcy
    from src.unet_model import Unet3D

    cfg = O.unet_config(dim=32, channels=2)
    model = Unet3D(dim=32, channels=2, padding_mode='circular')
    model.load_state_dict(circular_state_dict(O.make_test_state_dict(cfg, seed=0)), strict=True)
    MG.save('unet_circular_keys.pt', dict(keys=list(model.state_dict().keys())))

    # ---- forward + taps on the inputs of unet_darcy_fwd.pt ---------------------------------------------------------
    fw = torch.load(os.path.join(MG.OUT, 'unet_darcy_fwd.pt'), weights_only=True)
    x, t = fw['x'], fw['t']
    taps = {}

    def hook(name):
        def f(mod, inp, out):
            taps[name] = out.detach().squeeze(2).clone()
        return f
    hs = [model.init_conv.register_forward_hook(hook('init_conv')),
          model.downs[0][0].register_forward_hook(hook('downs.0.0')),
          model.downs[0][2].register_forward_hook(hook('downs.0.2')),
          model.mid_spatial_attn.register_forward_hook(hook('mid_attn')),
          model.ups[0][3].register_forward_hook(hook('ups.0'))]
    model.eval()
    with torch.no_grad():
        y = model(x, t)
    for h in hs:
        h.remove()
    MG.save('unet_circular_fwd.pt', dict(x=x, t=t, y=y, **{'tap_' + k: O.golden_sample(v) for k, v in taps.items()}))

    def darcy(**kw):
        return ResidualsDarcy(model=model, fd_acc=2, pixels_per_dim=64, pixels_at_boundary=True, reverse_d1=True,
                              device='cpu', bcs='periodic', domain_length=1., **kw)

    # ---- training loss + gradients, mean mode (the darcy_loss_periodic.pt recipe) ------------------------------------
    res = darcy()
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
    keys = ['init_conv.weight', 'downs.0.0.block1.proj.weight', 'downs.1.3.weight', 'ups.0.3.conv_transpose.weight',
            'ups.2.3.conv_transpose.bias', 'ups.3.1.block2.proj.weight', 'final_conv.1.weight']
    named = dict(model.named_parameters())
    grads = {'grad_' + k: O.golden_sample(named[k].grad) for k in keys}
    gn = torch.sqrt(sum((p.grad.double() ** 2).sum() for p in model.parameters() if p.grad is not None)).float()
    MG.save('darcy_loss_circular.pt', dict(x0=x0, t=t_l, noise=e_l, loss=loss.detach(), data_loss=torch.tensor(data_l),
                                           residual_abs=torch.tensor(res_l), grad_norm=gn, **grads))

    # ---- residual-gradient guidance (the darcy_guidance.pt recipe, reference mask draw) ------------------------------
    res_g = darcy(residual_grad_guidance=True)
    x0g = MG.smooth_fields(4, seed=19)
    torch.manual_seed(55)
    loss_g, _, _, _, _ = diff.model_estimation_loss(x0g, residual_func=res_g, c_data=1., c_residual=1e-3, c_ineq=0.,
                                                    lambda_opt=0.)
    model.zero_grad()
    loss_g.backward()
    torch.manual_seed(55)
    t_g = torch.randint(0, 100, size=(4,))
    e_g = torch.randn_like(x0g)
    mask_g = torch.zeros((4,)).float().uniform_(0, 1) < 0.1
    MG.save('darcy_guidance_circular.pt', dict(x0=x0g, t=t_g, noise=e_g, null_mask=mask_g, loss=loss_g.detach(),
                                               grad_emb2=named['emb_conv.2.weight'].grad.clone(),
                                               grad_emb0=named['emb_conv.0.weight'].grad.clone(),
                                               grad_final_w=named['final_conv.1.weight'].grad.clone()))

    # ---- ancestral sampling loop, 6 diffusion steps, B=1 (the sample_loop_6.pt recipe) --------------------------------
    model.eval()
    d6 = DenoisingDiffusion(6, 'cpu')
    torch.manual_seed(77)
    (x_seq, interm), aux = d6.p_sample_loop(None, (1, 2, 64, 64), save_output=True, surpress_noise=True,
                                            residual_func=res, eval_residuals=True)
    torch.manual_seed(77)
    x_T = torch.randn(1, 2, 64, 64)
    zs = [torch.randn(1, 2, 64, 64) for _ in range(6)]
    MG.save('sample_loop_circular.pt', dict(x_T=x_T, noises=torch.stack(zs), x_final=x_seq[-1], x_after_first=x_seq[1],
                                            x0_pred_last=interm[-1], residual=aux['residual'].detach()))


if __name__ == '__main__':
    main()
