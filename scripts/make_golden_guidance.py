"""Golden vectors for one residual-gradient guidance training iteration.  TEST INFRASTRUCTURE ONLY; runs on CPU.

Runs the UNMODIFIED reference modules (checkout in PIDM_REFERENCE, imported through oracle/ref_shims/ exactly as
oracle/make_golden.py does) for one iteration of the training loop (reference main.py:158-179) with
residual_grad_guidance=True at B = 8, and writes NEW fixtures to tests/golden/ (every existing fixture is left as it is):

    darcy_guidance_step.pt             x0, t, eps, the classifier-free mask (both values occur), loss, data loss,
                                       mean|r|, a golden_sample(., 256) of the gradient of every parameter that receives
                                       one, and the global gradient norm that drives clipping
    params_without_grad_guidance.txt   the parameters whose .grad stays None under guidance

    PIDM_REFERENCE=<checkout of the original project> python scripts/make_golden_guidance.py
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

B = 8
GRAD_SAMPLE = 256


def draws(seed, x0):
    """the loop's three draws in order: t, eps (denoising_utils.py:625,636), the mask (unet_model.py:63-69)"""
    torch.manual_seed(seed)
    t = torch.randint(0, 100, size=(B,))
    e = torch.randn_like(x0)
    mask = torch.zeros((B,)).float().uniform_(0, 1) < 0.1
    return t, e, mask


def main():
    torch.set_num_threads(8)
    import src.unet_model as _um
    assert os.path.abspath(_um.__file__).startswith(os.path.abspath(MG.REF)), _um.__file__
    from src.denoising_utils import DenoisingDiffusion
    from src.residuals_darcy import ResidualsDarcy
    from src.unet_model import Unet3D

    cfg = O.unet_config(dim=32, channels=2)
    model = Unet3D(dim=32, channels=2)
    model.load_state_dict(O.make_test_state_dict(cfg, seed=0), strict=True)
    res = ResidualsDarcy(model=model, fd_acc=2, pixels_per_dim=64, pixels_at_boundary=True, reverse_d1=True,
                         device='cpu', bcs='none', domain_length=1., residual_grad_guidance=True)
    diff = DenoisingDiffusion(100, 'cpu', residual_grad_guidance=True)
    x0 = MG.smooth_fields(B, seed=29)
    seed = next(s for s in range(1000, 2000) if 0 < int(draws(s, x0)[2].sum()) < B)     # a mask with both values
    t, e, mask = draws(seed, x0)
    model.train()
    torch.manual_seed(seed)
    loss, data_l, rabs, _, _ = diff.model_estimation_loss(x0, residual_func=res, c_data=1., c_residual=1e-3, c_ineq=0.,
                                                          lambda_opt=0.)
    model.zero_grad()
    loss.backward()
    named = dict(model.named_parameters())
    grads = {'grad_' + k: O.golden_sample(p.grad, GRAD_SAMPLE) for k, p in named.items() if p.grad is not None}
    gn = torch.sqrt(sum((p.grad.double() ** 2).sum() for p in model.parameters() if p.grad is not None)).float()
    nograd = sorted(k for k, p in named.items() if p.grad is None)
    MG.save('darcy_guidance_step.pt', dict(x0=x0, t=t, noise=e, null_mask=mask, loss=loss.detach(),
                                           data_loss=torch.tensor(data_l), residual_abs=torch.tensor(rabs), grad_norm=gn,
                                           grad_sample=torch.tensor(GRAD_SAMPLE), **grads))
    with open(os.path.join(MG.OUT, 'params_without_grad_guidance.txt'), 'w') as f:
        f.write('\n'.join(nograd) + '\n')


if __name__ == '__main__':
    main()
