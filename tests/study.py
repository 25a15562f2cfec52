"""The Darcy study options as test data: their constructor options, the seeded weights of the dim-32 Darcy U-Net, one
builder of (model, diffusion, residuals) on the GPU, and fixed draws for the training step.  The product package is
imported inside the functions, so importing this module builds nothing."""
import contextlib
import functools

import torch

from oracle import pidm_oracle as O

DEV = 'cuda'

STUDIES = {
    'none': {},
    'periodic': dict(bcs='periodic'),
    'circular': dict(bcs='periodic', padding_mode='circular'),
    'guidance': dict(residual_grad_guidance=True),
}


def config(padding_mode='zeros'):
    return O.unet_config(dim=32, channels=2, padding_mode=padding_mode)


@functools.cache
def state_dict(padding_mode='zeros'):
    return O.make_test_state_dict(config(padding_mode), 0)


def build_darcy(study='none', n_steps=100, use_ddim_x0=False, **options):
    """(model, diffusion, residuals) on the GPU with the seeded weights, for a study of STUDIES; `options` (bcs,
    padding_mode, residual_grad_guidance) are added to the study's own"""
    from physicsinformeddiffusionmodels_b200.denoising_utils import DenoisingDiffusion
    from physicsinformeddiffusionmodels_b200.residuals_darcy import ResidualsDarcy
    from physicsinformeddiffusionmodels_b200.unet_model import Unet3D
    opts = {**STUDIES[study], **options}
    padding_mode = opts.get('padding_mode', 'zeros')
    guidance = opts.get('residual_grad_guidance', False)
    model = Unet3D(dim=32, channels=2, padding_mode=padding_mode).to(DEV)
    model.load_state_dict(state_dict(padding_mode))
    diff = DenoisingDiffusion(n_steps, DEV, residual_grad_guidance=guidance)
    res = ResidualsDarcy(model=model, fd_acc=2, pixels_per_dim=64, pixels_at_boundary=True, reverse_d1=True, device=DEV,
                         bcs=opts.get('bcs', 'none'), domain_length=1., residual_grad_guidance=guidance,
                         use_ddim_x0=use_ddim_x0, ddim_steps=0)
    return model, diff, res


@contextlib.contextmanager
def fixed_draws(t, e):
    """torch.randint / torch.randn_like return t / e (also under graph capture, where they become static inputs of the
    captured step)"""
    o1, o2 = torch.randint, torch.randn_like
    torch.randint, torch.randn_like = (lambda *a, **k: t), (lambda *a, **k: e)
    try:
        yield
    finally:
        torch.randint, torch.randn_like = o1, o2
