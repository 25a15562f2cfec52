"""The call sequence of the reference drivers (main.py:116-316, sample.py:112-150), written against the drop-in `src.*`
module names with the reference's own glue (torch DataLoader, optim.Adam, clip_grad_norm_, EMA register/update/ema/
restore, save_model/load_model, p_sample_loop), with bcs = 'none' and with bcs = 'periodic' and CoCoGen corrections in
the sampler.  Sizes are reduced (4 diffusion steps, 3 iterations)."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('bcs,M,N', [('none', 0, 0), ('periodic', 1, 1)])
def test_reference_driver_sequence_runs_on_the_drop_in_modules(tmp_path, bcs, M, N):
    import torch.optim as optim
    from torch.utils.data import DataLoader
    from src.data_utils import Dataset, cycle  # noqa: F401
    from src.denoising_utils import DenoisingDiffusion, EMA, device, exists, load_model, save_model  # noqa: F401
    from src.residuals_darcy import ResidualsDarcy
    from src.unet_model import Unet3D
    from physicsinformeddiffusionmodels_b200 import ops
    ops.set_precision('bf16')
    assert device.type == 'cuda'
    rng = np.random.default_rng(0)
    paths = []
    for name in ('p_data.csv', 'K_data.csv'):
        p = tmp_path / name
        np.savetxt(p, rng.standard_normal((6, 64 * 64)).astype(np.float32), delimiter=',')
        paths.append(str(p))
    ds = Dataset(tuple(paths), use_double=False)
    assert ds[0].shape == (2, 64, 64)
    dl = cycle(DataLoader(ds, batch_size=3, shuffle=False))
    diffusion_utils = DenoisingDiffusion(4, device, False)
    model = Unet3D(dim=32, channels=2, sigmoid_last_channel=False).to(device)
    ema = EMA(0.99)
    ema.register(model)
    assert sum(p.numel() for p in model.parameters() if p.requires_grad) == 10386482
    residuals = ResidualsDarcy(model=model, fd_acc=2, pixels_per_dim=64, pixels_at_boundary=True, reverse_d1=True,
                               device=device, bcs=bcs, domain_length=1., residual_grad_guidance=False,
                               use_ddim_x0=False, ddim_steps=0)
    optimizer = optim.Adam(model.parameters(), lr=1.e-4)
    w_before = model.final_conv[1].weight.detach().clone()
    losses = []
    for iteration in range(3):
        model.train()
        cur_batch = next(dl).to(device)
        loss, data_loss, residual_loss, ineq_loss, opt_loss = diffusion_utils.model_estimation_loss(
            cur_batch, residual_func=residuals, c_data=1, c_residual=0.001, c_ineq=0, lambda_opt=0)
        optimizer.zero_grad()
        loss.backward()
        torch.nn.utils.clip_grad_norm_(model.parameters(), 1.)
        optimizer.step()
        losses.append(loss.item())
        assert isinstance(data_loss, float) and isinstance(residual_loss, float)
        if iteration > 0:
            ema.update(model)
        model.eval()
        ema.ema(residuals.model)
        if iteration == 2:
            save_model({'gov_eqs': 'darcy', 'diff_steps': 4}, model, iteration, str(tmp_path / 'run'))
        ema.restore(residuals.model)
    assert all(np.isfinite(losses)) and not torch.equal(model.final_conv[1].weight.detach(), w_before)
    # sampling exactly as main.py:220-225 / sample.py:145-150
    output = diffusion_utils.p_sample_loop(None, (2, 2, 64, 64), save_output=True, surpress_noise=True,
                                           use_dynamic_threshold=False, residual_func=residuals, eval_residuals=True,
                                           return_optimizer=False, return_inequality=False, M_correction=M,
                                           N_correction=N, correction_mode='xt')
    seqs, aux = output
    assert torch.isfinite(aux['residual']).all()
    residual = aux['residual'].abs().mean(dim=tuple(range(1, aux['residual'].ndim)))
    assert residual.shape == (2,) and torch.isfinite(residual).all()
    seq = torch.stack(seqs[0], dim=0)
    assert seq.shape == (5 + M, 2, 2, 64, 64) and not seq.is_cuda and np.isfinite(seq[-1].numpy()).all()
    # checkpoint round trip in the reference's format
    ck = tmp_path / 'run' / 'model' / 'checkpoint_2.pt'
    assert ck.exists() and (tmp_path / 'run' / 'model' / 'model.yaml').exists()
    model2 = Unet3D(dim=32, channels=2).to(device)
    load_model(ck, model2)
    sd1, sd2 = torch.load(ck, map_location='cpu')['model'], model2.state_dict()
    assert len(sd1) == 317 and all(torch.equal(sd1[k], sd2[k].cpu()) for k in sd1)
