"""End-to-end parity of the engine (U-Net, loss, gradients, sampler, training step) against the golden
fixtures produced by the UNMODIFIED reference (tests/golden, oracle/make_golden.py) and against the CPU oracle.  The
training loss and the sampling engine are checked for each study option (tests/study.py) that has a fixture.

Two precision modes: 'fp32' activations (exact mode: only summation order differs from the reference -> tight
tolerances) and 'bf16' (production mode: bf16 GEMM operands / activations, fp32 accumulate and statistics)."""
import os

import pytest
import torch

from checks import rel
from oracle import pidm_oracle as O
from study import build_darcy, config, fixed_draws, state_dict

pytestmark = pytest.mark.gpu
DEV = 'cuda'


@pytest.fixture(scope='module')
def ops():
    from physicsinformeddiffusionmodels_b200 import ops
    yield ops
    ops.set_precision('bf16')


# fp32 mode: 1e-4 (accumulation order over K up to 4608 and ~60 layers); bf16 mode: 3e-2 (2^-9 per rounding)
@pytest.mark.parametrize('mode,tol', [('fp32', 1e-4), ('bf16', 3e-2)])
def test_unet_forward_matches_reference(ops, golden, mode, tol):
    ops.set_precision(mode)
    gd = golden('unet_darcy_fwd.pt')
    model, _, _ = build_darcy()
    with torch.no_grad():
        y = model(gd['x'].to(DEV), gd['t'].to(DEV))
        y2 = model(gd['x'].permute(0, 2, 3, 1).reshape(2, 4096, 2).to(DEV), gd['t'].to(DEV))
    assert y.shape == (2, 2, 64, 64) and y.dtype == torch.float32
    # [B,P*P,C] and [B,C,P,P] inputs are the same tensor.  Two runs differ only by the order of fp32 atomics
    # (GroupNorm / linear-attention partial sums, ~1e-7); in bf16 mode that noise flips 1-ulp roundings of the
    # activations which then propagate through ~60 layers (measured 6e-3), so run-to-run is held to `tol` as well.
    assert rel(y, y2) < tol, rel(y, y2)
    assert rel(y, gd['y']) < tol, rel(y, gd['y'])


def test_unet_forward_tcgen05_vs_cuda_core_path(ops, golden):
    """Same bf16 operands through the tensor-core (wgmma) kernels and through the CUDA-core implicit GEMM: both round the same
    activations to bf16, so they agree to accumulation order + 1-ulp bf16 flips that propagate through ~60 layers (2e-2)."""
    ops.set_precision('bf16')
    gd = golden('unet_darcy_fwd.pt')
    model, _, _ = build_darcy()
    with torch.no_grad():
        ops.set_tensor_core_conv(True)
        y_tc = model(gd['x'].to(DEV), gd['t'].to(DEV))
        ops.set_tensor_core_conv(False)
        y_cc = model(gd['x'].to(DEV), gd['t'].to(DEV))
        ops.set_tensor_core_conv(True)
    assert rel(y_tc, y_cc) < 2e-2, rel(y_tc, y_cc)


# golden: (study, dead-parameter list or None, {mode: (loss, gradient, grad-norm tolerance)}).  A fixture with
# 'null_mask' is a guidance step with that classifier-free mask; one with 'grad_sample' stores its gradients sampled
# with that n.
ZEROS_TOL = {'fp32': (5e-5, 1e-3, 1e-3), 'bf16': (3e-2, 8e-2, 8e-2)}
LOSS_ROWS = {
    'darcy_loss_mean': ('none', 'params_without_grad.txt', ZEROS_TOL),
    'darcy_loss_periodic': ('periodic', None, ZEROS_TOL),
    'darcy_loss_circular': ('circular', None, ZEROS_TOL),
    'darcy_guidance_step': ('guidance', 'params_without_grad_guidance.txt',
                            {'fp32': (5e-5, 2e-3, 1e-3), 'bf16': (3e-2, 1e-1, 8e-2)}),
}


@pytest.mark.parametrize('name,mode', [(n, m) for n in LOSS_ROWS for m in ('fp32', 'bf16')])
def test_training_loss_and_gradients_match_reference(ops, golden, name, mode):
    study, dead_list, tols = LOSS_ROWS[name]
    tol_loss, tol_grad, tol_norm = tols[mode]
    ops.set_precision(mode)
    gd = golden(name + '.pt')
    model, diff, res = build_darcy(study)
    model._null_mask_override = gd['null_mask'].to(DEV) if 'null_mask' in gd else None
    loss, data_l, rabs, _, _ = diff.darcy_loss_from_draws(gd['x0'].to(DEV), gd['t'].to(DEV), gd['noise'].to(DEV), res,
                                                          1.0, 1e-3)
    model._null_mask_override = None
    assert abs(loss.item() / gd['loss'].item() - 1) < tol_loss, (loss.item(), gd['loss'].item())
    assert abs(float(data_l) / gd['data_loss'].item() - 1) < tol_loss
    assert abs(float(rabs) / gd['residual_abs'].item() - 1) < tol_loss
    loss.backward()
    named = dict(model.named_parameters())
    n = {'n': int(gd['grad_sample'])} if 'grad_sample' in gd else {}
    worst = {k: rel(O.golden_sample(named[k[5:]].grad, **n), v) for k, v in gd.items()
             if k.startswith('grad_') and k not in ('grad_norm', 'grad_sample')}
    assert max(worst.values()) < tol_grad, sorted(worst.items(), key=lambda kv: -kv[1])[:5]
    gn = torch.sqrt(sum((p.grad.double() ** 2).sum() for p in model.parameters() if p.grad is not None)).item()
    assert abs(gn / gd['grad_norm'].item() - 1) < tol_norm
    if dead_list is not None:
        with open(os.path.join(os.path.dirname(__file__), 'golden', dead_list)) as f:
            ref_dead = sorted(k for k in f.read().split() if not k.endswith('rotary_emb.freqs'))
        dead = sorted(k for k, p in named.items() if p.requires_grad and p.grad is None)
        assert dead == ref_dead


def test_sample_mode_loss_matches_reference(ops, golden):
    ops.set_precision('fp32')
    gd = golden('darcy_loss_sample.pt')
    model, diff, res = build_darcy(use_ddim_x0=True)
    loss, _, _, _, _ = diff.darcy_loss_from_draws(gd['x0'].to(DEV), gd['t'].to(DEV), gd['noise'].to(DEV), res, 1.0, 1e-3)
    assert abs(loss.item() / gd['loss'].item() - 1) < 1e-4
    loss.backward()
    assert rel(model.final_conv[1].weight.grad, gd['grad_final_w']) < 2e-3
    assert rel(model.init_conv.weight.grad, gd['grad_init_w']) < 2e-3


def ddim_walk_case(golden):
    from oracle import make_golden
    gd = golden('darcy_loss_sample.pt')
    xt = make_golden.ddim_walk_input()
    assert torch.equal(xt.double().sum(), gd['walk_x_t_checksum'])
    return gd, xt.to(DEV), make_golden.DDIM_WALK


def check_ddim_walk(gd, sample, ddim_steps, cur_x, model_out):
    """the walk's result and first network output against the reference's, at the fp32 U-Net tolerance"""
    assert rel(O.golden_sample(model_out.cpu(), sample), gd[f'walk_model_out_{ddim_steps}']) < 1e-4
    assert rel(O.golden_sample(cur_x.cpu(), sample), gd[f'walk_cur_x_{ddim_steps}']) < 1e-4


@pytest.mark.parametrize('ddim_steps', [1, 3])
def test_ddim_walk_matches_reference(ops, golden, ddim_steps):
    """ddim_sample_x0 at ddim_steps > 0, per-sample t = 0, 2 (repeated grid points), 57 and n_steps - 1"""
    ops.set_precision('fp32')
    gd, xt, spec = ddim_walk_case(golden)
    model, diff, _ = build_darcy(n_steps=spec['n_steps'])
    model.eval()
    with torch.no_grad():
        cur_x, model_out = diff.ddim_sample_x0(xt, gd['walk_t'].to(DEV), model, xt.shape, ddim_steps, 0.)
    check_ddim_walk(gd, spec['sample'], ddim_steps, cur_x, model_out)


def test_sample_engine_ddim3_step_matches_reference(ops, golden):
    """one sample-mode SampleEngine step with ddim_steps = 3: its x0 estimate is the reference's walk, its residual is
    that of the walk's result and its posterior step takes the walk's first network output"""
    from physicsinformeddiffusionmodels_b200.engine import SampleEngine
    ops.set_precision('fp32')
    gd, xt, spec = ddim_walk_case(golden)
    model, diff, res = build_darcy(n_steps=spec['n_steps'], use_ddim_x0=True)
    res.ddim_steps = 3
    model.eval()
    walks = []
    walk = diff.ddim_sample_x0
    diff.ddim_sample_x0 = lambda *a, **k: walks.append(walk(*a, **k)) or walks[-1]
    se = SampleEngine(model, diff, res, batch=xt.shape[0], use_graph=False, external_noise=True)
    se.z.normal_()
    se.x.copy_(xt)
    t = gd['walk_t'].to(DEV)
    se.t.copy_(t)
    se._step_body()
    (cur_x, model_out), = walks
    check_ddim_walk(gd, spec['sample'], 3, cur_x, model_out)
    assert torch.equal(se.residual, ops.darcy_residual(cur_x, res.f_s_flat, *res.geometry))
    c1, c2, sig = se.c1[t].view(-1, 1, 1, 1), se.c2[t].view(-1, 1, 1, 1), se.sigma[t].view(-1, 1, 1, 1)
    assert torch.allclose(se.x, c1 * model_out + c2 * xt + sig * se.z[0], rtol=1e-5, atol=1e-5)
    assert torch.equal(se.t, t - 1)


def test_ddim_device_grid_is_the_reference_linspace():
    """the time grid ddim_sample_x0 builds on the device is int(np.linspace(0, t, s + 2)) for every t < 1000 and
    s <= 20: a stub network records the t of each call"""
    import numpy as np
    from physicsinformeddiffusionmodels_b200.denoising_utils import DenoisingDiffusion
    diff = DenoisingDiffusion(1000, DEV)
    t = torch.arange(1000, device=DEV)
    x = torch.zeros(1000, 2, 4, 4, device=DEV)
    for s in range(21):
        seen = []

        def stub(inp, tt, self_cond=None):
            seen.append(tt.cpu())
            return torch.zeros_like(inp)
        diff.ddim_sample_x0(x, t, stub, x.shape, s, 0.)
        got = torch.stack(seen).flip(0).T                              # [t, grid point], ascending
        want = torch.tensor([[int(v) for v in np.linspace(0, ti, s + 2, dtype=float)] for ti in range(1000)])
        assert torch.equal(got, want), (s, (got != want).nonzero()[:5].tolist())


def test_sampling_loop_matches_reference(ops, golden, monkeypatch):
    """p_sample_loop with the reference's own draws injected (x_T, then one z per step incl. t=0)."""
    ops.set_precision('fp32')
    gd = golden('sample_loop_6.pt')
    model, diff, res = build_darcy(n_steps=6)
    model.eval()
    draws = [gd['x_T']] + list(gd['noises'])
    it = iter(draws)
    monkeypatch.setattr(torch, 'randn', lambda *a, **k: next(it).to(DEV))
    monkeypatch.setattr(torch, 'randn_like', lambda *a, **k: next(it).to(DEV))
    (x_seq, interm), aux = diff.p_sample_loop(None, (1, 2, 64, 64), save_output=True, surpress_noise=True,
                                              residual_func=res, eval_residuals=True)
    monkeypatch.undo()
    assert len(x_seq) == 7 and len(interm) == 7 and not x_seq[-1].is_cuda
    assert rel(x_seq[1], gd['x_after_first']) < 1e-4
    assert rel(x_seq[-1], gd['x_final']) < 5e-4
    assert rel(aux['residual'], gd['residual']) < 5e-3      # residual amplifies x0 differences by 1/h^2


@pytest.mark.parametrize('name,study', [('sample_loop_6', 'none'), ('sample_loop_periodic', 'periodic'),
                                        ('sample_loop_circular', 'circular')])
def test_sample_engine_matches_reference_and_graph_replay(ops, golden, monkeypatch, name, study):
    """SampleEngine (device-side time index, one captured step replayed n_steps times) against the reference's
    trajectory with its own draws injected, and CUDA-graph replay against the eager loop on identical noise."""
    ops.set_precision('fp32')
    from physicsinformeddiffusionmodels_b200.engine import SampleEngine
    gd = golden(name + '.pt')
    model, diff, res = build_darcy(study, n_steps=6)
    model.eval()
    it = iter(list(gd['noises']))
    monkeypatch.setattr(torch, 'randn_like', lambda *a, **k: next(it).to(DEV))
    x, r, traj = SampleEngine(model, diff, res, batch=1, use_graph=False).sample(x_init=gd['x_T'].to(DEV), trajectory=True)
    monkeypatch.undo()
    assert traj.shape[0] == 7
    assert rel(traj[1], gd['x_after_first']) < 1e-4
    assert rel(x, gd['x_final']) < 5e-4
    assert rel(r, gd['residual']) < 5e-3
    zfix = gd['noises'][0].to(DEV)
    monkeypatch.setattr(torch, 'randn_like', lambda *a, **k: zfix)
    xe = SampleEngine(model, diff, res, batch=1, use_graph=False).sample(x_init=gd['x_T'].to(DEV))[0].clone()
    xg = SampleEngine(model, diff, res, batch=1, use_graph=True).sample(x_init=gd['x_T'].to(DEV))[0].clone()
    monkeypatch.undo()
    assert rel(xg, xe) < 1e-4, rel(xg, xe)


@pytest.mark.parametrize('mode,tol_loss,tol_grad', [('fp32', 5e-5, 2e-3), ('bf16', 3e-2, 1e-1)])
def test_residual_gradient_guidance_matches_reference(ops, golden, mode, tol_loss, tol_grad):
    """SURVEY 8f.3 (residuals_darcy.py:114-126, unet_model.py:530-540,585-603): training loss and the gradients of the
    guidance-only layers with the reference's classifier-free mask, the forced-null-mask variant, and sampling with
    guidance scale 3, against the unmodified reference."""
    ops.set_precision(mode)
    gd = golden('darcy_guidance.pt')
    model, diff, res = build_darcy('guidance')
    x0, t, e = gd['x0'].to(DEV), gd['t'].to(DEV), gd['noise'].to(DEV)
    model._null_mask_override = gd['null_mask'].to(DEV)
    loss, _, _, _, _ = diff.darcy_loss_from_draws(x0, t, e, res, 1.0, 1e-3)
    assert abs(loss.item() / gd['loss'].item() - 1) < tol_loss, (loss.item(), gd['loss'].item())
    loss.backward()
    named = dict(model.named_parameters())
    for k, g in (('emb_conv.0.weight', 'grad_emb0'), ('combine_conv.weight', 'grad_combine'),
                 ('final_conv.1.weight', 'grad_final_w')):
        assert rel(named[k].grad, gd[g]) < tol_grad, (k, rel(named[k].grad, gd[g]))
    model._null_mask_override = gd['forced_mask'].to(DEV)
    loss_f, _, _, _, _ = diff.darcy_loss_from_draws(x0, t, e, res, 1.0, 1e-3)
    assert abs(loss_f.item() / gd['loss_forced'].item() - 1) < tol_loss
    model._null_mask_override = None
    model.eval()
    with torch.no_grad():
        xin = gd['sample_in'].permute(0, 2, 3, 1).reshape(4, 4096, 2).to(DEV)
        out = res.compute_residual(((xin, t),), reduce='per-batch', return_model_out=True, sample=True)
    assert rel(out['model_out'], gd['sample_x0']) < (2e-4 if mode == 'fp32' else 5e-2)


def test_sampling_loop_with_cocogen_corrections(ops, golden, monkeypatch):
    """p_sample_loop with N_correction / M_correction (reference :516-541): the corrected trajectory equals the plain
    one followed by explicit corrections where the reference applies them (correction_mode 'xt')."""
    ops.set_precision('fp32')
    gd = golden('sample_loop_6.pt')
    model, diff, res = build_darcy(n_steps=6)
    model.eval()

    def run(**kw):
        it = iter([gd['x_T']] + list(gd['noises']))
        monkeypatch.setattr(torch, 'randn', lambda *a, **k: next(it).to(DEV))
        monkeypatch.setattr(torch, 'randn_like', lambda *a, **k: next(it).to(DEV))
        out = diff.p_sample_loop(None, (1, 2, 64, 64), save_output=True, surpress_noise=True, residual_func=res,
                                 eval_residuals=True, **kw)
        monkeypatch.undo()
        return out
    (xs0, _), aux0 = run()
    (xs1, _), aux1 = run(M_correction=2, N_correction=0, correction_mode='xt')
    assert len(xs1) == len(xs0) + 2 and rel(xs1[6], xs0[6]) < 1e-5          # (run-to-run: fp32 atomics, ~1e-7)
    manual = xs0[-1].clone().to(DEV)
    for _ in range(2):
        m, r = res.residual_correction(manual.permute(0, 2, 3, 1).reshape(1, 4096, 2).contiguous())
        manual = m.reshape(1, 64, 64, 2).permute(0, 3, 1, 2).contiguous()
    assert rel(xs1[-1], manual) < 1e-5 and rel(aux1['residual'], r) < 1e-4
    (xs2, _), aux2 = run(M_correction=0, N_correction=2, correction_mode='xt')
    assert len(xs2) == len(xs0) and rel(xs2[4], xs0[4]) < 1e-5 and rel(xs2[5], xs0[5]) > 1e-7
    assert torch.isfinite(aux2['residual']).all()


@pytest.mark.parametrize('B', [1, 3, 5, 16])
def test_unet_tensor_core_path_at_odd_batch_sizes(ops, B):
    """Tile / chunk / cluster planning depends on the batch size (TN samples per pixel tile, per-sample pixel chunks of
    the attention kernels, one-wave pixel splits of the wgrads ...).  bf16 tensor-core path vs the fp32 CUDA-core path
    of the same engine (itself pinned to the oracle above) on the same weights and inputs: forward and gradients."""
    g = torch.Generator().manual_seed(100 + B)
    x = torch.randn(B, 2, 64, 64, generator=g).to(DEV)
    t = torch.randint(0, 100, (B,), generator=g).to(DEV)
    cot = torch.randn(B, 2, 64, 64, generator=g).to(DEV)
    outs = {}
    for mode in ('fp32', 'bf16'):
        ops.set_precision(mode)
        model, _, _ = build_darcy()
        y = model(x, t)
        (y * cot).sum().backward()
        outs[mode] = (y.detach().clone(), model.init_conv.weight.grad.clone(),
                      model.downs[3][0].block1.proj.weight.grad.clone(), model.final_conv[1].weight.grad.clone())
    assert torch.isfinite(outs['bf16'][0]).all()
    for a, b in zip(outs['bf16'], outs['fp32']):
        assert rel(a, b) < 4e-2, rel(a, b)


def test_mechanics_training_loss_matches_oracle(ops, monkeypatch):
    """configs[2]: one loss evaluation + backward of the mechanics (topology-optimisation) branch -- q_sample on the
    65x65 fields, bilinear 65->64, Unet3D(channels=10, out_dim=3, sigmoid on the density channel), bilinear 64->65 of the
    displacements, matrix-free K(rho)u - f residual, compliance and volume-fraction terms (reference
    denoising_utils.py:629-710, residuals_mechanics_K.py:198-274) -- against the oracle composition in fp32."""
    ops.set_precision('fp32')
    from physicsinformeddiffusionmodels_b200.denoising_utils import DenoisingDiffusion
    from physicsinformeddiffusionmodels_b200.residuals_mechanics_K import ResidualsMechanics
    from physicsinformeddiffusionmodels_b200.unet_model import Unet3D
    cfg = O.unet_config(dim=32, channels=10, out_dim=3, sigmoid_last_channel=True)
    sd = O.make_test_state_dict(cfg, 3)
    model = Unet3D(dim=32, channels=10, out_dim=3, sigmoid_last_channel=True).to(DEV)
    model.load_state_dict(sd)
    diff = DenoisingDiffusion(100, DEV)
    res = ResidualsMechanics(model=model, pixels_per_dim=64, pixels_at_boundary=True, no_BC_folder='', device=DEV)
    g = torch.Generator().manual_seed(77)
    B = 2
    cond = torch.rand(B, 3, 65, 65, generator=g)
    cond[:, 0] = torch.tensor([0.4, 0.55])[:, None, None]                     # volume fraction plane
    x0 = torch.cat((0.2 * torch.randn(B, 2, 65, 65, generator=g), torch.rand(B, 1, 65, 65, generator=g)), dim=1)
    bcs = torch.zeros(B, 4, 65, 65)
    bcs[:, 0, :, 0] = 1.; bcs[:, 1, :, 0] = 1.                                # clamped left edge
    bcs[:, 3, 32, 64] = -1.                                                   # point load
    t = torch.tensor([17, 63])
    noise = torch.randn(B, 3, 65, 65, generator=g)
    c_data, c_res, lam = 1.0, 1e-2, 1e-3
    # ---- oracle (CPU, fp32)
    tabs = O.diffusion_tables(100)
    xt = O.q_sample(x0, t, noise, tabs)
    net_in = torch.cat((O.bilinear_resize(torch.cat((xt, cond), dim=1), 64), O.bilinear_resize(bcs, 64)), dim=1)
    params = {k: v.clone().requires_grad_(True) for k, v in sd.items() if v.is_floating_point()}
    y = O.unet_forward({**sd, **params}, cfg, net_in, t)
    r, comp, _ = O.mechanics_residual(y, bcs, cond[:, 0, 0, 0])
    mo = torch.cat((O.bilinear_resize(y[:, :2], 65), torch.nn.functional.pad(y[:, 2], (0, 1, 0, 1)).unsqueeze(1)), dim=1)
    mse = ((x0 - mo) ** 2).reshape(B, -1).mean(dim=1)
    p2w = tabs['p2_loss_weight'][t].float()
    var = tabs['posterior_variance_clipped'][t].float()
    loss_o = c_data * (mse * p2w).mean() + (c_res * 0.5 * r ** 2 / var[:, None]).mean() + (lam * comp).mean()
    loss_o.backward()
    # ---- engine
    monkeypatch.setattr(torch, 'randn_like', lambda *a, **k: noise.to(DEV))
    inp = torch.cat((cond, x0, bcs), dim=1).to(DEV)
    loss, data_l, rabs, _, opt = res.training_loss(diff, inp, t.to(DEV), c_data, c_res, 0., lam)
    monkeypatch.undo()
    assert abs(loss.item() / loss_o.item() - 1) < 2e-4, (loss.item(), loss_o.item())
    loss.backward()
    for name in ('final_conv.1.weight', 'init_conv.weight', 'mid_block1.block1.proj.weight'):
        p = dict(model.named_parameters())[name]
        assert rel(p.grad, params[name].grad) < 3e-3, (name, rel(p.grad, params[name].grad))


def test_engine_training_steps_match_oracle(ops):
    """3 optimizer steps of the flat-buffer engine (eager and CUDA-graph) vs the oracle's autograd + Adam + EMA."""
    ops.set_precision('fp32')
    from physicsinformeddiffusionmodels_b200.engine import TrainEngine
    B = 2
    g = torch.Generator().manual_seed(21)
    x0 = torch.randn(B, 2, 64, 64, generator=g)
    ts = [torch.tensor([3, 70]), torch.tensor([50, 9]), torch.tensor([99, 0])]
    es = [torch.randn(B, 2, 64, 64, generator=g) for _ in ts]
    tables = O.diffusion_tables(100)
    sd = state_dict()
    sdr = {k: v.clone().requires_grad_('freqs' not in k) for k, v in sd.items()}
    train = [v for k, v in sdr.items() if v.requires_grad]
    m = [torch.zeros_like(p) for p in train]
    v = [torch.zeros_like(p) for p in train]
    ema = [p.detach().clone() for p in train]
    ref_losses = []
    for step, (t, e) in enumerate(zip(ts, es), 1):
        for p in train:
            p.grad = None
        loss, _ = O.darcy_training_loss(sdr, config(), x0, t, e, tables)
        loss.backward()
        ref_losses.append(loss.item())
        with torch.no_grad():
            grads = [p.grad if p.grad is not None else torch.zeros_like(p) for p in train]
            O.adam_ema_step(train, grads, m, v, ema, step)
    model, diff, res = build_darcy()
    eng = TrainEngine(model, diff, res, use_graph=False)
    losses = []
    for t, e in zip(ts, es):
        with fixed_draws(t.to(DEV), e.to(DEV)):
            loss, _, _ = eng.step(x0.to(DEV))
        losses.append(loss.item())
    for a, b in zip(losses, ref_losses):
        assert abs(a / b - 1) < 2e-3, (losses, ref_losses)
    named = dict(model.named_parameters())
    for k in ('final_conv.1.weight', 'downs.0.0.block1.proj.weight', 'mid_spatial_attn.fn.fn.fn.to_qkv.weight'):
        # Adam normalises every coordinate to |update| ~ lr, so parameters are compared by their UPDATE
        upd = named[k].detach().cpu() - sd[k]
        upd_ref = sdr[k].detach() - sd[k]
        assert rel(upd, upd_ref) < 0.1, (k, rel(upd, upd_ref))
    sd_ema = eng.ema_state_dict()
    assert set(sd_ema.keys()) == set(sd.keys())


def test_engine_cuda_graph_replay_runs_and_learns(ops):
    ops.set_precision('bf16')
    from physicsinformeddiffusionmodels_b200.engine import TrainEngine
    model, diff, res = build_darcy()
    eng = TrainEngine(model, diff, res, use_graph=True, lr=1e-3)
    g = torch.Generator().manual_seed(22)
    x0 = (0.5 * torch.randn(4, 2, 64, 64, generator=g)).to(DEV)
    w0 = model.final_conv[1].weight.detach().clone()
    first = None
    for i in range(6):
        loss, data_l, rabs = eng.step(x0)
        if i == 0:
            first = loss.item()
    torch.cuda.synchronize()
    assert torch.isfinite(loss).all() and first is not None
    assert not torch.equal(model.final_conv[1].weight.detach(), w0)
    assert int(eng.fp.step_dev.item()) == eng.steps_done


def test_state_dict_roundtrip_and_cpu_rejection():
    model, diff, res = build_darcy()
    sd = model.state_dict()
    assert len(sd) == 317 and sum(v.numel() for v in sd.values()) == 10386514
    assert list(sd.keys()) == list(state_dict().keys())
    with pytest.raises(RuntimeError):
        model(torch.zeros(1, 2, 64, 64), torch.zeros(1, dtype=torch.long))     # CPU tensor: no fallback


def test_smoke_entry_point():
    import __graft_entry__
    __graft_entry__.smoke()
