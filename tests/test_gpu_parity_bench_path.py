"""Parity of the BENCHMARKED path: the configuration `bench.py` times is batch 32, bf16, CUDA-graph replay with the
weight-gradient side stream and programmatic dependent launch on, device-side Adam step counter.  The golden fixtures
are B=2 and eager, and tile planning depends on the batch size (conv_tc.cu tc_plan picks the n-tile width from the tile
count, the wgrads split pixels over one wave, attention chunks pixels per sample), so these tests pin exactly the
instantiations and the schedule the bench runs.  The graph-replayed step is checked against the eager step for every
study option (tests/study.py) and for the mechanics branch."""
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


GRAD_KEYS = ['init_conv.weight', 'time_mlp.1.weight', 'downs.0.0.block1.proj.weight', 'downs.0.0.mlp.1.weight',
             'downs.0.2.fn.fn.to_qkv.weight', 'downs.1.3.weight', 'downs.3.1.block2.proj.weight',
             'mid_spatial_attn.fn.fn.fn.to_qkv.weight', 'ups.0.3.weight', 'ups.3.2.fn.norm.gamma',
             'ups.1.0.res_conv.weight', 'final_conv.0.block1.proj.weight', 'final_conv.1.weight', 'final_conv.1.bias']


@pytest.fixture(scope='module')
def oracle_b32():
    """One oracle evaluation of the headline batch (32 samples, ~3 s of CPU): loss + gradients."""
    g = torch.Generator().manual_seed(3232)
    B = 32
    x0 = 0.7 * torch.randn(B, 2, 64, 64, generator=g)
    t = torch.randint(0, 100, (B,), generator=g)
    e = torch.randn(B, 2, 64, 64, generator=g)
    sdr = {k: v.clone().requires_grad_('freqs' not in k) for k, v in state_dict().items()}
    loss, aux = O.darcy_training_loss(sdr, config(), x0, t, e, O.diffusion_tables(100), 1.0, 1e-3)
    loss.backward()
    grads = {k: sdr[k].grad.clone() for k in GRAD_KEYS}
    gn = torch.sqrt(sum((v.grad.double() ** 2).sum() for v in sdr.values() if v.grad is not None)).item()
    return dict(x0=x0, t=t, e=e, loss=loss.item(), grads=grads, grad_norm=gn)


# fp32 mode: summation order only (K up to 4608, ~60 layers, 32-sample means); bf16: 2^-9 per rounding through ~60
# layers, run-to-run noise 6e-3 (DESIGN section 2).  Same tolerances as the B=2 golden tests.
@pytest.mark.parametrize('mode,tol_loss,tol_grad', [('fp32', 5e-5, 1e-3), ('bf16', 3e-2, 8e-2)])
def test_headline_batch32_loss_and_gradients_match_oracle(ops, oracle_b32, mode, tol_loss, tol_grad):
    ops.set_precision(mode)
    ob = oracle_b32
    model, diff, res = build_darcy()
    loss, data_l, rabs, _, _ = diff.darcy_loss_from_draws(ob['x0'].to(DEV), ob['t'].to(DEV), ob['e'].to(DEV), res,
                                                          1.0, 1e-3)
    assert abs(loss.item() / ob['loss'] - 1) < tol_loss, (loss.item(), ob['loss'])
    loss.backward()
    named = dict(model.named_parameters())
    worst = {k: rel(named[k].grad, v) for k, v in ob['grads'].items()}
    assert max(worst.values()) < tol_grad, worst
    gn = torch.sqrt(sum((p.grad.double() ** 2).sum() for p in model.parameters() if p.grad is not None)).item()
    assert abs(gn / ob['grad_norm'] - 1) < tol_grad


def darcy(study, B, seed, **options):
    """builder and batch of a Darcy row: x0, t and the noise of B samples from one seeded generator"""
    def batch():
        g = torch.Generator().manual_seed(seed)
        x0 = 0.7 * torch.randn(B, 2, 64, 64, generator=g)
        t = torch.randint(0, 100, (B,), generator=g)
        return x0, t, torch.randn(B, 2, 64, 64, generator=g)
    return dict(build=lambda: build_darcy(study, **options), batch=batch)


def guidance(B, **options):
    """a guidance row: the classifier-free mask is fixed, and the guidance layers lie in the exchanged prefix"""
    return dict(darcy('guidance', B, 700 + B, **options), mask=torch.arange(B) % 3 == 1,
                live=('emb_conv.0.weight', 'emb_conv.2.weight', 'combine_conv.weight'))


def mechanics():
    from test_gpu_mechanics import build, synthetic_batch
    return dict(build=lambda: build(O, 32, 3)[2:], batch=lambda: synthetic_batch(2, 12),
                engine=dict(c_data=1.0, c_residual=1e-2, c_ineq=0.5, lambda_opt=1e-3))


# row: (mode, loss tolerance, flat-gradient tolerance, builder and batch).  fp32 mode isolates scheduling bugs (a missing
# stream dependency shows up as a wrong or partial gradient) from bf16 rounding noise; the bf16 rows use the run-to-run
# tolerance of that mode.
FP32, BF16 = ('fp32', 1e-5, 1e-4), ('bf16', 2e-2, 6e-2)
STEP_ROWS = {
    'none-fp32-B4': (*FP32, darcy('none', 4, 504)),
    'none-fp32-B32': (*FP32, darcy('none', 32, 532)),
    'none-bf16-B32': (*BF16, darcy('none', 32, 532)),
    'periodic-fp32-B32': (*FP32, darcy('periodic', 32, 532)),
    # the transposed layers read the halo'd dy on the weight-gradient side stream
    'circular-fp32-B32': (*FP32, darcy('circular', 32, 565)),
    'circular-bf16-B32': (*BF16, darcy('circular', 32, 565)),
    'guidance-fp32-B32': (*FP32, guidance(32)),
    'guidance-fp32-B5': (*FP32, guidance(5)),
    'guidance-circular-fp32-B8': (*FP32, guidance(8, bcs='periodic', padding_mode='circular')),
    'mechanics-fp32-B2': (*FP32, mechanics()),
}


def _worst(eng, model, ga, gb):
    """the three parameters whose gradients differ most between two flat gradients"""
    names = {id(p): k for k, p in model.named_parameters()}
    errs = [(rel(gb[o:o + p.numel()], ga[o:o + p.numel()]), names[id(p)]) for p, o in zip(eng.fp.params, eng.fp.offsets)]
    return sorted(errs, reverse=True)[:3]


@pytest.mark.parametrize('row', list(STEP_ROWS))
def test_graph_replayed_step_equals_eager_step(ops, row):
    """The step bench.py times (CUDA graph; wgrads on the forked stream; PDL; weight packing on its own stream) against
    the plain eager step on one stream, same weights / batch / draws: loss and the whole flat gradient, then the
    parameters after the update, for every study option and the mechanics branch."""
    mode, tol_loss, tol_grad, r = STEP_ROWS[row]
    ops.set_precision(mode)
    from physicsinformeddiffusionmodels_b200.engine import TrainEngine
    x0, t, e = (a.to(DEV) for a in r['batch']())
    mask = r['mask'].to(DEV) if 'mask' in r else None
    out = {}
    for use_graph in (False, True):
        model, diff, res = r['build']()
        model._null_mask_override = mask
        eng = TrainEngine(model, diff, res, use_graph=use_graph, snapshot_grad=True, **r.get('engine', {}))
        p0 = eng.fp.flat.clone()
        with fixed_draws(t, e):
            loss, _, _ = eng.step(x0)
        torch.cuda.synchronize()
        assert int(eng.fp.step_dev.item()) == 1          # warm-up steps of the capture are rolled back
        if mask is not None:
            assert torch.equal(model._null_mask_last, mask)
        named = dict(model.named_parameters())
        offsets = {id(p): o for p, o in zip(eng.fp.params, eng.fp.offsets)}
        for n in r.get('live', ()):
            assert offsets[id(named[n])] < eng.fp.live_total, n
        out[use_graph] = (loss.item(), eng.grad_snapshot.clone(), eng.fp.flat.clone() - p0, eng.fp.ema.clone() - p0)
        if use_graph:                                     # second replay: counter and moments advance on the device
            with fixed_draws(t, e):
                eng.step(x0)
            torch.cuda.synchronize()
            assert int(eng.fp.step_dev.item()) == 2
    (le, ge, pe, ee), (lg, gg, pg, eg) = out[False], out[True]
    assert abs(lg / le - 1) < tol_loss, (lg, le)
    assert rel(gg, ge) < tol_grad, (rel(gg, ge), _worst(eng, model, ge, gg))
    assert (ge != 0).float().mean().item() > 0.8          # the flat gradient really is populated
    assert pe.abs().max() > 0 and pg.abs().max() > 0      # the optimizer moved the weights
    # Adam normalises the update to ~lr per coordinate (sign-like for tiny gradients): compare the UPDATES, loosely
    assert rel(pg, pe) < (2e-2 if mode == 'fp32' else 0.5), rel(pg, pe)
    assert rel(eg, ee) < (2e-2 if mode == 'fp32' else 0.5), rel(eg, ee)


def test_device_step_counter_bias_correction():
    """pidm_adam_ema_step with the DEVICE step counter (the CUDA-graph path) vs the oracle at steps 1, 2 and 1000:
    the bias corrections 1 - beta^step are evaluated in double on the device like torch.optim.Adam does on the host
    (in fp32, 1 - 0.999^1 alone is off by 6e-5 relative)."""
    from physicsinformeddiffusionmodels_b200._lib import call, stream
    g = torch.Generator().manual_seed(15)
    n = 65536 + 3
    for step in (1, 2, 1000):
        for zero_p in (True, False):
            # zero_p: parameters start at 0, so the new parameter IS the (negated) update and can be compared to 1e-6
            # relative; with p = O(1) the update (1e-4) sits 3 decimal digits below one ulp of p, so that case is held
            # to "within one ulp of the fp32 parameter" instead
            p = torch.zeros(n) if zero_p else torch.randn(n, generator=g)
            gr = torch.randn(n, generator=g) * 0.01
            m, v = torch.randn(n, generator=g) * 0.01, torch.rand(n, generator=g) * 1e-4
            ema = p + 0.01 * torch.randn(n, generator=g)
            pr, mr, vr, er = p.clone(), m.clone(), v.clone(), ema.clone()
            O.adam_ema_step([pr], [gr], [mr], [vr], [er], step)
            pd, gd, md, vd, ed = (a.to(DEV) for a in (p, gr, m, v, ema))
            counter = torch.full((1,), step - 1, device=DEV, dtype=torch.int32)     # steps done so far
            nsq = torch.zeros(1, device=DEV)
            call('pidm_sumsq', gd, n, nsq, torch.zeros(1 + 148 * 8, device=DEV), stream())
            call('pidm_adam_ema_step', pd, gd, md, vd, ed, n, 1e-4, 0.9, 0.999, 1e-8, 0, counter, nsq, 1.0, 1.0, 0.99, 1,
                 0, stream())
            assert int(counter.item()) == step
            if zero_p:
                assert rel(pd.cpu(), pr) < 2e-6, (step, rel(pd.cpu(), pr))
            else:
                assert ((pd.cpu() - pr).abs() <= 1.2e-7 * pr.abs().clamp_min(1.0)).all(), step
            assert torch.allclose(ed.cpu(), er, rtol=1e-6, atol=2e-7), step
            assert torch.allclose(md.cpu(), mr, rtol=1e-5, atol=1e-9) and torch.allclose(vd.cpu(), vr, rtol=1e-5, atol=1e-12)


def test_ema_start_is_honoured_on_the_device(ops):
    """reference main.py:52,178: the shadow is first updated at the 0-based iteration ema_start + 1."""
    ops.set_precision('bf16')
    from physicsinformeddiffusionmodels_b200.engine import TrainEngine
    model, diff, res = build_darcy()
    eng = TrainEngine(model, diff, res, use_graph=True, ema_start=1, lr=1e-3)
    x0 = (0.5 * torch.randn(2, 2, 64, 64)).to(DEV)
    ema0 = eng.fp.ema.clone()
    eng.step(x0); eng.step(x0)                 # iterations 0 and 1: no EMA update yet
    torch.cuda.synchronize()
    assert torch.equal(eng.fp.ema, ema0)
    eng.step(x0)                               # iteration 2 > ema_start
    torch.cuda.synchronize()
    assert not torch.equal(eng.fp.ema, ema0)
    with pytest.raises(ValueError):
        eng.step(x0[:1])                       # captured for B=2: no silent broadcast of a smaller batch


def test_sample_engine_100_steps_matches_reference(ops, golden, monkeypatch):
    """The reference's default 100-step ancestral loop at B=1 with its own draws (regenerated from the stored seed)
    through SampleEngine, eager and CUDA-graph replay."""
    from test_oracle_golden import replay_draws_100
    ops.set_precision('fp32')
    from physicsinformeddiffusionmodels_b200.engine import SampleEngine
    gd = golden('sample_loop_100.pt')
    draws = replay_draws_100(gd).to(DEV)
    model, diff, res = build_darcy(n_steps=100)
    model.eval()
    it = iter(list(draws[1:]))
    monkeypatch.setattr(torch, 'randn_like', lambda *a, **k: next(it))
    x, r, traj = SampleEngine(model, diff, res, batch=1, use_graph=False).sample(x_init=draws[0], trajectory=True)
    x, r = x.clone(), r.clone()
    monkeypatch.undo()
    assert traj.shape[0] == 101
    for k in (25, 50, 75):
        assert rel(traj[k], gd[f'x_{k}']) < 1e-3, (k, rel(traj[k], gd[f'x_{k}']))
    assert rel(x, gd['x_final']) < 2e-3, rel(x, gd['x_final'])
    assert abs(r.abs().mean().item() / gd['residual_abs_mean'].item() - 1) < 2e-2
    # graph replay: the per-step noise is a static input buffer refreshed between replays
    eng = SampleEngine(model, diff, res, batch=1, use_graph=True, external_noise=True)     # 10 steps per graph
    assert eng.k == 10
    xg = eng.sample(x_init=draws[0], noises=draws[1:])[0]
    assert rel(xg, gd['x_final']) < 2e-3, rel(xg, gd['x_final'])


def test_darcy_loss_backward_twice_does_not_rescale(ops):
    """ADVICE r1: the fused loss kernel produces its gradient in forward; backward must scale a COPY."""
    ops.set_precision('fp32')
    from physicsinformeddiffusionmodels_b200.residuals_darcy import ResidualsDarcy
    from physicsinformeddiffusionmodels_b200.denoising_utils import DenoisingDiffusion
    diff = DenoisingDiffusion(100, DEV)
    res = ResidualsDarcy(model=None, fd_acc=2, pixels_per_dim=64, pixels_at_boundary=True, reverse_d1=True, device=DEV)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 2, 64, 64, generator=g).to(DEV).requires_grad_(True)
    tgt = torch.randn(2, 2, 64, 64, generator=g).to(DEV)
    t = torch.tensor([4, 80], device=DEV)
    dd = diff.diff_dict
    loss, _ = ops.darcy_pidm_loss(x, None, tgt, t, res.f_s_flat, dd['p2_loss_weight'], dd['posterior_variance_clipped'],
                                  1.0, 1e-3)
    (2.0 * loss).backward(retain_graph=True)
    g1 = x.grad.clone()
    x.grad = None
    (2.0 * loss).backward()
    assert torch.equal(x.grad, g1)
    with pytest.raises((AssertionError, RuntimeError)):
        ops.darcy_pidm_loss(x, None, tgt, t, res.f_s_flat, dd['p2_loss_weight'].double(),
                            dd['posterior_variance_clipped'], 1.0, 1e-3)
