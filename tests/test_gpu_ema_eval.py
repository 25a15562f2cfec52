"""Validation and sampling on the EMA weights during TrainEngine training (reference main.py:181-226): the flat-buffer
swap kernel, TrainEngine.ema_weights(), TrainEngine.validate() against the eager drop-in loss and the CPU oracle, the
reference loop's cadence eager and graph-replayed, SampleEngine inside the context, and the loss-only mode of the
mechanics loss kernel."""
import pytest
import torch

import mech_sample_inputs as MI
from checks import rel
from oracle import pidm_oracle as O
from study import build_darcy, config

pytestmark = pytest.mark.gpu
DEV = 'cuda'
MECH_CFG = dict(dim=32, channels=10, out_dim=3, sigmoid_last_channel=True)


@pytest.fixture(scope='module')
def ops():
    from physicsinformeddiffusionmodels_b200 import ops
    yield ops
    ops.set_precision('bf16')


def build_mechanics(n_steps=100, use_ddim_x0=False):
    from physicsinformeddiffusionmodels_b200.denoising_utils import DenoisingDiffusion
    from physicsinformeddiffusionmodels_b200.residuals_mechanics_K import ResidualsMechanics
    from physicsinformeddiffusionmodels_b200.unet_model import Unet3D
    model = Unet3D(**MECH_CFG).to(DEV)
    model.load_state_dict(O.make_test_state_dict(O.unet_config(**MECH_CFG), 3))
    res = ResidualsMechanics(model=model, pixels_per_dim=64, pixels_at_boundary=True, no_BC_folder='', device=DEV,
                             use_ddim_x0=use_ddim_x0, ddim_steps=0)
    return model, DenoisingDiffusion(n_steps, DEV), res


def mech_batch(B, seed):
    """[B, 10, 65, 65] = (conditioning | disp_x, disp_y, E | bcs) of the topology-optimisation study"""
    cond, bcs, _ = MI.conditioning_batch()
    g = torch.Generator().manual_seed(seed)
    rows = [i % 2 for i in range(B)]
    x0 = torch.cat((0.2 * torch.randn(B, 2, 65, 65, generator=g), torch.rand(B, 1, 65, 65, generator=g)), dim=1)
    return torch.cat((cond[rows], x0, bcs[rows]), dim=1).to(DEV)


def darcy_batch(B, seed):
    g = torch.Generator().manual_seed(seed)
    return (0.7 * torch.randn(B, 2, 64, 64, generator=g)).to(DEV)


# study -> (builder, engine options, batch maker)
STUDIES = {
    'mean': (lambda **k: build_darcy(**k), {}, darcy_batch),
    'sample': (lambda **k: build_darcy(use_ddim_x0=True, **k), {}, darcy_batch),
    'guidance': (lambda **k: build_darcy('guidance', **k), {}, darcy_batch),
    'periodic': (lambda **k: build_darcy('periodic', **k), {}, darcy_batch),
    'circular': (lambda **k: build_darcy('circular', **k), {}, darcy_batch),
    'mechanics': (lambda **k: build_mechanics(**k), dict(c_residual=1e-2, c_ineq=1.0, lambda_opt=1e-3), mech_batch),
}


def trained_engine(study, steps=2, use_graph=False, ema_start=-1, **kw):
    from physicsinformeddiffusionmodels_b200.engine import TrainEngine
    build, opts, batch = STUDIES[study]
    model, diff, res = build(**kw)
    eng = TrainEngine(model, diff, res, lr=1e-3, use_graph=use_graph, ema_start=ema_start, **opts)
    torch.cuda.manual_seed(5)
    for i in range(steps):
        eng.step(batch(2, 10 + i))
    torch.cuda.synchronize()
    return eng


def fresh_copy(study, sd, **kw):
    model, diff, res = STUDIES[study][0](**kw)
    model.load_state_dict(sd)
    return model, diff, res


def swap(a, b, n):
    from physicsinformeddiffusionmodels_b200._lib import call, stream
    return call('pidm_swap_f32', a, b, n, stream())


# ---- 1. the swap kernel ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize('n', [4, 1020, 4 * (256 * 7 + 3), 4 * 148 * 8 * 256 + 36])
def test_swap_is_an_exact_exchange(n):
    a = torch.randn(n, device=DEV)
    b = torch.randn(n, device=DEV)
    a0, b0 = a.clone(), b.clone()
    swap(a, b, n)
    assert torch.equal(a, b0) and torch.equal(b, a0)
    swap(a, b, n)
    assert torch.equal(a, a0) and torch.equal(b, b0)


def test_swap_rejects_misuse_without_launching():
    a = torch.randn(64, device=DEV)
    b = torch.randn(64, device=DEV)
    a0, b0 = a.clone(), b.clone()
    with pytest.raises(RuntimeError, match='multiple of 4'):
        swap(a, b, 62)
    with pytest.raises(RuntimeError, match='16-byte aligned'):
        swap(a[1:], b[1:], 60)
    torch.cuda.synchronize()
    assert torch.equal(a, a0) and torch.equal(b, b0)


# ---- 2. + 7. the context: exactness and guards ----------------------------------------------------------------------

def test_ema_context_is_exact_and_leaves_training_unchanged(ops):
    """Inside the context every parameter is the EMA weight; on exit every training buffer is bitwise what it was, and
    the next graph-replayed step is that of the same state without the context (bitwise where replays from one state
    agree bitwise; otherwise to the run-to-run spread of the fp32 atomics)."""
    ops.set_precision('fp32')
    x = darcy_batch(2, 1)
    eng = trained_engine('mean', steps=3, use_graph=True)
    fp = eng.fp
    bufs = (fp.flat, fp.ema, fp.exp_avg, fp.exp_avg_sq, fp.step_dev, fp.grad)
    before = [v.clone() for v in bufs]
    assert not torch.equal(fp.flat, fp.ema)
    ema_sd = eng.ema_state_dict()
    with eng.ema_weights():
        torch.cuda.synchronize()
        for name, p in eng.model.named_parameters():
            assert torch.equal(p.detach(), ema_sd[name].to(p.device)), name
        inside = eng.ema_state_dict()             # where main.py:312-313 saves its checkpoint
        assert inside.keys() == ema_sd.keys() and all(torch.equal(v, ema_sd[k]) for k, v in inside.items())
    torch.cuda.synchronize()
    for v, k in zip(bufs, before):
        assert torch.equal(v, k)

    def next_step(enter):
        for v, k in zip(bufs, before):
            v.copy_(k)
        if enter:
            with eng.ema_weights():
                pass
        torch.cuda.manual_seed(77)
        out = torch.stack(eng.step(x))
        torch.cuda.synchronize()
        return torch.cat((out, fp.flat, fp.ema, fp.exp_avg, fp.exp_avg_sq)).clone()
    # The run-to-run spread of the fp32 atomics (GroupNorm statistics, weight-gradient splits) is not one value: two
    # replays may agree bitwise, differ in a few small elements, or differ by an ulp of the loss, which dominates the
    # norm.  So the spread is taken over every pair of replays within each group, five interleaved replays with and
    # five without the context, and every replay with the context must lie within 4x of it from every replay
    # without: bitwise where all within-group pairs agree bitwise.
    runs = {enter: [] for enter in (False, True)}
    for _ in range(5):
        for enter in (False, True):
            runs[enter].append(next_step(enter))
    spread = max(rel(a, b) for g in runs.values() for i, a in enumerate(g) for b in g[i + 1:])
    cross = max(rel(e, p) for e in runs[True] for p in runs[False])
    assert cross <= 4 * spread, (cross, spread)


def test_ema_context_guards(ops):
    ops.set_precision('bf16')
    eng = trained_engine('mean', steps=2)
    flat0, ema0 = eng.fp.flat.clone(), eng.fp.ema.clone()
    with eng.ema_weights():
        with pytest.raises(RuntimeError, match='ema_weights'):
            eng.step(darcy_batch(2, 3))
        with pytest.raises(RuntimeError, match='nest'):
            with eng.ema_weights():
                pass
        assert torch.equal(eng.fp.flat, ema0)
    assert torch.equal(eng.fp.flat, flat0) and torch.equal(eng.fp.ema, ema0)
    with pytest.raises(ValueError, match='inside'):
        with eng.ema_weights():
            raise ValueError('inside')
    assert torch.equal(eng.fp.flat, flat0) and torch.equal(eng.fp.ema, ema0)
    with eng.ema_weights():                        # usable again after the exception
        pass
    assert eng.step(darcy_batch(2, 3))[0].isfinite()


# ---- 3. validate against the eager drop-in loss on a model loaded from ema_state_dict() ------------------------------

@pytest.mark.parametrize('study', list(STUDIES))
def test_validate_on_ema_matches_dropin_loss(ops, study):
    """fp32 activations: the same kernels on the same weights; only the order of fp32 atomics differs (1e-4, the
    engine-versus-eager tolerance of test_gpu_e2e.py).  Negative control: the loss of the live weights, validated just
    before entering and just after leaving the context, differs from the EMA loss by far more than that tolerance, so
    packed operands left stale by the swap in or out would fail the test."""
    ops.set_precision('fp32')
    eng = trained_engine(study)

    def live_loss():
        torch.cuda.manual_seed(1234)
        return eng.validate(xv)[0].item()
    model, diff, res = fresh_copy(study, eng.ema_state_dict())
    opts = STUDIES[study][1]
    xv = STUDIES[study][2](3, 99)
    torch.cuda.manual_seed(1234)
    with torch.no_grad():
        ref = diff.model_estimation_loss(xv, residual_func=res, c_data=1.0, c_residual=opts.get('c_residual', 1e-3),
                                         c_ineq=opts.get('c_ineq', 0.), lambda_opt=opts.get('lambda_opt', 0.),
                                         sync_scalars=False)
    rng_ref = torch.cuda.get_rng_state()
    live_before = live_loss()
    torch.cuda.manual_seed(1234)
    with eng.ema_weights():
        got = eng.validate(xv)
    assert torch.equal(torch.cuda.get_rng_state(), rng_ref)
    got = [v.clone() for v in got]
    live_after = live_loss()
    assert abs(live_after - live_before) <= 1e-4 * abs(live_before), (live_before, live_after)
    assert abs(got[0].item() - live_before) > 1e-3 * abs(live_before), (got[0].item(), live_before)
    assert len(got) == 5 and all(isinstance(v, torch.Tensor) and v.is_cuda for v in got)
    for g, r in zip(got, ref):
        r = torch.as_tensor(r, device=DEV, dtype=torch.float32)
        assert abs(g.item() - r.item()) <= 1e-4 * abs(r.item()) + 1e-12, (study, [v.item() for v in got], ref)
    if study != 'mechanics':
        assert got[3].item() == 0. and got[4].item() == 0.
    else:
        assert got[3].item() != 0. and got[4].item() != 0.


@pytest.mark.parametrize('study', ['mean', 'guidance', 'mechanics'])
def test_validate_graph_replay_equals_eager(ops, study):
    """one captured graph per input shape (a ragged last batch included); the RNG stream advances as in the eager call"""
    ops.set_precision('fp32')
    eng = trained_engine(study, use_graph=True)
    batch = STUDIES[study][2]
    with eng.ema_weights():
        for B, seed in ((4, 50), (3, 51), (4, 52)):
            xv = batch(B, seed)
            eng.use_graph = False
            torch.cuda.manual_seed(seed)
            ve = torch.stack(eng.validate(xv)).clone()
            rng_e = torch.cuda.get_rng_state()
            eng.use_graph = True
            torch.cuda.manual_seed(seed)
            vg = torch.stack(eng.validate(xv)).clone()
            assert torch.equal(torch.cuda.get_rng_state(), rng_e)
            assert rel(vg, ve) < 1e-5, (B, vg, ve)
    assert len(eng._val_graphs) == 2


# ---- 4. the CPU oracle on the EMA weights ---------------------------------------------------------------------------

def test_validate_on_ema_matches_oracle(ops):
    """injected t and eps; fp32 tolerance of the loss goldens (5e-5)"""
    ops.set_precision('fp32')
    eng = trained_engine('mean')
    sd = {k: v.cpu() for k, v in eng.ema_state_dict().items()}
    g = torch.Generator().manual_seed(3)
    x0 = 0.7 * torch.randn(2, 2, 64, 64, generator=g)
    t = torch.tensor([7, 61])
    e = torch.randn(2, 2, 64, 64, generator=g)
    with torch.no_grad():
        loss_o, aux = O.darcy_training_loss(sd, config(), x0, t, e, O.diffusion_tables(100))
    rng = torch.cuda.get_rng_state()
    with eng.ema_weights():
        loss, data_l, rabs, _, _ = eng.validate(x0.to(DEV), t=t.to(DEV), noise=e.to(DEV))
    assert torch.equal(torch.cuda.get_rng_state(), rng)          # injected draws: nothing drawn
    assert abs(loss.item() / loss_o.item() - 1) < 5e-5, (loss.item(), loss_o.item())
    assert abs(data_l.item() / aux['data'].item() - 1) < 5e-5
    assert abs(rabs.item() / aux['residual_abs'].item() - 1) < 5e-5


# ---- 5. the reference loop's cadence --------------------------------------------------------------------------------

@pytest.mark.parametrize('study', ['mean', 'guidance'])
def test_training_loop_cadence_graph_equals_eager(ops, study):
    """main.py:157-198 with ema_start=1 and validation inside ema_weights() every 2 iterations, 6 iterations, training
    at batch 4 and validating at batch 3: before iteration ema_start + 1 the shadow still holds the initial weights, and
    that is what the first validations see.  Under guidance the captured training step writes its classifier-free mask
    into model._null_mask_last: a validation at another batch size leaves that tensor in place (were it replaced and
    freed, the replayed steps would write through a dangling pointer and drift from the eager run).  Tolerance: graph
    and eager differ by the order of fp32 atomics (1e-5); under guidance the network's condition is sign(r) of the noisy
    sample's residual, which turns those last bits into a drift of ~2e-5 over the six steps (measured), hence 1e-4."""
    ops.set_precision('fp32')
    from physicsinformeddiffusionmodels_b200.engine import TrainEngine
    runs = {}
    for use_graph in (False, True):
        model, diff, res = STUDIES[study][0]()
        eng = TrainEngine(model, diff, res, lr=1e-3, use_graph=use_graph, ema_start=1)
        ema0 = eng.fp.ema.clone()
        torch.cuda.manual_seed(11)
        vals = []
        train_mask = None
        for it in range(6):
            vals.append(torch.stack(eng.step(darcy_batch(4, 20 + it))).clone())
            if study == 'guidance':
                if it == 0:
                    train_mask = model._null_mask_last
                assert model._null_mask_last is train_mask and train_mask.shape == (4,)
                vals.append(train_mask.float().clone())
            if it < 2:
                assert torch.equal(eng.fp.ema, ema0) and not torch.equal(eng.fp.flat, ema0)
            if it % 2 == 0:
                with eng.ema_weights():
                    vals.append(torch.stack(eng.validate(darcy_batch(3, 40 + it))).clone())
                if study == 'guidance':
                    assert model._null_mask_last is train_mask
        torch.cuda.synchronize()
        assert not torch.equal(eng.fp.ema, ema0)
        runs[use_graph] = (vals, eng.fp.flat.clone(), eng.fp.ema.clone())
        eng.close()
    (ve, fe, ee), (vg, fg, eg) = runs[False], runs[True]
    assert len(ve) == len(vg) == (15 if study == 'guidance' else 9)
    tol = 1e-4 if study == 'guidance' else 1e-5
    for i, (a, b) in enumerate(zip(vg, ve)):
        assert rel(a, b) < tol, (i, a, b)
    assert rel(fg, fe) < tol and rel(eg, ee) < tol


# ---- 6. SampleEngine inside the context -----------------------------------------------------------------------------

def _darcy_sampler(model, diff, res):
    from physicsinformeddiffusionmodels_b200.engine import SampleEngine
    return SampleEngine(model, diff, res, batch=2, use_graph=True, external_noise=True)


def _mech_sampler(model, diff, res):
    from physicsinformeddiffusionmodels_b200.engine import SampleEngine
    return SampleEngine(model, diff, res, batch=2, image_shape=(3, 65, 65), use_graph=True, external_noise=True)


@pytest.mark.parametrize('study', ['mean', 'mechanics'])
def test_sample_engine_inside_the_context_samples_the_ema_weights(ops, study):
    """fp32 activations; two sampling runs differ by the order of fp32 atomics only (GroupNorm and attention partial
    sums), so runs are compared to 1e-5 (measured bitwise equal or ~1e-7 apart)"""
    ops.set_precision('fp32')
    eng = trained_engine(study, n_steps=6)
    mech = study == 'mechanics'
    make = _mech_sampler if mech else _darcy_sampler
    g = torch.Generator().manual_seed(8)
    shape = (2, 3, 65, 65) if mech else (2, 2, 64, 64)
    x_T = torch.randn(*shape, generator=g).to(DEV)
    zs = torch.randn(6, *shape, generator=g).to(DEV)
    kw = {}
    if mech:
        cond, bcs, _ = MI.conditioning_batch()
        kw = dict(conditioning_input=(cond.to(DEV), bcs.to(DEV), None))

    def run(se):
        x, r, _ = se.sample(x_init=x_T, noises=zs, **kw)
        return x.clone(), (r['residual'] if mech else r).clone()
    se = make(eng.model, eng.diffusion, eng.residuals)
    live = run(se)
    with eng.ema_weights():
        on_ema = run(se)
    after = run(se)
    ref = run(make(*fresh_copy(study, eng.ema_state_dict(), n_steps=6)))
    assert rel(on_ema[0], live[0]) > 1e-3
    for a, b in zip(on_ema, ref):
        assert rel(a, b) < 1e-5, rel(a, b)
    for a, b in zip(after, live):
        assert rel(a, b) < 1e-5, rel(a, b)


# ---- 8. loss-only mode of the mechanics loss kernel -----------------------------------------------------------------

@pytest.mark.parametrize('B', [1, 3])
def test_mechanics_loss_only_mode_sums_are_those_of_the_gradient_call(B):
    """one CTA per sample adds its terms into the sums with atomics: with one sample the sums are bitwise those of the
    gradient-writing call, with more they may differ in the order of the CTAs' additions (a few ulp)"""
    from physicsinformeddiffusionmodels_b200._lib import call, stream
    g = torch.Generator().manual_seed(4)
    nel = 64
    n = (nel + 1) ** 2
    u = torch.randn(B, 2, n, generator=g).to(DEV)
    rho = torch.rand(B, nel, nel, generator=g).to(DEV)
    x0 = torch.randn(B, 3, n, generator=g).to(DEV)
    r = torch.randn(B, 2 * n, generator=g).to(DEV)
    comp = torch.rand(B, generator=g).to(DEV)
    vf = torch.rand(B, generator=g).to(DEV)
    t = torch.tensor([3, 50, 97][:B], device=DEV)
    tabs = O.diffusion_tables(100)
    p2 = tabs['p2_loss_weight'].float().to(DEV)
    var = tabs['posterior_variance_clipped'].float().to(DEV)
    grads = [torch.empty_like(u), torch.empty_like(rho), torch.empty_like(r), torch.empty_like(comp)]

    def sums_of(gs):
        s = torch.empty(6, device=DEV)
        call('pidm_mech_pidm_loss', u, rho, x0, r, comp, vf, t, p2, var, 1.0, 1e-2, 0.5, 1e-3, s, *gs, B, nel, stream())
        return s
    with_grads = sums_of(grads)
    loss_only = sums_of([None] * 4)
    if B == 1:
        assert torch.equal(with_grads, loss_only)
    else:
        assert torch.allclose(with_grads, loss_only, rtol=1e-6, atol=0), (with_grads, loss_only)
    with pytest.raises(RuntimeError, match='all set or all NULL'):
        sums_of(grads[:2] + [None, None])
