"""CoCoGen residual corrections on the GPU: `pidm_darcy_cocogen` (all corrections of a batch in one launch) against the
unmodified reference's fixtures, against the multi-launch composition it replaces and against the fp64 oracle, its
device-side predication, and the corrected `SampleEngine` (graph and eager) against the drop-in
`DenoisingDiffusion.p_sample_loop` and the reference's corrected sampling loop."""
import pytest
import torch

from checks import rel
from oracle import pidm_oracle as O
from study import build_darcy

pytestmark = pytest.mark.gpu
DEV = 'cuda'
P = 64


@pytest.fixture(scope='module')
def ops():
    from physicsinformeddiffusionmodels_b200 import ops
    yield ops
    ops.set_precision('bf16')


def build(study='none', use_ddim_x0=False):
    model, diff, res = build_darcy(study, n_steps=6, use_ddim_x0=use_ddim_x0)
    model.eval()
    return model, diff, res


def compose(res, x, steps):
    """`steps` corrections as the multi-launch composition residual_correction used to be: residual, cotangent 2r,
    adjoint, Jacobian maximum, step size, update, and the residual of the result"""
    from physicsinformeddiffusionmodels_b200._lib import call, stream
    x = x.clone()
    B = x.shape[0]
    geo = res._abi_geometry()
    mx = torch.empty(B, device=DEV)
    call('pidm_darcy_jacobian_max', x, mx, B, P, *geo, stream())
    eps = 1.e-6 / torch.clamp(mx, max=1e12)
    r = torch.empty(B, P * P, 3, device=DEV)
    gx = torch.empty_like(x)
    for _ in range(steps):
        call('pidm_darcy_residual_fwd', x, res.f_s_flat, r, B, P, *geo, stream())
        call('pidm_darcy_residual_bwd', x, res.f_s_flat, (2.0 * r).contiguous(), gx, B, P, *geo, stream())
        x[:, 0] -= eps.view(B, 1, 1) * gx[:, 0]
    call('pidm_darcy_residual_fwd', x, res.f_s_flat, r, B, P, *geo, stream())
    return x, r


def kernel(res, x, steps, t=None, n_active=0, residual=None):
    x = x.to(DEV).float().contiguous().clone()
    r = torch.full((x.shape[0], P * P, 3), float('nan'), device=DEV) if residual is None else residual.clone()
    res.cocogen(x, r, steps, t, n_active)
    torch.cuda.synchronize()
    return x, r


# ---- kernel, one step: the reference's residual_correction ----------------------------------------------------------
@pytest.mark.parametrize('study,fixture', [('none', 'cocogen.pt'), ('periodic', 'cocogen_periodic.pt')])
def test_one_step_matches_reference(golden, study, fixture):
    """the kernel, and residual_correction, which applies it in place on the [B, P*P, 2] tensor like the reference"""
    gd = golden(fixture)
    res = build(study)[2]
    x, r = kernel(res, gd['x0_pred'], 1)
    xin = gd['x0_pred'].permute(0, 2, 3, 1).reshape(2, P * P, 2).clone().to(DEV)
    x_corr, r_corr = res.residual_correction(xin)
    assert x_corr is xin
    d_ref = gd['corrected'] - gd['x0_pred']
    for xc, rc in ((x.cpu(), r), (xin.reshape(2, P, P, 2).permute(0, 3, 1, 2).cpu(), r_corr)):
        assert rel(xc - gd['x0_pred'], d_ref) < 1e-3, rel(xc - gd['x0_pred'], d_ref)
        assert torch.equal(xc[:, 1], gd['x0_pred'][:, 1])
        assert rel(rc, gd['residual_corrected']) < 1e-5


# ---- kernel, several steps ------------------------------------------------------------------------------------------
# Against the composition: each step does the same fp32 arithmetic in the same order, apart from the residual that
# forms the cotangent (the composition takes it from the forward kernel's vectorised stencil, the correction kernel
# from the adjoint kernel's per-pixel one; they differ in the last bit).  A 1-ulp change of one step's p-increment can
# round p to the neighbouring float, an error of ulp(p) against an accumulated increment many ulps large, so the
# accumulated change of p is held to 1e-4 and the residual (a fixed linear map of that change plus f_s) to 1e-5.
# Against the reference (fp32 vmap(jacfwd) path) and the fp64 oracle: the 1e-3 / 1e-5 of the one-step test.
@pytest.mark.parametrize('steps', [2, 5, 200])
@pytest.mark.parametrize('study,fixture', [('none', 'cocogen.pt'), ('periodic', 'cocogen_periodic.pt')])
def test_steps_match_composition_and_reference(golden, study, fixture, steps):
    res = build(study)[2]
    x0 = golden(fixture)['x0_pred']
    x, r = kernel(res, x0, steps)
    xc, rc = compose(res, x0.to(DEV), steps)
    d = (x - x0.to(DEV))[:, 0]
    dc = (xc - x0.to(DEV))[:, 0]
    assert dc.abs().max() > 0
    assert torch.equal(x[:, 1], xc[:, 1])
    assert rel(d, dc) < 1e-4, rel(d, dc)
    assert rel(r, rc) < 1e-5, rel(r, rc)
    if study == 'none' and steps <= 5:
        gd = golden('cocogen_steps.pt')
        d_ref = gd['p_iterates'][steps - 1] - gd['x0_pred'][:, 0]
        assert rel(d, d_ref) < 1e-3, rel(d, d_ref)
        if steps == gd['p_iterates'].shape[0]:
            assert rel(r, gd['residual_final']) < 1e-5
    if study == 'none' and steps == 200:
        # fp64 oracle: p is rounded to fp32 after each of the 200 steps, and the residual, a small difference of
        # second-difference terms of order K p / h^2, magnifies those roundings (measured 1.0e-4 on an H100)
        xo, ro, _ = O.cocogen_steps(x0.double(), steps)
        d_o = xo[:, 0] - x0.double()[:, 0]
        assert rel(d, d_o) < 1e-3, rel(d, d_o)
        assert rel(r, ro) < 3e-4, rel(r, ro)


def test_zero_steps_is_the_residual(ops, golden):
    res = build()[2]
    x0 = golden('cocogen.pt')['x0_pred'].to(DEV)
    x, r = kernel(res, x0, 0)
    assert torch.equal(x, x0)
    assert torch.equal(r, ops.darcy_residual(x0, res.f_s_flat, *res.geometry))


# ---- predication ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('study', ['none', 'periodic'])
def test_inactive_samples_are_left_untouched(study):
    res = build(study)[2]
    g = torch.Generator().manual_seed(5)
    B = 6
    x0 = torch.randn(B, 2, P, P, generator=g)
    x0[:, 1] = (0.5 * x0[:, 1]).exp()
    r0 = torch.randn(B, P * P, 3, generator=g).to(DEV)
    t = torch.tensor([0, 5, 1, 9, 2, 0], dtype=torch.long, device=DEV)
    x, r = kernel(res, x0, 3, t=t, n_active=2, residual=r0)
    active = (t < 2).cpu()
    x0d = x0.to(DEV)
    for b in range(B):
        if active[b]:
            xc, rc = compose(res, x0d[b:b + 1], 3)
            assert not torch.equal(x[b, 0], x0d[b, 0])
            assert rel(x[b:b + 1] - x0d[b:b + 1], xc - x0d[b:b + 1]) < 1e-4
            assert rel(r[b:b + 1], rc) < 1e-5
        else:
            assert torch.equal(x[b], x0d[b]) and torch.equal(r[b], r0[b]), b
    x, r = kernel(res, x0, 3, t=t, n_active=0, residual=r0)          # nothing active: nothing written
    assert torch.equal(x, x0d) and torch.equal(r, r0)


def test_abi_rejects_bad_arguments():
    from physicsinformeddiffusionmodels_b200._lib import call, stream
    res = build()[2]
    x = torch.zeros(1, 2, P, P, device=DEV)
    r = torch.zeros(1, P * P, 3, device=DEV)
    geo = res._abi_geometry()
    with pytest.raises(Exception):
        call('pidm_darcy_cocogen', x, res.f_s_flat, r, None, 0, -1, 1, P, *geo, stream())
    with pytest.raises(Exception):
        call('pidm_darcy_cocogen', x, res.f_s_flat, r, None, 0, 1, 1, 32, *geo, stream())
    with pytest.raises(Exception):
        call('pidm_darcy_cocogen', x, res.f_s_flat, r, None, 0, 1, 1, P, geo[0], geo[1], 16, stream())


# ---- SampleEngine against the drop-in loop ---------------------------------------------------------------------------
def dropin(diff, res, x_T, zs, monkeypatch, **kw):
    draws = [x_T]
    for z in zs:
        if res.use_ddim_x0:                # the DDIM walk draws (and discards) one noise tensor before the step's z
            draws.append(torch.zeros_like(z))
        draws.append(z)
    it = iter(draws)
    monkeypatch.setattr(torch, 'randn', lambda *a, **k: next(it).clone())
    monkeypatch.setattr(torch, 'randn_like', lambda *a, **k: next(it).clone())
    try:
        (xs, _), aux = diff.p_sample_loop(None, tuple(x_T.shape), save_output=False, surpress_noise=True,
                                          residual_func=res, eval_residuals=True, **kw)
    finally:
        monkeypatch.undo()
    return xs, aux['residual']


def engine(model, diff, res, x_T, zs, use_graph, trajectory=False, **kw):
    from physicsinformeddiffusionmodels_b200.engine import SampleEngine
    eng = SampleEngine(model, diff, res, batch=x_T.shape[0], use_graph=use_graph, external_noise=True,
                       steps_per_graph=1 if trajectory else None, **kw)
    x, r, traj = eng.sample(x_init=x_T, noises=zs, trajectory=trajectory)
    return x.clone(), r.clone(), traj


CASES = {
    'xt_N2': dict(kw=dict(N_correction=2, correction_mode='xt')),
    'x0_N2': dict(kw=dict(N_correction=2, correction_mode='x0')),
    'M5': dict(kw=dict(M_correction=5)),
    'periodic_xt_N3_M3': dict(study='periodic', kw=dict(N_correction=3, M_correction=3, correction_mode='xt')),
    'sample_mode_x0_N2_M2': dict(use_ddim_x0=True, kw=dict(N_correction=2, M_correction=2, correction_mode='x0')),
    'guidance_xt_N2_M1': dict(study='guidance', kw=dict(N_correction=2, M_correction=1, correction_mode='xt')),
}


@pytest.mark.parametrize('case', list(CASES))
def test_engine_matches_dropin(ops, monkeypatch, case):
    c = CASES[case]
    ops.set_precision('fp32')
    model, diff, res = build(c.get('study', 'none'), c.get('use_ddim_x0', False))
    g = torch.Generator().manual_seed(21)
    x_T = torch.randn(2, 2, P, P, generator=g).to(DEV)
    zs = torch.randn(6, 2, 2, P, P, generator=g).to(DEV)
    xs, r_d = dropin(diff, res, x_T, zs, monkeypatch, **c['kw'])
    x_d = xs[-1]
    for use_graph in (False, True):
        x, r, _ = engine(model, diff, res, x_T, zs, use_graph, **c['kw'])
        assert rel(x, x_d) < 1e-4, (use_graph, rel(x, x_d))
        assert rel(r, r_d) < 1e-3, (use_graph, rel(r, r_d))
    # the corrections did something: the uncorrected loop ends elsewhere
    x0, _, _ = engine(model, diff, res, x_T, zs, False)
    assert rel(x0, x_d) > 1e-7


@pytest.mark.parametrize('tag,N,M', [('xt', 2, 3), ('x0', 2, 0)])
def test_engine_and_dropin_match_reference(ops, golden, monkeypatch, tag, N, M):
    ops.set_precision('fp32')
    gd = golden('sample_loop_cocogen.pt')
    model, diff, res = build()
    kw = dict(N_correction=N, M_correction=M, correction_mode=tag)
    x_T, zs = gd['x_T'].to(DEV), gd['noises'].to(DEV)
    xs, r_d = dropin(diff, res, x_T, zs, monkeypatch, **kw)
    assert len(xs) == int(gd[f'{tag}_len'])
    tail = gd[f'{tag}_tail']
    for k in range(tail.shape[0]):
        assert rel(xs[len(xs) - tail.shape[0] + k], tail[k]) < 5e-4, k
    assert rel(r_d, gd[f'{tag}_residual']) < 5e-3         # residual amplifies x0 differences by 1/h^2
    for use_graph in (False, True):
        x, r, _ = engine(model, diff, res, x_T, zs, use_graph, **kw)
        assert rel(x, gd[f'{tag}_x_final']) < 5e-4, (use_graph, rel(x, gd[f'{tag}_x_final']))
        assert rel(r, gd[f'{tag}_residual']) < 5e-3, (use_graph, rel(r, gd[f'{tag}_residual']))
    # trajectory: one entry per step plus ONE for all post-loop corrections
    x, r, traj = engine(model, diff, res, x_T, zs, False, trajectory=True, **kw)
    assert traj.shape[0] == 7 + (1 if M else 0)
    assert torch.equal(traj[-1], x)
    assert rel(traj[6], tail[1]) < 5e-4                    # the state after the t = 0 step


# ---- launches and validation ---------------------------------------------------------------------------------------
@pytest.mark.parametrize('use_graph', [False, True])
def test_engine_launch_count(ops, monkeypatch, use_graph):
    from physicsinformeddiffusionmodels_b200 import _lib
    from physicsinformeddiffusionmodels_b200.engine import SampleEngine
    ops.set_precision('fp32')
    model, diff, res = build()
    calls = []
    real = _lib.call

    def counting(name, *a):
        calls.append(name)
        return real(name, *a)
    monkeypatch.setattr(_lib, 'call', counting)
    x_T = torch.randn(1, 2, P, P, device=DEV)

    def count(**kw):
        calls.clear()
        eng = SampleEngine(model, diff, res, batch=1, use_graph=use_graph, **kw)
        eng.sample(x_init=x_T)
        eng.sample(x_init=x_T)                             # a second loop replays without new launches from Python
        return calls.count('pidm_darcy_cocogen'), eng.k
    n, _ = count()
    assert n == 0
    n, k = count(N_correction=2, correction_mode='xt')
    # eager: every step of both loops; graph: the two warm-up steps and the k captured ones, then replays only
    assert n == (2 + k if use_graph else 2 * diff.n_steps), (n, k)
    n, k = count(N_correction=2, M_correction=4, correction_mode='x0')
    assert n == (2 + k if use_graph else 2 * diff.n_steps) + 2, (n, k)


def test_engine_rejects_bad_corrections():
    from physicsinformeddiffusionmodels_b200.engine import SampleEngine
    from physicsinformeddiffusionmodels_b200.residuals_mechanics_K import ResidualsMechanics
    model, diff, res = build()
    for mode in ('none', 'bad'):
        with pytest.raises(ValueError):
            SampleEngine(model, diff, res, batch=1, N_correction=1, correction_mode=mode)
    with pytest.raises(ValueError):
        SampleEngine(model, diff, res, batch=1, M_correction=-1)
    mech = ResidualsMechanics.__new__(ResidualsMechanics)
    mech.gov_eqs = 'mechanics'
    for kw in (dict(N_correction=1, correction_mode='xt'), dict(M_correction=2)):
        with pytest.raises(ValueError, match='only implemented for the Darcy'):
            SampleEngine(model, diff, mech, batch=1, image_shape=(3, 65, 65), **kw)
