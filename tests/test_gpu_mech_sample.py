"""Conditional sampling of the topology-optimisation model (configs[2]) on the graph-replayed SampleEngine and its
evaluation solve, against the unmodified reference (tests/golden/mechanics_sample_loop.pt, mechanics_eval.pt) and the
fp64 sparse direct solve of oracle/pidm_oracle.py.  The four kernels of these steps (sample input, posterior step, PCG
solve, floating-material flag) are checked per element in tests/test_gpu_mech_eval_census.py."""
import pytest
import torch

import mech_sample_inputs as MI
from checks import rel

pytestmark = pytest.mark.gpu
DEV = 'cuda'
METRICS = ('rel_CE_error_full_batch', 'vf_error_full_batch', 'fm_error_full_batch')


@pytest.fixture(scope='module')
def env():
    from oracle import pidm_oracle as O
    from physicsinformeddiffusionmodels_b200 import ops
    yield dict(O=O, ops=ops)
    ops.set_precision('bf16')


def build(O, mode='mean', n_steps=6, topopt_eval=True):
    from physicsinformeddiffusionmodels_b200.denoising_utils import DenoisingDiffusion
    from physicsinformeddiffusionmodels_b200.residuals_mechanics_K import ResidualsMechanics
    from physicsinformeddiffusionmodels_b200.unet_model import Unet3D
    cfg = O.unet_config(dim=32, channels=10, out_dim=3, sigmoid_last_channel=True)
    model = Unet3D(dim=32, channels=10, out_dim=3, sigmoid_last_channel=True).to(DEV)
    model.load_state_dict(O.make_test_state_dict(cfg, seed=3))
    model.eval()
    res = ResidualsMechanics(model=model, pixels_per_dim=64, pixels_at_boundary=True, no_BC_folder='', device=DEV,
                             topopt_eval=topopt_eval, use_ddim_x0=mode == 'sample', ddim_steps=0)
    return model, DenoisingDiffusion(n_steps, DEV), res


def engine(env, mode, batch=2, **kw):
    from physicsinformeddiffusionmodels_b200.engine import SampleEngine
    model, diff, res = build(env['O'], mode)
    return SampleEngine(model, diff, res, batch=batch, image_shape=(3, 65, 65), **kw)


def cond_input(gd, rows=(0, 1)):
    return tuple(t[list(rows)].to(DEV) for t in MI.inputs(gd))


def draws(gd, mode):
    """(x_T, the posterior z of every step) of the reference run, on the device"""
    x_T, zs, _ = MI.replay_draws(gd, mode)
    return x_T.to(DEV), zs.to(DEV)


def reference_draws(gd, mode):
    """the reference's draws after x_T, in its order (the DDIM walk draws before the posterior z in 'sample' mode)"""
    _, zs, ddim = MI.replay_draws(gd, mode)
    out = []
    for k in range(int(gd['n_steps'])):
        if mode == 'sample':
            out.append(ddim[k])
        out.append(zs[k])
    return [d.to(DEV) for d in out]


def rel_sampled(t, ref):
    """relative error on the elements the fixture keeps (oracle.pidm_oracle.golden_sample)"""
    from oracle import pidm_oracle as O
    return rel(O.golden_sample(t.detach().cpu(), MI.SAMPLE), ref)


def check_metrics_against_reference(aux, gd, mode, x0_eng):
    """Compliance / volume-fraction / floating-material metrics against the reference's (dense LU).  A pixel whose x0
    density sits within 1e-3 of the 0.5 threshold may binarise differently in fp32 on another device: such samples are
    reported by name and their metrics are not compared; every other sample must match."""
    rho_ref = gd[f'{mode}_rho_last']
    rho_eng = x0_eng[:, 2].cpu()
    flips = (rho_eng > 0.5) != (rho_ref > 0.5)
    assert ((rho_ref[flips] - 0.5).abs() < 1e-3).all(), 'a pixel away from the threshold binarised differently'
    compared = 0
    for b in range(rho_ref.shape[0]):
        if flips[b].any():
            print(f'[{mode}] sample {b}: {int(flips[b].sum())} pixel(s) with |rho_ref - 0.5| < 1e-3 binarise '
                  f'differently; its metrics are not compared')
            continue
        compared += 1
        ce, ce_ref = aux['rel_CE_error_full_batch'][b].item(), gd[f'{mode}_rel_CE_error'][b].item()
        assert abs(ce - ce_ref) <= 5e-2 * abs(ce_ref), (mode, b, ce, ce_ref)
        assert abs(aux['vf_error_full_batch'][b].item() - gd[f'{mode}_vf_error'][b].item()) < 1e-6
        assert int(aux['fm_error_full_batch'][b]) == int(gd[f'{mode}_fm_error'][b])
    return compared


@pytest.mark.parametrize('mode', ['mean', 'sample'])
def test_mech_sample_engine_matches_reference(env, golden, monkeypatch, mode):
    """fp32 engine with the reference's draws injected, B = 2, 6 steps, both x0 modes: the samples, the residual terms of
    the last step and the end-to-end evaluation metrics (fused solver) against the unmodified reference."""
    env['ops'].set_precision('fp32')
    gd = golden('mechanics_sample_loop.pt')
    eng = engine(env, mode, use_graph=False)
    it = iter(reference_draws(gd, mode))
    monkeypatch.setattr(torch, 'randn_like', lambda *a, **k: next(it))
    x, aux, traj = eng.sample(x_init=draws(gd, mode)[0], trajectory=True, conditioning_input=cond_input(gd))
    monkeypatch.undo()
    assert next(it, None) is None, 'the engine consumed fewer draws than the reference'
    assert rel_sampled(traj[1], gd[f'{mode}_x_first']) < 1e-4, rel_sampled(traj[1], gd[f'{mode}_x_first'])
    assert rel_sampled(x, gd[f'{mode}_x_final']) < 5e-4, rel_sampled(x, gd[f'{mode}_x_final'])
    assert rel_sampled(eng.x0_pred, gd[f'{mode}_x0_pred_last']) < 5e-4
    assert rel(eng.x0_pred[:, 2], gd[f'{mode}_rho_last']) < 5e-4
    r_err = rel_sampled(aux['residual'], gd[f'{mode}_residual'])
    assert r_err < 5e-3, r_err
    assert rel(aux['optimized_quant'], gd[f'{mode}_compliance']) < 5e-3
    assert rel(aux['inequality_quant'], gd[f'{mode}_inequality']) < 5e-3
    assert all(aux[k].is_cuda for k in ('residual', 'optimized_quant', 'inequality_quant') + METRICS)
    check_metrics_against_reference(aux, gd, mode, eng.x0_pred)


@pytest.mark.parametrize('mode', ['mean', 'sample'])
def test_mech_sample_graph_equals_eager(env, golden, mode):
    """CUDA-graph replay (2 steps per graph) against the eager loop on identical noise; the bf16 path runs and stays
    finite."""
    env['ops'].set_precision('fp32')
    gd = golden('mechanics_sample_loop.pt')
    x_T, z = draws(gd, mode)
    out = {}
    for use_graph in (False, True):
        eng = engine(env, mode, use_graph=use_graph, external_noise=True)
        x, aux, _ = eng.sample(x_init=x_T, noises=z, conditioning_input=cond_input(gd))
        out[use_graph] = (x.clone(), {k: v.clone() for k, v in aux.items()})
    assert eng.k == 2
    (xe, ae), (xg, ag) = out[False], out[True]
    assert rel(xg, xe) < 1e-4, rel(xg, xe)
    for k in ('residual', 'optimized_quant', 'inequality_quant'):
        assert rel(ag[k], ae[k]) < 1e-4, (k, rel(ag[k], ae[k]))
    env['ops'].set_precision('bf16')
    eng = engine(env, mode, use_graph=True)
    x, aux, _ = eng.sample(conditioning_input=cond_input(gd))
    assert torch.isfinite(x).all() and torch.isfinite(aux['residual']).all()
    assert torch.isfinite(aux['optimized_quant']).all() and torch.isfinite(aux['rel_CE_error_full_batch']).all()


def test_mech_sample_conditioning_swap_and_partial_batch(env, golden):
    """A second sample() with other conditioning equals a fresh engine's result (no recapture needed), and a final batch
    smaller than the engine's batch is padded and sliced: it equals an engine built for that batch."""
    env['ops'].set_precision('fp32')
    gd = golden('mechanics_sample_loop.pt')
    x_T, z = draws(gd, 'mean')
    swap = [1, 0]                                        # the two samples' conditioning exchanged
    eng = engine(env, 'mean', use_graph=True, external_noise=True)
    eng.sample(x_init=x_T, noises=z, conditioning_input=cond_input(gd))
    x2, a2, _ = eng.sample(x_init=x_T, noises=z, conditioning_input=cond_input(gd, swap))
    x2, a2 = x2.clone(), {k: v.clone() for k, v in a2.items()}
    fresh = engine(env, 'mean', use_graph=True, external_noise=True)
    xf, af, _ = fresh.sample(x_init=x_T, noises=z, conditioning_input=cond_input(gd, swap))
    # two engines agree to the run-to-run spread of the network's fp32 atomic reductions, not bit for bit
    assert rel(x2, xf) < 1e-5, rel(x2, xf)
    for k in ('residual', 'optimized_quant', 'rel_CE_error_full_batch'):
        assert rel(a2[k], af[k]) < 1e-5, (k, rel(a2[k], af[k]))
    # partial batch: 1 sample through the B = 2 engine against a B = 1 engine
    xp, ap, _ = eng.sample(x_init=x_T[1:], noises=z[:, 1:], conditioning_input=cond_input(gd, [1]))
    xp, ap = xp.clone(), {k: v.clone() for k, v in ap.items()}
    one = engine(env, 'mean', batch=1, use_graph=True, external_noise=True)
    x1, a1, _ = one.sample(x_init=x_T[1:], noises=z[:, 1:], conditioning_input=cond_input(gd, [1]))
    assert xp.shape == (1, 3, 65, 65) and all(v.shape[0] == 1 for v in ap.values())
    assert rel(xp, x1) < 1e-4, rel(xp, x1)
    for k in ('residual', 'optimized_quant', 'inequality_quant'):
        assert rel(ap[k], a1[k]) < 1e-4, (k, rel(ap[k], a1[k]))
    # and the same sample inside the full batch (samples are independent)
    xfull = eng.sample(x_init=x_T, noises=z, conditioning_input=cond_input(gd))[0]
    assert rel(xp, xfull[1:]) < 1e-4, rel(xp, xfull[1:])


def test_mech_sample_and_fused_solve_do_not_sync(env, golden):
    """sample() (graph replay, metrics with the fused solver included) and fem_solve_fused issue no host synchronisation."""
    env['ops'].set_precision('bf16')
    gd = golden('mechanics_sample_loop.pt')
    for mode in ('mean', 'sample'):
        eng = engine(env, mode, use_graph=True)
        ci = cond_input(gd)
        rho = gd['solution'][:, 2, :-1, :-1].to(DEV)
        eng.sample(conditioning_input=ci)                 # capture outside the checked region
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode('error')
        try:
            x, aux, _ = eng.sample(conditioning_input=ci)
            u, iters, rr = eng.residuals.fem_solve_fused(rho, ci[1])
        finally:
            torch.cuda.set_sync_debug_mode(0)
        assert set(METRICS) <= set(aux)
        assert (iters.cpu() < 6000).all() and torch.isfinite(u).all()


# ---- the fused solver ------------------------------------------------------------------------------------------------

def test_fused_solver_against_sparse_direct_solve(env, golden):
    """fem_solve_fused against the fp64 sparse direct solve on the mechanics_eval.pt designs (its data density and the
    binarised x0 of its golden) and on 12 binarised designs under four support / load cases, next to fem_solve on the
    same systems: every sample converges and the fused solve is at least as accurate as fem_solve."""
    from physicsinformeddiffusionmodels_b200.residuals_mechanics_K import ResidualsMechanics, compute_fm, floating_material
    ev = golden('mechanics_eval.pt')
    res = ResidualsMechanics(model=None, pixels_per_dim=64, pixels_at_boundary=True, no_BC_folder='', device=DEV)
    x0 = ev['x0_pred'][:, 2]
    rho_bin, bcs = MI.binarised_designs(12, seed=5)
    cases = [('eval_rho_simp', ev['solution'][:, 2, :-1, :-1], ev['bcs']),
             ('eval_x0_binarised', torch.where(x0 > 0.5, torch.ones_like(x0), torch.full_like(x0, 1e-3)), ev['bcs']),
             ('binarised', rho_bin, bcs)]
    KE = res.KE.double().cpu()
    report = {}
    for name, rho, bc in cases:
        u_ref = env['O'].fem_solve(rho, bc, KE)
        rho_d, bc_d = rho.contiguous().to(DEV), bc.contiguous().to(DEV)
        u_t = res.fem_solve(rho_d, bc_d)
        u_f, iters, relres = res.fem_solve_fused(rho_d, bc_d)
        iters, relres = iters.cpu(), relres.cpu()
        assert (iters < 6000).all() and (relres < 1e-6).all(), (name, iters, relres)
        for b in range(rho.shape[0]):
            e_t, e_f = rel(u_t[b], u_ref[b]), rel(u_f[b], u_ref[b])
            report[f'{name}[{b}]'] = (int(iters[b]), e_f, e_t)
            assert e_f <= e_t, (name, b, e_f, e_t)
        if name == 'binarised':
            assert len(set(iters.tolist())) > 1, iters          # samples stop on their own
            assert torch.equal(floating_material(rho_d).cpu(), compute_fm(rho_d).long())
    for k, v in report.items():
        print(f'{k}: iterations {v[0]}, rel. error fused {v[1]:.3e}, torch {v[2]:.3e}')


def test_fused_metrics_on_reference_golden(env, golden):
    """topopt_metrics with the fused solver on mechanics_eval.pt: rel_CE_error within the existing 5e-2, the volume
    fraction and floating-material errors equal to the torch path's and the reference's."""
    from physicsinformeddiffusionmodels_b200.residuals_mechanics_K import ResidualsMechanics
    gd = golden('mechanics_eval.pt')
    res = ResidualsMechanics(model=None, pixels_per_dim=64, pixels_at_boundary=True, no_BC_folder='', device=DEV,
                             topopt_eval=True)
    rho = gd['x0_pred'][:, 2].contiguous().to(DEV)
    args = (rho, gd['bcs'].to(DEV), gd['vf'].to(DEV), gd['solution'].to(DEV))
    fused, torch_ = res.topopt_metrics(*args, solver='fused'), res.topopt_metrics(*args)
    assert torch.allclose(fused['rel_CE_error_full_batch'].cpu(), gd['rel_CE_error'], rtol=5e-2)
    assert torch.equal(fused['vf_error_full_batch'], torch_['vf_error_full_batch'])
    assert torch.allclose(fused['vf_error_full_batch'].cpu(), gd['vf_error'], atol=1e-6)
    assert torch.equal(fused['fm_error_full_batch'].cpu(), gd['fm_error'].long())
    # a solution that does not solve its system: the torch path raises, the fused path marks the batch NaN
    bad = gd['solution'].clone()
    bad[:, :2] *= 1.5
    with pytest.raises(AssertionError):
        res.topopt_metrics(*args[:3], bad.to(DEV))
    assert torch.isnan(res.topopt_metrics(*args[:3], bad.to(DEV), solver='fused')['rel_CE_error_full_batch']).all()
