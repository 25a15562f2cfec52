"""The CPU oracle (oracle/pidm_oracle.py) against fixtures produced by the UNMODIFIED reference
(oracle/make_golden.py), plus analytic known-answer tests (SURVEY.md section 4).  The training loss, the sampling loop
and the CoCoGen correction are checked for each study option (tests/study.py) that has a fixture."""
import math
import os

import pytest
import torch

import study
from checks import rel
from oracle import make_golden
from oracle import pidm_oracle as O


def oracle_study(name):
    """(config, seeded weights, periodic flag) of the oracle for a study of study.STUDIES"""
    opts = study.STUDIES[name]
    padding_mode = opts.get('padding_mode', 'zeros')
    return study.config(padding_mode), study.state_dict(padding_mode), opts.get('bcs') == 'periodic'


def test_every_golden_file_has_a_recipe():
    """The recipe table of oracle/make_golden.py (importable without a reference checkout) names every file under
    tests/golden exactly once, so no fixture exists that the recipes cannot rewrite."""
    files = [f for _, names in make_golden.RECIPES.values() for f in names]
    assert len(files) == len(set(files))
    assert sorted(files) == sorted(os.listdir(os.path.join(os.path.dirname(__file__), 'golden')))


@pytest.mark.parametrize('n', [100, 250])
def test_schedule_tables_match_reference(golden, n):
    ref = golden(f'schedule_{n}.pt')
    mine = O.diffusion_tables(n)
    assert list(mine.keys()) == list(ref.keys())
    for k in ref:
        assert torch.allclose(mine[k], ref[k], rtol=1e-6, atol=1e-7, equal_nan=True), k


def test_schedule_spot_values():
    d = O.diffusion_tables(100)                       # SURVEY.md section 8a row A1
    assert abs(d['betas'][0].item() - 6.3127e-4) < 1e-7
    assert abs(d['betas'][99].item() - 0.999) < 1e-6
    assert abs(d['posterior_variance_clipped'][0].item() - 4.0349e-4) < 1e-7
    assert d['posterior_variance_clipped'][0] == d['posterior_variance_clipped'][1]
    assert d['p2_loss_weight'][0].item() == 5.0


def test_unet_forward_matches_reference(golden):
    gd = golden('unet_darcy_fwd.pt')
    cfg = O.unet_config(dim=32, channels=2)
    sd = O.make_test_state_dict(cfg, 0)
    assert len(sd) == 317 and sum(v.numel() for v in sd.values()) == 10386514
    with torch.no_grad():
        y, taps = O.unet_forward(sd, cfg, gd['x'], gd['t'], return_taps=True)
        y2 = O.unet_forward(sd, cfg, gd['x'].permute(0, 2, 3, 1).reshape(2, 4096, 2), gd['t'])
    assert torch.equal(y, y2)
    for k in ('init_conv', 'time_emb', 'downs.0.0', 'downs.0.2', 'mid_attn', 'ups.0'):
        assert rel(O.golden_sample(taps[k]), gd['tap_' + k]) < 2e-5, k
    assert rel(y, gd['y']) < 5e-5


def test_darcy_residual_matches_reference(golden):
    gd = golden('darcy_residual.pt')
    assert torch.equal(O.darcy_source(64), gd['f_s'])
    r = O.darcy_residual(gd['x0_pred'])
    assert rel(r, gd['residual']) < 1e-5
    x = gd['x0_pred'].clone().requires_grad_(True)
    (O.darcy_residual(x) * gd['cotangent']).sum().backward()
    assert rel(x.grad, gd['grad_x0_pred']) < 1e-5


def test_darcy_source_layout():
    f = O.darcy_source(64)
    assert (f != 0).sum() == 128 and (f[:8, :8] == 10).all() and (f[56:, 56:] == -10).all()


def test_darcy_residual_manufactured_quadratic():
    """p = x^2 + xy + y^2, K = 1 + x + 2y on x=i/63, y=(63-j)/63: second-order FD (one-sided at the
    boundary) is exact on quadratics, so eq_0 + f_s = -(K(p_xx+p_yy) + K_x p_x + K_y p_y) in closed form."""
    i = torch.arange(64, dtype=torch.float64) / 63
    X, Yr = torch.meshgrid(i, i, indexing='ij')
    Y = 1.0 - Yr
    p = X * X + X * Y + Y * Y
    K = 1 + X + 2 * Y
    r = O.darcy_residual(torch.stack([p, K])[None]).reshape(64, 64, 3)
    exact = -(K * 4.0 + 1.0 * (2 * X + Y) + 2.0 * (X + 2 * Y)) - O.darcy_source(64, dtype=torch.float64)
    assert (r[..., 0] - exact).abs().max() < 1e-8
    px, py = 2 * X + Y, X + 2 * Y
    assert (r[0, :, 1] + px[0]).abs().max() < 1e-9 and (r[-1, :, 1] - px[-1]).abs().max() < 1e-9
    # reverse_d1: stored column derivative is d/d(col*h1) with h1<0 == d/dy
    assert (r[:, 0, 2] - py[:, 0]).abs().max() < 1e-9 and (r[:, -1, 2] + py[:, -1]).abs().max() < 1e-9
    assert r[1:-1, :, 1].abs().max() == 0 and r[:, 1:-1, 2].abs().max() == 0


# golden: (study, gradient tolerance, extra assertions).  A fixture with 'null_mask' is a guidance step with that
# classifier-free mask; one with 'grad_sample' stores its gradients sampled with that n.
LOSS_ROWS = {
    'darcy_loss_mean': ('none', 5e-4, dict(dead='params_without_grad.txt', dead_numel=1464432)),   # SURVEY.md 3.2
    'darcy_loss_periodic': ('periodic', 5e-4, {}),
    'darcy_loss_circular': ('circular', 5e-4, {}),
    'darcy_guidance_step': ('guidance', 1e-3, dict(keys=('grad_emb_conv.0.weight', 'grad_combine_conv.bias'))),
}


@pytest.mark.parametrize('name', list(LOSS_ROWS))
def test_training_loss_and_grads_match_reference(golden, name):
    s, tol_grad, extra = LOSS_ROWS[name]
    gd = golden(name + '.pt')
    cfg, sd0, periodic = oracle_study(s)
    sd = {k: v.clone().requires_grad_(v.is_floating_point() and 'freqs' not in k) for k, v in sd0.items()}
    mask = gd.get('null_mask')
    if mask is not None:
        assert 0 < int(mask.sum()) < len(mask)                       # both branches of the mask are exercised
    loss, aux = O.darcy_training_loss(sd, cfg, gd['x0'], gd['t'], gd['noise'], O.diffusion_tables(100),
                                      guidance_null_mask=mask, periodic=periodic)
    assert abs(loss.item() / gd['loss'].item() - 1) < 2e-5
    assert abs(aux['data'].item() / gd['data_loss'].item() - 1) < 2e-5
    assert abs(aux['residual_abs'].item() / gd['residual_abs'].item() - 1) < 2e-5
    loss.backward()
    n = {'n': int(gd['grad_sample'])} if 'grad_sample' in gd else {}
    worst = {k: rel(O.golden_sample(sd[k[5:]].grad, **n), v) for k, v in gd.items()
             if k.startswith('grad_') and k not in ('grad_norm', 'grad_sample')}
    assert all(k in worst for k in extra.get('keys', ())), sorted(worst)
    assert max(worst.values()) < tol_grad, sorted(worst.items(), key=lambda kv: -kv[1])[:5]
    gn = math.sqrt(sum((p.grad.double() ** 2).sum().item() for p in sd.values() if p.grad is not None))
    assert abs(gn / gd['grad_norm'].item() - 1) < 1e-4
    if 'dead' in extra:
        dead = sorted(k for k, p in sd.items() if p.requires_grad and p.grad is None)
        with open(os.path.join(os.path.dirname(__file__), 'golden', extra['dead'])) as f:
            ref_dead = [k for k in f.read().split() if not k.endswith('rotary_emb.freqs')]   # frozen, never trainable
        assert dead == ref_dead
        assert sum(sd[k].numel() for k in dead) == extra['dead_numel']


def test_sample_mode_loss_matches_reference(golden):
    gd = golden('darcy_loss_sample.pt')
    cfg = O.unet_config(dim=32, channels=2)
    sd = {k: v.clone().requires_grad_('freqs' not in k) for k, v in O.make_test_state_dict(cfg, 0).items()}
    tables = O.diffusion_tables(100)
    loss, aux = O.darcy_training_loss(sd, cfg, gd['x0'], gd['t'], gd['noise'], tables, use_ddim_x0=True)
    assert abs(loss.item() / gd['loss'].item() - 1) < 5e-5
    loss.backward()
    assert rel(sd['final_conv.1.weight'].grad, gd['grad_final_w']) < 5e-4
    assert rel(sd['init_conv.weight'].grad, gd['grad_init_w']) < 5e-4


@pytest.mark.parametrize('ddim_steps', [1, 3])
def test_ddim_walk_matches_reference(golden, ddim_steps):
    """the oracle's DDIM walk (ddim_sample_x0, eta = 0) at ddim_steps > 0 and per-sample t whose grids repeat points"""
    gd = golden('darcy_loss_sample.pt')
    xt = make_golden.ddim_walk_input()
    assert torch.equal(xt.double().sum(), gd['walk_x_t_checksum'])
    cfg = O.unet_config(dim=32, channels=2)
    with torch.no_grad():
        cur_x, model_out = O.ddim_x0(O.make_test_state_dict(cfg, 0), cfg, xt, gd['walk_t'], O.diffusion_tables(100),
                                     ddim_steps=ddim_steps)
    n = make_golden.DDIM_WALK['sample']
    assert rel(O.golden_sample(model_out, n), gd[f'walk_model_out_{ddim_steps}']) < 1e-5
    assert rel(O.golden_sample(cur_x, n), gd[f'walk_cur_x_{ddim_steps}']) < 1e-5


@pytest.mark.parametrize('name,s', [('sample_loop_6', 'none'), ('sample_loop_periodic', 'periodic'),
                                    ('sample_loop_circular', 'circular')])
def test_sampling_loop_matches_reference(golden, name, s):
    gd = golden(name + '.pt')
    cfg, sd, periodic = oracle_study(s)
    with torch.no_grad():
        x, r = O.p_sample_loop(sd, cfg, gd['x_T'], list(gd['noises']), O.diffusion_tables(6), 6, periodic=periodic)
    assert rel(x, gd['x_final']) < 2e-4
    assert rel(r, gd['residual']) < 2e-3          # residual amplifies x0 differences by 1/h^2


def replay_draws_100(gd):
    """the 101 draws of the 100-step reference run (x_T, then one z per step), regenerated from the stored seed"""
    torch.manual_seed(int(gd['seed']))
    draws = torch.stack([torch.randn(1, 2, 64, 64) for _ in range(101)])
    assert torch.equal(draws.double().sum(dim=(1, 2, 3, 4)), gd['noise_checksum']), \
        'CPU generator does not reproduce the draws of the golden run (torch version mismatch?)'
    return draws


def test_sampling_loop_100_steps_matches_reference(golden):
    """The reference's default 100-step ancestral loop at B=1 (denoising_utils.py:494-545): errors of the x0
    estimate are re-injected at every step, so this is the long-horizon check of the sampler algebra."""
    gd = golden('sample_loop_100.pt')
    cfg = O.unet_config(dim=32, channels=2)
    sd = O.make_test_state_dict(cfg, 0)
    tables = O.diffusion_tables(100)
    draws = replay_draws_100(gd)
    with torch.no_grad():
        x, r = O.p_sample_loop(sd, cfg, draws[0], list(draws[1:]), tables, 100)
    assert rel(x, gd['x_final']) < 1e-3, rel(x, gd['x_final'])
    assert abs(r.abs().mean().item() / gd['residual_abs_mean'].item() - 1) < 1e-2


def test_q4_stiffness_known_answer(golden):
    """Closed-form 99-line-topopt KE (E=1, nu=0.3) == the Gauss-integrated Q4 used by the reference run."""
    KE = O.q4_plane_stress_stiffness()
    assert torch.allclose(KE, KE.T) and KE.sum(dim=1).abs().max() < 1.0     # symmetric
    assert abs(KE[0, 0].item() - (0.5 - 0.05) / 0.91) < 1e-12
    assert torch.allclose(KE.float(), golden('mechanics_residual.pt')['KE'], atol=1e-6)
    # rigid-body translations produce no force
    tx = torch.tensor([1., 0, 1, 0, 1, 0, 1, 0], dtype=torch.float64)
    assert (KE @ tx).abs().max() < 1e-12


def test_mechanics_residual_matches_reference(golden):
    gd = golden('mechanics_residual.pt')
    x = gd['x0_pred'].clone().requires_grad_(True)
    r, c, q = O.mechanics_residual(x, gd['bcs'], gd['vf'])
    assert rel(r, gd['residual']) < 2e-5
    assert rel(c, gd['compliance']) < 2e-5
    assert torch.allclose(q, gd['inequality'], atol=1e-6)
    ((r * gd['cotangent']).sum() + 0.3 * c.sum() + 2.0 * q.sum()).backward()
    assert rel(x.grad, gd['grad_x0_pred']) < 5e-5


def test_mechanics_training_loss_matches_reference(golden):
    """The reference's own model_estimation_loss for gov_eqs='mechanics' (dense 8450 x 8450 assembly, B = 2, all four loss
    terms on; c_ineq > 0 pins the [B,1] x [B] broadcast of denoising_utils.py:679,694) vs the matrix-free oracle."""
    gd = golden('mechanics_loss.pt')
    cfg = O.unet_config(dim=32, channels=10, out_dim=3, sigmoid_last_channel=True)
    sd = O.make_test_state_dict(cfg, 3)
    sdr = {k: v.clone().requires_grad_(v.is_floating_point() and 'freqs' not in k) for k, v in sd.items()}
    c_data, c_res, c_ineq, lam = gd['coefs'].tolist()
    loss, aux = O.mechanics_training_loss(sdr, cfg, gd['input'], gd['t'], gd['noise'], O.diffusion_tables(100), c_data, c_res,
                                          c_ineq, lam)
    assert abs(loss.item() / gd['loss'].item() - 1) < 2e-5
    assert abs(aux['data'].item() / gd['data_loss'].item() - 1) < 2e-5
    assert abs(aux['residual_abs'].item() / gd['residual_abs'].item() - 1) < 2e-5
    assert abs(aux['inequality'].item() - gd['inequality'].item()) < 1e-6
    assert abs(aux['compliance'].item() / gd['compliance'].item() - 1) < 2e-5
    loss.backward()
    assert rel(sdr['final_conv.1.weight'].grad, gd['grad_final_w']) < 1e-4
    assert rel(sdr['init_conv.weight'].grad, gd['grad_init_w']) < 1e-4
    assert rel(sdr['downs.1.0.block1.proj.weight'].grad, gd['grad_mid_w']) < 1e-4


@pytest.mark.parametrize('tag,mode,ddim', [('x0_mean', 'x0', False), ('x0_sample', 'x0', True), ('eps_sample', 'eps', True)])
def test_toy_loss_matches_reference(golden, tag, mode, ddim):
    """configs[0] (main_toy.py): the toy study's PIDM loss through the unmodified reference module vs the oracle."""
    gd = golden('toy.pt')
    sd = {k[3:]: v.clone().requires_grad_(True) for k, v in gd.items() if k.startswith('sd_')}
    tables = O.diffusion_tables(100)
    loss, tracked = O.toy_training_loss(sd, gd['x0'], gd['t'], gd['noise'], tables, mode, ddim, 1.0, 0.005, 0.3, 0.01)
    assert abs(loss.item() / gd[tag + '_loss'].item() - 1) < 1e-5
    for a, b in zip(tracked, gd[tag + '_tracked'].tolist()):
        assert abs(a.item() - b) < 1e-5 * max(1.0, abs(b))
    loss.backward()
    assert rel(sd['lin3.weight'].grad, gd[tag + '_grad_lin3']) < 1e-4
    assert rel(sd['lin1.lin.weight'].grad, gd[tag + '_grad_lin1']) < 1e-4
    assert rel(sd['lin2.embed.weight'].grad, gd[tag + '_grad_embed2']) < 1e-4


@pytest.mark.parametrize('name,s', [('cocogen', 'none'), ('cocogen_periodic', 'periodic')])
def test_cocogen_correction_matches_reference(golden, name, s):
    """SURVEY 8f.3: ResidualsDarcy.residual_correction through the reference's vmap(jacfwd) Jacobian vs the oracle."""
    gd = golden(name + '.pt')
    xc, rc = O.cocogen_correction(gd['x0_pred'], periodic=oracle_study(s)[2])
    # the correction itself is tiny (step 1e-6 / max|J|): compare the CHANGE, not the field
    d_ref = gd['corrected'] - gd['x0_pred']
    assert d_ref.abs().max() > 0
    assert rel(xc - gd['x0_pred'], d_ref) < 1e-3
    assert torch.equal(xc[:, 1], gd['x0_pred'][:, 1])                 # K is never touched
    assert rel(rc, gd['residual_corrected']) < 1e-5


def test_residual_gradient_guidance_matches_reference(golden):
    """SURVEY 8f.3: the guidance branch (cond = d mean|r(x_t)| / d x_t -> emb_conv -> combine_conv, classifier-free mask;
    residuals_darcy.py:114-126, unet_model.py:530-540,585-603) through the unmodified reference vs the oracle: training
    loss + gradients of the guidance-only layers, the forced-null-mask variant, and the guidance-scale-3 sample path."""
    gd = golden('darcy_guidance.pt')
    cfg = O.unet_config(dim=32, channels=2)
    sd = O.make_test_state_dict(cfg, 0)
    sdr = {k: v.clone().requires_grad_('freqs' not in k) for k, v in sd.items()}
    tables = O.diffusion_tables(100)
    loss, _ = O.darcy_training_loss(sdr, cfg, gd['x0'], gd['t'], gd['noise'], tables, guidance_null_mask=gd['null_mask'])
    assert abs(loss.item() / gd['loss'].item() - 1) < 2e-5
    loss.backward()
    assert rel(sdr['emb_conv.0.weight'].grad, gd['grad_emb0']) < 1e-4
    assert rel(sdr['combine_conv.weight'].grad, gd['grad_combine']) < 1e-4
    assert rel(sdr['final_conv.1.weight'].grad, gd['grad_final_w']) < 1e-4
    loss_f, _ = O.darcy_training_loss(sd, cfg, gd['x0'], gd['t'], gd['noise'], tables, guidance_null_mask=gd['forced_mask'])
    assert abs(loss_f.item() / gd['loss_forced'].item() - 1) < 2e-5
    with torch.no_grad():
        c = O.darcy_residual_gradient(gd['sample_in'])
        B = c.shape[0]
        lo = O.unet_forward(sd, cfg, gd['sample_in'], gd['t'], cond=c, null_mask=torch.zeros(B, dtype=torch.bool))
        nu = O.unet_forward(sd, cfg, gd['sample_in'], gd['t'], cond=c, null_mask=torch.ones(B, dtype=torch.bool))
    assert rel(nu + (lo - nu) * 3.0, gd['sample_x0']) < 2e-5
