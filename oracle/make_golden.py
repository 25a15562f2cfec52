"""Golden-vector generator.  TEST INFRASTRUCTURE ONLY; runs on the CPU, not on the GPU box.

Imports the UNMODIFIED reference modules from a checkout of the original project (path in PIDM_REFERENCE) through
the import shims in oracle/ref_shims/ (SURVEY.md section 8c), runs them on seeded CPU inputs and writes small fixtures
to tests/golden/.  The weights are not stored: both sides rebuild them with
oracle.pidm_oracle.make_test_state_dict(cfg, seed).  Large tensors are stored as oracle.pidm_oracle.golden_sample().
RECIPES maps every file under tests/golden/ to the recipe family that writes it.

    PIDM_REFERENCE=<checkout of the original project> python oracle/make_golden.py [--out DIR] [FAMILY ...]

With no FAMILY every fixture is written; --out defaults to tests/golden.  Recipes whose inputs come from another fixture
(darcy_residual.pt, cocogen.pt, unet_darcy_fwd.pt) read them from the committed tests/golden/.
"""
import argparse
import contextlib
import importlib.util
import os
import sys
import tempfile
import types
import warnings

import numpy as np
import torch
from torch.nn.functional import pad as F_pad

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(ROOT, 'tests', 'golden')


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


O = _load('pidm_oracle', os.path.join(HERE, 'pidm_oracle.py'))


def import_reference():
    """Make `src` the reference checkout named by PIDM_REFERENCE and the absent third-party modules the shims.  The
    repository root must NOT be importable here: its `src/` drop-in package (a regular package) would shadow the
    reference's `src/` (a namespace package) regardless of path order."""
    ref = os.environ['PIDM_REFERENCE']
    sys.path = [p for p in sys.path if os.path.abspath(p or '.') != ROOT]
    sys.path.insert(0, os.path.join(HERE, 'ref_shims'))
    sys.path.insert(0, ref)
    warnings.filterwarnings('ignore')
    import findiff
    import src.unet_model
    assert os.path.abspath(src.unet_model.__file__).startswith(os.path.abspath(ref)), src.unet_model.__file__
    assert os.path.abspath(findiff.__file__).startswith(os.path.join(HERE, 'ref_shims')), findiff.__file__


def save(out, name, obj):
    os.makedirs(out, exist_ok=True)
    torch.save(obj, os.path.join(out, name))
    n = sum(v.numel() * v.element_size() for v in obj.values() if torch.is_tensor(v))
    print(f'wrote {name}: {n / 1024:.1f} KiB')


def save_names(out, name, names):
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, name), 'w') as f:
        f.write('\n'.join(names) + '\n')


def load_golden(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=True)


def smooth_fields(B, seed, P=64):
    """Smooth positive-K / smooth-p fields (a few Fourier modes) used as x0 / x0_pred."""
    g = torch.Generator().manual_seed(seed)
    i = torch.arange(P, dtype=torch.float32) / (P - 1)
    X, Y = torch.meshgrid(i, i, indexing='ij')
    out = torch.zeros(B, 2, P, P)
    for b in range(B):
        for c in range(2):
            f = torch.zeros(P, P)
            for _ in range(4):
                a, kx, ky, ph = torch.randn(1, generator=g), *torch.randint(1, 4, (2,), generator=g), torch.rand(1, generator=g)
                f += a * torch.sin(np.pi * kx * X + ph) * torch.cos(np.pi * ky * Y)
            out[b, c] = f if c == 0 else torch.exp(0.5 * f)
    return out


@contextlib.contextmanager
def mesh_folder(nel=64):
    """A temporary folder with the unit-square 65x65-node / 64x64-element mesh files in the solidspy text format read
    at residuals_mechanics_K.py:43-49; convention documented in oracle.pidm_oracle.mechanics_mesh."""
    with tempfile.TemporaryDirectory() as folder:
        nn_ = nel + 1
        rows, cols = np.meshgrid(np.arange(nn_), np.arange(nn_), indexing='ij')
        ids = (rows * nn_ + cols).reshape(-1)
        nodes = np.stack([ids, cols.reshape(-1) / nel, (nel - rows.reshape(-1)) / nel, 0 * ids, 0 * ids], axis=1)
        np.savetxt(os.path.join(folder, 'nodes.txt'), nodes, fmt='%d %.8f %.8f %d %d')
        er, ec = np.meshgrid(np.arange(nel), np.arange(nel), indexing='ij')
        er, ec = er.reshape(-1), ec.reshape(-1)
        eles = np.stack([er * nel + ec, 0 * er + 1, 0 * er, (er + 1) * nn_ + ec, (er + 1) * nn_ + ec + 1,
                         er * nn_ + ec + 1, er * nn_ + ec], axis=1)
        np.savetxt(os.path.join(folder, 'eles.txt'), eles, fmt='%d')
        np.savetxt(os.path.join(folder, 'mater.txt'), np.array([[1.0, 0.3]]), fmt='%.4f')
        np.savetxt(os.path.join(folder, 'loads.txt'), np.array([[0, 0.0, 0.0]]), fmt='%d %.2f %.2f')
        yield folder + '/'


# ---- the reference objects of the recipes ---------------------------------------------------------------------------

MECHANICS_CFG = dict(channels=10, out_dim=3, sigmoid_last_channel=True)


def reference_unet(seed, **cfg):
    """the reference Unet3D(dim=32, **cfg) with the weights make_test_state_dict(unet_config(dim=32, **cfg), seed)"""
    from src.unet_model import Unet3D
    model = Unet3D(dim=32, **cfg)
    model.load_state_dict(O.make_test_state_dict(O.unet_config(dim=32, **cfg), seed=seed), strict=True)
    return model


def darcy_model(padding_mode='zeros'):
    return reference_unet(0, channels=2, padding_mode=padding_mode)


def darcy_residuals(model, bcs='none', **kw):
    from src.residuals_darcy import ResidualsDarcy
    return ResidualsDarcy(model=model, fd_acc=2, pixels_per_dim=64, pixels_at_boundary=True, reverse_d1=True,
                          device='cpu', bcs=bcs, domain_length=1., **kw)


def mechanics_residuals(folder, model=None, topopt_eval=False, **kw):
    from src.residuals_mechanics_K import ResidualsMechanics
    return ResidualsMechanics(model=model, pixels_per_dim=64, pixels_at_boundary=True, no_BC_folder=folder,
                              device='cpu', topopt_eval=topopt_eval, **kw)


def diffusion(n_steps, **kw):
    from src.denoising_utils import DenoisingDiffusion
    return DenoisingDiffusion(n_steps, 'cpu', **kw)


def loss_draws(seed, x0, mask=False):
    """the training loss's draws after torch.manual_seed(seed), in order: t and eps (denoising_utils.py:625,636), then
    with `mask` the classifier-free mask of the guidance branch (unet_model.py:63-69)"""
    torch.manual_seed(seed)
    B = x0.shape[0]
    t = torch.randint(0, 100, size=(B,))
    e = torch.randn_like(x0)
    if not mask:
        return t, e
    return t, e, torch.zeros((B,)).float().uniform_(0, 1) < 0.1


def darcy_loss(x0, res, seed, backward=True):
    """(loss, data loss, mean |r|) of model_estimation_loss with the Darcy study's coefficients after
    torch.manual_seed(seed); with `backward` the model's .grad are the gradients of this loss"""
    diff = diffusion(100, residual_grad_guidance=res.residual_grad_guidance)
    torch.manual_seed(seed)
    loss, data_l, res_l, _, _ = diff.model_estimation_loss(x0, residual_func=res, c_data=1., c_residual=1e-3, c_ineq=0.,
                                                           lambda_opt=0.)
    if backward:
        res.model.zero_grad()
        loss.backward()
    return loss, data_l, res_l


def grad_norm(model):
    return torch.sqrt(sum((p.grad.double() ** 2).sum() for p in model.parameters() if p.grad is not None)).float()


# ---- recipes shared by several families -----------------------------------------------------------------------------

def forward_fixture(out, name, model, x, t, time_emb=False):
    """forward output and golden samples of the tapped activations.  With `time_emb` the time embedding is tapped too,
    and the [B, P*P, C] input layout must give the same output (the taps are those of that second call)."""
    taps = {}

    def hook(tap, squeeze=True):
        def f(mod, inp, o):
            taps[tap] = (o.detach().squeeze(2) if squeeze else o.detach()).clone()
        return f
    mods = {'init_conv': model.init_conv, 'downs.0.0': model.downs[0][0], 'downs.0.2': model.downs[0][2],
            'mid_attn': model.mid_spatial_attn, 'ups.0': model.ups[0][3]}
    hs = [m.register_forward_hook(hook(k)) for k, m in mods.items()]
    if time_emb:
        hs.append(model.time_mlp.register_forward_hook(hook('time_emb', squeeze=False)))
    model.eval()
    with torch.no_grad():
        y = model(x, t)
        if time_emb:
            assert torch.equal(y, model(x.permute(0, 2, 3, 1).reshape(2, 4096, 2), t))
    for h in hs:
        h.remove()
    save(out, name, dict(x=x, t=t, y=y, **{'tap_' + k: O.golden_sample(v) for k, v in taps.items()}))


def residual_vjp(res, x0p, g):
    """(residual, cotangent drawn from g, VJP of the residual with that cotangent) of the fields x0p"""
    r = res.compute_residual(x0p, pass_through=True)['residual']
    xg = x0p.clone().requires_grad_(True)
    rg = res.compute_residual(xg, pass_through=True)['residual']
    wgt = torch.randn(rg.shape, generator=g)
    (rg * wgt).sum().backward()
    return r.detach(), wgt, xg.grad.clone()


def cocogen_fixture(out, name, res, x0p):
    """one residual_correction (8f.3, through the reference's vmap(jacfwd) Jacobian) of the first two fields of x0p"""
    xc = x0p[:2].clone()
    xin = xc.permute(0, 2, 3, 1).reshape(2, 4096, 2).clone()
    x_corr, r_corr = res.residual_correction(xin)
    save(out, name, dict(x0_pred=xc, corrected=x_corr.reshape(2, 64, 64, 2).permute(0, 3, 1, 2).contiguous().clone(),
                         residual_corrected=r_corr.detach().clone()))


def loss_fixture(out, name, model, res, keys, nograd_name=None):
    """mean-mode training loss (A3) on smooth_fields(2, seed=9) with the seed-123 draws: the loss terms, golden samples
    of the gradients of the parameters `keys` and the global gradient norm; with `nograd_name` also the list of the
    parameters whose .grad stays None"""
    model.train()
    x0 = smooth_fields(2, seed=9)
    loss, data_l, res_l = darcy_loss(x0, res, 123)
    t, e = loss_draws(123, x0)
    named = dict(model.named_parameters())
    grads = {'grad_' + k: O.golden_sample(named[k].grad) for k in keys}
    save(out, name, dict(x0=x0, t=t, noise=e, loss=loss.detach(), data_loss=torch.tensor(data_l),
                         residual_abs=torch.tensor(res_l), grad_norm=grad_norm(model), **grads))
    if nograd_name:
        save_names(out, nograd_name, sorted(k for k, p in named.items() if p.grad is None))


def guidance_fixture(out, name, model, bcs, grads, forced_mask=None):
    """residual-gradient guidance (8f.3: residuals_darcy.py:114-126, unet_model.py:530-540,585-603): the training loss
    on smooth_fields(4, seed=19) with the seed-55 draws (t, eps, the classifier-free mask) and the gradients `grads`
    ({fixture key: parameter}).  The mask draw rarely drops a sample at B = 4: `forced_mask` adds the loss under that
    mask, which covers the null branch, and the guidance-scale-3 x0 estimate of a noisy sample."""
    res = darcy_residuals(model, bcs, residual_grad_guidance=True)
    x0 = smooth_fields(4, seed=19)
    model.train()
    loss = darcy_loss(x0, res, 55)[0]
    t, e, mask = loss_draws(55, x0, mask=True)
    extra = {}
    if forced_mask is not None:
        import src.unet_model as um
        draw = um.prob_mask_like
        um.prob_mask_like = lambda shape, prob, device: forced_mask.clone()
        loss_f = darcy_loss(x0, res, 55, backward=False)[0]
        um.prob_mask_like = draw
        model.eval()
        xs_in = (x0 * 0.6 + 0.3 * e)                        # (the reference needs autograd on here: no no_grad, :491-492)
        og = res.compute_residual((((xs_in.permute(0, 2, 3, 1).reshape(4, 4096, 2)).clone(), t),), reduce='per-batch',
                                  return_model_out=True, sample=True)
        extra = dict(forced_mask=forced_mask, loss_forced=loss_f.detach(), sample_in=xs_in,
                     sample_x0=og['model_out'].detach().clone())
    named = dict(model.named_parameters())
    save(out, name, dict(x0=x0, t=t, noise=e, null_mask=mask, loss=loss.detach(),
                         **{k: named[p].grad.clone() for k, p in grads.items()}, **extra))


def sample_loop(res, n_steps=6, seed=77, **corrections):
    """((x_seq, x0 estimates), aux) of the reference's ancestral loop (A11) at B = 1 after torch.manual_seed(seed)"""
    res.model.eval()
    d = diffusion(n_steps)
    torch.manual_seed(seed)
    return d.p_sample_loop(None, (1, 2, 64, 64), save_output=True, surpress_noise=True, residual_func=res,
                           eval_residuals=True, **corrections)


def sample_loop_draws():
    """the draws of sample_loop(): x_T, then one z per step (corrections draw none)"""
    torch.manual_seed(77)
    x_T = torch.randn(1, 2, 64, 64)
    zs = [torch.randn(1, 2, 64, 64) for _ in range(6)]
    return dict(x_T=x_T, noises=torch.stack(zs))


def sample_loop_fixture(out, name, res):
    """the sample_loop_6 recipe: 6 diffusion steps, B = 1, seed-77 draws"""
    (x_seq, interm), aux = sample_loop(res)
    save(out, name, dict(**sample_loop_draws(), x_final=x_seq[-1], x_after_first=x_seq[1], x0_pred_last=interm[-1],
                         residual=aux['residual'].detach()))


def consistent_solution(st, rho_simp, bcs):
    """[1,3,65,65] = (u_x, u_y, rho_simp padded) with u solving K(rho_simp) u = f, the reference's modified dense
    system assembled with its own helper, in fp64"""
    Kd = torch.zeros(st.neq, st.neq, dtype=torch.float64)
    kl = st.tot_local_stiffness.double() * rho_simp.reshape(-1).double()[:, None, None]
    idx = st.glob_assembler_idcs
    Kd.index_put_((idx[:, :, 0].reshape(-1), idx[:, :, 1].reshape(-1)),
                  kl[:, st.indices_ext[:, 0], st.indices_ext[:, 1]].reshape(-1), accumulate=True)
    bcx = st.image_to_stiffness_coord(bcs[:, 0], 0) + st.image_to_stiffness_coord(bcs[:, 1], 1)
    fg = (st.image_to_stiffness_coord(bcs[:, 2], 0) + st.image_to_stiffness_coord(bcs[:, 3], 1))[0].double()
    mk = bcx[0] != 0
    Kd[mk] = 0
    Kd[mk, mk] = 1
    fg[mk] = 0
    u = torch.linalg.solve(Kd, fg).float()[None]
    sol = torch.stack((st.stiffness_to_image_coord(u, 0), st.stiffness_to_image_coord(u, 1)), dim=1)
    return torch.cat((sol, F_pad(rho_simp, (0, 1, 0, 1)).unsqueeze(1)), dim=1)


# ---- the families ---------------------------------------------------------------------------------------------------

DARCY_LOSS_KEYS = ['init_conv.weight', 'time_mlp.1.weight', 'downs.0.0.block1.proj.weight', 'downs.0.0.mlp.1.weight',
                   'downs.0.2.fn.fn.to_qkv.weight', 'downs.1.3.weight', 'mid_spatial_attn.fn.fn.fn.to_qkv.weight',
                   'ups.0.3.weight', 'ups.3.2.fn.norm.gamma', 'final_conv.1.weight', 'final_conv.1.bias',
                   'downs.3.1.block2.norm.weight', 'ups.1.0.res_conv.weight']


def darcy_fixtures(out):
    """the Darcy study with bcs='none': schedule tables (A1), default-init checksums, U-Net forward (A6), residual
    (A7-A9), CoCoGen correction, mean- and sample-mode losses (A3, A12), guidance, 6- and 100-step sampling (A11)"""
    from src.unet_model import Unet3D
    for n in (100, 250):
        save(out, f'schedule_{n}.pt', {k: v.clone() for k, v in diffusion(n).diff_dict.items()})

    # default-init checksums under seed 0 (holder construction order = RNG order)
    torch.manual_seed(0)
    m0 = Unet3D(dim=32, channels=2)
    save(out, 'unet_init_seed0.pt', {k: torch.stack([v.double().sum(), v.double().abs().sum()])
                                     for k, v in m0.state_dict().items()})

    model = darcy_model()
    g = torch.Generator().manual_seed(11)
    x = torch.randn(2, 2, 64, 64, generator=g)
    forward_fixture(out, 'unet_darcy_fwd.pt', model, x, torch.tensor([3, 77]), time_emb=True)

    res = darcy_residuals(model)
    x0p = smooth_fields(3, seed=5)
    x0p[2] = torch.randn(2, 64, 64, generator=g)          # one rough sample
    r, wgt, grad = residual_vjp(res, x0p, g)
    save(out, 'darcy_residual.pt', dict(x0_pred=x0p, residual=r, f_s=res.f_s.reshape(64, 64).clone(), cotangent=wgt,
                                        grad_x0_pred=grad))
    cocogen_fixture(out, 'cocogen.pt', res, x0p)
    loss_fixture(out, 'darcy_loss_mean.pt', model, res, DARCY_LOSS_KEYS, nograd_name='params_without_grad.txt')

    # sample-mode loss (A12: ddim_sample_x0, ddim_steps=0) and the DDIM walk at ddim_steps = 1, 3
    x0 = smooth_fields(2, seed=9)
    loss_s, data_s, res_abs_s = darcy_loss(x0, darcy_residuals(model, use_ddim_x0=True, ddim_steps=0), 321)
    t_s, e_s = loss_draws(321, x0)
    named = dict(model.named_parameters())
    save(out, 'darcy_loss_sample.pt', dict(x0=x0, t=t_s, noise=e_s, loss=loss_s.detach(), data_loss=torch.tensor(data_s),
                                           residual_abs=torch.tensor(res_abs_s),
                                           grad_final_w=named['final_conv.1.weight'].grad.clone(),
                                           grad_init_w=named['init_conv.weight'].grad.clone(),
                                           **ddim_walk_keys(model)))

    guidance_fixture(out, 'darcy_guidance.pt', model, 'none',
                     dict(grad_emb0='emb_conv.0.weight', grad_combine='combine_conv.weight',
                          grad_final_w='final_conv.1.weight'),
                     forced_mask=torch.tensor([False, True, False, False]))
    sample_loop_fixture(out, 'sample_loop_6.pt', res)

    # the reference's default 100 diffusion steps.  The 101 draws are not stored (3.3 MB): tests replay them with
    # torch.manual_seed(78) on the CPU generator and check `noise_checksum` first, so a generator mismatch is reported
    # as such and not as a parity failure.
    (x_seq, _), aux = sample_loop(res, n_steps=100, seed=78)
    torch.manual_seed(78)
    draws = torch.stack([torch.randn(1, 2, 64, 64) for _ in range(101)])
    assert torch.equal(draws[0], x_seq[0])
    save(out, 'sample_loop_100.pt', dict(seed=torch.tensor(78), noise_checksum=draws.double().sum(dim=(1, 2, 3, 4)),
                                         x_25=x_seq[25], x_50=x_seq[50], x_75=x_seq[75], x_final=x_seq[-1],
                                         residual_abs_mean=aux['residual'].detach().abs().mean()))


def mechanics_fixtures(out):
    """the topology-optimisation study: residual (A13), evaluation metrics (8f.4) and training loss (A3 + A13)"""
    with mesh_folder() as folder:
        mres = mechanics_residuals(folder)
        KE = mres.stiffs.tot_local_stiffness[0].clone()
        gm = torch.Generator().manual_seed(4)
        xm = torch.randn(1, 3, 64, 64, generator=gm) * 0.1
        xm[:, 2] = torch.sigmoid(torch.randn(1, 64, 64, generator=gm))
        bcs = torch.zeros(1, 4, 65, 65)
        bcs[:, 0, :, 0] = 1.
        bcs[:, 1, :, 0] = 1.
        bcs[:, 1, 64, 10:20] = 1.
        bcs[:, 3, 20:24, 64] = -1.
        bcs[:, 2, 0, 30] = 0.5
        vf = torch.tensor([0.4])
        xmg = xm.clone().requires_grad_(True)
        o = mres.compute_residual((xmg, bcs, vf, None), reduce='per-batch', return_optimizer=True,
                                  return_inequality=True, pass_through=True)
        wr = torch.randn(o['residual'].shape, generator=gm)
        ((o['residual'] * wr).sum() + 0.3 * o['optimizer'].sum() + 2.0 * o['inequality'].sum()).backward()
        save(out, 'mechanics_residual.pt', dict(x0_pred=xm, bcs=bcs, vf=vf, residual=o['residual'].detach(),
                                                compliance=o['optimizer'].detach(), inequality=o['inequality'].detach(),
                                                KE=KE, cotangent=wr,
                                                grad_x0_pred=xmg.grad.clone()))

        # evaluation metrics (reference :276-354) on a consistent data sample
        ge = torch.Generator().manual_seed(8)
        i64 = torch.arange(64, dtype=torch.float32) / 63
        Xe, Ye = torch.meshgrid(i64, i64, indexing='ij')
        rho_simp = (0.55 + 0.45 * torch.sin(3.1 * Xe + 0.4) * torch.cos(2.3 * Ye)).clamp(0.05, 1.0)[None]
        bce = torch.zeros(1, 4, 65, 65)
        bce[:, 0, :, 0] = 1.
        bce[:, 1, :, 0] = 1.
        bce[:, 3, 30:34, 64] = -0.25
        sol = consistent_solution(mres.stiffs, rho_simp, bce)
        x_eval = torch.zeros(1, 3, 64, 64)
        x_eval[:, :2] = 0.05 * torch.randn(1, 2, 64, 64, generator=ge)
        x_eval[:, 2] = (rho_simp + 0.25 * torch.randn(1, 64, 64, generator=ge)).clamp(0, 1)
        vfe = torch.tensor([0.5])
        oe = mechanics_residuals(folder, topopt_eval=True).compute_residual(
            (x_eval, bce, vfe, sol), reduce='per-batch', return_optimizer=True, return_inequality=True, sample=True,
            pass_through=True)
        save(out, 'mechanics_eval.pt', dict(x0_pred=x_eval, bcs=bce, vf=vfe, solution=sol,
                                            rel_CE_error=oe['rel_CE_error_full_batch'].clone(),
                                            vf_error=oe['vf_error_full_batch'].clone(),
                                            fm_error=oe['fm_error_full_batch'].clone()))

        # training loss through the reference's model_estimation_loss (configs[2] glue), B = 2 with all four terms on
        # (c_ineq > 0 pins the [B,1] x [B] broadcast of :679,:694)
        model = reference_unet(3, **MECHANICS_CFG)
        model.train()
        mres_t = mechanics_residuals(folder, model)
        gt = torch.Generator().manual_seed(77)
        B = 2
        cond = torch.rand(B, 3, 65, 65, generator=gt)
        cond[:, 0] = torch.tensor([0.4, 0.55])[:, None, None]
        x0m = torch.cat((0.2 * torch.randn(B, 2, 65, 65, generator=gt), torch.rand(B, 1, 65, 65, generator=gt)), dim=1)
        bcm = torch.zeros(B, 4, 65, 65)
        bcm[:, 0, :, 0] = 1.
        bcm[:, 1, :, 0] = 1.
        bcm[:, 3, 32, 64] = -1.
        inp = torch.cat((cond, x0m, bcm), dim=1)
        coefs = dict(c_data=1.0, c_residual=1e-2, c_ineq=0.5, lambda_opt=1e-3)
        diff = diffusion(100)
        torch.manual_seed(99)
        loss, data_l, res_l, ineq_l, opt_l = diff.model_estimation_loss(inp, residual_func=mres_t, **coefs)
        model.zero_grad()
        loss.backward()
        t, e = loss_draws(99, x0m)
        named = dict(model.named_parameters())
        save(out, 'mechanics_loss.pt', dict(input=inp, t=t, noise=e, loss=loss.detach(), data_loss=torch.tensor(data_l),
                                            residual_abs=torch.tensor(res_l), inequality=torch.tensor(ineq_l),
                                            compliance=torch.tensor(opt_l), coefs=torch.tensor(list(coefs.values())),
                                            grad_final_w=named['final_conv.1.weight'].grad.clone(),
                                            grad_init_w=named['init_conv.weight'].grad.clone(),
                                            grad_mid_w=named['downs.1.0.block1.proj.weight'].grad.clone()))


def toy_fixtures(out):
    """configs[0]: the toy study's loss (src/denoising_toy_utils.py:436-511) through the unmodified reference module, with
    the residual / inequality / optimisation callables of main_toy.py:48-79."""
    import src.denoising_toy_utils as T
    T.device = torch.device('cpu')

    def residual_func(x):
        return torch.sum(x ** 2, dim=1) - 1.0

    def ineq_func(x):
        density = torch.sum(torch.abs(x), dim=1)
        return torch.relu(density - 1.0), density

    def opt_func(x):
        return x[:, 0]
    torch.manual_seed(5)
    np.random.seed(5)
    model = T.ConditionalModel(2, 100)
    dd = T.create_diff_dict(100, 'cpu')
    x0 = torch.tensor(T.sample_hypersphere(128, 2)).float()
    fx = {'x0': x0, **{'sd_' + k: v.clone() for k, v in model.state_dict().items()}}
    for tag, mode, ddim in (('x0_mean', 'x0', False), ('x0_sample', 'x0', True), ('eps_sample', 'eps', True)):
        torch.manual_seed(17)
        loss, data_l, res_l, ineq_l, opt_l = T.model_estimation_loss(
            model, x0, 100, dd, model_pred_mode=mode, residual_func=residual_func, ineq_func=ineq_func, opt_func=opt_func,
            c_data=1.0, c_residual=0.005, c_ineq=0.3, lambda_opt=0.01, use_ddim_x0=ddim, reduced_ddim_steps=0)
        model.zero_grad()
        loss.backward()
        fx[tag + '_loss'] = loss.detach().clone()
        fx[tag + '_tracked'] = torch.tensor([data_l, res_l, ineq_l, opt_l])
        fx[tag + '_grad_lin3'] = model.lin3.weight.grad.clone()
        fx[tag + '_grad_lin1'] = model.lin1.lin.weight.grad.clone()
        fx[tag + '_grad_embed2'] = model.lin2.embed.weight.grad.clone()
    torch.manual_seed(17)                                  # replay the draws (:440-441, :447)
    t = torch.randint(0, 100, size=(128 // 2 + 1,))
    fx['t'] = torch.cat([t, 100 - t - 1], dim=0)[:128].long()
    fx['noise'] = torch.randn_like(x0)
    # short ancestral loop (x0 mode), draws replayed by the test: x_T then one z per step
    model.eval()
    d8 = T.create_diff_dict(8, 'cpu')
    torch.manual_seed(23)
    xs, _, _ = T.p_sample_loop(model, [64, 2], 8, d8, model_pred_mode='x0', save_output=False, surpress_noise=True)
    torch.manual_seed(23)
    fx['loop_draws'] = torch.stack([torch.randn(64, 2) for _ in range(9)])
    fx['loop_final'] = xs[-1]
    save(out, 'toy.pt', fx)


def periodic_fixtures(out):
    """ResidualsDarcy(bcs='periodic'):

    darcy_residual_periodic.pt   residual, VJP and the five stencil_gradients modes on the fields of darcy_residual.pt
    cocogen_periodic.pt          residual_correction (vmap(jacfwd) Jacobian) on two of those fields
    darcy_loss_periodic.pt       mean-mode model_estimation_loss, loss terms and the gradients of darcy_loss_mean.pt
    sample_loop_periodic.pt      the sample_loop_6 recipe"""
    model = darcy_model()
    res = darcy_residuals(model, 'periodic')
    assert res.periodic
    x0p = load_golden('darcy_residual.pt')['x0_pred']
    r, wgt, grad = residual_vjp(res, x0p, torch.Generator().manual_seed(31))
    with torch.no_grad():
        sg = {'stencil_' + m: res.grads.stencil_gradients(x0p[:, 0].clone(), mode=m).clone()
              for m in ('d_d0', 'd_d1', 'd_d00', 'd_d11', 'd_d01')}
    save(out, 'darcy_residual_periodic.pt', dict(x0_pred=x0p, residual=r, cotangent=wgt, grad_x0_pred=grad, **sg))
    cocogen_fixture(out, 'cocogen_periodic.pt', res, x0p)
    loss_fixture(out, 'darcy_loss_periodic.pt', model, res, DARCY_LOSS_KEYS)
    sample_loop_fixture(out, 'sample_loop_periodic.pt', res)


def circular_fixtures(out):
    """Unet3D(padding_mode='circular') with ResidualsDarcy(bcs='periodic'):

    unet_circular_keys.pt        the circular state_dict key list, in order
    unet_circular_fwd.pt         forward output + taps on the unet_darcy_fwd.pt inputs
    darcy_loss_circular.pt       mean-mode loss, loss terms, grad-norm and gradients
    darcy_guidance_circular.pt   residual-gradient guidance loss + gradients (emb_conv[2] stays zero-padded)
    sample_loop_circular.pt      the sample_loop_6 recipe"""
    model = darcy_model('circular')
    save(out, 'unet_circular_keys.pt', dict(keys=list(model.state_dict().keys())))
    fw = load_golden('unet_darcy_fwd.pt')
    forward_fixture(out, 'unet_circular_fwd.pt', model, fw['x'], fw['t'])
    res = darcy_residuals(model, 'periodic')
    loss_fixture(out, 'darcy_loss_circular.pt', model, res,
                 ['init_conv.weight', 'downs.0.0.block1.proj.weight', 'downs.1.3.weight', 'ups.0.3.conv_transpose.weight',
                  'ups.2.3.conv_transpose.bias', 'ups.3.1.block2.proj.weight', 'final_conv.1.weight'])
    guidance_fixture(out, 'darcy_guidance_circular.pt', model, 'periodic',
                     dict(grad_emb2='emb_conv.2.weight', grad_emb0='emb_conv.0.weight', grad_final_w='final_conv.1.weight'))
    sample_loop_fixture(out, 'sample_loop_circular.pt', res)


def cocogen_fixtures(out):
    """CoCoGen residual corrections:

    cocogen_steps.pt         five successive residual_correction calls (vmap(jacfwd) Jacobian) on the two fields of
                             cocogen.pt: the p plane after every call and the residual after the last
    sample_loop_cocogen.pt   the sample_loop_6 recipe (6 steps, B=1, seed-0 test weights, seed-77 draws) run with
                             N_correction=2, M_correction=3, 'xt' and with N_correction=2, M_correction=0, 'x0'"""
    res = darcy_residuals(darcy_model())
    x0p = load_golden('cocogen.pt')['x0_pred']
    xin = x0p.permute(0, 2, 3, 1).reshape(2, 4096, 2).clone()
    p_iterates, r = [], None
    for _ in range(5):
        xin, r = res.residual_correction(xin)                # in place, like p_sample_loop's post-loop corrections
        p_iterates.append(xin[:, :, 0].reshape(2, 64, 64).detach().clone())
    save(out, 'cocogen_steps.pt', dict(x0_pred=x0p, p_iterates=torch.stack(p_iterates), residual_final=r.detach().clone()))

    fx = {}
    for tag, kw in (('xt', dict(N_correction=2, M_correction=3, correction_mode='xt')),
                    ('x0', dict(N_correction=2, M_correction=0, correction_mode='x0'))):
        (x_seq, _), aux = sample_loop(res, **kw)
        r = aux['residual'].detach().clone()
        M = kw['M_correction']
        # On the CPU `.cpu()` returns the tensor itself, so the reference's trajectory entries of the t = 0 step and of
        # the post-loop corrections all alias one tensor that the in-place corrections keep updating.  The tail (the
        # last two loop states, then one state per post-loop correction) is therefore rebuilt from the loop without
        # post-loop corrections and M explicit residual_correction calls, and checked against the aliased final state.
        if M:
            (tail, _), _ = sample_loop(res, **dict(kw, M_correction=0))
            tail = [v.clone() for v in tail[-2:]]
            cur = tail[-1].permute(0, 2, 3, 1).reshape(1, 4096, 2).clone()
            for _ in range(M):
                cur, r_m = res.residual_correction(cur)
                tail.append(cur.reshape(1, 64, 64, 2).permute(0, 3, 1, 2).detach().clone())
            assert torch.equal(tail[-1], x_seq[-1]) and torch.equal(r_m, r)
        else:
            tail = [v.clone() for v in x_seq[-2:]]
        fx[f'{tag}_x_final'] = x_seq[-1].clone()
        fx[f'{tag}_residual'] = r
        fx[f'{tag}_tail'] = torch.stack(tail)
        fx[f'{tag}_len'] = torch.tensor(len(x_seq))
    save(out, 'sample_loop_cocogen.pt', dict(**sample_loop_draws(), **fx))


def guidance_step_fixtures(out):
    """one iteration of the training loop (reference main.py:158-179) with residual_grad_guidance=True at B = 8:

    darcy_guidance_step.pt             x0, t, eps, the classifier-free mask (both values occur), loss, data loss,
                                       mean|r|, a golden_sample(., 256) of the gradient of every parameter that receives
                                       one, and the global gradient norm that drives clipping
    params_without_grad_guidance.txt   the parameters whose .grad stays None under guidance"""
    B, n_sample = 8, 256
    model = darcy_model()
    res = darcy_residuals(model, residual_grad_guidance=True)
    x0 = smooth_fields(B, seed=29)
    seed = next(s for s in range(1000, 2000) if 0 < int(loss_draws(s, x0, mask=True)[2].sum()) < B)   # both values
    t, e, mask = loss_draws(seed, x0, mask=True)
    model.train()
    loss, data_l, rabs = darcy_loss(x0, res, seed)
    named = dict(model.named_parameters())
    grads = {'grad_' + k: O.golden_sample(p.grad, n_sample) for k, p in named.items() if p.grad is not None}
    save(out, 'darcy_guidance_step.pt', dict(x0=x0, t=t, noise=e, null_mask=mask, loss=loss.detach(),
                                             data_loss=torch.tensor(data_l), residual_abs=torch.tensor(rabs),
                                             grad_norm=grad_norm(model), grad_sample=torch.tensor(n_sample), **grads))
    save_names(out, 'params_without_grad_guidance.txt', sorted(k for k, p in named.items() if p.grad is None))


def mech_sample_fixtures(out):
    """conditional sampling of the topology-optimisation model: `DenoisingDiffusion.p_sample_loop` with a
    `conditioning_input` (reference denoising_utils.py:388-545, sample.py:244-262) at B = 2 over 6 diffusion steps, with
    `eval_residuals`, `return_optimizer`, `return_inequality` and `topopt_eval=True` (dense LU of the binarised designs
    at t = 0), for both x0 estimates ('mean': one network call; 'sample': `use_ddim_x0=True, ddim_steps=0`).  The data
    samples are consistent (their displacements solve K(rho_simp) u = f), so the reference's data-residual check passes.
    The inputs and the draws are rebuilt by tests/mech_sample_inputs.py and only checksummed here; large outputs are
    stored as oracle.pidm_oracle.golden_sample(., 4096).  Keys of mechanics_sample_loop.pt:

    seed, n_steps, input_checksum, solution      the loop's seed, the inputs' checksums, the consistent data samples
per mode (prefix 'mean_' / 'sample_'):
    noise_checksum                               per-draw sums of x_T, the posterior z and (in 'sample' mode) the DDIM
                                                 walk's draws, in the reference's order
    x_first, x_final, x0_pred_last, residual     golden samples of the sample after the first / last step, the last x0
                                                 estimate (the last network output) and the residual of the last step
    rho_last                                     the density channel of that x0 estimate, whole (binarisation checks)
    compliance, inequality, rel_CE_error, vf_error, fm_error    the aux outputs of the last step"""
    MI = _load('mech_sample_inputs', os.path.join(ROOT, 'tests', 'mech_sample_inputs.py'))
    n_steps, seed = 6, 2024
    model = reference_unet(3, **MECHANICS_CFG)
    model.eval()
    last = {}
    model.register_forward_hook(lambda m, i, o: last.__setitem__('y', o.detach().clone()))
    cond, bcs, rho = MI.conditioning_batch()
    fx = {'n_steps': torch.tensor(n_steps), 'seed': torch.tensor(seed),
          'input_checksum': torch.stack([cond.double().sum(), bcs.double().sum(), rho.double().sum()])}
    gs = lambda t: O.golden_sample(t, MI.SAMPLE)  # noqa: E731
    with mesh_folder() as folder:
        for mode in ('mean', 'sample'):
            res = mechanics_residuals(folder, model, topopt_eval=True, use_ddim_x0=mode == 'sample', ddim_steps=0)
            if mode == 'mean':
                sol = torch.cat([consistent_solution(res.stiffs, rho[b][None], bcs[b:b + 1]) for b in range(MI.B)], dim=0)
                fx['solution'] = sol
            diff = diffusion(n_steps)
            torch.manual_seed(seed)
            with torch.no_grad():
                (x_seq, _), aux = diff.p_sample_loop((cond, bcs, sol), (MI.B, 3, 65, 65), save_output=True,
                                                     surpress_noise=True, residual_func=res, eval_residuals=True,
                                                     return_optimizer=True, return_inequality=True)
            x_T, zs, ddim = MI.draws(seed, n_steps, mode)     # replay the draws in the reference's order
            assert torch.equal(x_T, x_seq[0])
            fx.update({f'{mode}_{k}': v for k, v in dict(
                noise_checksum=MI.checksums(x_T, zs, ddim), x_first=gs(x_seq[1]), x_final=gs(x_seq[-1]),
                x0_pred_last=gs(last['y']), rho_last=last['y'][:, 2].clone(), residual=gs(aux['residual'].detach()),
                compliance=aux['optimized_quant'].detach(), inequality=aux['inequality_quant'].detach(),
                rel_CE_error=aux['rel_CE_error_full_batch'].detach(), vf_error=aux['vf_error_full_batch'].detach(),
                fm_error=aux['fm_error_full_batch']).items()})
            print(mode, 'rel_CE_error', aux['rel_CE_error_full_batch'].tolist(), 'fm', aux['fm_error_full_batch'].tolist(),
                  '|rho - 0.5| min', (last['y'][:, 2] - 0.5).abs().min().item())
    save(out, 'mechanics_sample_loop.pt', fx)


def darcy_gen_fixtures(out):
    """the reference's src/darcy_data_generation.py, in fp64:

    eigenvalues [64]   the q = 64 largest covariance eigenvalues (compute_eigenpairs on complete_covariance_matrix)
    f_s [4096], int_cond [4096]   create_f_s and the trapezoid weights of create_int_cond
    seed [4], z [4, 64], K [4, 4096], p [4, 4096], res [4]   generate_sample on four argument tuples

    geometry_*         the same generate_sample at pixels_at_boundary=False, reverse_dy=False, domain_length=2 (its own
                       eigenpairs, grid, source and weights): the three options, f_s, int_cond, seed [2], K, p [2, 4096],
                       res [2]

    generate_sample draws its seed from os.getpid() * time.time(); the recipe replaces the module's `os` and `time`
    names by stand-ins (pid = seed, clock = 1 ms), so that unique_seed = seed.  The reference file itself is not
    touched."""
    import src.darcy_data_generation as G
    P, dl, l, q, acc = 64, 1., 0.1, 64, 2
    shape = (P, P)
    pts = G.uniform_points_pixelwise(P, dl, True)
    d0 = dl / (P - 1)
    d1 = -d0
    eigenvalues, eigenvectors = G.compute_eigenpairs(G.complete_covariance_matrix(pts, l), q)
    f_s = G.create_f_s(pts[:, 0], pts[:, 1])
    xmin_bd, xmax_bd, ymin_bd, ymax_bd = G.create_boundary_idcs(shape)
    int_cond = G.create_int_cond(True, shape, d0)

    fx = dict(seed=[], z=[], K=[], p=[], res=[])
    for s in (1, 20231, 777, 4242424):
        G.os = types.SimpleNamespace(getpid=lambda s=s: s)
        G.time = types.SimpleNamespace(time=lambda: 0.001)
        args = (0, eigenvalues, eigenvectors, q, P, shape, acc, d0, d1, f_s, int_cond, xmin_bd, xmax_bd, ymin_bd,
                ymax_bd, True)
        K, p, res, seed = G.generate_sample(args)
        assert seed == s, (seed, s)
        np.random.seed(s)
        z = G.norm.rvs(size=q)
        fx['seed'].append(seed)
        fx['z'].append(z)
        fx['K'].append(K)
        fx['p'].append(p)
        fx['res'].append(res)
        print(f'seed {s}: res {res:.6e}  max|p| {np.abs(p).max():.4f}')
    t = lambda a: torch.tensor(np.asarray(a), dtype=torch.float64)  # noqa: E731
    out_fx = dict(eigenvalues=t(eigenvalues), f_s=t(f_s), int_cond=t(int_cond).reshape(-1),
                  seed=torch.tensor(fx['seed'], dtype=torch.int64), z=t(fx['z']), K=t(fx['K']), p=t(fx['p']),
                  res=t(fx['res']))

    # geometry_*: the same generate_sample away from the default geometry (pixel centres, h = L / P, the plain-mean
    # integral row, d1 = +h with the -D1 | +D1 BC rows), two samples
    pab, reverse_dy, dl = False, False, 2.
    pts = G.uniform_points_pixelwise(P, dl, pab)
    d0 = d1 = dl / P
    eigenvalues, eigenvectors = G.compute_eigenpairs(G.complete_covariance_matrix(pts, l), q)
    f_s = G.create_f_s(pts[:, 0], pts[:, 1])
    int_cond = G.create_int_cond(pab, shape, d0)
    fx = dict(seed=[], K=[], p=[], res=[])
    for s in (3, 90210):
        G.os = types.SimpleNamespace(getpid=lambda s=s: s)
        G.time = types.SimpleNamespace(time=lambda: 0.001)
        args = (0, eigenvalues, eigenvectors, q, P, shape, acc, d0, d1, f_s, int_cond, xmin_bd, xmax_bd, ymin_bd,
                ymax_bd, reverse_dy)
        K, p, res, seed = G.generate_sample(args)
        assert seed == s, (seed, s)
        for k, v in zip(('seed', 'K', 'p', 'res'), (seed, K, p, res)):
            fx[k].append(v)
        print(f'geometry seed {s}: res {res:.6e}  max|p| {np.abs(p).max():.4f}')
    geometry = dict(pixels_at_boundary=torch.tensor(pab), reverse_dy=torch.tensor(reverse_dy),
                    domain_length=torch.tensor(dl, dtype=torch.float64), f_s=t(f_s), int_cond=t(int_cond).reshape(-1),
                    seed=torch.tensor(fx['seed'], dtype=torch.int64), K=t(fx['K']), p=t(fx['p']), res=t(fx['res']))
    out_fx.update({f'geometry_{k}': v for k, v in geometry.items()})
    save(out, 'darcy_gen.pt', out_fx)


DDIM_WALK = dict(n_steps=100, t=(0, 2, 57, 99), seed=13, sample=4096)


def ddim_walk_input():
    """x_t [4,2,64,64] of the DDIM walk in darcy_loss_sample.pt, regenerated from its seed (the fixture keeps its
    checksum)"""
    return torch.randn(len(DDIM_WALK['t']), 2, 64, 64, generator=torch.Generator().manual_seed(DDIM_WALK['seed']))


def ddim_walk_keys(model):
    """the walk_* keys of darcy_loss_sample.pt: the reference's DenoisingDiffusion.ddim_sample_x0 (eta = 0) on the Darcy
    test model for ddim_steps = 1 and 3 at per-sample t = 0, 2 (the grids repeat points: linspace(0, 2, 5) -> 0, 0, 1,
    1, 2), 57 and n_steps - 1; golden_sample(cur_x) and golden_sample(model_out) per ddim_steps"""
    diff = diffusion(DDIM_WALK['n_steps'])
    xt = ddim_walk_input()
    t = torch.tensor(DDIM_WALK['t'])
    fx = dict(walk_t=t, walk_seed=torch.tensor(DDIM_WALK['seed']), walk_x_t_checksum=xt.double().sum())
    with torch.no_grad():
        for s in (1, 3):
            cur_x, model_out = diff.ddim_sample_x0(xt, t, model, xt.shape, s, 0.)
            fx[f'walk_cur_x_{s}'] = O.golden_sample(cur_x, DDIM_WALK['sample'])
            fx[f'walk_model_out_{s}'] = O.golden_sample(model_out, DDIM_WALK['sample'])
    return fx


# family -> (recipe, the files under tests/golden/ it writes)
RECIPES = {
    'darcy': (darcy_fixtures, ('schedule_100.pt', 'schedule_250.pt', 'unet_init_seed0.pt', 'unet_darcy_fwd.pt',
                               'darcy_residual.pt', 'cocogen.pt', 'darcy_loss_mean.pt', 'params_without_grad.txt',
                               'darcy_loss_sample.pt', 'darcy_guidance.pt', 'sample_loop_6.pt', 'sample_loop_100.pt')),
    'mechanics': (mechanics_fixtures, ('mechanics_residual.pt', 'mechanics_eval.pt', 'mechanics_loss.pt')),
    'toy': (toy_fixtures, ('toy.pt',)),
    'periodic': (periodic_fixtures, ('darcy_residual_periodic.pt', 'cocogen_periodic.pt', 'darcy_loss_periodic.pt',
                                     'sample_loop_periodic.pt')),
    'circular': (circular_fixtures, ('unet_circular_keys.pt', 'unet_circular_fwd.pt', 'darcy_loss_circular.pt',
                                     'darcy_guidance_circular.pt', 'sample_loop_circular.pt')),
    'cocogen': (cocogen_fixtures, ('cocogen_steps.pt', 'sample_loop_cocogen.pt')),
    'guidance': (guidance_step_fixtures, ('darcy_guidance_step.pt', 'params_without_grad_guidance.txt')),
    'mech_sample': (mech_sample_fixtures, ('mechanics_sample_loop.pt',)),
    'darcy_gen': (darcy_gen_fixtures, ('darcy_gen.pt',)),
}


def main(argv=None):
    ap = argparse.ArgumentParser(description='Write the golden fixtures from the unmodified reference '
                                             '(checkout in PIDM_REFERENCE).')
    ap.add_argument('--out', default=GOLDEN, help='output directory (default: tests/golden)')
    ap.add_argument('families', nargs='*', choices=list(RECIPES), metavar='FAMILY',
                    help=f'recipe families to run (default: all of {", ".join(RECIPES)})')
    args = ap.parse_args(argv)
    import_reference()
    torch.set_num_threads(8)
    for family in args.families or RECIPES:
        RECIPES[family][0](args.out)


if __name__ == '__main__':
    main()
