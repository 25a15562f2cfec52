"""Golden-vector generator.  TEST INFRASTRUCTURE ONLY; runs in the build container, not on the GPU box.

Imports the UNMODIFIED reference modules from a checkout of the original project (path in PIDM_REFERENCE) through
the import shims in oracle/ref_shims/ (SURVEY.md section 8c), runs them on seeded CPU inputs and writes small fixtures
to tests/golden/.  The weights are not stored: both sides rebuild them with
oracle.pidm_oracle.make_test_state_dict(cfg, seed).  Large tensors are stored as oracle.pidm_oracle.golden_sample().

    PIDM_REFERENCE=<checkout of the original project> python oracle/make_golden.py      # rewrites tests/golden/*.pt
"""
import os
import sys
import tempfile
import warnings

import numpy as np
import torch
from torch.nn.functional import pad as F_pad

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.environ['PIDM_REFERENCE']
# NOTE: the repo root must NOT be importable here: its `src/` drop-in package (a regular package) would shadow
# the reference's `src/` (a namespace package) regardless of path order.
sys.path = [p for p in sys.path if os.path.abspath(p or '.') != ROOT]
sys.path.insert(0, os.path.join(HERE, 'ref_shims'))
sys.path.insert(0, REF)
warnings.filterwarnings('ignore')

import importlib.util  # noqa: E402

_spec = importlib.util.spec_from_file_location('pidm_oracle', os.path.join(HERE, 'pidm_oracle.py'))
O = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(O)

OUT = os.path.join(ROOT, 'tests', 'golden')


def save(name, obj):
    os.makedirs(OUT, exist_ok=True)
    torch.save(obj, os.path.join(OUT, name))
    n = sum(v.numel() * v.element_size() for v in obj.values() if torch.is_tensor(v))
    print(f'wrote {name}: {n / 1024:.1f} KiB')


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


def write_mesh(folder, nel=64):
    """Unit-square 65x65-node / 64x64-element mesh files in the solidspy text format read at
    residuals_mechanics_K.py:43-49; convention documented in oracle.pidm_oracle.mechanics_mesh."""
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


def main():
    torch.set_num_threads(8)
    from src.unet_model import Unet3D
    import src.unet_model as _ref_mod
    assert os.path.abspath(_ref_mod.__file__).startswith(os.path.abspath(REF)), _ref_mod.__file__
    from src.denoising_utils import DenoisingDiffusion
    from src.residuals_darcy import ResidualsDarcy
    from src.residuals_mechanics_K import ResidualsMechanics

    # ---- schedule tables (A1) -----------------------------------------------------------------
    for n in (100, 250):
        d = DenoisingDiffusion(n, 'cpu')
        save(f'schedule_{n}.pt', {k: v.clone() for k, v in d.diff_dict.items()})

    # ---- default-init checksums under seed 0 (holder construction order = RNG order) --------------
    torch.manual_seed(0)
    m0 = Unet3D(dim=32, channels=2)
    save('unet_init_seed0.pt', {k: torch.stack([v.double().sum(), v.double().abs().sum()]) for k, v in m0.state_dict().items()})

    # ---- U-Net forward with taps (A6) ---------------------------------------------------------
    cfg = O.unet_config(dim=32, channels=2)
    sd = O.make_test_state_dict(cfg, seed=0)
    model = Unet3D(dim=32, channels=2)
    model.load_state_dict(sd, strict=True)
    model.eval()
    g = torch.Generator().manual_seed(11)
    x = torch.randn(2, 2, 64, 64, generator=g)
    t = torch.tensor([3, 77])
    taps = {}

    def hook(name):
        def f(mod, inp, out):
            taps[name] = out.detach().squeeze(2).clone()
        return f
    hs = [model.init_conv.register_forward_hook(hook('init_conv')),
          model.time_mlp.register_forward_hook(lambda m, i, o: taps.__setitem__('time_emb', o.detach().clone())),
          model.downs[0][0].register_forward_hook(hook('downs.0.0')),
          model.downs[0][2].register_forward_hook(hook('downs.0.2')),
          model.mid_spatial_attn.register_forward_hook(hook('mid_attn')),
          model.ups[0][3].register_forward_hook(hook('ups.0'))]
    with torch.no_grad():
        y = model(x, t)
        y_bxyc = model(x.permute(0, 2, 3, 1).reshape(2, 4096, 2), t)
    for h in hs:
        h.remove()
    assert torch.equal(y, y_bxyc)
    save('unet_darcy_fwd.pt', dict(x=x, t=t, y=y, **{'tap_' + k: O.golden_sample(v) for k, v in taps.items()}))

    # ---- Darcy residual on given fields (A7-A9) -----------------------------------------------
    res = ResidualsDarcy(model=model, fd_acc=2, pixels_per_dim=64, pixels_at_boundary=True, reverse_d1=True,
                         device='cpu', bcs='none', domain_length=1.)
    x0p = smooth_fields(3, seed=5)
    x0p[2] = torch.randn(2, 64, 64, generator=g)          # one rough sample
    r = res.compute_residual(x0p, pass_through=True)['residual']
    xg = x0p.clone().requires_grad_(True)
    rg = res.compute_residual(xg, pass_through=True)['residual']
    wgt = torch.randn(rg.shape, generator=g)
    (rg * wgt).sum().backward()
    save('darcy_residual.pt', dict(x0_pred=x0p, residual=r.detach(), f_s=res.f_s.reshape(64, 64).clone(),
                                   cotangent=wgt, grad_x0_pred=xg.grad.clone()))

    # ---- CoCoGen residual correction (8f.3), through the reference's vmap(jacfwd) Jacobian -------
    xc = generalized_cocogen_input = x0p[:2].clone()
    xin = xc.permute(0, 2, 3, 1).reshape(2, 4096, 2).clone()
    x_corr, r_corr = res.residual_correction(xin)
    save('cocogen.pt', dict(x0_pred=xc, corrected=x_corr.reshape(2, 64, 64, 2).permute(0, 3, 1, 2).contiguous().clone(),
                            residual_corrected=r_corr.detach().clone()))

    # ---- full training loss + gradients, mean mode (A3) ---------------------------------------
    diff = DenoisingDiffusion(100, 'cpu')
    model.train()
    x0 = smooth_fields(2, seed=9)
    torch.manual_seed(123)
    loss, data_l, res_l, _, _ = diff.model_estimation_loss(x0, residual_func=res, c_data=1., c_residual=1e-3,
                                                           c_ineq=0., lambda_opt=0.)
    model.zero_grad()
    loss.backward()
    torch.manual_seed(123)                                  # replay the two RNG draws (:625,:636)
    t_l = torch.randint(0, 100, size=(2,))
    e_l = torch.randn_like(x0)
    keys = ['init_conv.weight', 'time_mlp.1.weight', 'downs.0.0.block1.proj.weight', 'downs.0.0.mlp.1.weight',
            'downs.0.2.fn.fn.to_qkv.weight', 'downs.1.3.weight', 'mid_spatial_attn.fn.fn.fn.to_qkv.weight',
            'ups.0.3.weight', 'ups.3.2.fn.norm.gamma', 'final_conv.1.weight', 'final_conv.1.bias',
            'downs.3.1.block2.norm.weight', 'ups.1.0.res_conv.weight']
    named = dict(model.named_parameters())
    grads = {'grad_' + k: O.golden_sample(named[k].grad) for k in keys}
    gn = torch.sqrt(sum((p.grad.double() ** 2).sum() for p in model.parameters() if p.grad is not None)).float()
    nograd = sorted(k for k, p in named.items() if p.grad is None)
    save('darcy_loss_mean.pt', dict(x0=x0, t=t_l, noise=e_l, loss=loss.detach(), data_loss=torch.tensor(data_l),
                                    residual_abs=torch.tensor(res_l), grad_norm=gn, **grads))
    with open(os.path.join(OUT, 'params_without_grad.txt'), 'w') as f:
        f.write('\n'.join(nograd) + '\n')

    # ---- sample-mode loss (A12: ddim_sample_x0, ddim_steps=0) ---------------------------------
    res_s = ResidualsDarcy(model=model, fd_acc=2, pixels_per_dim=64, pixels_at_boundary=True, reverse_d1=True,
                           device='cpu', bcs='none', domain_length=1., use_ddim_x0=True, ddim_steps=0)
    torch.manual_seed(321)
    loss_s, data_s, res_abs_s, _, _ = diff.model_estimation_loss(x0, residual_func=res_s, c_data=1.,
                                                                 c_residual=1e-3, c_ineq=0., lambda_opt=0.)
    model.zero_grad()
    loss_s.backward()
    torch.manual_seed(321)
    t_s = torch.randint(0, 100, size=(2,))
    e_s = torch.randn_like(x0)
    save('darcy_loss_sample.pt', dict(x0=x0, t=t_s, noise=e_s, loss=loss_s.detach(),
                                      data_loss=torch.tensor(data_s), residual_abs=torch.tensor(res_abs_s),
                                      grad_final_w=named['final_conv.1.weight'].grad.clone(),
                                      grad_init_w=named['init_conv.weight'].grad.clone()))

    # ---- residual-gradient guidance (8f.3: residuals_darcy.py:114-126, unet_model.py:530-540,585-603) -----------------
    res_g = ResidualsDarcy(model=model, fd_acc=2, pixels_per_dim=64, pixels_at_boundary=True, reverse_d1=True,
                           device='cpu', bcs='none', domain_length=1., residual_grad_guidance=True)
    x0g = smooth_fields(4, seed=19)
    model.train()
    torch.manual_seed(55)
    loss_g, data_g, res_abs_g, _, _ = diff.model_estimation_loss(x0g, residual_func=res_g, c_data=1., c_residual=1e-3,
                                                                 c_ineq=0., lambda_opt=0.)
    model.zero_grad()
    loss_g.backward()
    torch.manual_seed(55)                                   # replay: t, eps, then the classifier-free mask (unet_model.py:69)
    t_g = torch.randint(0, 100, size=(4,))
    e_g = torch.randn_like(x0g)
    mask_g = torch.zeros((4,)).float().uniform_(0, 1) < 0.1
    mask_forced = torch.tensor([False, True, False, False])
    # the draw above rarely drops a sample at B = 4: a second evaluation with a forced mask covers the null branch
    import src.unet_model as _um
    _orig_mask = _um.prob_mask_like
    _um.prob_mask_like = lambda shape, prob, device: mask_forced.clone()
    torch.manual_seed(55)
    loss_f, _, _, _, _ = diff.model_estimation_loss(x0g, residual_func=res_g, c_data=1., c_residual=1e-3, c_ineq=0., lambda_opt=0.)
    _um.prob_mask_like = _orig_mask
    model.eval()
    xs_in = (x0g * 0.6 + 0.3 * e_g)                        # (the reference needs autograd on here: no no_grad, :491-492)
    og = res_g.compute_residual((((xs_in.permute(0, 2, 3, 1).reshape(4, 4096, 2)).clone(), t_g),), reduce='per-batch',
                                return_model_out=True, sample=True)
    og = {k: v.detach() for k, v in og.items()}
    save('darcy_guidance.pt', dict(x0=x0g, t=t_g, noise=e_g, null_mask=mask_g, loss=loss_g.detach(),
                                   grad_emb0=named['emb_conv.0.weight'].grad.clone(),
                                   grad_combine=named['combine_conv.weight'].grad.clone(),
                                   grad_final_w=named['final_conv.1.weight'].grad.clone(),
                                   forced_mask=mask_forced, loss_forced=loss_f.detach(),
                                   sample_in=xs_in, sample_x0=og['model_out'].clone()))
    model.train()

    # ---- ancestral sampling loop (A11), 6 diffusion steps, B=1 --------------------------------
    model.eval()
    d6 = DenoisingDiffusion(6, 'cpu')
    torch.manual_seed(77)
    (x_seq, interm), aux = d6.p_sample_loop(None, (1, 2, 64, 64), save_output=True, surpress_noise=True,
                                            residual_func=res, eval_residuals=True)
    torch.manual_seed(77)
    x_T = torch.randn(1, 2, 64, 64)
    zs = [torch.randn(1, 2, 64, 64) for _ in range(6)]
    save('sample_loop_6.pt', dict(x_T=x_T, noises=torch.stack(zs), x_final=x_seq[-1], x_after_first=x_seq[1],
                                  x0_pred_last=interm[-1], residual=aux['residual'].detach()))

    # ---- ancestral sampling loop, the reference's default 100 diffusion steps, B=1 ---------------
    # The 101 draws are not stored (3.3 MB): tests replay them with torch.manual_seed(78) on the CPU generator and
    # check `noise_checksum` first, so a generator mismatch is reported as such and not as a parity failure.
    d100 = DenoisingDiffusion(100, 'cpu')
    torch.manual_seed(78)
    (x_seq, _), aux = d100.p_sample_loop(None, (1, 2, 64, 64), save_output=True, surpress_noise=True,
                                         residual_func=res, eval_residuals=True)
    torch.manual_seed(78)
    draws = torch.stack([torch.randn(1, 2, 64, 64) for _ in range(101)])
    assert torch.equal(draws[0], x_seq[0])
    save('sample_loop_100.pt', dict(seed=torch.tensor(78), noise_checksum=draws.double().sum(dim=(1, 2, 3, 4)),
                                    x_25=x_seq[25], x_50=x_seq[50], x_75=x_seq[75], x_final=x_seq[-1],
                                    residual_abs_mean=aux['residual'].detach().abs().mean()))

    # ---- mechanics residual on given fields (A13) ---------------------------------------------
    with tempfile.TemporaryDirectory() as td:
        write_mesh(td)
        mres = ResidualsMechanics(model=None, pixels_per_dim=64, pixels_at_boundary=True, no_BC_folder=td + '/',
                                  device='cpu', topopt_eval=False)
        KE_ref = mres.stiffs.tot_local_stiffness[0].clone()
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
        out = mres.compute_residual((xmg, bcs, vf, None), reduce='per-batch', return_optimizer=True,
                                    return_inequality=True, pass_through=True)
        wr = torch.randn(out['residual'].shape, generator=gm)
        ((out['residual'] * wr).sum() + 0.3 * out['optimizer'].sum() + 2.0 * out['inequality'].sum()).backward()
        save('mechanics_residual.pt', dict(x0_pred=xm, bcs=bcs, vf=vf, residual=out['residual'].detach(),
                                           compliance=out['optimizer'].detach(), inequality=out['inequality'].detach(),
                                           KE=KE_ref, cotangent=wr, grad_x0_pred=xmg.grad.clone()))

        # ---- evaluation metrics of the topology-optimisation study (8f.4; reference :276-354) -------------------------
        # a consistent data sample: u_data solves K(rho_simp) u = f (dense assembly with the reference's own helper, fp64)
        st = mres.stiffs
        ge = torch.Generator().manual_seed(8)
        i64 = torch.arange(64, dtype=torch.float32) / 63
        Xe, Ye = torch.meshgrid(i64, i64, indexing='ij')
        rho_simp = (0.55 + 0.45 * torch.sin(3.1 * Xe + 0.4) * torch.cos(2.3 * Ye)).clamp(0.05, 1.0)[None]
        bce = torch.zeros(1, 4, 65, 65)
        bce[:, 0, :, 0] = 1.
        bce[:, 1, :, 0] = 1.
        bce[:, 3, 30:34, 64] = -0.25
        Kd = torch.zeros(st.neq, st.neq, dtype=torch.float64)
        kl = (st.tot_local_stiffness.double() * rho_simp.reshape(-1).double()[:, None, None])
        idx = st.glob_assembler_idcs
        Kd.index_put_((idx[:, :, 0].reshape(-1), idx[:, :, 1].reshape(-1)),
                      kl[:, st.indices_ext[:, 0], st.indices_ext[:, 1]].reshape(-1), accumulate=True)
        bcx = st.image_to_stiffness_coord(bce[:, 0], 0) + st.image_to_stiffness_coord(bce[:, 1], 1)
        fg = (st.image_to_stiffness_coord(bce[:, 2], 0) + st.image_to_stiffness_coord(bce[:, 3], 1))[0].double()
        mk = bcx[0] != 0
        Kd[mk] = 0
        Kd[mk, mk] = 1
        fg[mk] = 0
        u_data = torch.linalg.solve(Kd, fg).float()[None]
        sol = torch.stack((st.stiffness_to_image_coord(u_data, 0), st.stiffness_to_image_coord(u_data, 1)), dim=1)
        sol = torch.cat((sol, F_pad(rho_simp, (0, 1, 0, 1)).unsqueeze(1)), dim=1)              # [1,3,65,65]
        x_eval = torch.zeros(1, 3, 64, 64)
        x_eval[:, :2] = 0.05 * torch.randn(1, 2, 64, 64, generator=ge)
        x_eval[:, 2] = (rho_simp + 0.25 * torch.randn(1, 64, 64, generator=ge)).clamp(0, 1)
        mres_e = ResidualsMechanics(model=None, pixels_per_dim=64, pixels_at_boundary=True, no_BC_folder=td + '/',
                                    device='cpu', topopt_eval=True)
        vfe = torch.tensor([0.5])
        oe = mres_e.compute_residual((x_eval, bce, vfe, sol), reduce='per-batch', return_optimizer=True,
                                     return_inequality=True, sample=True, pass_through=True)
        save('mechanics_eval.pt', dict(x0_pred=x_eval, bcs=bce, vf=vfe, solution=sol,
                                       rel_CE_error=oe['rel_CE_error_full_batch'].clone(),
                                       vf_error=oe['vf_error_full_batch'].clone(),
                                       fm_error=oe['fm_error_full_batch'].clone()))

        # ---- mechanics training loss through the reference's model_estimation_loss (A3 + A13, configs[2] glue) ------
        # B = 2 with all four terms switched on (c_ineq > 0 pins the [B,1] x [B] broadcast of :679,:694)
        cfg_m = O.unet_config(dim=32, channels=10, out_dim=3, sigmoid_last_channel=True)
        sd_m = O.make_test_state_dict(cfg_m, seed=3)
        model_m = Unet3D(dim=32, channels=10, out_dim=3, sigmoid_last_channel=True)
        model_m.load_state_dict(sd_m, strict=True)
        model_m.train()
        mres_t = ResidualsMechanics(model=model_m, pixels_per_dim=64, pixels_at_boundary=True, no_BC_folder=td + '/',
                                    device='cpu', topopt_eval=False)
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
        torch.manual_seed(99)
        loss_m, data_m, res_m, ineq_m, opt_m = diff.model_estimation_loss(inp, residual_func=mres_t, **coefs)
        model_m.zero_grad()
        loss_m.backward()
        torch.manual_seed(99)
        t_m = torch.randint(0, 100, size=(B,))
        e_m = torch.randn_like(x0m)
        named_m = dict(model_m.named_parameters())
        save('mechanics_loss.pt', dict(input=inp, t=t_m, noise=e_m, loss=loss_m.detach(), data_loss=torch.tensor(data_m),
                                       residual_abs=torch.tensor(res_m), inequality=torch.tensor(ineq_m),
                                       compliance=torch.tensor(opt_m), coefs=torch.tensor(list(coefs.values())),
                                       grad_final_w=named_m['final_conv.1.weight'].grad.clone(),
                                       grad_init_w=named_m['init_conv.weight'].grad.clone(),
                                       grad_mid_w=named_m['downs.1.0.block1.proj.weight'].grad.clone()))


def toy_golden():
    """configs[0]: the toy study's loss (src/denoising_toy_utils.py:436-511) through the unmodified reference module, with
    the residual / inequality / optimisation callables of main_toy.py:48-79."""
    import src.denoising_toy_utils as T
    assert os.path.abspath(T.__file__).startswith(os.path.abspath(REF)), T.__file__
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
    out = {'x0': x0, **{'sd_' + k: v.clone() for k, v in model.state_dict().items()}}
    for tag, mode, ddim in (('x0_mean', 'x0', False), ('x0_sample', 'x0', True), ('eps_sample', 'eps', True)):
        torch.manual_seed(17)
        loss, data_l, res_l, ineq_l, opt_l = T.model_estimation_loss(
            model, x0, 100, dd, model_pred_mode=mode, residual_func=residual_func, ineq_func=ineq_func, opt_func=opt_func,
            c_data=1.0, c_residual=0.005, c_ineq=0.3, lambda_opt=0.01, use_ddim_x0=ddim, reduced_ddim_steps=0)
        model.zero_grad()
        loss.backward()
        out[tag + '_loss'] = loss.detach().clone()
        out[tag + '_tracked'] = torch.tensor([data_l, res_l, ineq_l, opt_l])
        out[tag + '_grad_lin3'] = model.lin3.weight.grad.clone()
        out[tag + '_grad_lin1'] = model.lin1.lin.weight.grad.clone()
        out[tag + '_grad_embed2'] = model.lin2.embed.weight.grad.clone()
    torch.manual_seed(17)                                  # replay the draws (:440-441, :447)
    t = torch.randint(0, 100, size=(128 // 2 + 1,))
    out['t'] = torch.cat([t, 100 - t - 1], dim=0)[:128].long()
    out['noise'] = torch.randn_like(x0)
    # short ancestral loop (x0 mode), draws replayed by the test: x_T then one z per step
    model.eval()
    d8 = T.create_diff_dict(8, 'cpu')
    torch.manual_seed(23)
    xs, _, _ = T.p_sample_loop(model, [64, 2], 8, d8, model_pred_mode='x0', save_output=False, surpress_noise=True)
    torch.manual_seed(23)
    out['loop_draws'] = torch.stack([torch.randn(64, 2) for _ in range(9)])
    out['loop_final'] = xs[-1]
    save('toy.pt', out)


if __name__ == '__main__':
    main()
    toy_golden()
