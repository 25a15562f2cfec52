"""Toy study of the reference (`main_toy.py`, `src/denoising_toy_utils.py`; BASELINE.json configs[0]): diffusion on
2-D points with a user-supplied residual / inequality / optimisation callable, same function surface, so that the
reference's `main_toy.py` runs unchanged on top of `src/denoising_toy_utils.py`.

What runs where.  The point model (`ConditionalModel`, a 2 -> 128 -> 128 -> 2 MLP with per-timestep gains) and the three
callables defined by the driver are ordinary torch modules -- they are user code by design.  The diffusion algebra around
them goes through libpidm like the image path: q_sample (`pidm_qsample`), the DDIM jump (`pidm_axpby_per_sample`), the
ancestral step (`pidm_posterior_step` / `pidm_axpby_per_sample`) and the whole PIDM loss -- p2-weighted data term, clamped
Gaussian NLL of residual and inequality, optimisation term -- with its gradients in ONE kernel (`pidm_toy_pidm_loss`).
Like the rest of the package it needs CUDA tensors: there is no CPU fallback (the reference picks `cuda:0` when present).

`model_pred_mode`: 'x0' (the reference default) and 'eps' are implemented; 'mu' (variational loss) raises."""
import os

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import ops
from ._lib import call, stream
from .denoising_utils import _axpby, _AxpbyPerSample, _cosine_betas, default, exists, extract, fix_seeds, noop  # noqa: F401

device = torch.device('cuda:0' if torch.cuda.is_available() else 'cpu')


# ---- data ------------------------------------------------------------------------------------------------------------
def sample_zeros(size):
    return np.zeros((size, 2))


def sample_gaussian(size, dim=2):
    return np.random.randn(size, dim)


def sample_hypersphere(size, dim):
    """points on the unit hypersphere surface (reference :111-120)"""
    x = np.random.normal(0, 1, (size, dim))
    return x / np.linalg.norm(x, axis=1, keepdims=True)


def sample_two_points(size):
    x = np.array([[-0.5, -0.5], [0.5, 0.5]])
    return x[np.random.randint(2, size=size)]


def sample_four_points(size):
    x = np.array([[-1., -1.], [-1., 1.], [1., -1.], [1., 1.]])
    return x[np.random.randint(4, size=size)]


def right_pad_dims_to(x, t):
    padding_dims = x.ndim - t.ndim
    return t if padding_dims <= 0 else t.view(*t.shape, *((1,) * padding_dims))


# ---- schedule (reference :42-89; the same cosine tables as the image path) -------------------------------------------
def make_beta_schedule(schedule='linear', n_timesteps=1000, start=1e-5, end=1e-2):
    if schedule == 'linear':
        return torch.linspace(start, end, n_timesteps)
    if schedule == 'quad':
        return torch.linspace(start ** 0.5, end ** 0.5, n_timesteps) ** 2
    if schedule == 'sigmoid':
        return torch.sigmoid(torch.linspace(-6, 6, n_timesteps)) * (end - start) + start
    if schedule == 'cosine':
        return _cosine_betas(n_timesteps)
    raise ValueError(schedule)


def create_diff_dict(n_steps, device):
    b = make_beta_schedule('cosine', n_steps)
    d = {'betas': b}
    a = 1. - b
    d['alphas'] = a
    d['sqrt_recip_alphas'] = torch.sqrt(1. / a)
    ap = torch.cumprod(a, 0)
    d['alphas_prod'] = ap
    d['alphas_prod_p'] = torch.cat([torch.ones(1), ap[:-1]], 0)
    d['alphas_bar_sqrt'] = torch.sqrt(ap)
    d['sqrt_recip_alphas_cumprod'] = torch.sqrt(1. / ap)
    d['sqrt_recipm1_alphas_cumprod'] = torch.sqrt(1. / ap - 1)
    d['one_minus_alphas_bar_log'] = torch.log(1 - ap)
    d['one_minus_alphas_bar_sqrt'] = torch.sqrt(1 - ap)
    app = F.pad(ap[:-1], (1, 0), value=1.)
    d['alphas_prod_prev'] = app
    d['posterior_mean_coef1'] = b * torch.sqrt(app) / (1. - ap)
    d['posterior_mean_coef2'] = (1. - app) * torch.sqrt(a) / (1. - ap)
    d['noise_mean_coeff'] = torch.sqrt(1. / a) * (1. - a) / torch.sqrt(1. - ap)
    pv = b * (1. - app) / (1. - ap)
    d['posterior_variance'] = pv
    pvc = pv.clone()
    pvc[0] = pv[1]
    d['posterior_variance_clipped'] = pvc
    d['posterior_log_variance_clipped'] = torch.log(pvc)
    snr = ap / (1. - ap)
    d['p2_loss_weight'] = torch.minimum(snr, torch.ones_like(snr) * 5.0)
    return {k: v.to(device).float().contiguous() for k, v in d.items()}


# ---- model (user-side torch modules; state_dict keys as in the reference :171-199) -----------------------------------
class ConditionalLinear(nn.Module):
    def __init__(self, num_in, num_out, n_steps):
        super().__init__()
        self.num_out = num_out
        self.lin = nn.Linear(num_in, num_out)
        self.embed = nn.Embedding(n_steps, num_out)
        self.embed.weight.data.uniform_()

    def forward(self, x, y):
        return self.embed(y).view(-1, self.num_out) * self.lin(x)


class ConditionalModel(nn.Module):
    def __init__(self, dim, n_steps):
        super().__init__()
        self.lin1 = ConditionalLinear(dim, 128, n_steps)
        self.lin2 = ConditionalLinear(128, 128, n_steps)
        self.lin3 = nn.Linear(128, dim)

    def forward(self, x, y):
        x = F.softplus(self.lin1(x, y))
        x = F.softplus(self.lin2(x, y))
        return self.lin3(x)


# ---- diffusion algebra through libpidm --------------------------------------------------------------------------------
def _need_cuda(x):
    if not x.is_cuda:
        raise RuntimeError('physicsinformeddiffusionmodels_b200 (toy study) runs on CUDA tensors only: no CPU fallback')


def q_sample(x_0, t, alphas_bar_sqrt, one_minus_alphas_bar_sqrt, noise=None):
    if noise is None:
        noise = torch.randn_like(x_0)
    if len(t) == 1 and len(x_0) != 1:
        t = t.expand(len(x_0))
    return ops.q_sample(x_0, noise, t, alphas_bar_sqrt, one_minus_alphas_bar_sqrt)


def predict_start_from_noise(x_t, t, noise, diff_dict):
    """x0 = sqrt(1/abar) x_t - sqrt(1/abar - 1) eps  (differentiable w.r.t. both tensors)"""
    a = diff_dict['sqrt_recip_alphas_cumprod'][t].contiguous()
    b = (-diff_dict['sqrt_recipm1_alphas_cumprod'][t]).contiguous()
    return _AxpbyPerSample.apply(a, x_t, b, noise)


def predict_noise_from_mean(x_t, t, mean_t, diff_dict):
    inv = 1. / diff_dict['noise_mean_coeff'][t]
    return _AxpbyPerSample.apply((diff_dict['sqrt_recip_alphas'][t] * inv).contiguous(), x_t, (-inv).contiguous(), mean_t)


def gaussian_log_likelihood(x, means, variance, return_full=False):
    """-0.5 (x - mu)^2 / var, clamped at -27.631 (reference :372-383; used by user code, the loss below is fused)"""
    ll = -0.5 * ((x - means) ** 2) / variance
    if return_full:
        ll = ll - 0.5 * (torch.log(variance) + np.log(2 * np.pi))
    return torch.clamp(ll, min=-27.6310211159)


class _ToyPidmLoss(torch.autograd.Function):
    """All loss terms of reference :453-511 and their gradients w.r.t. (output, residual, ineq, opt) in one launch."""

    @staticmethod
    def forward(ctx, target, output, residual, ineq, opt, t, p2w, pvar, coefs):
        B, D = output.shape
        sums = torch.empty(7, device=output.device, dtype=torch.float32)
        g_out, g_r = torch.empty_like(output), torch.empty_like(residual)
        g_q = None if ineq is None else torch.empty_like(ineq)
        g_o = None if opt is None else torch.empty_like(opt)
        call('pidm_toy_pidm_loss', target, output, residual, ineq, opt, t, p2w, pvar, *[float(c) for c in coefs], sums,
             g_out, g_r, g_q, g_o, B, D, stream())
        ctx.save_for_backward(g_out, g_r, g_q, g_o)
        ctx.mark_non_differentiable(sums)
        return sums[0] + sums[1] + sums[2] + sums[3], sums

    @staticmethod
    def backward(ctx, g, _unused):
        g = g.contiguous().float()
        outs = []
        for t_ in ctx.saved_tensors:
            if t_ is None:
                outs.append(None)
                continue
            o = torch.empty_like(t_)
            call('pidm_scale', t_, g, o, t_.numel(), stream())
            outs.append(o)
        return (None, outs[0], outs[1], outs[2], outs[3], None, None, None, None)


def model_estimation_loss(model, x_0, n_steps, diff_dict, model_pred_mode='eps', residual_func=None, ineq_func=None,
                          opt_func=None, c_data=1., c_residual=0., c_ineq=0., lambda_opt=0., use_ddim_x0=False,
                          reduced_ddim_steps=0):
    """Reference :436-511.  RNG draws in the reference's order: antithetic t (randint of B//2+1, mirrored), then eps."""
    _need_cuda(x_0)
    batch_size = x_0.shape[0]
    t = torch.randint(0, n_steps, size=(batch_size // 2 + 1,), device=x_0.device)
    t = torch.cat([t, n_steps - t - 1], dim=0)[:batch_size].long().contiguous()
    x_0 = x_0.contiguous().float()
    e = torch.randn_like(x_0)
    x = ops.q_sample(x_0, e, t, diff_dict['alphas_bar_sqrt'], diff_dict['one_minus_alphas_bar_sqrt'])
    output = model(x, t)
    if model_pred_mode == 'eps':
        target, p2w = e, None
        x_0_pred = predict_start_from_noise(x, t, output, diff_dict)
    elif model_pred_mode == 'x0':
        target, p2w = x_0, diff_dict['p2_loss_weight']
        x_0_pred = output
    elif model_pred_mode == 'mu':
        raise NotImplementedError("model_pred_mode='mu' (variational loss, reference :385-434) is not built; use 'x0' "
                                  "(the reference default) or 'eps'")
    else:
        raise ValueError('model_pred_mode not recognized.')
    if use_ddim_x0:
        eval_x0 = ddim_sample_x0(x, t, model, x.shape, reduced_ddim_steps, 0, diff_dict, model_pred_mode=model_pred_mode)
    else:
        eval_x0 = x_0_pred
    residual = residual_func(eval_x0).contiguous().float()
    ineq = ineq_func(eval_x0)[0].contiguous().float() if ineq_func is not None else None
    opt = opt_func(eval_x0).contiguous().float() if opt_func is not None else None
    loss, sums = _ToyPidmLoss.apply(target.contiguous(), output.contiguous().float(), residual, ineq, opt, t, p2w,
                                    diff_dict['posterior_variance_clipped'], (c_data, c_residual, c_ineq, lambda_opt))
    s = sums.tolist()                      # one host sync for the four tracked scalars (the reference does four .item())
    # reference quirk kept (:477-478,:491): `data_loss = loss` aliases the tensor that `loss += ...` updates in place, so
    # the second return value is the TOTAL loss, not the data term
    return loss, s[0] + s[1] + s[2] + s[3], s[4], s[5], s[6]


def ddim_sample_x0(xt, t, model, shape, reduced_n_steps, ddim_sampling_eta, diff_dict, model_pred_mode='eps'):
    """x0 estimate by a short deterministic DDIM walk (reference :267-333), time grids built on the device.  Unlike the
    image path (whose reference feeds the original x_t to every call) the toy reference advances cur_x."""
    if ddim_sampling_eta != 0:
        raise NotImplementedError('only eta = 0 (the reference call sites) is implemented')
    batch, dev = shape[0], diff_dict['alphas'].device
    batch_t = (torch.ones(batch, device=dev, dtype=torch.long) * t) if len(t) == 1 else t
    n_pts = reduced_n_steps + 2
    k = torch.arange(n_pts, device=dev, dtype=torch.float64)
    # int() truncation of np.linspace, whose step is t / (n_pts - 1): divided by a device tensor, since a CUDA
    # tensor divided by a Python scalar is multiplied by its reciprocal, which can round the step low and a grid
    # point one lower (t = 14 on 7 points gives 6 for 7)
    step = batch_t.double() / torch.full_like(batch_t, n_pts - 1, dtype=torch.float64)
    grid = (k[None, :] * step[:, None]).long()
    grid[:, -1] = batch_t
    cur_times = grid.flip(1).T.contiguous()
    next_times = torch.cat([grid.new_full((batch, 1), -1), grid[:, :-1]], dim=1).flip(1).T.contiguous()
    cur_x, x0_pred = xt, None
    dd = diff_dict
    for idx in range(n_pts):
        tt, tn = cur_times[idx], next_times[idx]
        out = model(cur_x, tt)
        if model_pred_mode == 'eps':
            eps_theta = out
            x0_pred = predict_start_from_noise(cur_x, tt, out, dd)
        elif model_pred_mode == 'x0':
            x0_pred = out
            eps_theta = None
        else:
            raise NotImplementedError("model_pred_mode='mu' is not built")
        if idx == n_pts - 1:
            cur_x = x0_pred
            continue
        a_next = dd['alphas_prod'][tn.clamp_min(0)]
        c = (1 - a_next).sqrt()
        keep = (tt == tn).float()
        _ = torch.randn_like(cur_x)                     # RNG parity: the reference draws noise even when sigma = 0
        if model_pred_mode == 'x0':
            # eps = (sra x - (c1 x0 + c2 x)) / nmc  ->  x' = (sqrt(a') - c c1 / nmc) x0 + c (sra - c2) / nmc x
            c1, c2 = dd['posterior_mean_coef1'][tt], dd['posterior_mean_coef2'][tt]
            sra, nmc = dd['sqrt_recip_alphas'][tt], dd['noise_mean_coeff'][tt]
            coef_a = (1 - keep) * (a_next.sqrt() - c * c1 / nmc)
            coef_x = keep + (1 - keep) * (c * (sra - c2) / nmc)
            cur_x = _AxpbyPerSample.apply(coef_a.contiguous(), x0_pred, coef_x.contiguous(), cur_x)
        else:
            # x' = sqrt(a') x0 + c eps with x0 = ra x - rm eps  ->  x' = sqrt(a') ra x + (c - sqrt(a') rm) eps
            ra, rm = dd['sqrt_recip_alphas_cumprod'][tt], dd['sqrt_recipm1_alphas_cumprod'][tt]
            coef_x = keep + (1 - keep) * a_next.sqrt() * ra
            coef_e = (1 - keep) * (c - a_next.sqrt() * rm)
            cur_x = _AxpbyPerSample.apply(coef_x.contiguous(), cur_x, coef_e.contiguous(), eps_theta)
    return cur_x


def p_sample(model, x, t, diff_dict, model_pred_mode='eps', save_output=False, surpress_noise=False,
             use_dynamic_threshold=False, reduced_ddim_steps=0):
    """One ancestral step (reference :201-265) -> (sample, model_output, x0_estimation)."""
    if use_dynamic_threshold:
        raise NotImplementedError('dynamic thresholding is not used by the reference driver')
    _need_cuda(x)
    ti = int(t)
    t = torch.tensor([ti], device=x.device)
    tb = t.expand(len(x))
    dd = diff_dict
    out = model(x, t)
    model_output = out.clone().detach() if save_output else None
    z = torch.randn_like(x)
    sigma = float(dd['betas'][ti].sqrt()) if not (surpress_noise and ti == 0) else 0.
    if model_pred_mode == 'x0':
        x0_pred = out
        sample = ops.posterior_step(x, out.detach(), z, float(dd['posterior_mean_coef1'][ti]),
                                    float(dd['posterior_mean_coef2'][ti]), sigma)
    elif model_pred_mode == 'eps':
        x0_pred = predict_start_from_noise(x, tb, out, dd)
        ia = float(1. / dd['alphas'][ti].sqrt())
        ef = float((1 - dd['alphas'][ti]) / dd['one_minus_alphas_bar_sqrt'][ti])
        B = len(x)
        full = lambda v: torch.full((B,), v, device=x.device, dtype=torch.float32)   # noqa: E731
        sample = _axpby(full(ia), x, full(-ia * ef), out.detach(), full(sigma), z)
    else:
        raise NotImplementedError("model_pred_mode='mu' is not built")
    x0_estimation = None
    if save_output:
        x0_estimation = ddim_sample_x0(x, t, model, x.shape, reduced_ddim_steps, 0, dd, model_pred_mode=model_pred_mode) \
            if ti > 0 else x0_pred
    return sample, model_output, x0_estimation


def p_sample_loop(model, shape, n_steps, diff_dict, model_pred_mode='x0', save_output=False, surpress_noise=True,
                  use_dynamic_threshold=False, reduced_ddim_steps=0):
    """Reference :267-288; the trajectory stays on the device and is copied to the host ONCE at the end."""
    dev = diff_dict['alphas'].device
    cur_x = torch.randn(shape, device=dev)
    xs, mos, x0s = [cur_x], [], []
    with torch.no_grad():
        for i in reversed(range(n_steps)):
            cur_x, mo, x0e = p_sample(model, cur_x.detach(), i, diff_dict, model_pred_mode, save_output, surpress_noise,
                                      use_dynamic_threshold, reduced_ddim_steps=reduced_ddim_steps)
            xs.append(cur_x)
            if save_output:
                mos.append(mo)
                x0s.append(x0e)
    x_seq = list(torch.stack(xs).cpu().unbind(0))
    if save_output:
        model_outputs = [torch.zeros(shape)] + list(torch.stack(mos).cpu().unbind(0))
        x0_estimations = [torch.zeros(shape)] + list(torch.stack(x0s).cpu().unbind(0))
    else:
        model_outputs, x0_estimations = [], []
    return x_seq, model_outputs, x0_estimations


# ---- checkpoints (reference :527-594: weights by torch.save, the three callables by dill) ----------------------------
def save_model(model, name, diff_dict, step, n_steps, dim, model_pred_mode, residual_func, ineq_func, opt_func):
    import dill
    save_dir = './trained_models/toy/' + name + '/model'
    os.makedirs(save_dir, exist_ok=True)
    base = save_dir + '/checkpoint_' + str(step)
    with open(base + '.pt', 'wb') as f:
        torch.save(dict(model=model.state_dict(), n_steps=n_steps, dim=dim, model_pred_mode=model_pred_mode,
                        diff_dict=diff_dict), f)
    for tag, fn in (('residual_func', residual_func), ('ineq_func', ineq_func), ('opt_func', opt_func)):
        with open(f'{base}_{tag}.pkl', 'wb') as f:
            dill.dump(fn, f)
    print(f'checkpoint saved to {save_dir}')


def load_model(path, strict=True):
    import dill
    with open(path, 'rb') as f:
        obj = torch.load(f, map_location='cpu')
    model = ConditionalModel(obj['dim'], obj['n_steps'])
    model.load_state_dict(obj['model'], strict=strict)
    fns = []
    for tag in ('residual_func', 'ineq_func', 'opt_func'):
        with open(path.replace('.pt', f'_{tag}.pkl'), 'rb') as f:
            fns.append(dill.load(f))
    return (model, obj['diff_dict'], obj['n_steps'], obj['dim'], obj['model_pred_mode'], *fns)


def remove_outliers(data, percentile=0.01, also_lower_bound=False):
    percentile *= 100
    if data.size == 0:
        return data
    norms = np.linalg.norm(data, axis=1)
    lower = np.percentile(norms, percentile) if also_lower_bound else 0.
    upper = np.percentile(norms, 100 - percentile)
    return data[(norms > lower) & (norms < upper)]


def array_to_gif(data, output_save_dir, x_lim, y_lim, label=None, duration=0.05, s=10):
    raise NotImplementedError('GIF export is visualisation only and outside the built hot path (SURVEY.md section 2)')
