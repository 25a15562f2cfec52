"""Diffusion process with the reference's class surface (`DenoisingDiffusion`, `EMA`, `save_model`,
`load_model`, `fix_seeds`, layout helpers; reference src/denoising_utils.py), executed by libpidm kernels.

RNG: the draws (`randint` for t, `randn_like` for eps / z, `randn` for x_T) stay torch calls in the
reference's order so that identical seeds give identical draws on the same device type; everything
downstream of the draws is libpidm."""
import os
from pathlib import Path

import numpy as np
import torch
import torch.nn as nn
import yaml

from . import ops
from .grad_utils import generalized_b_xy_c_to_image, generalized_image_to_b_xy_c

device = torch.device('cuda' if torch.cuda.is_available() else 'cpu')


def fix_seeds(seed=42):
    torch.manual_seed(seed)
    torch.cuda.manual_seed(seed)
    np.random.seed(seed)


def image_to_b_xy_c(tensor):
    """[B, C, X, Y] -> [B, X*Y, C] (a view; reference :36-42)."""
    assert len(tensor.shape) == 4, 'Input tensor must have shape [batch, channels, x, y].'
    b, c, px, py = tensor.shape
    return torch.permute(tensor, (0, 2, 3, 1)).reshape(b, px * py, c)


def b_xy_c_to_image(tensor, pixels_x=None, pixels_y=None):
    """[B, X*Y, C] -> [B, C, X, Y] (reference :44-55)."""
    assert len(tensor.shape) == 3, 'Input tensor must have shape [batch, x*y, channels].'
    b, n, c = tensor.shape
    if pixels_x is None and pixels_y is None:
        assert np.sqrt(n) % 1 == 0, 'Number of pixels must be a perfect square.'
        pixels_x = pixels_y = int(np.sqrt(n))
    else:
        assert pixels_x * pixels_y == n, 'Number of given pixels must match dim 1 of input tensor.'
    return torch.permute(tensor.reshape(b, pixels_x, pixels_y, c), (0, 3, 1, 2))


def noop(*args, **kwargs):
    pass


def exists(x):
    return x is not None


def default(val, d):
    if exists(val):
        return val
    return d() if callable(d) else d


def image_array_to_gif(image_array, output_file, frame_duration=0.05, normalization_mode='final_pred',
                       given_min_max=None):
    raise NotImplementedError('GIF export is visualisation only and outside the built hot path (SURVEY.md section 2)')


class EMA(object):
    """Per-tensor EMA shadow with backup/restore (reference :163-205), as multi-tensor (foreach) updates.
    The flat-buffer engine (engine.py) fuses the same update into its Adam kernel."""

    def __init__(self, mu=0.999):
        self.mu = mu
        self.shadow = {}
        self.backup = {}

    def _named(self, module):
        return [(n, p) for n, p in module.named_parameters() if p.requires_grad]

    def register(self, module):
        for name, param in self._named(module):
            self.shadow[name] = param.data.clone()

    def update(self, module):
        named = self._named(module)
        sh = [self.shadow[n] for n, _ in named]
        torch._foreach_mul_(sh, self.mu)
        torch._foreach_add_(sh, [p.data for _, p in named], alpha=1. - self.mu)

    def ema(self, module, backup=True):
        named = self._named(module)
        for name, _ in named:
            assert name in self.shadow
        if backup:
            self.backup = {n: b for (n, _), b in zip(named, torch._foreach_add([p.data for _, p in named], 0.0))}
        torch._foreach_copy_([p.data for _, p in named], [self.shadow[n] for n, _ in named])

    def restore(self, module):
        named = self._named(module)
        for name, _ in named:
            assert name in self.backup
        torch._foreach_copy_([p.data for _, p in named], [self.backup[n] for n, _ in named])
        self.backup = {}

    def state_dict(self):
        return self.shadow

    def load_state_dict(self, state_dict):
        self.shadow = state_dict


def save_model(config, model, train_iterations, output_save_dir):
    """Weights-only checkpoint in the reference's format (reference :273-287)."""
    os.makedirs(Path(output_save_dir, 'model/'), exist_ok=True)
    with open(output_save_dir + '/model/model.yaml', 'w') as yaml_file:
        yaml.dump(dict(config), yaml_file, default_flow_style=False)
    path = output_save_dir + '/model/checkpoint_' + str(train_iterations) + '.pt'
    with open(path, 'wb') as f:
        torch.save(dict(model=model.state_dict()), f)
    print(f'\ncheckpoint saved to {output_save_dir}/.')


def load_model(path, model, strict=True):
    with open(path, 'rb') as f:
        loaded_obj = torch.load(f, map_location='cpu')
    try:
        model.load_state_dict(loaded_obj['model'], strict=strict)
    except RuntimeError:
        print('Failed loading state dict.')
    print('\nCheckpoint loaded from {}'.format(path))
    return model


def extract(input, t, x):
    out = torch.gather(input, 0, t.to(input.device))
    return out.reshape(t.shape[0], *([1] * (len(x.shape) - 1)))


def _cosine_betas(n_timesteps, s=0.008):
    x = torch.linspace(0, n_timesteps, n_timesteps + 1)
    ac = torch.cos(((x / n_timesteps) + s) / (1 + s) * torch.pi * 0.5) ** 2
    ac = ac / ac[0]
    return torch.clip(1 - (ac[1:] / ac[:-1]), 0, 0.999)


class _AxpbyPerSample(torch.autograd.Function):
    """out = a_b * x + b_b * y (+ c_b * z) with per-sample fp32 coefficients (DDIM jump of ddim_sample_x0)."""

    @staticmethod
    def forward(ctx, a, x, b, y):
        ctx.save_for_backward(a, b)
        zero = torch.zeros_like(a)
        return _axpby(a, x, b, y, zero, x)

    @staticmethod
    def backward(ctx, g):
        a, b = ctx.saved_tensors
        zero = torch.zeros_like(a)
        g = g.contiguous()
        return None, _axpby(a, g, zero, g, zero, g), None, _axpby(b, g, zero, g, zero, g)


def _axpby(a, x, b, y, c, z):
    from ._lib import call, stream
    out = torch.empty_like(x)
    call('pidm_axpby_per_sample', a, x.contiguous(), b, y.contiguous(), c, z.contiguous(), out, x.shape[0],
         x[0].numel(), stream())
    return out


def draw_t_and_noise(n_steps, x_0, draw_shard=None):
    """The two RNG draws of the training loss in the reference's order (denoising_utils.py:625,636): t ~ U{0..n_steps-1}
    per sample, then eps ~ N(0,1) of x_0's shape.  draw_shard=(rank, world): both are drawn for the GLOBAL batch
    (world * len(x_0) rows) and this rank's rows are sliced out, so that ranks with identical generator states consume
    exactly the random numbers of the one-process run on the concatenated batch (SURVEY 8e)."""
    B = len(x_0)
    rank, world = draw_shard if draw_shard is not None else (0, 1)
    lo, hi = rank * B, (rank + 1) * B
    t = torch.randint(0, n_steps, size=(B * world,), device=x_0.device)[lo:hi]
    if world == 1:
        e = torch.randn_like(x_0)
    else:
        e = torch.randn((B * world,) + tuple(x_0.shape[1:]), device=x_0.device, dtype=x_0.dtype)[lo:hi]
    return t, e


class DenoisingDiffusion(nn.Module):
    def __init__(self, n_steps, device, residual_grad_guidance=False):
        # like the reference, nn.Module.__init__ is deliberately not called (no parameters are owned)
        self.n_steps = n_steps
        self.device = device
        self.diff_dict = self.create_diff_dict()
        self.residual_grad_guidance = residual_grad_guidance
        self.sync_scalars = True     # False: tracked scalars are returned as device tensors (no host sync)

    # ---- A1: schedule tables (reference :315-370), computed once on the host in fp32, then moved -----------
    def create_diff_dict(self):
        d = {}
        b = _cosine_betas(self.n_steps)
        d['betas'] = b
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
        app = torch.cat([torch.ones(1), ap[:-1]], 0)
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
        self._host_tables = {k: v.clone() for k, v in d.items()}
        return {k: v.to(self.device).contiguous() for k, v in d.items()}

    # ---- A4 ---------------------------------------------------------------------------------------------------
    def q_sample(self, x_0, t, alphas_bar_sqrt, one_minus_alphas_bar_sqrt, noise=None):
        if noise is None:
            noise = torch.randn_like(x_0)
        return ops.q_sample(x_0, noise, t, alphas_bar_sqrt, one_minus_alphas_bar_sqrt)

    # ---- A3: training loss (reference :616-710) ------------------------------------------------------------
    def model_estimation_loss(self, input, residual_func=None, c_data=1., c_residual=0., c_ineq=0., lambda_opt=0.,
                              sync_scalars=None, draw_shard=None):
        """Reference signature plus two keyword extensions used by engine.TrainEngine:
        sync_scalars=False returns the tracked scalars as device tensors (no host sync; default: self.sync_scalars);
        draw_shard=(rank, world): t / eps are drawn for the GLOBAL batch (world * len(input) rows) and sliced to this
        rank's rows -- with identical generator states on all ranks the data-parallel job consumes the same random
        numbers as the one-process run on the concatenated batch (SURVEY 8e)."""
        sync = self.sync_scalars if sync_scalars is None else sync_scalars
        if residual_func.gov_eqs == 'darcy':
            t, e = draw_t_and_noise(self.n_steps, input, draw_shard)
            return self.darcy_loss_from_draws(input, t, e, residual_func, c_data, c_residual, sync_scalars=sync,
                                              draw_shard=draw_shard)
        if residual_func.gov_eqs == 'mechanics':
            return residual_func.training_loss(self, input, None, c_data, c_residual, c_ineq, lambda_opt,
                                               sync_scalars=sync, draw_shard=draw_shard)
        raise ValueError('Unknown governing equations.')

    def darcy_loss_from_draws(self, x_0, t, e, residual_func, c_data=1., c_residual=0., sync_scalars=None,
                              draw_shard=None):
        """The body of model_estimation_loss for Darcy after the t / eps draws: q_sample -> U-Net (-> DDIM walk) ->
        fused residual + loss kernel.  Returns (loss, data_loss, mean|r|, 0., 0.).  With residual-gradient guidance the
        network draws the classifier-free mask (for the global batch under draw_shard)."""
        dd = self.diff_dict
        x = ops.q_sample(x_0, e, t, dd['alphas_bar_sqrt'], dd['one_minus_alphas_bar_sqrt'])
        kw = {} if draw_shard is None else {'draw_shard': draw_shard}
        x0_hat, model_out = residual_func.predict_x0((image_to_b_xy_c(x), t), ddim_func=self.ddim_sample_x0, **kw)
        loss, sums = ops.darcy_pidm_loss(x0_hat, model_out, x_0, t, residual_func.f_s_flat, dd['p2_loss_weight'],
                                         dd['posterior_variance_clipped'], c_data, c_residual, *residual_func.geometry)
        if self.sync_scalars if sync_scalars is None else sync_scalars:
            s = sums.tolist()                   # one host sync (the reference does two .item() calls here)
            return loss, s[0], s[2], 0., 0.
        return loss, sums[0], sums[2], 0., 0.

    # ---- A11: ancestral sampling (reference :388-545) -----------------------------------------------------
    def p_sample(self, x, conditioning_input, t, save_output=False, surpress_noise=False, use_dynamic_threshold=False,
                 residual_func=None, eval_residuals=False, return_optimizer=False, return_inequality=False,
                 residual_correction=False, correction_mode='none'):
        assert correction_mode in ['x0', 'xt'] or not residual_correction, 'Correction mode unknown or not given.'
        if residual_correction and residual_func.gov_eqs != 'darcy':
            raise ValueError('CoCoGen correction is only implemented for the Darcy flow study (reference main.py:37-38).')
        if use_dynamic_threshold:
            raise NotImplementedError('dynamic thresholding is not used by the reference drivers')
        dd = self.diff_dict
        x_init = x.detach()
        batch_size = len(x)
        t_vec = torch.full((batch_size,), int(t), device=x.device, dtype=torch.long)
        if residual_func.gov_eqs == 'darcy':
            model_in = (image_to_b_xy_c(x_init), t_vec)
            out_dict = residual_func.compute_residual((model_in,), reduce='per-batch', return_model_out=True,
                                                      return_optimizer=return_optimizer,
                                                      return_inequality=return_inequality, sample=True,
                                                      ddim_func=self.ddim_sample_x0)
        else:
            out_dict = residual_func.sampling_residual(self, x_init, conditioning_input, t_vec, return_optimizer,
                                                       return_inequality, sample=(int(t) == 0))
        model_out, residual = out_dict['model_out'], out_dict['residual']
        if len(model_out.shape) == 3:
            model_out = generalized_b_xy_c_to_image(model_out)
        if residual_correction and correction_mode == 'x0':                   # CoCoGen on the x0 estimate (reference :433-435)
            mo, residual = residual_func.residual_correction(generalized_image_to_b_xy_c(model_out.detach().clone()))
            model_out = generalized_b_xy_c_to_image(mo)
        model_intermediate = model_out.detach() if save_output else None
        z = torch.randn_like(x_init)                                  # drawn even at t == 0 (reference :447)
        ht = self._host_tables
        sigma = float(ht['betas'][t].sqrt())
        if surpress_noise and int(t) == 0:
            sigma = 0.
        sample = ops.posterior_step(x_init, model_out.detach(), z, float(ht['posterior_mean_coef1'][t]),
                                    float(ht['posterior_mean_coef2'][t]), sigma)
        if residual_correction and correction_mode == 'xt':                   # CoCoGen on the new sample (reference :455-457)
            sm, residual = residual_func.residual_correction(generalized_image_to_b_xy_c(sample))
            sample = generalized_b_xy_c_to_image(sm).contiguous()
        if int(t) == 0 and eval_residuals:
            aux_out = {'residual': residual}
            if return_optimizer:
                aux_out['optimized_quant'] = out_dict['optimizer']
            if return_inequality:
                aux_out['inequality_quant'] = out_dict['inequality']
            for k in ('rel_CE_error_full_batch', 'vf_error_full_batch', 'fm_error_full_batch'):
                if k in out_dict:
                    aux_out[k] = out_dict[k]
            return (sample, model_intermediate), aux_out
        return (sample, model_intermediate), None

    def p_sample_loop(self, conditioning_input, shape, save_output=False, surpress_noise=True,
                      use_dynamic_threshold=False, residual_func=None, eval_residuals=False, return_optimizer=False,
                      return_inequality=False, M_correction=0, N_correction=0, correction_mode='none'):
        dev = self.diff_dict['alphas'].device
        cur_x = torch.randn(shape, device=dev)
        # the trajectory stays on the device during the loop; ONE device->host transfer at the end
        dev_seq = [cur_x]
        dev_interm = []
        output = None
        with torch.no_grad():
            for i in reversed(range(self.n_steps)):
                residual_correction = False
                if i < N_correction:                                           # CoCoGen: correct during the last N steps
                    residual_correction = True
                    eval_residuals = True
                output = self.p_sample(cur_x, conditioning_input, i, save_output, surpress_noise, use_dynamic_threshold,
                                       residual_func=residual_func, eval_residuals=eval_residuals,
                                       return_optimizer=return_optimizer, return_inequality=return_inequality,
                                       residual_correction=residual_correction, correction_mode=correction_mode)
                cur_x, interm_img = output[0]
                dev_seq.append(cur_x)
                if interm_img is not None:
                    dev_interm.append(interm_img)
            for i in range(M_correction):                                      # CoCoGen: M extra corrections of x_0
                # (the correction works in place: keep the trajectory entry recorded above intact)
                cm, residual = residual_func.residual_correction(generalized_image_to_b_xy_c(cur_x.clone()))
                cur_x = generalized_b_xy_c_to_image(cm).contiguous()
                dev_seq.append(cur_x)
                if eval_residuals and i == M_correction - 1:
                    output[1]['residual'] = residual
        x_seq = list(torch.stack(dev_seq).cpu().unbind(0))
        interm_imgs = [torch.zeros(shape)] if save_output else []
        if dev_interm:
            interm_imgs += list(torch.stack(dev_interm).cpu().unbind(0))
        if eval_residuals:
            return (x_seq, interm_imgs), output[1]
        return x_seq, interm_imgs

    def gaussian_log_likelihood(self, x, means, variance):
        return -0.5 * ((x - means) ** 2) / variance

    def predict_noise_from_mean(self, x_t, t, mean_t):
        dd = self.diff_dict
        return (extract(dd['sqrt_recip_alphas'], t, mean_t) * x_t - mean_t) / extract(dd['noise_mean_coeff'], t, mean_t)

    # ---- A12: x0 estimate by a short DDIM walk (reference :712-787) -------------------------------------------
    def ddim_sample_x0(self, xt, t, model, shape, reduced_n_steps, ddim_sampling_eta, gov_eqs=None, self_cond=None):
        """Per-sample time grids linspace(0, t, steps+2) built ON THE DEVICE (the reference loops over the batch on
        the host).  Reference quirk kept: every network call sees the ORIGINAL x_t; only `t` advances (:741-753)."""
        if ddim_sampling_eta != 0.:
            raise NotImplementedError('only eta = 0 (deterministic DDIM, the reference call sites) is implemented')
        dd = self.diff_dict
        batch = shape[0]
        dev = dd['alphas'].device
        batch_t = (torch.ones(batch, device=dev, dtype=torch.long) * t) if len(t) == 1 else t
        n_pts = reduced_n_steps + 2
        k = torch.arange(n_pts, device=dev, dtype=torch.float64)
        # int() truncation of np.linspace, whose step is t / (n_pts - 1): divided by a device tensor, since a CUDA
        # tensor divided by a Python scalar is multiplied by its reciprocal, which can round the step low and a grid
        # point one lower (t = 14 on 7 points gives 6 for 7)
        step = batch_t.double() / torch.full_like(batch_t, n_pts - 1, dtype=torch.float64)
        grid = (k[None, :] * step[:, None]).long()
        grid[:, -1] = batch_t
        cur_times = grid.flip(1).T.contiguous()                                        # [n_pts, B]: t, ..., 0
        next_times = torch.cat([grid.new_full((batch, 1), -1), grid[:, :-1]], dim=1).flip(1).T.contiguous()
        if len(xt.shape) == 3:
            xt = generalized_b_xy_c_to_image(xt)
        model_input = xt
        cur_x = xt[:, :3] if gov_eqs == 'mechanics' else xt
        model_out = None
        for idx in range(n_pts):
            tt, tn = cur_times[idx], next_times[idx]
            x0_pred = model(model_input, tt, self_cond)
            if idx == 0:
                model_out = x0_pred
            if idx == n_pts - 1:                       # t_next == -1 for every sample: the walk ends on x0_pred
                cur_x = x0_pred
                continue
            # mean = c1 x0 + c2 x ; eps = (sra x - mean)/nmc ; x' = sqrt(a_next) x0 + sqrt(1-a_next) eps   (eta = 0):
            # the per-sample coefficients of x0 and x in ONE launch (pidm_ddim_coefs)
            from ._lib import call, stream
            coef_x0 = torch.empty(batch, device=dev, dtype=torch.float32)
            coef_x = torch.empty(batch, device=dev, dtype=torch.float32)
            call('pidm_ddim_coefs', tt, tn, dd['posterior_mean_coef1'], dd['posterior_mean_coef2'], dd['sqrt_recip_alphas'],
                 dd['noise_mean_coeff'], dd['alphas_prod'], coef_x0, coef_x, batch, stream())
            _ = torch.randn_like(cur_x)                # RNG parity: the reference draws noise even when sigma = 0
            cur_x = _AxpbyPerSample.apply(coef_x0, x0_pred, coef_x, cur_x)
        assert model_out is not None, 'Model output not given.'
        return cur_x, model_out
