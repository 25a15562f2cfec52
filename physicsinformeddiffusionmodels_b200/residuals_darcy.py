"""`ResidualsDarcy` with the reference's constructor / method surface (reference src/residuals_darcy.py),
backed by the fused Darcy kernels of libpidm (csrc/darcy.cu)."""
import torch

from . import ops
from .grad_utils import GradientsHelper, generalized_b_xy_c_to_image, generalized_image_to_b_xy_c  # noqa: F401


class ResidualsDarcy:
    def __init__(self, model, fd_acc, pixels_per_dim, pixels_at_boundary, reverse_d1, device='cpu', bcs='none',
                 domain_length=1., residual_grad_guidance=False, use_ddim_x0=False, ddim_steps=0):
        self.gov_eqs = 'darcy'
        self.model = model
        self.pixels_at_boundary = pixels_at_boundary
        # bcs='periodic': wrapped central stencils at every pixel (reference grad_utils.py:76-81); h, f_s, the two BC
        # channels and the trapezoid weights are the same as with 'none'
        self.periodic = bcs == 'periodic'
        self.input_dim = 2
        d0 = domain_length / (pixels_per_dim - 1) if pixels_at_boundary else domain_length / pixels_per_dim
        d1 = -d0 if reverse_d1 else d0
        self.reverse_d1 = reverse_d1
        self.domain_length = domain_length
        self.grads = GradientsHelper(d0=d0, d1=d1, fd_acc=fd_acc, periodic=self.periodic, device=device)
        self.pixels_per_dim = pixels_per_dim
        self.device = device
        # stationary source field on the pixel-centre grid (reference :40-53,95-104)
        w, r = 0.125, 10.0
        ps = 1.0 / pixels_per_dim
        c = torch.linspace(ps / 2, 1.0 - ps / 2, steps=pixels_per_dim)
        X, Y = torch.meshgrid(c, c, indexing='ij')
        f = torch.zeros_like(X)
        f[torch.logical_and(torch.abs(X - 0.5 * w) <= 0.5 * w, torch.abs(Y - 0.5 * w) <= 0.5 * w)] = r
        f[torch.logical_and(torch.abs(X - 1 + 0.5 * w) <= 0.5 * w, torch.abs(Y - 1 + 0.5 * w) <= 0.5 * w)] = -r
        self.f_s = f.reshape(1, -1, 1).to(device)                 # [1, P*P, 1] like the reference
        self.f_s_flat = self.f_s.reshape(-1).contiguous()
        self.use_trapezoid = bool(pixels_at_boundary)
        if self.use_trapezoid:
            self.trapezoidal_weights = self.create_trapezoidal_weights()
        self.residual_grad_guidance = residual_grad_guidance
        self.use_ddim_x0 = use_ddim_x0
        self.ddim_steps = ddim_steps
        # (domain_length, reverse_d1, pixels_at_boundary, periodic): trailing arguments of ops.darcy_residual / _pidm_loss
        self.geometry = (float(domain_length), bool(reverse_d1), bool(pixels_at_boundary), self.periodic)

    def _abi_geometry(self):
        """(domain_length, reverse_d1, flags) as the Darcy C entry points take them"""
        dl, rev, pab, per = self.geometry
        return float(dl), int(rev), ops.darcy_flags(pab, per)

    def create_trapezoidal_weights(self):
        P = self.pixels_per_dim
        w = torch.full((1, P, P), 4.)
        w[..., 0, :] = 2.
        w[..., -1, :] = 2.
        w[..., :, 0] = 2.
        w[..., :, -1] = 2.
        for i in (0, -1):
            for j in (0, -1):
                w[..., i, j] = 1.
        w *= (1. / P) ** 2 / 4.
        return w.reshape(1, -1).to(self.device)

    # (x0_pred, model_out) for the residual / loss kernels
    def residual_gradient(self, noisy_in, world=1):
        """d mean|r(x_t)| / d x_t for x_t [B, P*P, 2] (reference :117-120), the residual evaluated on x_t itself: one
        kernel forms the cotangent sign(r) / n in registers and applies the adjoint stencils.  Returned in the b_xy_c
        layout of the input; it is data for the network (no graph is attached, as in the reference's
        torch.autograd.grad call).  world > 1: x_t is one of `world` equal shards of a global batch and the mean runs over
        the global batch (n = world * B * P*P * 3), as in the one-process run on that batch."""
        from ._lib import call, stream
        with torch.no_grad():
            img = generalized_b_xy_c_to_image(noisy_in.detach()).contiguous().float()
            B, _, P, _ = img.shape
            cond = torch.empty(B, P * P, 2, device=img.device, dtype=torch.float32)
            call('pidm_darcy_abs_residual_grad', img, self.f_s_flat, cond, B, world * B * P * P * 3, P,
                 *self._abi_geometry(), stream())
        return cond

    def predict_x0(self, model_input, ddim_func=None, sample=False, draw_shard=None):
        """draw_shard=(rank, world) (training only): the batch is this rank's shard of a global batch; the guidance
        gradient is normalised by the global count and the classifier-free mask is drawn for the global batch."""
        noisy_in, time = model_input
        if self.residual_grad_guidance:
            assert not self.use_ddim_x0, 'Residual gradient guidance is not implemented with sample estimation for residual.'
            dr_dx = self.residual_gradient(noisy_in, 1 if draw_shard is None else draw_shard[1])
            if sample:
                # NOTE (reference): "There is no mentioning of value for the guidance scale in the paper and repo"
                out = self.model.forward_with_guidance_scale(noisy_in, time, cond=dr_dx, guidance_scale=3.)
            elif draw_shard is not None:
                out = self.model(noisy_in, time, cond=dr_dx, null_cond_prob=0.1, draw_shard=draw_shard)
            else:
                out = self.model(noisy_in, time, cond=dr_dx, null_cond_prob=0.1)
            return out, out
        if self.use_ddim_x0:
            return ddim_func(noisy_in, time, self.model, noisy_in.shape, self.ddim_steps, 0.)
        out = self.model(noisy_in, time)
        return out, out

    def compute_residual(self, input, reduce='none', return_model_out=False, return_optimizer=False,
                         return_inequality=False, sample=False, ddim_func=None, pass_through=False):
        if pass_through:
            assert isinstance(input, torch.Tensor), 'Input is assumed to directly be given output.'
            x0_pred = model_out = input
        else:
            assert len(input[0]) == 2 and isinstance(input[0], tuple), \
                'Input[0] must be a tuple consisting of noisy signal and time.'
            x0_pred, model_out = self.predict_x0(input[0], ddim_func, sample=sample)
        assert len(x0_pred.shape) == 4, \
            'Model output must be a tensor shaped as an image (with explicit axes for the spatial dimensions).'
        residual = ops.darcy_residual(x0_pred, self.f_s_flat, *self.geometry)       # [B, P*P, 3]
        output = {'residual': residual}
        if return_model_out:
            output['model_out'] = model_out
        if reduce == 'full':
            return {k: v.mean() for k, v in output.items()}
        elif reduce == 'per-batch':
            return {k: v.mean(dim=tuple(range(1, v.ndim))) if v.ndim > 1 and (k != 'model_out' and k != 'residual') else v
                    for k, v in output.items()}
        elif reduce == 'none':
            return output
        raise ValueError('Unknown reduction method.')

    def cocogen(self, x, residual, steps, t=None, n_active=0):
        """`steps` CoCoGen corrections of x [B,2,P,P] (contiguous fp32, updated in place) in one launch
        (`pidm_darcy_cocogen`); residual [B,P*P,3] receives the residual of the corrected fields.  With t [B] int64 on
        the device only the samples with t[b] < n_active are corrected, and the other rows of x and residual are left
        as they are.  The step size 1e-6 / max dr/dp is computed once per launch: the corrections leave K unchanged."""
        from ._lib import call, stream
        ops._need_cuda(x, residual, t)
        ops._need_f32(x=x, residual=residual)
        B, C, P, _ = x.shape
        assert C == 2 and residual.shape == (B, P * P, 3), (x.shape, residual.shape)
        assert t is None or (t.dtype == torch.int64 and t.shape == (B,) and t.is_contiguous()), 't must be int64 [B]'
        call('pidm_darcy_cocogen', x, self.f_s_flat, residual, t, int(n_active), int(steps), B, P, *self._abi_geometry(),
             stream())
        return x, residual

    def residual_correction(self, x0_pred_in):
        """CoCoGen correction step (reference :209-240): p <- p - (1e-6 / max|dr/dp|) * d(sum r^2)/dp, residual re-evaluated.
        x0_pred_in [B, P*P, 2] is updated IN PLACE like the reference and returned with the corrected residual.
        The reference materialises the per-sample Jacobian dr/dp (12288 x 4096, vmap(jacfwd)) to take its maximum; the
        residual is linear in p, so the maximum is evaluated analytically from the stencil coefficients and K, and the
        whole step is one `pidm_darcy_cocogen` launch with steps = 1."""
        assert len(x0_pred_in.shape) == 3, 'Model output must be a tensor shaped as b_xy_c.'
        with torch.no_grad():
            img = generalized_b_xy_c_to_image(x0_pred_in).contiguous().float()          # [B,2,P,P]
            B, _, P, _ = img.shape
            residual_corrected = torch.empty(B, P * P, 3, device=img.device, dtype=torch.float32)
            self.cocogen(img, residual_corrected, 1)
            if img.data_ptr() != x0_pred_in.data_ptr():      # a copy was corrected: write p back into the caller's tensor
                x0_pred_in[:, :, 0] = img[:, 0].reshape(B, -1)
        return x0_pred_in, residual_corrected
