"""`ResidualsMechanics` with the reference's constructor / method surface (reference
src/residuals_mechanics_K.py), evaluated MATRIX-FREE by libpidm (csrc/mechanics.cu): the reference's dense
B x 8450 x 8450 stiffness assembly (285.6 MB per sample) is never formed.

Mesh convention (the authors' mesh files are an external download, SURVEY.md section 8c): the structured
unit-square mesh with node id = row*65 + col, dof = 2*node + d and counter-clockwise Q4 elements
n1=(er+1,ec), n2=(er+1,ec+1), n3=(er,ec+1), n4=(er,ec); with it the element->dof map is implicit and
`no_BC_folder` is not read.  Element stiffness: closed-form plane-stress Q4, E = 1, nu = 0.3 (the reference
overrides the material file with exactly these values, residuals_mechanics_K.py:30-33)."""
import torch
import torch.nn.functional as F  # noqa: F401  (re-exported name of the reference module)

from ._lib import call, stream
from .grad_utils import generalized_b_xy_c_to_image, generalized_image_to_b_xy_c  # noqa: F401


def q4_plane_stress_stiffness(E=1.0, nu=0.3):
    k = [1 / 2 - nu / 6, 1 / 8 + nu / 8, -1 / 4 - nu / 12, -1 / 8 + 3 * nu / 8,
         -1 / 4 + nu / 12, -1 / 8 - nu / 8, nu / 6, 1 / 8 - 3 * nu / 8]
    idx = [[0, 1, 2, 3, 4, 5, 6, 7], [1, 0, 7, 6, 5, 4, 3, 2], [2, 7, 0, 5, 6, 3, 4, 1], [3, 6, 5, 0, 7, 2, 1, 4],
           [4, 5, 6, 7, 0, 1, 2, 3], [5, 4, 3, 2, 1, 0, 7, 6], [6, 3, 4, 1, 2, 7, 0, 5], [7, 2, 1, 4, 3, 6, 5, 0]]
    return torch.tensor([[k[j] for j in row] for row in idx], dtype=torch.float64) * (E / (1 - nu ** 2))


def check_floating_material(image):
    """True if the binarised design is not exactly one connected piece of material (reference :376-380: cv2
    connectedComponents, 8-connectivity, `labels != 2`)."""
    import numpy as np
    solid = np.asarray(image) > 0.5
    try:
        import cv2
        n = cv2.connectedComponents(solid.astype(np.uint8))[0]
    except ImportError:                                   # same labelling with scipy
        from scipy import ndimage
        n = ndimage.label(solid, structure=np.ones((3, 3)))[1] + 1
    return n != 2


def compute_fm(gen):
    """floating-material flag per sample (host side, like the reference: evaluation only)"""
    g = gen.detach().cpu().numpy()
    return torch.tensor([int(check_floating_material(g[i])) for i in range(len(g))])


def floating_material(rho):
    """compute_fm on the device: rho [B,nel,nel] -> int64 [B] (one libpidm launch, no host synchronisation)."""
    rho = rho.contiguous().float()
    fm = torch.empty(rho.shape[0], device=rho.device, dtype=torch.int64)
    call('pidm_mech_floating_material', rho, fm, rho.shape[0], rho.shape[-1], stream())
    return fm


class _Resize(torch.autograd.Function):
    """Bilinear resize of [B, C, S, S] fp32 planes, align_corners=False, antialias=False (reference :10-21)."""

    @staticmethod
    def forward(ctx, x, size):
        B, C, S, _ = x.shape
        y = torch.empty(B, C, size, size, device=x.device, dtype=torch.float32)
        call('pidm_bilinear_resize_fwd', x, y, B * C, S, size, stream())
        ctx.dims = (B, C, S, size)
        return y

    @staticmethod
    def backward(ctx, dy):
        B, C, S, size = ctx.dims
        dx = torch.empty(B, C, S, S, device=dy.device, dtype=torch.float32)
        call('pidm_bilinear_resize_bwd', dy.contiguous(), dx, B * C, S, size, stream())
        return dx, None


def resize_image(tensor, target_size):
    assert len(tensor.shape) > 3, f'Expected image, got {tensor.shape}'
    shp = tensor.shape
    flat = tensor.reshape(shp[0], -1, shp[-2], shp[-1]).contiguous().float()
    return _Resize.apply(flat, target_size).reshape(*shp[:-2], target_size, target_size)


class _MechResidual(torch.autograd.Function):
    @staticmethod
    def forward(ctx, u, rho, bcs, KE):
        B, _, nn_, _ = u.shape
        nel = nn_ - 1
        r = torch.empty(B, 2 * nn_ * nn_, device=u.device, dtype=torch.float32)
        c = torch.empty(B, device=u.device, dtype=torch.float32)
        call('pidm_mechanics_residual_fwd', u, rho, bcs, KE, r, c, B, nel, stream())
        ctx.save_for_backward(u, rho, bcs, KE)
        return r, c

    @staticmethod
    def backward(ctx, gr, gc):
        u, rho, bcs, KE = ctx.saved_tensors
        B, _, nn_, _ = u.shape
        gu = torch.empty_like(u)
        grho = torch.empty_like(rho)
        ws = torch.empty(B * 2 * nn_ * nn_, device=u.device, dtype=torch.float32)
        call('pidm_mechanics_residual_bwd', u, rho, bcs, KE, None if gr is None else gr.contiguous(),
             None if gc is None else gc.contiguous(), gu, grho, ws, B, nn_ - 1, stream())
        return gu, grho, None, None


class _MechPidmLoss(torch.autograd.Function):
    """Data + residual + inequality + optimisation terms of the mechanics PIDM loss and their gradients in ONE libpidm
    launch (csrc/mechanics.cu mech_loss_kernel; reference denoising_utils.py:669-710).  Like the Darcy loss the gradients
    are produced in forward and only scaled (out of place) in backward.  Returns (loss, sums6)."""

    @staticmethod
    def forward(ctx, u, rho, residual, compliance, x0, vf, t, p2w, pvar, coefs):
        B, _, nn_, _ = u.shape
        c_data, c_res, c_ineq, lam = coefs
        sums = torch.empty(6, device=u.device, dtype=torch.float32)
        gu = grho = gr = gc = None                          # loss only (validation under no_grad): no gradient written
        if any(x.requires_grad for x in (u, rho, residual, compliance)):
            gu, grho, gr, gc = (torch.empty_like(u), torch.empty_like(rho), torch.empty_like(residual),
                                torch.empty_like(compliance))
        call('pidm_mech_pidm_loss', u, rho, x0, residual, compliance, vf, t, p2w, pvar, float(c_data), float(c_res),
             float(c_ineq), float(lam), sums, gu, grho, gr, gc, B, nn_ - 1, stream())
        ctx.save_for_backward(gu, grho, gr, gc)
        ctx.mark_non_differentiable(sums)
        return sums[0] + sums[1] + sums[2] + sums[3], sums

    @staticmethod
    def backward(ctx, g, _unused):
        g = g.contiguous().float()
        outs = []
        for t_ in ctx.saved_tensors:
            o = torch.empty_like(t_)
            call('pidm_scale', t_, g, o, t_.numel(), stream())
            outs.append(o)
        return (*outs, None, None, None, None, None, None)


class ResidualsMechanics:
    def __init__(self, model, pixels_per_dim, pixels_at_boundary, no_BC_folder, device='cpu', bcs='none', E=1.0,
                 nu=0.3, topopt_eval=False, use_ddim_x0=False, ddim_steps=0):
        self.gov_eqs = 'mechanics'
        self.model = model
        self.pixels_at_boundary = pixels_at_boundary
        self.E, self.nu = E, nu
        # the reference only stores the flag (residuals_mechanics_K.py:122-125): 'periodic' computes what 'none' computes
        self.periodic = bcs == 'periodic'
        self.device = device
        self.pixels_per_dim = pixels_per_dim
        self.KE = q4_plane_stress_stiffness(1.0, 0.3).float().to(device).contiguous()
        self.topopt_eval = topopt_eval
        self.use_ddim_x0 = use_ddim_x0
        self.ddim_steps = ddim_steps

    def compute_residual(self, input_tuple, reduce='none', return_model_out=False, return_optimizer=False,
                         return_inequality=False, sample=False, ddim_func=None, pass_through=False):
        input, bcs, vf = input_tuple[0], input_tuple[1], input_tuple[2]
        bcs = bcs.contiguous().float()
        if pass_through:
            assert isinstance(input, torch.Tensor), 'Input is assumed to directly be given output.'
            x0_pred = model_out = input
        else:
            assert len(input) == 2 and isinstance(input, tuple), \
                'Input must be a tuple consisting of noisy signal and time.'
            noisy_in, time = input
            noisy_in = generalized_b_xy_c_to_image(noisy_in)
            net_in = torch.cat((resize_image(noisy_in, 64), resize_image(bcs, 64)), dim=1)
            if self.use_ddim_x0:
                x0_pred, model_out = ddim_func(net_in, time, self.model, noisy_in.shape, self.ddim_steps, 0.,
                                               gov_eqs='mechanics')
            else:
                x0_pred = model_out = self.model(net_in, time)
        assert len(x0_pred.shape) == 4, \
            'Model output must be a tensor shaped as an image (with explicit axes for the spatial dimensions).'
        P = x0_pred.shape[-1]
        u = resize_image(x0_pred[:, :-1], P + 1)
        rho = x0_pred[:, -1].contiguous().float()
        residual, compliance = _MechResidual.apply(u, rho, bcs, self.KE)
        output = {'residual': residual}
        if return_model_out:
            u_mo = u if model_out is x0_pred else resize_image(model_out[:, :-1], P + 1)
            rho_pad = F.pad(model_out[:, -1], pad=(0, 1, 0, 1), mode='constant', value=0)
            output['model_out'] = torch.cat((u_mo, rho_pad.unsqueeze(1)), dim=1)
        if return_optimizer:
            output['optimizer'] = compliance
        if return_inequality:
            output['inequality'] = rho.reshape(rho.shape[0], -1).mean(1) - vf
        if self.topopt_eval and sample:
            with torch.no_grad():
                output.update(self.topopt_metrics(rho.detach(), bcs, vf, input_tuple[3]))
        if reduce == 'full':
            return {k: v.mean() for k, v in output.items()}
        elif reduce == 'per-batch':
            return {k: v.mean(dim=tuple(range(1, v.ndim))) if v.ndim > 1 and (k != 'model_out' and k != 'residual') else v
                    for k, v in output.items()}
        elif reduce == 'none':
            return output
        raise ValueError('Unknown reduction method.')

    # ---- evaluation metrics of the topology-optimisation study (reference :276-354) -----------------------------
    def _apply_K(self, v, rho, masks):
        """A v for nodal fields v [B,2,nn,nn]: (K(rho) v) on the free dofs, v itself on the Dirichlet dofs (the reference's
        identity rows) -- one matrix-free libpidm launch; masks = bcs with the load planes zeroed."""
        B, _, nn_, _ = v.shape
        r = torch.empty(B, 2 * nn_ * nn_, device=v.device, dtype=torch.float32)
        call('pidm_mechanics_residual_fwd', v, rho, masks, self.KE, r, None, B, nn_ - 1, stream())
        return r.view(B, nn_ * nn_, 2).permute(0, 2, 1).reshape(B, 2, nn_, nn_)

    def fem_solve(self, rho, bcs, tol=1e-6, max_iter=6000):
        """u with K(rho) u = f on the free dofs, u = 0 on the Dirichlet dofs: Jacobi-preconditioned conjugate gradients on
        the matrix-free operator, all samples at once (the reference assembles a dense 8450 x 8450 matrix per sample and
        calls torch.linalg.solve in a Python loop, :322-325).  Returns u [B,2,nn,nn]."""
        B, _, nn_, _ = bcs.shape
        rho = rho.contiguous().float()
        free = (bcs[:, :2] == 0).float()
        f = (bcs[:, 2:4] * free).contiguous()
        masks = torch.cat((bcs[:, :2], torch.zeros_like(bcs[:, 2:4])), dim=1).contiguous()
        # diag K = KE[0,0] * (sum of the adjacent element densities): all eight diagonal entries of the Q4 matrix are equal
        node_rho = F.conv2d(F.pad(rho[:, None], (1, 1, 1, 1)), torch.ones(1, 1, 2, 2, device=rho.device))
        dinv = free / (self.KE[0, 0] * node_rho).clamp_min(1e-12)

        def dot(a, b):
            return (a.double() * b.double()).sum(dim=(1, 2, 3))
        u = torch.zeros_like(f)
        r = f.clone()
        z = dinv * r
        p = z.clone()
        rz = dot(r, z)
        f2 = dot(f, f).clamp_min(1e-300)
        for it in range(max_iter):
            Ap = self._apply_K(p.contiguous(), rho, masks) * free
            alpha = (rz / dot(p, Ap).clamp_min(1e-300)).float().view(B, 1, 1, 1)
            u = u + alpha * p
            r = r - alpha * Ap
            if it % 50 == 49 and bool(((dot(r, r) / f2).sqrt() < tol).all()):
                break
            z = dinv * r
            rz_new = dot(r, z)
            p = z + (rz_new / rz.clamp_min(1e-300)).float().view(B, 1, 1, 1) * p
            rz = rz_new
        return u

    def fem_solve_fused(self, rho, bcs, tol=1e-6, max_iter=6000):
        """The system of fem_solve, solved by one libpidm launch for the whole batch (csrc/mechanics.cu mech_pcg_kernel:
        one CTA per sample, fp64 Jacobi-PCG, the stopping rule tested at every iteration, no host synchronisation).
        Returns (u [B,2,nn,nn] fp32, iterations [B] int32, final ||r|| / ||f|| [B] fp64), all on the device: a sample
        that did not converge shows iterations == max_iter and relres >= tol."""
        B, _, nn_, _ = bcs.shape
        rho = rho.contiguous().float()
        bcs = bcs.contiguous().float()
        u = torch.empty(B, 2, nn_, nn_, device=rho.device, dtype=torch.float32)
        iters = torch.empty(B, device=rho.device, dtype=torch.int32)
        relres = torch.empty(B, device=rho.device, dtype=torch.float64)
        call('pidm_mech_fem_pcg', rho, bcs, self.KE, u, iters, relres, float(tol), int(max_iter), B, nn_ - 1, stream())
        return u, iters, relres

    def topopt_metrics(self, rho, bcs, vf, solution, solver='torch'):
        """rel_CE_error (compliance of the binarised design, FEM-solved, vs the compliance of the data), vf_error and the
        floating-material flag of reference :276-346, per sample.
        solver='torch': fem_solve, the host floating-material check and the reference's assert on the data residual.
        solver='fused': fem_solve_fused and the floating-material kernel, without a host synchronisation: the data
        residual check cannot raise there, so a failing batch gets rel_CE_error = NaN instead."""
        assert solver in ('torch', 'fused'), solver
        bcs = bcs.contiguous().float()
        nn_ = bcs.shape[-1]
        B = bcs.shape[0]
        free = (bcs[:, :2] == 0).float()
        f = bcs[:, 2:4] * free
        opt_disp = solution[:, :2].contiguous().float()
        rho_simp = solution[:, 2, :-1, :-1].contiguous().float()                 # remove the padding
        r_data, _ = _MechResidual.apply(opt_disp, rho_simp, bcs, self.KE)
        data_ok = torch.isclose(r_data.abs().mean(), torch.zeros((), device=r_data.device), atol=1.e-5)
        if solver == 'torch':
            assert data_ok, 'Residual of opt_disp is not zero.'
        compliance_data = (opt_disp * f).sum(dim=(1, 2, 3))
        rho_bin = torch.where(rho > 0.5, torch.ones_like(rho), torch.full_like(rho, 1.e-3)).contiguous()
        u_sol = self.fem_solve(rho_bin, bcs) if solver == 'torch' else self.fem_solve_fused(rho_bin, bcs)[0]
        compliance_true = (u_sol * f).sum(dim=(1, 2, 3))
        rel_ce = (compliance_true - compliance_data) / compliance_data
        if solver == 'fused':
            rel_ce = torch.where(data_ok, rel_ce, torch.full_like(rel_ce, float('nan')))
        out = {'rel_CE_error_full_batch': rel_ce,
               'vf_error_full_batch': torch.abs(rho_bin.reshape(B, -1).mean(1) - vf) / vf,
               'fm_error_full_batch': compute_fm(rho_bin) if solver == 'torch' else floating_material(rho_bin)}
        return out

    # ---- hooks used by DenoisingDiffusion (mechanics branch of the reference's loss / sampler) ------------------
    def training_loss(self, diffusion, input, t, c_data, c_residual, c_ineq, lambda_opt, sync_scalars=True,
                      draw_shard=None, noise=None):
        """model_estimation_loss for gov_eqs='mechanics' (reference denoising_utils.py:629-710).
        input [B,10,65,65] = (vf, strain energy, von Mises | disp_x, disp_y, E | bc_x, bc_y, load_x, load_y).
        Mean-mode x0 (the reference default): q_sample, the two resamplings, the matrix-free residual and ONE fused loss
        kernel are libpidm launches; no host synchronisation unless sync_scalars (the reference reads four .item()s).
        t=None: draw it here (the normal path); a given t is used as is (tests).  With t and noise [B,3,65,65] both given
        nothing is drawn (injected draws)."""
        from . import ops
        from .denoising_utils import image_to_b_xy_c
        dd = diffusion.diff_dict
        conditioning, x_0, bcs = torch.tensor_split(input, (3, 6), dim=1)
        x_0 = x_0.contiguous().float()
        from .denoising_utils import draw_t_and_noise
        if t is None or noise is None:
            t_drawn, e = draw_t_and_noise(diffusion.n_steps, x_0, draw_shard)  # reference order: t, then eps (:625,:636)
            if t is None:
                t = t_drawn
        if noise is not None:
            e = noise
        x = ops.q_sample(x_0, e, t, dd['alphas_bar_sqrt'], dd['one_minus_alphas_bar_sqrt'])
        x = torch.cat((x, conditioning), dim=1)
        vf = conditioning[:, 0, 0, 0].contiguous().float()
        if not self.use_ddim_x0:
            bcs = bcs.contiguous().float()
            net_in = torch.cat((resize_image(x, 64), resize_image(bcs, 64)), dim=1)
            y = self.model(net_in, t)                                        # [B,3,64,64]: u_x, u_y, rho (sigmoid)
            P = y.shape[-1]
            u = resize_image(y[:, :-1], P + 1)
            rho = y[:, -1].contiguous()
            residual, compliance = _MechResidual.apply(u, rho, bcs, self.KE)
            loss, sums = _MechPidmLoss.apply(u, rho, residual, compliance, x_0, vf, t.to(torch.int64).contiguous(),
                                             dd['p2_loss_weight'], dd['posterior_variance_clipped'],
                                             (c_data, c_residual, c_ineq, lambda_opt))
            # tracked scalars of the reference: data loss, mean|r|, mean inequality (only if c_ineq > 0), mean compliance
            tracked = (sums[0], sums[4], sums[5] if c_ineq > 0. else 0., compliance.detach().mean())
        else:
            out = self.compute_residual(((image_to_b_xy_c(x), t), bcs, vf, x_0), reduce='per-batch', return_model_out=True,
                                        return_optimizer=True, return_inequality=c_ineq > 0.,
                                        ddim_func=diffusion.ddim_sample_x0)
            residual, output = out['residual'], out['model_out']
            B = x_0.shape[0]
            mse = ((x_0 - output) ** 2).reshape(B, -1).mean(dim=1)
            data_loss = c_data * (mse * dd['p2_loss_weight'][t]).mean()
            var = dd['posterior_variance_clipped'][t]
            loss = data_loss + (c_residual * 0.5 * residual ** 2 / var[:, None]).mean()
            ineq_track = 0.
            if c_ineq > 0.:
                # reference quirk kept (:679,:694): `var` is extracted with the residual's rank ([B,1]) while the
                # inequality is [B], so the quotient broadcasts to [B,B]: mean_i(1/var_i) * mean_j(ineq_j^2) * c_ineq / 2
                loss = loss + (c_ineq * 0.5 * out['inequality'][None, :] ** 2 / var[:, None]).mean()
                ineq_track = out['inequality'].detach().mean()
            loss = loss + (lambda_opt * out['optimizer']).mean()
            tracked = (data_loss.detach(), residual.detach().abs().mean(), ineq_track, out['optimizer'].detach().mean())
        if sync_scalars:
            tracked = tuple(float(v) for v in tracked)
        return (loss,) + tracked

    def sampling_residual(self, diffusion, x, conditioning_input, t_vec, return_optimizer, return_inequality, sample):
        from .denoising_utils import image_to_b_xy_c
        conditioning, bcs, solution = conditioning_input
        xin = torch.cat((x, conditioning), dim=1)
        vf = conditioning[:, 0, 0, 0]
        return self.compute_residual(((image_to_b_xy_c(xin), t_vec), bcs, vf, solution), reduce='per-batch',
                                     return_model_out=True, return_optimizer=return_optimizer,
                                     return_inequality=return_inequality, sample=sample,
                                     ddim_func=diffusion.ddim_sample_x0)
