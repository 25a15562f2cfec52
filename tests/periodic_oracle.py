"""CPU oracle for bcs='periodic' (reference src/grad_utils.py:76-81).  TEST INFRASTRUCTURE ONLY.

The periodic counterparts of the Darcy functions of oracle/pidm_oracle.py, in plain PyTorch (float32 or float64, CPU).
With periodic=True the reference pads by one pixel with mode='circular' and applies the interior ('C', 'C') stencil, so
every pixel, boundary pixels included, uses the central second-order stencil with wrapped neighbours.  Everything else
is kept as with bcs='none': h = domain_length / (P-1) when pixels_at_boundary, f_s, and the two BC channels on rows 0 /
P-1 and columns 0 / P-1 with the same signs (built from the wrapped p_0 / p_1).  The U-Net, schedule tables, loss
algebra and posterior step are the ones of oracle/pidm_oracle.py.  Pinned against the reference by
tests/test_oracle_periodic.py (fixtures from scripts/make_golden_periodic.py).
"""
import torch

from oracle import pidm_oracle as O


def fd_first(u, axis, h):
    """central first derivative along `axis`, neighbours wrapped"""
    return (torch.roll(u, -1, axis) - torch.roll(u, 1, axis)) * (0.5 / h)


def fd_second(u, axis, h):
    """central second derivative [1, -2, 1] / h^2 along `axis`, neighbours wrapped"""
    return (torch.roll(u, -1, axis) - 2.0 * u + torch.roll(u, 1, axis)) / (h * h)


def stencil_gradients(u, mode, d0, d1):
    """StencilGradients(periodic=True).forward for one mode on [..., P, P]"""
    if mode == 'd_d0':
        return fd_first(u, -2, d0)
    if mode == 'd_d1':
        return fd_first(u, -1, d1)
    if mode == 'd_d00':
        return fd_second(u, -2, d0)
    if mode == 'd_d11':
        return fd_second(u, -1, d1)
    if mode == 'd_d01':
        return fd_first(fd_first(u, -1, d1), -2, d0)
    raise ValueError(mode)


def spacing(P, domain_length=1.0, reverse_d1=True, pixels_at_boundary=True):
    d0 = domain_length / (P - 1) if pixels_at_boundary else domain_length / P
    return d0, (-d0 if reverse_d1 else d0)


def darcy_residual(x0_pred, domain_length=1.0, reverse_d1=True, pixels_at_boundary=True):
    """ResidualsDarcy(bcs='periodic').compute_residual on x0_pred [B,2,P,P] -> [B, P*P, 3] = (eq_0, bc_x0, bc_x1)."""
    B, C, P, _ = x0_pred.shape
    d0, d1 = spacing(P, domain_length, reverse_d1, pixels_at_boundary)
    p, K = x0_pred[:, 0], x0_pred[:, 1]
    p0, p1 = fd_first(p, -2, d0), fd_first(p, -1, d1)
    p00, p11 = fd_second(p, -2, d0), fd_second(p, -1, d1)
    K0, K1 = fd_first(K, -2, d0), fd_first(K, -1, d1)
    fs = O.darcy_source(P, dtype=x0_pred.dtype).to(x0_pred.device)
    eq0 = (-K * p00 - K0 * p0) + (-K * p11 - K1 * p1) - fs
    bc0 = torch.zeros_like(p)
    bc1 = torch.zeros_like(p)
    bc0[:, 0, :] = -p0[:, 0, :]
    bc0[:, -1, :] = p0[:, -1, :]
    sgn = 1.0 if reverse_d1 else -1.0
    bc1[:, :, 0] = sgn * p1[:, :, 0]
    bc1[:, :, -1] = -sgn * p1[:, :, -1]
    return torch.stack([eq0, bc0, bc1], dim=-1).reshape(B, P * P, 3)


def darcy_residual_gradient(x_t):
    """d mean|r(x_t)| / d x_t with the periodic residual (residuals_darcy.py:117-120)"""
    with torch.enable_grad():
        x = x_t.detach().clone().requires_grad_(True)
        return torch.autograd.grad(darcy_residual(x).abs().mean(), x)[0]


def darcy_training_loss(sd, cfg, x0, t, noise, tables, c_data=1.0, c_residual=1e-3, guidance_null_mask=None):
    """model_estimation_loss for gov_eqs='darcy', mean mode, bcs='periodic' (t and eps supplied)."""
    xt = O.q_sample(x0, t, noise, tables)
    if guidance_null_mask is not None:
        model_out = O.unet_forward(sd, cfg, xt, t, cond=darcy_residual_gradient(xt), null_mask=guidance_null_mask)
    else:
        model_out = O.unet_forward(sd, cfg, xt, t)
    r = darcy_residual(model_out)
    loss, data, rabs = O.pidm_loss_from_x0pred(x0, model_out, r, t, tables, c_data, c_residual)
    return loss, dict(data=data, residual_abs=rabs, model_out=model_out, residual=r, x_t=xt)


def cocogen_correction(x0_pred):
    """ResidualsDarcy(bcs='periodic').residual_correction on [B,2,P,P]; Jacobian columns from the unit fields as in
    oracle.pidm_oracle.cocogen_correction."""
    B, _, P, _ = x0_pred.shape
    x = x0_pred.detach().clone().requires_grad_(True)
    dr_dp = torch.autograd.grad((darcy_residual(x) ** 2).sum(), x)[0][:, 0]
    out = x0_pred.detach().clone()
    for b in range(B):
        out[b, 0] = out[b, 0] - (1e-6 / jacobian_max(x0_pred[b:b + 1])[0]) * dr_dp[b]
    return out, darcy_residual(out)


def jacobian_max(x0_pred):
    """[B]: largest entry (signed, zeros included) of d residual / d p per sample, clamped at 1e12 like the reference"""
    B, _, P, _ = x0_pred.shape
    out = torch.empty(B, dtype=x0_pred.dtype)
    for b in range(B):
        basis = torch.zeros(P * P + 1, 2, P, P, dtype=x0_pred.dtype)
        basis[:, 1] = x0_pred[b, 1].detach()
        basis[torch.arange(P * P), 0, torch.arange(P * P) // P, torch.arange(P * P) % P] = 1.0
        rr = darcy_residual(basis)
        out[b] = torch.clamp((rr[:-1] - rr[-1:]).max(), max=1e12)
    return out


def p_sample_loop(sd, cfg, x_T, noises, tables, n_steps):
    """ancestral loop for Darcy, mean-mode x0, periodic residual of the last x0 estimate"""
    x = x_T
    r = None
    for k, i in enumerate(reversed(range(n_steps))):
        tt = torch.full((x.shape[0],), i, dtype=torch.long)
        x0p = O.unet_forward(sd, cfg, x, tt)
        r = darcy_residual(x0p)
        x = O.posterior_step(x, x0p, noises[k], i, tables)
    return x, r
