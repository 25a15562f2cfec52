"""CPU oracle for CoCoGen residual corrections (reference src/residuals_darcy.py:209-240 and the correction branches of
src/denoising_utils.py:433-459,517-540).  TEST INFRASTRUCTURE ONLY.

Builds on oracle/pidm_oracle.py: the Jacobian maximum comes from the residuals of the 4096 unit fields, as in
pidm_oracle.cocogen_correction, and the gradient of sum r^2 from autograd through pidm_oracle.darcy_residual.  A
correction changes p only, so K and the step size stay fixed over successive corrections of a field.  Pinned against
the reference by tests/test_oracle_cocogen.py (fixtures from scripts/make_golden_cocogen.py).
"""
import torch

from oracle import pidm_oracle as O


def jacobian_max(x0_pred):
    """max_dr_dp [B] (signed, as torch.max) of d residual / d p, with the reference's clamp(max=1e12)"""
    B, _, P, _ = x0_pred.shape
    out = torch.empty(B, dtype=x0_pred.dtype)
    for b in range(B):
        basis = torch.zeros(P * P + 1, 2, P, P, dtype=x0_pred.dtype)
        basis[:, 1] = x0_pred[b, 1].detach()
        basis[torch.arange(P * P), 0, torch.arange(P * P) // P, torch.arange(P * P) % P] = 1.0
        rr = O.darcy_residual(basis)
        out[b] = torch.clamp((rr[:-1] - rr[-1:]).max(), max=1e12)
    return out


def cocogen_steps(x0_pred, steps):
    """`steps` successive residual_correction calls on x0_pred [B,2,P,P].  Returns (x, residual of x, [p after each
    correction])."""
    eps = (1e-6 / jacobian_max(x0_pred)).view(-1, 1, 1)
    x = x0_pred.detach().clone()
    p_iterates = []
    for _ in range(steps):
        with torch.enable_grad():
            xg = x.clone().requires_grad_(True)
            dr_dp = torch.autograd.grad((O.darcy_residual(xg) ** 2).sum(), xg)[0][:, 0]
        x[:, 0] = x[:, 0] - eps * dr_dp
        p_iterates.append(x[:, 0].clone())
    return x, O.darcy_residual(x), p_iterates


def p_sample_loop(sd, cfg, x_T, noises, tables, n_steps, N_correction=0, M_correction=0, correction_mode='none'):
    """pidm_oracle.p_sample_loop with CoCoGen corrections: while t < N_correction the x0 estimate ('x0') or the new
    sample ('xt') is corrected once and the step's residual is the corrected one; then M_correction corrections of the
    final sample.  Returns (trajectory [x_T, ..., one entry per post-loop correction], residual of the last step or
    correction)."""
    x = x_T
    seq = [x]
    r = None
    for k, i in enumerate(reversed(range(n_steps))):
        tt = torch.full((x.shape[0],), i, dtype=torch.long)
        x0p = O.unet_forward(sd, cfg, x, tt)
        r = O.darcy_residual(x0p)
        correct = i < N_correction
        if correct and correction_mode == 'x0':
            x0p, r, _ = cocogen_steps(x0p, 1)
        x = O.posterior_step(x, x0p, noises[k], i, tables)
        if correct and correction_mode == 'xt':
            x, r, _ = cocogen_steps(x, 1)
        seq.append(x)
    for _ in range(M_correction):
        x, r, _ = cocogen_steps(x, 1)
        seq.append(x)
    return seq, r
