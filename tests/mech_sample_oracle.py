"""CPU oracle for conditional sampling of the topology-optimisation model and for its evaluation solve.  TEST
INFRASTRUCTURE ONLY.

* `p_sample_loop`: the reference's ancestral loop with a conditioning input (denoising_utils.py:388-545 with
  residuals_mechanics_K.py:176-205), restated on the U-Net of oracle/pidm_oracle.py (`unet_forward`) and its matrix-free
  mechanics residual (`mechanics_residual`), float32 or float64.  The DDIM walk of the 'sample' x0 estimate draws a noise
  tensor that eta = 0 never uses (the reference draws it for RNG parity), so only the posterior draws are inputs here.
* `fem_solve`: fp64 sparse assembly of K(rho) with the reference's modification (Dirichlet rows replaced by identity
  rows, columns kept, f zeroed on the Dirichlet dofs; residuals_mechanics_K.py:296-325) and scipy's sparse direct
  solve: the ground truth for the iterative solvers.
Pinned against the reference by tests/test_oracle_mech_sample.py."""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla
import torch
import torch.nn.functional as F

from oracle import pidm_oracle as O


def ddim_x0(sd, cfg, net_in, t, tables, ddim_steps=0):
    """ddim_sample_x0 with eta = 0 and gov_eqs='mechanics' (denoising_utils.py:712-787): the walk runs on the three
    solution channels, every network call sees the ORIGINAL input.  Returns (x0 at the end of the walk, first output)."""
    B, dt = net_in.shape[0], net_in.dtype
    seqs, seqs_next = [], []
    for ti in t.tolist():
        seq = [int(v) for v in torch.linspace(0, ti, ddim_steps + 2, dtype=torch.float64).tolist()]
        seqs.append(list(reversed(seq)))
        seqs_next.append(list(reversed([-1] + seq[:-1])))
    cur_t, nxt_t = torch.tensor(seqs).T, torch.tensor(seqs_next).T
    v4 = lambda name, idx: tables[name].to(dt)[idx].view(B, 1, 1, 1)
    cur_x, model_out = net_in[:, :3], None
    for k in range(cur_t.shape[0]):
        tt, tn = cur_t[k], nxt_t[k]
        x0p = O.unet_forward(sd, cfg, net_in, tt)
        if k == 0:
            model_out = x0p
        if int(tn[0]) < 0:
            cur_x = x0p
            continue
        mean = v4('posterior_mean_coef1', tt) * x0p + v4('posterior_mean_coef2', tt) * cur_x
        eps = (v4('sqrt_recip_alphas', tt) * cur_x - mean) / v4('noise_mean_coeff', tt)
        a_next = v4('alphas_prod', tn)
        new_x = x0p * a_next.sqrt() + (1 - a_next).sqrt() * eps
        mask = (tt == tn).to(dt).view(B, 1, 1, 1)
        cur_x = mask * cur_x + (1 - mask) * new_x
    return cur_x, model_out


def p_sample_loop(sd, cfg, x_T, noises, conditioning, bcs, tables, n_steps, use_ddim_x0=False, ddim_steps=0):
    """x_T [B,3,65,65], noises[k] = the posterior z of loop iteration k (drawn at t = 0 too), conditioning [B,3,65,65],
    bcs [B,4,65,65].  Returns dict(x_first, x_final, x0_pred_last, residual, compliance, inequality); the residual terms
    are those of the last step (t = 0)."""
    x, out = x_T, {}
    vf = conditioning[:, 0, 0, 0]
    bcs_red = O.bilinear_resize(bcs, 64)
    for k, i in enumerate(reversed(range(n_steps))):
        tt = torch.full((x.shape[0],), i, dtype=torch.long)
        net_in = torch.cat((O.bilinear_resize(torch.cat((x, conditioning), dim=1), 64), bcs_red), dim=1)
        if use_ddim_x0:
            x0p, mo = ddim_x0(sd, cfg, net_in, tt, tables, ddim_steps)
        else:
            x0p = mo = O.unet_forward(sd, cfg, net_in, tt)
        model_out = torch.cat((O.bilinear_resize(mo[:, :2], 65), F.pad(mo[:, 2], (0, 1, 0, 1)).unsqueeze(1)), dim=1)
        x = O.posterior_step(x, model_out, noises[k], i, tables)
        if k == 0:
            out['x_first'] = x
    r, comp, ineq = O.mechanics_residual(x0p, bcs, vf)
    out.update(x_final=x, x0_pred_last=x0p, residual=r, compliance=comp, inequality=ineq)
    return out


def reduced_system(rho, bcs, KE=None):
    """rho [nel,nel], bcs [4,nel+1,nel+1] -> (K scipy CSC fp64, f fp64) in the dof order 2*node + d."""
    rho = np.asarray(rho, dtype=np.float64)
    bcs = np.asarray(bcs, dtype=np.float64)
    nel = rho.shape[-1]
    n = 2 * (nel + 1) ** 2
    KE = (O.q4_plane_stress_stiffness() if KE is None else torch.as_tensor(KE)).double().numpy()
    dofs = O.mechanics_mesh(nel).numpy()                                          # [nel^2, 8]
    vals = rho.reshape(-1)[:, None, None] * KE[None]
    rows = np.broadcast_to(dofs[:, :, None], vals.shape)
    cols = np.broadcast_to(dofs[:, None, :], vals.shape)
    K = sp.coo_matrix((vals.ravel(), (rows.ravel(), cols.ravel())), shape=(n, n)).tocsr()
    fixed = np.stack((bcs[0].ravel(), bcs[1].ravel()), axis=1).ravel() != 0
    f = np.stack((bcs[2].ravel(), bcs[3].ravel()), axis=1).ravel()
    f[fixed] = 0.
    K = sp.diags((~fixed).astype(np.float64)) @ K + sp.diags(fixed.astype(np.float64))
    return K.tocsc(), f


def fem_solve(rho, bcs, KE=None):
    """u [B,2,nel+1,nel+1] fp64 with K(rho) u = f on the free dofs, u = 0 on the Dirichlet dofs (sparse direct)."""
    rho, bcs = torch.as_tensor(rho), torch.as_tensor(bcs)
    out = []
    for b in range(rho.shape[0]):
        K, f = reduced_system(rho[b].cpu().numpy(), bcs[b].cpu().numpy(), KE)
        nn_ = bcs.shape[-1]
        out.append(torch.from_numpy(spla.spsolve(K, f).reshape(nn_ * nn_, 2).T.reshape(2, nn_, nn_).copy()))
    return torch.stack(out)
