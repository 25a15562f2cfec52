"""The topology-optimisation sampling and evaluation kernels of mechanics.cu, replayed element by element against fp64:
the batched Jacobi-PCG solve (pidm_mech_fem_pcg), the floating-material flag (pidm_mech_floating_material), the U-Net
input of a conditional sampling step (pidm_mech_sample_input) and its posterior step (pidm_mech_posterior_step).

pidm_mech_fem_pcg runs one 512-thread CTA per sample for the whole solve, nine node slots per thread ((nel+1)^2 <= 4608,
so 2 <= nel <= 66), in fp64 on the fp32 rho and KE; `rel_CE_error` of topopt_metrics(solver='fused') comes straight
from its u.  pidm_mech_floating_material labels the solid pixels (> 0.5) of one design per 1024-thread CTA in shared
memory (nel^2 ints, above 48 KB from nel = 111).  The two sampling kernels are grid-stride loops capped at 8 CTAs of 256
threads per SM.  Here, in the five parts of the other census files:

  1. census: the distinct keys of the four entry points in census.census_sampling() (conditional mechanics sampling in
     mean and sample mode and the evaluation of its last x0 prediction) must equal the tables below;
  2. replay, through the C ABI between NaN guards:
        pcg         tol = 0 runs exactly max_iter iterations, so truncated trajectories are compared with pcg_ref, an
                    fp64 PCG on the kernel's own operator (fp32 KE and rho widened, dinv formed in fp64 and rounded to
                    fp32, the Dirichlet dofs masked in A p, the loads on fixed dofs dropped):
                      iters == max_iter,
                      |u - u_ref| <= u32 |u_ref| + C_PCG k u64 sum_j |alpha_j p_j|,
                      |relres - relres_ref| <= C_PCG k u64 || sum_j |alpha_j| |A| |p_j| ||_2 / ||f||_2;
                    the stopping rule at a tol strictly between two reference iterates; converged solves (tol 1e-6)
                    against the residual of the returned u and against the sparse direct solve (fem_solve);
        fm          exactly the flag of scipy.ndimage.label with 8-connectivity under check_floating_material's rule;
        mech_input  channels >= 3 bitwise the planes, channels 0..2 within the resize bound (checks.resize_bounds);
        mech_post   C_MPOST u32 (|c1 mo| + |c2 x| + |sigma z|) + |c1| (the resize bound of mo), bitwise the same in place
                    and out of place;
     with u32 = 2^-24 and u64 = 2^-53;
  3. mutants: the same predicates reject the fp64 references edited the way a subtle kernel bug would change them;
  4. plan coverage: the launch arithmetic, restated below, shows that the rows reach both states of the ninth node slot,
     the largest PCG shared-memory plan, the fm opt-in above 48 KB at 1 and 16 pixels per thread and several grid-stride
     passes of both sampling kernels;
  5. completeness is the sampling census's closure test: these four are keyed, so census.CHECKED_ELSEWHERE names none.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F
from scipy import ndimage

import mech_sample_inputs as MI
from census import assert_census_in_tables, assert_tables_in_census
from checks import GUARD, U, call_sync, gen, guarded, guards_intact, note, ratio, resize_bounds, sms
from oracle import pidm_oracle as O

pytestmark = pytest.mark.gpu

DEV = 'cuda'
TAG = 'mech eval census'
U64 = 2.0 ** -53
# Worst |err| / bound on an H100 80GB HBM3 (700 W) in brackets (DESIGN.md section 2); C_PCG was not minimised
C_PCG = 2 ** 18     # fp64 trajectory of the PCG: order-dependent roundings of the sums, amplified by CG itself (u 0.997,
                    # the fp32 output rounding; relres 4e-7)
C_MPOST = 4         # two products and two adds (contracted or not) after the resized model output (0.67)
C_RESIZE = 4        # the physics census's resize constant: the same bil_sample
SUM_DEPTH = 64      # the fp32 addition chain of torch's CUDA sum over the 2 (nel+1)^2 dofs of one sample

# ----------------------------------------------------------------------------------------------------------------------
# the committed census tables (`python tests/census.py --print-table`); distinct keys per workload:
#   mech_sample_mean_b2, mech_sample_sample_b2: mech_input 1, mech_post 1
#   mech_aux_b2: pcg 1, fm 1
#   the other sampling workloads: none of the four
#   distinct: mech_input 1, mech_post 1, pcg 1, fm 1
# ----------------------------------------------------------------------------------------------------------------------
# mech_input: B, nc, P;  mech_post: B, P;  pcg: B, nel, tol, max_iter;  fm: B, nel
MECH_INPUT_TABLE = [
    (2, 7, 64),  # mech_sample_mean_b2 mech_sample_sample_b2
]
MECH_POST_TABLE = [
    (2, 64),  # mech_sample_mean_b2 mech_sample_sample_b2
]
PCG_TABLE = [
    (2, 64, 1e-06, 6000),  # mech_aux_b2
]
FM_TABLE = [
    (2, 64),  # mech_aux_b2
]
TABLES = {'mech_input': MECH_INPUT_TABLE, 'mech_post': MECH_POST_TABLE, 'pcg': PCG_TABLE, 'fm': FM_TABLE}


def test_census_is_covered_by_the_table():
    assert_census_in_tables(TABLES)


def test_every_table_row_is_produced_by_the_census():
    assert_tables_in_census(TABLES)


# ----------------------------------------------------------------------------------------------------------------------
# launch arithmetic (restated from mechanics.cu; the kernels have no plan query)
# ----------------------------------------------------------------------------------------------------------------------
PCG_THREADS, PCG_NPT = 512, 9       # mech_pcg_kernel: one CTA per sample, node tid + k * 512 in slot k < 9
FM_THREADS = 1024                   # mech_fm_kernel: one CTA per sample, pixel i, i + 1024, ...
SMEM_DEFAULT = 48 * 1024            # dynamic shared memory without the opt-in


def pcg_smem(nel):                  # pidm_mech_fem_pcg: p and u (fp64, two planes each), 4 x 16 fp64 sums, rho (fp32)
    nn = nel + 1
    return (4 * nn * nn + 4 * (PCG_THREADS // 32)) * 8 + nel * nel * 4


def pcg_ninth_slot_filled(nel):     # slot 8 holds nodes 4096 .. (nel+1)^2 - 1
    return (nel + 1) ** 2 > (PCG_NPT - 1) * PCG_THREADS


def fm_smem(nel):
    return nel * nel * 4


def grid_passes(total, n_sms):      # the sampling kernels: 256 threads, min(ceil(total / 256), 8 SMs) CTAs
    grid = min(-(-total // 256), 8 * n_sms)
    return -(-total // (grid * 256))


def input_total(B, nc, P):
    return B * (3 + nc) * P * P


def post_total(B, P):
    return B * 3 * (P + 1) ** 2


def _wrap_batch(per_sample):
    """a batch whose capped grid takes three grid-stride passes"""
    return -(-3 * 8 * sms() * 256 // per_sample)


def _batch(spec, per_sample=None):
    """an int, 'wide' (2 x SMs + 5: past two waves of one-CTA-per-sample launches) or 'wrap'"""
    if isinstance(spec, int):
        return spec
    return 2 * sms() + 5 if spec == 'wide' else _wrap_batch(per_sample)


# ----------------------------------------------------------------------------------------------------------------------
# pcg
# ----------------------------------------------------------------------------------------------------------------------
def ke():
    from physicsinformeddiffusionmodels_b200.residuals_mechanics_K import q4_plane_stress_stiffness
    return q4_plane_stress_stiffness(1.0, 0.3).float().to(DEV).contiguous()


def pcg_operands(B, nel, seed, case='mixed'):
    """(rho [B,nel,nel], bcs [B,4,nn,nn]) fp32.  'mixed': rho in [1e-3, 1], a clamped left edge (value 1) for even
    samples and pinned bottom corners (values 0.5 and -1) for odd ones, sparse random loads that also land on fixed
    dofs, and a load on the free top-right corner.  'no_load': the same without loads; 'all_fixed': every dof fixed,
    loads everywhere; 'rho_min': rho = 1e-3 everywhere."""
    g = gen((B, nel, seed, case))
    nn = nel + 1
    rho = 1e-3 + (1 - 1e-3) * torch.rand(B, nel, nel, generator=g, device=DEV)
    if case == 'rho_min':
        rho = torch.full_like(rho, 1e-3)
    bcs = torch.zeros(B, 4, nn, nn, device=DEV)
    bcs[0::2, 0, :, 0] = 1.
    bcs[0::2, 1, :, 0] = 1.
    bcs[1::2, 0, nel, 0] = 0.5
    bcs[1::2, 1, nel, 0] = 0.5
    bcs[1::2, 1, nel, nel] = -1.
    loads = torch.randn(B, 2, nn, nn, generator=g, device=DEV)
    bcs[:, 2:4] = loads * (torch.rand(B, 2, nn, nn, generator=g, device=DEV) < 0.2)
    bcs[:, 2:4, :, 0] = loads[..., :, 0]                  # loads on the clamped edge (ignored) and left column
    bcs[:, 3, 0, nel] = -1.
    if case == 'no_load':
        bcs[:, 2:4] = 0.
    elif case == 'all_fixed':
        bcs[:, :2] = 1.
        bcs[:, 2:4] = loads
    return rho.contiguous(), bcs.contiguous()


def guarded_int(n, dtype, fill):
    """(buffer, its middle n elements) of an integer output, every element `fill`"""
    buf = torch.full((n + 2 * GUARD,), fill, device=DEV, dtype=dtype)
    return buf, buf[GUARD:GUARD + n]


def int_guards_intact(buf, fill):
    return bool((buf[:GUARD] == fill).all() and (buf[-GUARD:] == fill).all())


def pcg_launch(rho, bcs, tol, max_iter):
    """(u [B,2,nn,nn], iters [B], relres [B]) of one launch, each output between guards"""
    B, nel = rho.shape[0], rho.shape[-1]
    nn = nel + 1
    ub, u = guarded(B * 2 * nn * nn)
    ib, it = guarded_int(B, torch.int32, -7)
    rb, rr = guarded(B, torch.float64)
    call_sync('pidm_mech_fem_pcg', rho, bcs, ke(), u, it, rr, float(tol), int(max_iter), B, nel)
    assert guards_intact(ub) and guards_intact(rb), 'a store landed outside u / relres'
    assert int_guards_intact(ib, -7), 'a store landed outside iters'
    return u.view(B, 2, nn, nn), it.long(), rr


def pcg_system(rho, bcs, KE):
    """the kernel's operator in fp64: (K v and |K| |v| for v [B,2,nn,nn], f, dinv, fixed)"""
    B, nel = rho.shape[0], rho.shape[-1]
    nn = nel + 1
    rho_d, KE_d = rho.double(), KE.double()
    fixed = bcs[:, :2] != 0
    f = torch.where(fixed, 0., bcs[:, 2:4].double())
    # the sum of <= 4 adjacent fp32 densities is exact in fp64; KE[0,0] * sum, 1 / max(., 1e-12) round once each
    node_rho = F.conv2d(F.pad(rho_d[:, None], (1, 1, 1, 1)), torch.ones(1, 1, 2, 2, dtype=torch.float64,
                                                                         device=rho.device))
    dinv = (1.0 / (KE_d[0, 0] * node_rho).clamp_min(1e-12)).float().double().expand(B, 2, nn, nn)
    zero = torch.zeros(B, 4, nn, nn, dtype=torch.float64, device=rho.device)

    def K(v, absolute=False):
        r = O.mechanics_matfree(v, rho_d, zero, KE_d, absolute=absolute)[0]
        return r.view(B, nn, nn, 2).permute(0, 3, 1, 2)
    return K, f, dinv, fixed


PCG_EDITS = ('dirichlet_dof_free', 'load_on_fixed_dof', 'identity_preconditioner', 'beta_unpreconditioned',
             'stop_late', 'previous_iterate')


def pcg_ref(rho, bcs, KE, k, tol=0.0, edit=None):
    """fp64 Jacobi-PCG of mech_pcg_kernel with at most k[b] iterations for sample b (k: int or [B]) and the stopping
    test rel < tol after each iteration.  Returns dict(u, relres, iters, hist [B, kmax + 1] (relres after each
    iteration, NaN past the stop), Tu = sum_j |alpha_j p_j|, Tr = || sum_j |alpha_j| |A| |p_j| ||_2 / ||f||_2).
    edit: one of PCG_EDITS (mutants)"""
    B = rho.shape[0]
    K, f, dinv, fixed = pcg_system(rho, bcs, KE)
    mask = fixed
    if edit == 'dirichlet_dof_free':                      # the first fixed dof of every sample left free in A p
        flat = fixed.reshape(B, -1).clone()
        first = flat.float().argmax(dim=1)
        flat[torch.arange(B, device=rho.device), first] = False
        mask = flat.view_as(fixed)
    if edit == 'load_on_fixed_dof':
        f = bcs[:, 2:4].double()
    if edit == 'identity_preconditioner':
        dinv = torch.ones_like(dinv)
    k = torch.as_tensor(k, device=rho.device).expand(B).long()

    def dot(a, b):
        return (a * b).sum(dim=(1, 2, 3))

    def bc(v):
        return v.view(B, 1, 1, 1)
    u = torch.zeros_like(f)
    r = f.clone()
    p = dinv * r
    rz = dot(r, p)
    rr_old = dot(r, r)
    f2 = rr_old.clamp_min(1e-300)
    rel = torch.sqrt(rr_old / f2)
    it = torch.zeros(B, dtype=torch.long, device=rho.device)
    done = k <= 0
    crossed = torch.zeros(B, dtype=torch.bool, device=rho.device)
    hist = [rel.clone()]
    Tu, TA = torch.zeros_like(u), torch.zeros_like(u)
    u_prev = u.clone()
    for _ in range(int(k.max())):
        live = ~done
        if not bool(live.any()):
            break
        Ap = torch.where(mask, 0., K(p))
        alpha = rz / dot(p, Ap).clamp_min(1e-300)
        a = bc(alpha)
        L = bc(live)
        u_prev = torch.where(L, u, u_prev)
        u = torch.where(L, u + a * p, u)
        Tu = torch.where(L, Tu + (a * p).abs(), Tu)
        TA = torch.where(L, TA + a.abs() * torch.where(mask, 0., K(p, absolute=True)), TA)
        r = torch.where(L, r - a * Ap, r)
        rr, rzn = dot(r, r), dot(dinv * r, r)
        it = it + live.long()
        rel = torch.where(live, torch.sqrt(rr / f2), rel)
        hist.append(torch.where(live, rel, float('nan')))
        below = rel < tol
        stop = live & ((crossed if edit == 'stop_late' else below) | (it >= k))
        crossed = crossed | (live & below)
        beta = (rr / rr_old.clamp_min(1e-300)) if edit == 'beta_unpreconditioned' else rzn / rz.clamp_min(1e-300)
        go = live & ~stop
        p = torch.where(bc(go), dinv * r + bc(beta) * p, p)
        rz = torch.where(go, rzn, rz)
        rr_old = torch.where(go, rr, rr_old)
        done = done | stop
    fn = torch.sqrt(f2)
    return dict(u=u_prev if edit == 'previous_iterate' else u, relres=rel, iters=it, hist=torch.stack(hist, 1), Tu=Tu,
                Tr=torch.sqrt((TA * TA).sum(dim=(1, 2, 3))) / fn)


def pcg_ratios(out, ref):
    """(worst u ratio, worst relres ratio, iteration counts equal) of a launch against pcg_ref"""
    u, it, rr = out
    k = ref['iters'].double()
    qu = ratio((u.double() - ref['u']).abs(), U * ref['u'].abs() + C_PCG * k.view(-1, 1, 1, 1) * U64 * ref['Tu'])
    qr = ratio((rr - ref['relres']).abs(), C_PCG * k * U64 * ref['Tr'])
    return qu, qr, torch.equal(it, ref['iters'])


# (B, nel, max_iter, case): every edge nel at every truncation, B = 1 and past two waves, the edge designs
PCG_NELS = (2, 3, 7, 31, 63, 64, 66)
PCG_TRUNC = (0, 1, 2, 3, 10, 50)
# At nel = 7 and k = 50 the fp64 trajectory is chaotic: its distance from the reference was 1.3 x 10^5 and then
# 8.4 x 10^5 times k u64 sum |alpha p| in two runs of the same code (DESIGN.md section 2), so that pair is left out
PCG_ROWS = ([(3, nel, k, 'mixed') for nel in PCG_NELS for k in PCG_TRUNC if (nel, k) != (7, 50)]
            + [(1, 66, 50, 'mixed'), (1, 2, 3, 'mixed'), ('wide', 7, 10, 'mixed'), ('wide', 64, 3, 'mixed')]
            + [(2, nel, k, case) for case in ('no_load', 'all_fixed') for nel, k in ((3, 3), (64, 10))]
            + [(2, nel, k, 'rho_min') for nel, k in ((7, 10), (64, 50))])


def pcg_id(row):
    return f'B{row[0]}_nel{row[1]}_k{row[2]}_{row[3]}'


@pytest.mark.parametrize('row', PCG_ROWS, ids=pcg_id)
def test_pcg_truncated_replay(row):
    B, nel, k, case = _batch(row[0]), row[1], row[2], row[3]
    rho, bcs = pcg_operands(B, nel, 500 + nel + k, case)
    out = pcg_launch(rho, bcs, 0.0, k)
    ref = pcg_ref(rho, bcs, ke(), k)
    qu, qr, same = pcg_ratios(out, ref)
    note(TAG, f'pcg {pcg_id(row)} u', qu)
    note(TAG, f'pcg {pcg_id(row)} relres', qr)
    assert same and bool((out[1] == k).all()), (out[1], k)
    assert qu <= 1.0 and qr <= 1.0, (qu, qr)
    u, _, rr = out
    if k == 0 or case in ('no_load', 'all_fixed'):
        assert bool((u == 0).all()), 'u must be 0 before the first iteration and without a load'
        assert bool((rr == (1.0 if k == 0 and case not in ('no_load', 'all_fixed') else 0.0)).all()), rr
    if case == 'mixed':                                   # the load on the fixed dofs of the left edge is ignored
        assert bool(((bcs[:, 2:4] != 0) & (bcs[:, :2] != 0)).any())
        assert bool((u[bcs[:, :2] != 0] == 0).all()), 'a fixed dof moved'


STOP_ROWS = [(3, 7, 4), (3, 31, 10), (2, 64, 25), (1, 66, 10)]      # B, nel, the first iteration j to stop at
STOP_MARGIN = 1e-6                                                   # relative gap between tol and every iterate


def stop_tol(rho, bcs, j):
    """(tol, j'): j' >= j the first iteration at which sample 0's relres falls below every earlier value (PCG's
    residual norm is not monotone), tol the geometric mean of that value and the smallest earlier one"""
    h = pcg_ref(rho, bcs, ke(), 8 * j)['hist'][0]
    for jj in range(j, len(h)):
        lo = float(h[:jj].min())
        if float(h[jj]) < lo:
            return (lo * float(h[jj])) ** 0.5, jj
    raise AssertionError('no new minimum of the relative residual after iteration j')


def stop_ref(rho, bcs, tol, edit=None):
    """pcg_ref under the stopping rule, with the margin between tol and every iterate it saw asserted (for the
    unedited rule)"""
    ref = pcg_ref(rho, bcs, ke(), 6000, tol=tol, edit=edit)
    if edit is not None:
        return ref
    h = ref['hist'][:, 1:]
    seen = torch.isfinite(h)
    assert bool(((h - tol).abs() > STOP_MARGIN * tol)[seen].all()), 'tol too close to an iterate'
    assert bool((ref['relres'] < tol).all()), 'a sample does not reach tol'
    return ref


@pytest.mark.parametrize('row', STOP_ROWS, ids=lambda r: f'B{r[0]}_nel{r[1]}_j{r[2]}')
def test_pcg_stopping_rule(row):
    B, nel, j = row
    rho, bcs = pcg_operands(B, nel, 700 + nel)
    tol, jj = stop_tol(rho, bcs, j)
    ref = stop_ref(rho, bcs, tol)
    assert int(ref['iters'][0]) == jj
    out = pcg_launch(rho, bcs, tol, 6000)
    qu, qr, same = pcg_ratios(out, ref)
    note(TAG, f'pcg stop nel={nel} j={jj} u', qu)
    note(TAG, f'pcg stop nel={nel} j={jj} relres', qr)
    assert same, (out[1], ref['iters'])
    assert qu <= 1.0 and qr <= 1.0, (qu, qr)
    assert bool((out[2] < tol).all())


def converged_cases(ev):
    """(name, rho [B,64,64], bcs [B,4,65,65]) on the host: the data density and the binarised x0 of mechanics_eval.pt
    (ev), and 12 binarised designs under four support / load cases"""
    x0 = ev['x0_pred'][:, 2]
    rho_bin, bcs = MI.binarised_designs(12, seed=5)
    return [('eval_rho_simp', ev['solution'][:, 2, :-1, :-1].contiguous(), ev['bcs']),
            ('eval_x0_binarised', torch.where(x0 > 0.5, torch.ones_like(x0), torch.full_like(x0, 1e-3)), ev['bcs']),
            ('binarised', rho_bin, bcs)]


def converged_ratios(rho, bcs, u, iters, relres, u_star):
    """(relres ratio, metric ratio, metric bound, f^T u) of converged solves, in fp64 on the device:
    relres is honest  ||f - K u||_2 <= relres ||f||_2 + (u32 + C_PCG iters u64) || |K| |u| ||_2
    the metric        |f^T u - f^T u*| <= ||u*||_2 (||f - K u||_2 + ||r*||_2) + ||r*||_2 ||u - u*||_2 + slack,
    from f^T (u - u*) = u*^T (K u - f) + r*^T (u - u*) on the free dofs (u and u* are 0 on the fixed ones), r* = f - K u*
    the residual of the direct solve, slack = 8 n u64 |f|^T (|u| + |u*|) for the fp64 evaluation"""
    K, f, _, fixed = pcg_system(rho, bcs, ke())
    ud = u.double()
    us = torch.where(fixed, 0., u_star.to(DEV))

    def nrm(v):
        return torch.sqrt((v * v).sum(dim=(1, 2, 3)))
    res = torch.where(fixed, 0., f - K(ud))
    Aabs = torch.where(fixed, 0., K(ud, absolute=True))
    bound_r = relres * nrm(f) + (U + C_PCG * iters.double() * U64) * nrm(Aabs) + 16 * U64 * nrm(Aabs)
    q_r = ratio(nrm(res), bound_r)
    rs = torch.where(fixed, 0., f - K(us))
    n = f[0].numel()
    fu, fus = (f * ud).sum(dim=(1, 2, 3)), (f * us).sum(dim=(1, 2, 3))
    slack = 8 * n * U64 * (f.abs() * (ud.abs() + us.abs())).sum(dim=(1, 2, 3))
    bound_m = nrm(us) * (nrm(res) + nrm(rs)) + nrm(rs) * nrm(ud - us) + slack
    return q_r, ratio((fu - fus).abs(), bound_m), bound_m, fu, fus


@pytest.fixture(scope='module')
def converged(golden):
    """the converged solves of converged_cases(): kernel outputs and the direct solution"""
    out = []
    for name, rho, bcs in converged_cases(golden('mechanics_eval.pt')):
        rho_d, bcs_d = rho.float().contiguous().to(DEV), bcs.float().contiguous().to(DEV)
        u, it, rr = pcg_launch(rho_d, bcs_d, 1e-6, 6000)
        out.append((name, rho_d, bcs_d, u, it, rr, O.fem_solve(rho.double(), bcs.double(), ke().double().cpu())))
    return out


def test_pcg_converged_solves(converged):
    for name, rho, bcs, u, it, rr, u_star in converged:
        assert bool((it < 6000).all() and (it > 0).all() and (rr < 1e-6).all()), (name, it, rr)
        q_r, q_m, _, _, _ = converged_ratios(rho, bcs, u, it, rr, u_star)
        note(TAG, f'pcg converged {name} relres honest', q_r)
        note(TAG, f'pcg converged {name} f^T u', q_m)
        assert q_r <= 1.0 and q_m <= 1.0, (name, q_r, q_m)


def test_pcg_table_row_and_rel_ce_error(converged, golden):
    """the recorded launch (B = 2, nel = 64, tol 1e-6, 6000) and topopt_metrics(solver='fused') on mechanics_eval.pt:
    rel_CE_error within the metric bound plus the fp32 sums of f^T u and of the data compliance, against fp64"""
    from physicsinformeddiffusionmodels_b200.residuals_mechanics_K import ResidualsMechanics
    B, nel, tol, max_iter = PCG_TABLE[0]
    _, rho, bcs, _, _, _, _ = converged[2]
    rho, bcs = rho[:B].contiguous(), bcs[:B].contiguous()
    u, it, rr = pcg_launch(rho, bcs, tol, max_iter)
    q_r, q_m, _, _, _ = converged_ratios(rho, bcs, u, it, rr, O.fem_solve(rho.cpu().double(), bcs.cpu().double(),
                                                                             ke().double().cpu()))
    note(TAG, f'pcg {PCG_TABLE[0]} relres honest', q_r)
    note(TAG, f'pcg {PCG_TABLE[0]} f^T u', q_m)
    assert q_r <= 1.0 and q_m <= 1.0
    gd = golden('mechanics_eval.pt')
    res = ResidualsMechanics(model=None, pixels_per_dim=64, pixels_at_boundary=True, no_BC_folder='', device=DEV,
                             topopt_eval=True)
    sol = gd['solution'].to(DEV)
    m = res.topopt_metrics(gd['x0_pred'][:, 2].contiguous().to(DEV), gd['bcs'].to(DEV), gd['vf'].to(DEV), sol,
                           solver='fused')
    name, rho_b, bcs_b, u_b, it_b, rr_b, us_b = converged[1]          # the same binarised system, solved once more
    u2, it2, rr2 = pcg_launch(rho_b, bcs_b, 1e-6, 6000)
    assert torch.equal(u2.view(torch.int32), u_b.view(torch.int32)) and torch.equal(it2, it_b), 'not deterministic'
    _, _, bound_m, fu, fus = converged_ratios(rho_b, bcs_b, u_b, it_b, rr_b, us_b)
    f = torch.where(bcs_b[:, :2] != 0, 0., bcs_b[:, 2:4]).double()
    opt = sol[:, :2].double()
    cd = (opt * f).sum(dim=(1, 2, 3))
    gam = (SUM_DEPTH + 1) * U
    rel_ref = (fus - cd) / cd
    e_ct = bound_m + gam * (u_b.double() * f).abs().sum(dim=(1, 2, 3))
    e_cd = gam * (opt * f).abs().sum(dim=(1, 2, 3))
    bound = e_ct / cd.abs() + (fu.abs() + e_ct) * e_cd / (cd * cd) + 4 * U * rel_ref.abs()
    q = ratio((m['rel_CE_error_full_batch'].double() - rel_ref).abs(), bound)
    note(TAG, 'rel_CE_error (fused) vs fp64', q)
    assert q <= 1.0, q


# ----------------------------------------------------------------------------------------------------------------------
# fm: the floating-material flag
# ----------------------------------------------------------------------------------------------------------------------
FM_NELS = (1, 2, 31, 33, 64, 110, 111, 127, 128)


def snake(n):
    d = np.zeros((n, n))
    for k in range(0, n, 2):
        d[k] = 1.
        if k + 1 < n:
            d[k + 1, n - 1 if (k // 2) % 2 == 0 else 0] = 1.
    return d


def spiral(n):
    """a one-pixel-wide square spiral with one-pixel gaps between its turns, walked in from the corner"""
    d = np.zeros((n, n))
    r, c, dr, dc = 0, 0, 0, 1
    d[0, 0] = 1.

    def free(rr, cc):
        return 0 <= rr < n and 0 <= cc < n and d[rr, cc] == 0

    turns = 0
    while turns < 2:
        if free(r + dr, c + dc) and (not (0 <= r + 2 * dr < n and 0 <= c + 2 * dc < n) or d[r + 2 * dr, c + 2 * dc] == 0):
            r, c = r + dr, c + dc
            d[r, c] = 1.
            turns = 0
        else:
            dr, dc = dc, -dr
            turns += 1
    return d


def fm_designs(nel, seed):
    """[D, nel, nel] fp32 designs: empty, full, one pixel, a diagonal line (contacts across corners only), a
    checkerboard (one 8-connected component), vertical stripes, the snake and the spiral, random fields at densities
    0.2 / 0.45 / 0.6 / 0.8, and the full design with pixels exactly at 0.5 and NaN pixels (not solid)"""
    rng = np.random.default_rng(seed)
    i = np.arange(nel)
    ds = [np.zeros((nel, nel)), np.ones((nel, nel))]
    one = np.zeros((nel, nel))
    one[nel // 2, nel // 3] = 1.
    ds.append(one)
    ds.append(np.eye(nel))
    ds.append(((i[:, None] + i[None, :]) % 2 == 0).astype(float))
    stripes = np.zeros((nel, nel))
    stripes[:, ::2] = 1.
    ds += [stripes, snake(nel), spiral(nel)]
    for dens in (0.2, 0.45, 0.6, 0.8):
        ds.append(np.where(rng.random((nel, nel)) < dens, 0.5 + 0.5 * rng.random((nel, nel)), 0.5 * rng.random((nel, nel))))
    half = np.ones((nel, nel))
    half[:, nel // 2] = 0.5                               # a column exactly at the threshold splits the design
    ds.append(half)
    nan = np.ones((nel, nel))
    nan[nel // 3, :] = np.nan                             # a NaN row splits it too
    ds.append(nan)
    return torch.tensor(np.stack(ds), dtype=torch.float32)


def fm_ref(rho, edit=None):
    """check_floating_material's rule with scipy labelling: flag = the solid pixels (> 0.5) do not form exactly one
    8-connected component.  edit: 'four_connected', 'threshold_ge', 'flag_roots_gt_1' (mutants)"""
    out = []
    for img in rho.cpu().numpy():
        solid = img >= 0.5 if edit == 'threshold_ge' else img > 0.5
        n = ndimage.label(solid, structure=None if edit == 'four_connected' else np.ones((3, 3)))[1]
        out.append(int(n > 1) if edit == 'flag_roots_gt_1' else int(n != 1))
    return torch.tensor(out)


def fm_launch(rho):
    B, nel = rho.shape[0], rho.shape[-1]
    buf, fm = guarded_int(B, torch.int64, -5)
    call_sync('pidm_mech_floating_material', rho.contiguous().to(DEV), fm, B, nel)
    assert int_guards_intact(buf, -5), 'a store landed outside fm'
    return fm.cpu()


def fm_batch(nel, spec, seed):
    """the designs of fm_designs, or B random designs (spec an int or 'wide')"""
    if spec == 'designs':
        return fm_designs(nel, seed)
    B = _batch(spec)
    g = torch.Generator().manual_seed(seed)
    dens = torch.rand(B, 1, 1, generator=g)
    return torch.rand(B, nel, nel, generator=g) * (torch.rand(B, nel, nel, generator=g) < dens) * 1.2


FM_ROWS = ([(spec, nel) for nel in FM_NELS for spec in ('designs', 1)] + [('wide', 33), ('wide', 128)]
           + [(r[0], r[1]) for r in FM_TABLE])


@pytest.mark.parametrize('row', FM_ROWS, ids=lambda r: f'{r[0]}_nel{r[1]}')
def test_fm_replay(row):
    spec, nel = row
    rho = fm_batch(nel, spec, 40 + nel)
    got, want = fm_launch(rho), fm_ref(rho)
    bad = int((got != want).sum())
    print(f'[{TAG}] fm {spec} nel={nel}: {rho.shape[0]} designs, {int(want.sum())} flagged, {bad} mismatches')
    assert bad == 0, (got, want)
    if spec == 'designs' and nel > 2:
        assert want[:3].tolist() == [1, 0, 0] and want[3:5].tolist() == [0, 0], 'the design table lost its meaning'


@pytest.mark.parametrize('edit', ['four_connected', 'threshold_ge', 'flag_roots_gt_1'])
def test_mutant_fm(edit):
    rho = fm_designs(33, 73)
    got = fm_launch(rho)
    assert torch.equal(got, fm_ref(rho))
    bad = int((got != fm_ref(rho, edit)).sum())
    print(f'[{TAG}] fm mutant {edit}: {bad} of {rho.shape[0]} flags differ')
    assert bad > 0, edit


# ----------------------------------------------------------------------------------------------------------------------
# mech_input and mech_post: the two kernels around the network call of a sampling step
# ----------------------------------------------------------------------------------------------------------------------
SAMPLE_PS = (2, 3, 16, 64, 127)
MECH_INPUT_ROWS = (MECH_INPUT_TABLE + [(b, nc, P) for P in SAMPLE_PS for b, nc in ((1, 0), (3, 7))]
                   + [('wrap', 7, 64), ('wrap', 0, 16), ('wrap', 7, 3)])
MECH_POST_ROWS = (MECH_POST_TABLE + [(b, P) for P in SAMPLE_PS for b in (1, 4)] + [('wrap', 64), ('wrap', 3)])


def mech_input_case(row, seed):
    B = _batch(row[0], input_total(1, row[1], row[2]))
    nc, P = row[1], row[2]
    g = gen(seed)
    x = torch.randn(B, 3, P + 1, P + 1, generator=g, device=DEV)
    planes = torch.randn(B, nc, P, P, generator=g, device=DEV)
    buf, out = guarded(input_total(B, nc, P))
    call_sync('pidm_mech_sample_input', x, planes, out, B, nc, P)
    assert guards_intact(buf), 'a store landed outside out'
    return x, planes, out.view(B, 3 + nc, P, P)


def mech_input_ratio(x, planes, out, edit=None):
    """(worst ratio of channels 0..2, planes bitwise equal) against fp64; edit 'planes_shifted' (mutant)"""
    B, _, n_in, _ = x.shape
    P = n_in - 1
    want = planes.roll(-1, dims=1) if edit == 'planes_shifted' else planes
    same = torch.equal(out[:, 3:].view(torch.int32), want.view(torch.int32))
    xd = x.double().cpu().reshape(B * 3, n_in, n_in)
    r = F.interpolate(xd[:, None], size=(P, P), mode='bilinear', align_corners=False)[:, 0]
    A, coord = resize_bounds(xd, P)
    return ratio((out[:, :3].double().cpu().reshape(B * 3, P, P) - r).abs(), C_RESIZE * U * A + coord), same


@pytest.mark.parametrize('row', MECH_INPUT_ROWS, ids=lambda r: 'B{}_nc{}_P{}'.format(*r))
def test_mech_input_replay(row):
    x, planes, out = mech_input_case(row, 900 + row[1] + row[2])
    q, same = mech_input_ratio(x, planes, out)
    note(TAG, f'mech_input {row}', q)
    assert same, 'channels >= 3 are not the planes bit for bit'
    assert q <= 1.0, q


N_STEPS = 100


def post_tables():
    """(c1, c2, sigma) fp32 on the device as SampleEngine passes them for a 100-step schedule (sigma[0] = 0)"""
    tab = O.diffusion_tables(N_STEPS)
    sig = tab['betas'].sqrt().float()
    sig[0] = 0.
    return (tab['posterior_mean_coef1'].float().to(DEV).contiguous(),
            tab['posterior_mean_coef2'].float().to(DEV).contiguous(), sig.to(DEV).contiguous())


def mech_post_case(row, seed):
    """operands and the out-of-place result of one launch; the same launch in place must equal it bit for bit"""
    B = _batch(row[0], post_total(1, row[1]))
    P = row[1]
    g = gen(seed)
    y = torch.randn(B, 3, P, P, generator=g, device=DEV)
    y[:, 2] = torch.rand(B, P, P, generator=g, device=DEV)
    x, z = (torch.randn(B, 3, P + 1, P + 1, generator=g, device=DEV) for _ in range(2))
    t = torch.randint(0, N_STEPS, (B,), generator=g, device=DEV)
    t[0] = 0
    t[-1] = N_STEPS - 1 if B > 1 else 0
    c1, c2, sig = post_tables()
    n = post_total(B, P)
    buf, xo = guarded(n)
    call_sync('pidm_mech_posterior_step', y, x, z, t, c1, c2, sig, xo, B, P)
    assert guards_intact(buf), 'a store landed outside x_out'
    ibuf, xi = guarded(n)
    xi.copy_(x.reshape(-1))
    call_sync('pidm_mech_posterior_step', y, xi, z, t, c1, c2, sig, xi, B, P)
    assert guards_intact(ibuf), 'a store landed outside x (in place)'
    assert torch.equal(xi.view(torch.int32), xo.view(torch.int32)), 'in place differs from out of place'
    return (y, x, z, t, c1, c2, sig), xo.view(B, 3, P + 1, P + 1)


def mech_post_ref(y, x, z, t, c1, c2, sig, edit=None):
    """fp64 (x', bound) on the host: model_out = (u_x, u_y resized P -> P + 1, rho zero-padded at row and column P).
    edit: 'c1_c2_swapped', 'pad_replicated', 'align_corners' (mutants)"""
    B, _, P, _ = y.shape
    yd, xd, zd = y.double().cpu(), x.double().cpu(), z.double().cpu()
    a, b, s = (v.double().cpu()[t.cpu()].view(B, 1, 1, 1) for v in (c1, c2, sig))
    if edit == 'c1_c2_swapped':
        a, b = b, a
    mo01 = F.interpolate(yd[:, :2], size=(P + 1, P + 1), mode='bilinear', align_corners=edit == 'align_corners')
    mo2 = F.pad(yd[:, 2:], (0, 1, 0, 1), mode='replicate' if edit == 'pad_replicated' else 'constant')
    mo = torch.cat((mo01, mo2), dim=1)
    A, coord = resize_bounds(yd[:, :2].reshape(B * 2, P, P), P + 1)
    e_mo = torch.cat(((C_RESIZE * U * A + coord).view(B, 2, P + 1, P + 1), torch.zeros(B, 1, P + 1, P + 1,
                                                                                         dtype=torch.float64)), dim=1)
    r = a * mo + b * xd + s * zd
    return r, C_MPOST * U * ((a * mo).abs() + (b * xd).abs() + (s * zd).abs()) + a.abs() * e_mo


@pytest.mark.parametrize('row', MECH_POST_ROWS, ids=lambda r: 'B{}_P{}'.format(*r))
def test_mech_post_replay(row):
    ops_, y = mech_post_case(row, 950 + row[1])
    r, bound = mech_post_ref(*ops_)
    q = ratio((y.double().cpu() - r).abs(), bound)
    note(TAG, f'mech_post {row}', q)
    assert q <= 1.0, q


# ----------------------------------------------------------------------------------------------------------------------
# mutants: the predicates above reject references edited the way a subtle kernel bug would change them
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('edit', [e for e in PCG_EDITS if e != 'stop_late'])
def test_mutant_pcg(edit):
    rho, bcs = pcg_operands(3, 31, 811)
    out = pcg_launch(rho, bcs, 0.0, 10)
    qu, qr, same = pcg_ratios(out, pcg_ref(rho, bcs, ke(), 10))
    assert same and max(qu, qr) <= 1.0
    qu, qr, _ = pcg_ratios(out, pcg_ref(rho, bcs, ke(), 10, edit=edit))
    note(TAG, f'pcg mutant {edit} u / relres', max(qu, qr))
    assert max(qu, qr) > 1.0, edit


def test_mutant_pcg_stop_late():
    B, nel, j = STOP_ROWS[1]
    rho, bcs = pcg_operands(B, nel, 700 + nel)
    tol, _ = stop_tol(rho, bcs, j)
    out = pcg_launch(rho, bcs, tol, 6000)
    assert max(pcg_ratios(out, stop_ref(rho, bcs, tol))[:2]) <= 1.0
    late = stop_ref(rho, bcs, tol, edit='stop_late')
    qu, qr, same = pcg_ratios(out, late)
    note(TAG, 'pcg mutant stop_late u / relres', max(qu, qr))
    assert not same and max(qu, qr) > 1.0


@pytest.mark.parametrize('edit', ['c1_c2_swapped', 'pad_replicated', 'align_corners'])
def test_mutant_mech_post(edit):
    ops_, y = mech_post_case((4, 16), 951)
    r, bound = mech_post_ref(*ops_)
    assert ratio((y.double().cpu() - r).abs(), bound) <= 1.0
    r, _ = mech_post_ref(*ops_, edit=edit)
    q = ratio((y.double().cpu() - r).abs(), bound)
    note(TAG, f'mech_post mutant {edit}', q)
    assert q > 1.0, edit


def test_mutant_mech_input_planes_shifted():
    x, planes, out = mech_input_case((3, 7, 16), 901)
    q, same = mech_input_ratio(x, planes, out)
    assert same and q <= 1.0
    _, same = mech_input_ratio(x, planes, out, edit='planes_shifted')
    assert not same


# ----------------------------------------------------------------------------------------------------------------------
# plan coverage
# ----------------------------------------------------------------------------------------------------------------------
def test_plan_coverage():
    n_sms = sms()
    nels = {r[1] for r in PCG_ROWS} | {r[1] for r in STOP_ROWS} | {r[1] for r in PCG_TABLE} | {64}
    batches = {_batch(r[0]) for r in PCG_ROWS}
    cases = {'pcg: the ninth node slot filled': any(pcg_ninth_slot_filled(n) for n in nels),
             'pcg: the ninth node slot empty': any(not pcg_ninth_slot_filled(n) for n in nels),
             'pcg: nel = 66, (nel+1)^2 <= 9 x 512 at its largest': 66 in nels and 67 ** 2 <= PCG_NPT * PCG_THREADS < 68 ** 2,
             'pcg: 161,584 B of shared memory at nel = 66': pcg_smem(66) == 161584,
             'pcg: B = 1': 1 in batches, 'pcg: more than two waves of CTAs': any(B > 2 * n_sms for B in batches),
             'pcg: nel = 2': 2 in nels}
    fnels = {r[1] for r in FM_ROWS}
    fbatches = {_batch(r[0]) for r in FM_ROWS if r[0] != 'designs'}
    cases.update({'fm: above 48 KB (opt-in)': any(fm_smem(n) > SMEM_DEFAULT for n in fnels),
                  'fm: the last nel below the opt-in': any(fm_smem(n) <= SMEM_DEFAULT < fm_smem(n + 1) for n in fnels),
                  'fm: one pixel per thread': any(n * n <= FM_THREADS for n in fnels),
                  'fm: 16 pixels per thread': any(-(-n * n // FM_THREADS) == 16 for n in fnels),
                  'fm: nel = 1': 1 in fnels, 'fm: B = 1': 1 in fbatches,
                  'fm: more than two waves': any(B > 2 * n_sms for B in fbatches)})
    ipasses = [grid_passes(input_total(_batch(r[0], input_total(1, r[1], r[2])), r[1], r[2]), n_sms)
               for r in MECH_INPUT_ROWS]
    ppasses = [grid_passes(post_total(_batch(r[0], post_total(1, r[1])), r[1]), n_sms) for r in MECH_POST_ROWS]
    cases.update({'mech_input: >= 2 grid-stride passes': max(ipasses) >= 2, 'mech_input: one pass': min(ipasses) == 1,
                  'mech_input: nc = 0 and 7': {r[1] for r in MECH_INPUT_ROWS} >= {0, 7},
                  'mech_post: >= 2 grid-stride passes': max(ppasses) >= 2, 'mech_post: one pass': min(ppasses) == 1,
                  'mech_post: P = 64 past the wrap (B >= 22 at 132 SMs)':
                      any(r[1] == 64 and grid_passes(post_total(_batch(r[0], post_total(1, 64)), 64), n_sms) >= 2
                          for r in MECH_POST_ROWS)})
    for P in SAMPLE_PS:
        cases[f'P = {P}'] = any(r[2] == P for r in MECH_INPUT_ROWS) and any(r[1] == P for r in MECH_POST_ROWS)
    missing = [c for c, ok in cases.items() if not ok]
    assert not missing, f'rows miss {missing}'
