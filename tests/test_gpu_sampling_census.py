"""The sampling-side kernels, replayed element by element against fp64: the DDIM jump coefficients, the ancestral
posterior step, the CoCoGen corrections and the toy PIDM loss.

pidm_ddim_coefs folds the mean / eps / jump algebra of the DDIM walk (ddim_sample_x0) into two per-sample coefficients
and must return exactly (0, 1) where a time grid repeats a point (t == t_next); pidm_posterior_step has a float4 path and
a scalar path for n % 4 != 0 (the toy study's odd batches); pidm_darcy_cocogen runs every correction of a sample in one
CTA with a per-sample step size, updates p in place, leaves inactive samples (t >= n_active) unread and unwritten and
re-evaluates the residual; pidm_toy_pidm_loss is one CTA of 256 threads looping over the batch with a clamped-NLL
branch of zero gradient and optional ineq / opt / p2 pointers.  Their other tests compare norm ratios, which a wrong tail
element, a wrong inactive sample or a wrong branch cannot move.  Here, in the five parts of the other census files:

  1. census: the distinct keys of the four entry points in one eager step of every sampling-side workload
     (census.census_sampling(): bench.py's sample-mode step, a DDIM walk with ddim_steps = 3, CoCoGen steps, the
     drop-in p_sample, conditional mechanics sampling and the toy study) must equal the tables below (`python
     tests/census.py --print-table` regenerates them).  The other kernels those steps launch (convolutions, norms,
     attention, glue) are checked at entry-point level only: their families replay the benchmarked shapes;
  2. replay: every table row plus synthetic rows, through the C ABI between NaN guards, on seeded operands, against fp64
     evaluated from the fp32 values the kernel reads.  With u = 2^-24 and A the same chain on absolute values:
        ddim        |c - r| <= C_DDIM u A, and bitwise (0, 1) where t == t_next
        posterior   |y - r| <= C_POST u (|c1 x0| + |c2 x| + |sigma z|)
        cocogen     p: see cocogen_ref; residual: C_DARCY u A against the fp64 residual of the kernel's own p; K,
                    inactive samples and their residual rows bitwise untouched
        toy_loss    sums: (C_TOY + depth) u A, depth the kernel's fp32 accumulation chain; gradients C_TOY u |r|
  3. mutants: the same predicates reject the fp64 references edited the way a subtle kernel bug would change them;
  4. plan coverage: the launch arithmetic, restated below, shows that the rows reach a ragged last CTA of the DDIM
     launch, both posterior paths and their grid-stride wrap, more CoCoGen CTAs than SMs and a partial last warp of the
     toy loop;
  5. completeness: every entry point census_sampling() calls is keyed, launches nothing or is named in
     census.CHECKED_ELSEWHERE with a test that exists.
"""
import numpy as np
import pytest
import torch

from census import (CHECKED_ELSEWHERE, assert_census_in_tables, assert_checked_or_listed, assert_tables_in_census,
                    census_exact, census_sampling)
from checks import P, U, call_sync, gen, guarded, guards_intact, note, ratio, sms
from oracle import pidm_oracle as O
from test_gpu_physics_census import C_DARCY, _fields, _geom, fs_dev, jacobian_max_ref

pytestmark = pytest.mark.gpu

DEV = 'cuda'
TAG = 'sampling census'
# The smallest powers of two that passed on an H100 80GB HBM3 (700 W), worst |err| / bound in brackets (DESIGN.md
# section 2): C_DDIM 2 (0.66), C_POST 4 (0.66), C_COCO 16 (0.83, the only value tried), C_TOY 4 (0.77 for the gradients)
C_DDIM = 2          # sqrt, two quotients, a product and a difference per coefficient
C_POST = 4          # two products and two adds (contracted or not)
C_COCO = 16         # roundings of one step's increment eps * dp, relative to its absolute chain
C_TOY = 4           # products and quotients before each term enters its sum

# ----------------------------------------------------------------------------------------------------------------------
# the committed census tables (`python tests/census.py --print-table`); distinct keys per workload:
#   darcy_sample_ddim0_b16, darcy_sample_ddim3_b4, mech_sample_sample_b2: ddim 1
#   cocogen_{xt,x0,M3}_{none,periodic}_b4: cocogen 1
#   p_sample_b2, toy_p_sample_b63: posterior 1
#   toy_loss_x0_b128, toy_loss_eps_b128: toy_loss 1
#   mech_sample_mean_b2, mech_aux_b2: none of the four
#   distinct: ddim 3, posterior 2, cocogen 4, toy_loss 2
# ----------------------------------------------------------------------------------------------------------------------
# ddim: B;  posterior: n;  cocogen: B, P, domain_length, reverse_d1, flags, steps, n_active, t set;
# toy_loss: B, D, ineq set, opt set, p2w set
DDIM_TABLE = [
    (2,),  # mech_sample_sample_b2
    (4,),  # darcy_sample_ddim3_b4
    (16,),  # darcy_sample_ddim0_b16
]
POSTERIOR_TABLE = [
    (126,),  # toy_p_sample_b63
    (16384,),  # p_sample_b2
]
COCOGEN_TABLE = [
    (4, 64, 1.0, 1, 1, 1, 2, 1),  # cocogen_x0_none_b4 cocogen_xt_none_b4
    (4, 64, 1.0, 1, 1, 3, 0, 0),  # cocogen_M3_none_b4
    (4, 64, 1.0, 1, 3, 1, 2, 1),  # cocogen_x0_periodic_b4 cocogen_xt_periodic_b4
    (4, 64, 1.0, 1, 3, 3, 0, 0),  # cocogen_M3_periodic_b4
]
TOY_LOSS_TABLE = [
    (128, 2, 0, 0, 0),  # toy_loss_eps_b128
    (128, 2, 1, 1, 1),  # toy_loss_x0_b128
]
TABLES = {'ddim': DDIM_TABLE, 'posterior': POSTERIOR_TABLE, 'cocogen': COCOGEN_TABLE, 'toy_loss': TOY_LOSS_TABLE}


# ----------------------------------------------------------------------------------------------------------------------
# census
# ----------------------------------------------------------------------------------------------------------------------
def test_census_is_covered_by_the_table():
    assert_census_in_tables(TABLES)


def test_every_table_row_is_produced_by_the_census():
    assert_tables_in_census(TABLES)


def test_every_sampling_entry_point_is_checked_or_listed():
    assert_checked_or_listed(census_sampling()[1], 'the sampling steps')
    stale = sorted(set(CHECKED_ELSEWHERE) - census_exact()[1] - census_sampling()[1])
    assert not stale, f'CHECKED_ELSEWHERE lists entry points that neither recording calls: {stale}'


# ----------------------------------------------------------------------------------------------------------------------
# launch arithmetic (restated from elementwise.cu and darcy.cu; the kernels have no plan query)
# ----------------------------------------------------------------------------------------------------------------------
def grid_for(n, block, n_sms):      # elementwise.cu grid_for: ceil(n / block) CTAs, capped at 16 per SM
    return min(max(-(-n // block), 1), 16 * n_sms)


def posterior_plan(n, n_sms):       # pidm_posterior_step: (float4 path, grid-stride passes over n/4 or n items)
    vec = n % 4 == 0
    items = n // 4 if vec else n
    return vec, -(-items // (grid_for(items, 256, n_sms) * 256))


TOY_THREADS = 256                   # pidm_toy_pidm_loss: one CTA; thread i takes samples i, i + 256, ...


def toy_depth(B, D):
    """the longest fp32 addition chain into one of the seven sums: a thread's own samples (D terms each for the data
    term), the five warp_sum levels, then the sum over the eight warp partials"""
    return -(-B // TOY_THREADS) * D + 5 + TOY_THREADS // 32


# ----------------------------------------------------------------------------------------------------------------------
# ddim: every (t, t_next) pair of the device time grids of ddim_sample_x0
# ----------------------------------------------------------------------------------------------------------------------
DDIM_NSTEPS = (100, 250)
DDIM_STEPS = (0, 1, 3, 10)
DDIM_SYNTH = [(1,), (127,), (128,), (129,), (1000,)]


def ddim_grid(t, s):
    """the reference's grid: list(map(int, np.linspace(0, t, s + 2)))"""
    return [int(v) for v in np.linspace(0, t, s + 2, endpoint=True, dtype=float)]


def ddim_pairs(n_steps):
    """every (t, t_next) pair the walk launches pidm_ddim_coefs with (t_next >= 0), for every t < n_steps and every
    ddim_steps of DDIM_STEPS"""
    pairs = set()
    for s in DDIM_STEPS:
        for t in range(n_steps):
            g = ddim_grid(t, s)
            pairs.update((g[k], g[k - 1]) for k in range(1, len(g)))
    return sorted(pairs)


def ddim_tables(n_steps):
    tab = O.diffusion_tables(n_steps)
    return {k: tab[k].float().to(DEV).contiguous() for k in
            ('posterior_mean_coef1', 'posterior_mean_coef2', 'sqrt_recip_alphas', 'noise_mean_coeff', 'alphas_prod')}


def ddim_ref(tt, tn, tab, edit=None):
    """fp64 (coef_x0, coef_x, A_x0, A_x) of the reference's jump from the fp32 tables: mean = c1 x0 + c2 x,
    eps = (sra x - mean) / nmc, x' = sqrt(a') x0 + sqrt(1 - a') eps with a' = alphas_prod[t_next], and x' = x where
    t == t_next.  edit: 'identity_dropped', 'a_next_at_t', 'c_from_a_t' (mutants)"""
    d = {k: v.double() for k, v in tab.items()}
    c1, c2, sra, nmc = (d[k][tt] for k in ('posterior_mean_coef1', 'posterior_mean_coef2', 'sqrt_recip_alphas',
                                           'noise_mean_coeff'))
    an = d['alphas_prod'][tt if edit == 'a_next_at_t' else tn]
    c = torch.sqrt(1 - (d['alphas_prod'][tt] if edit == 'c_from_a_t' else an))
    cx0 = torch.sqrt(an) - c * c1 / nmc
    cx = c * (sra - c2) / nmc
    A0 = torch.sqrt(an) + c * c1.abs() / nmc
    A1 = c * (sra.abs() + c2.abs()) / nmc
    if edit != 'identity_dropped':
        same = tt == tn
        cx0, cx = torch.where(same, 0., cx0), torch.where(same, 1., cx)
    return cx0, cx, A0, A1


def ddim_bound(tt, tn, A):
    """C_DDIM u A, and 0 where t == t_next: the identity branch is exact"""
    return torch.where(tt == tn, 0., C_DDIM * U * A)


def ddim_launch(tt, tn, tab, B):
    """coef_x0, coef_x of all pairs, launched B pairs at a time (the last launch padded with the first pairs)"""
    n = len(tt)
    pad = (-n) % B
    t_all, n_all = torch.cat([tt, tt[:pad]]), torch.cat([tn, tn[:pad]])
    out0, out1 = [], []
    for lo in range(0, n + pad, B):
        b0, c0 = guarded(B)
        b1, c1 = guarded(B)
        call_sync('pidm_ddim_coefs', t_all[lo:lo + B].contiguous(), n_all[lo:lo + B].contiguous(),
                  tab['posterior_mean_coef1'], tab['posterior_mean_coef2'], tab['sqrt_recip_alphas'],
                  tab['noise_mean_coeff'], tab['alphas_prod'], c0, c1, B)
        assert guards_intact(b0) and guards_intact(b1), 'a store landed outside coef_x0 / coef_x'
        out0.append(c0.clone())
        out1.append(c1.clone())
    return torch.cat(out0)[:n], torch.cat(out1)[:n]


def ddim_case(n_steps, B):
    pairs = torch.tensor(ddim_pairs(n_steps), dtype=torch.long, device=DEV)
    tt, tn = pairs[:, 0].contiguous(), pairs[:, 1].contiguous()
    tab = ddim_tables(n_steps)
    return tt, tn, tab, ddim_launch(tt, tn, tab, B)


def ddim_ratios(tt, tn, tab, y, edit=None):
    cx0, cx, A0, A1 = ddim_ref(tt, tn, tab, edit)
    return (ratio((y[0].double() - cx0).abs(), ddim_bound(tt, tn, A0)),
            ratio((y[1].double() - cx).abs(), ddim_bound(tt, tn, A1)))


@pytest.mark.parametrize('n_steps', DDIM_NSTEPS)
@pytest.mark.parametrize('row', DDIM_TABLE + DDIM_SYNTH, ids=lambda k: f'B{k[0]}')
def test_ddim_replay(row, n_steps):
    tt, tn, tab, y = ddim_case(n_steps, row[0])
    assert bool((tt == tn).any()), 'no repeated grid point among the pairs'
    q0, q1 = ddim_ratios(tt, tn, tab, y)
    note(TAG, f'ddim n_steps={n_steps} B={row[0]} coef_x0', q0)
    note(TAG, f'ddim n_steps={n_steps} B={row[0]} coef_x', q1)
    assert max(q0, q1) <= 1.0, (q0, q1)


def test_ddim_pairs_are_those_of_the_device_grid():
    """the pairs above are the device grid's (ddim_sample_x0 builds it as k * (t / (s + 1)) truncated, t last)"""
    for n_steps in DDIM_NSTEPS:
        for s in DDIM_STEPS:
            t = torch.arange(n_steps, dtype=torch.long)
            k = torch.arange(s + 2, dtype=torch.float64)
            grid = (k[None, :] * (t.double() / (s + 1))[:, None]).long()
            grid[:, -1] = t
            assert grid.tolist() == [ddim_grid(ti, s) for ti in range(n_steps)], (n_steps, s)


# ----------------------------------------------------------------------------------------------------------------------
# posterior: x_{t-1} = c1 x0 + c2 x_t + sigma z
# ----------------------------------------------------------------------------------------------------------------------
def _wrap(kind):
    """n that makes the capped grid of the float4 ('wrap4') or scalar ('wrap1') path take three grid-stride passes"""
    threads = grid_for(1 << 40, 256, sms()) * 256
    return 4 * 2 * threads + 4 if kind == 'wrap4' else 2 * threads + 1


# n % 4 = 0, 1, 2, 3, n < 4, the toy study's odd batch (126 = 63 x 2), and the two grid-stride wraps
POSTERIOR_SYNTH = [1, 2, 3, 4, 5, 6, 7, 126, 4097, 4098, 4099, 8192, 'wrap4', 'wrap1']



def posterior_coefs(t):
    """(c1, c2, sigma) as the drop-in p_sample passes them for a 100-step schedule (sigma = 0 at t = 0), rounded to the
    fp32 the C ABI takes"""
    tab = O.diffusion_tables(100)
    f = lambda v: float(torch.tensor(float(v), dtype=torch.float32))   # noqa: E731
    return f(tab['posterior_mean_coef1'][t]), f(tab['posterior_mean_coef2'][t]), (0. if t == 0 else
                                                                                   f(tab['betas'][t].sqrt()))


def posterior_ref(x, x0, z, c1, c2, sig, edit=None):
    if edit == 'c1_c2_swapped':
        c1, c2 = c2, c1
    x, x0, z = x.double(), x0.double(), z.double()
    r = c1 * x0 + c2 * x + sig * z
    return r, C_POST * U * ((c1 * x0).abs() + (c2 * x).abs() + (sig * z).abs())


def posterior_launch(n, t, seed):
    g = gen(seed)
    x, x0, z = (torch.randn(n, generator=g, device=DEV) for _ in range(3))
    c1, c2, sig = posterior_coefs(t)
    buf, y = guarded(n)
    call_sync('pidm_posterior_step', x, x0, z, y, c1, c2, sig, n)
    assert guards_intact(buf), 'a store landed past n'
    return (x, x0, z, c1, c2, sig), y


@pytest.mark.parametrize('t', [0, 57])
@pytest.mark.parametrize('n', [r[0] for r in POSTERIOR_TABLE] + POSTERIOR_SYNTH, ids=str)
def test_posterior_replay(n, t):
    n = _wrap(n) if isinstance(n, str) else n
    ops_, y = posterior_launch(n, t, 7 + n % 1000)
    r, bound = posterior_ref(*ops_)
    q = ratio((y.double() - r).abs(), bound)
    note(TAG, f'posterior n={n} t={t}', q)
    assert q <= 1.0, q


# ----------------------------------------------------------------------------------------------------------------------
# cocogen
# ----------------------------------------------------------------------------------------------------------------------
# Bound of the corrected p.  Step s computes delta_s = fl(eps * fl(dp_s)), dp_s = 2 J^T r(p_s), and p_{s+1} =
# fl(p_s - delta_s).  The kernel's eps = 1e-6 / max(dr/dp) carries the rounding of the maximum; dp_s carries the stencil
# roundings of r, which are relative to A_r = |stencils| (|K|, |p|, |f_s|) (the residual is a small difference of large
# terms), carried through |J|^T; the subtraction rounds p once per step.  The iteration is a fixed affine map close to
# the identity (eps |J^T J| is below one), so the errors of the steps add up:
#     |p_kernel - p_ref| <= u (S |p_S| + C_COCO sum_s (eps |J|^T (2 |r_s| + 2 A_r(p_s)) + |delta_s|))
# evaluated in fp64 along the reference's own iterates.  S = 0 makes the bound 0: p must come back bitwise.
COCOGEN_SYNTH = [
    (1, 64, 1.0, 1, 1, 1, 0, 0),            # one sample, one step
    (3, 64, 2.5, 0, 1, 5, 0, 0),            # domain_length != 1, reverse_d1 = 0
    (3, 64, 1.0, 1, 0, 2, 0, 0),            # pixels not at the boundary
    (3, 64, 1.0, 1, 1, 200, 0, 0),          # 200 steps
    (3, 64, 1.0, 1, 3, 200, 0, 0),          # 200 steps, periodic
    (3, 64, 1.0, 0, 3, 5, 0, 0),            # periodic, reverse_d1 = 0
    (5, 64, 2.5, 0, 3, 0, 2, 1),            # zero steps under a per-sample t
    (300, 64, 1.0, 1, 3, 2, 2, 1),          # more CTAs than SMs, mixed active and inactive samples
    (300, 64, 0.5, 0, 1, 1, 0, 0),
]
CHUNK = 100                                 # samples per fp64 reference chunk


def coco_t(B, n_active):
    """per-sample t: b mod (n_active + 2) mixes active (t < n_active) and inactive samples"""
    return torch.arange(B, device=DEV) % (n_active + 2)


def cocogen_ref(x, steps, per, geom, edit=None):
    """fp64 (p after `steps` corrections [B,P,P], bound [B,P,P]) of fp32 fields x [B,2,P,P]: the fp64 O.cocogen_steps
    at the geometry given (step size 1e-6 / jacobian max per sample).  edit: 'one_step_fewer', 'batch_max_step',
    'adjoint_wrap_dropped' (mutants)"""
    x = x.double()
    mx = jacobian_max_ref(x, per, geom)[0]
    if edit == 'batch_max_step':
        mx = mx.max().expand_as(mx)
    eps = (1e-6 / mx.clamp(max=1e12)).view(-1, 1, 1)
    stencils = O.darcy_stencils(P, per, **geom)
    adj = stencils
    if edit == 'adjoint_wrap_dropped':                      # row 0 of the p adjoint without its wrap to row P-1
        adj = list(stencils)
        adj[0], adj[1] = adj[0].clone(), adj[1].clone()
        adj[0][0, -1], adj[1][0, -1] = 0., 0.
    n = steps - 1 if edit == 'one_step_fewer' else steps
    acc = torch.zeros_like(x[:, 0])
    for _ in range(n):
        r = O.darcy_residual_matrix(x, per, stencils=stencils, **geom)
        Ar = O.darcy_residual_matrix(x, per, absolute=True, stencils=stencils, **geom)
        dp = O.darcy_residual_vjp(x, 2 * r, per, stencils=adj, **geom)[:, 0]
        dpa = O.darcy_residual_vjp(x, 2 * (r.abs() + Ar), per, absolute=True, stencils=stencils, **geom)[:, 0]
        delta = eps * dp
        acc += eps * dpa + delta.abs()
        x = x.clone()
        x[:, 0] = x[:, 0] - delta
    return x[:, 0], U * (steps * x[:, 0].abs() + C_COCO * acc)


def cocogen_launch(row, seed):
    """(fields x, t or None, x after the launch, residual after the launch, residual prefill)"""
    B, _, L, rev, flags, steps, n_active, tset = row
    x = _fields(B, seed)
    t = coco_t(B, n_active) if tset else None
    xbuf, xd = guarded(B * 2 * P * P)
    xd.copy_(x.reshape(-1))
    rbuf, rd = guarded(B * P * P * 3)
    prefill = torch.randn(B * P * P * 3, generator=gen(seed + 1), device=DEV)
    rd.copy_(prefill)
    call_sync('pidm_darcy_cocogen', xd, fs_dev(), rd, t, n_active, steps, B, P, float(L), int(rev), int(flags))
    assert guards_intact(xbuf) and guards_intact(rbuf), 'a store landed outside x / residual'
    return x, t, xd.view(B, 2, P, P), rd.view(B, P * P, 3), prefill.view(B, P * P, 3)


def cocogen_check(row, seed, edit=None, note_it=True):
    """worst (p ratio, residual ratio) of one row; asserts the bitwise parts"""
    B, _, L, rev, flags, steps, n_active, tset = row
    geom, per = _geom(L, rev, flags)
    x, t, y, res, prefill = cocogen_launch(row, seed)
    active = torch.ones(B, dtype=torch.bool, device=DEV) if t is None else t < n_active
    if edit == 'inactive_corrected':          # the reference corrects every sample; nothing is left to compare bitwise
        active = torch.ones_like(active)
    assert torch.equal(y[:, 1].view(torch.int32), x[:, 1].view(torch.int32)), 'K was written'
    qp = qr = 0.
    idx = active.nonzero().flatten()
    for lo in range(0, len(idx), CHUNK):
        i = idx[lo:lo + CHUNK]
        pr, bp = cocogen_ref(x[i], steps, per, geom, edit)
        qp = max(qp, ratio((y[i, 0].double() - pr).abs(), bp))
        yi = y[i].double()
        r = O.darcy_residual_matrix(yi, per, **geom)
        A = O.darcy_residual_matrix(yi, per, absolute=True, **geom)
        qr = max(qr, ratio((res[i].double() - r).abs(), C_DARCY * U * A))
    idle = (~active).nonzero().flatten()
    if len(idle):
        assert torch.equal(y[idle].view(torch.int32), x[idle].view(torch.int32)), 'an inactive sample was written'
        assert torch.equal(res[idle].view(torch.int32), prefill[idle].view(torch.int32)), \
            'the residual row of an inactive sample was written'
    if note_it:
        note(TAG, f'cocogen {row} p', qp)
        note(TAG, f'cocogen {row} residual', qr)
    return qp, qr


def coco_id(k):
    B, _, L, rev, flags, steps, n_active, tset = k
    return (f'B{B}_L{L}_rev{rev}_f{flags}_s{steps}' + (f'_t{n_active}' if tset else ''))


@pytest.mark.parametrize('row', COCOGEN_TABLE + COCOGEN_SYNTH, ids=coco_id)
def test_cocogen_replay(row):
    qp, qr = cocogen_check(row, 60 + row[0] + row[5])
    assert qp <= 1.0 and qr <= 1.0, (qp, qr)


# ----------------------------------------------------------------------------------------------------------------------
# toy_loss
# ----------------------------------------------------------------------------------------------------------------------
TOY_CLAMP = float(torch.tensor(27.6310211159, dtype=torch.float32))
# B, D, ineq set, opt set, p2w set: every batch and D, every pointer combination
TOY_SYNTH = [(1, 1, 0, 0, 0), (31, 2, 1, 0, 0), (256, 3, 0, 1, 0), (257, 2, 1, 1, 0), (1000, 1, 0, 0, 1),
             (31, 3, 1, 0, 1), (257, 1, 0, 1, 1), (1000, 2, 1, 1, 1), (256, 2, 1, 1, 1)]
TOY_COEFS = (1.0, 0.005, 0.3, 0.01)


def toy_inputs(key, seed):
    """target, output [B,D]; r, q with 0.5 v^2 / var below 13.8 or above 55 (both clamp branches, clear of 27.6); o; t"""
    B, D, qs, os_, ps = key
    g = gen(seed)
    from physicsinformeddiffusionmodels_b200 import denoising_toy_utils as T
    dd = T.create_diff_dict(100, DEV)
    pvar, p2w = dd['posterior_variance_clipped'].float().contiguous(), dd['p2_loss_weight'].float().contiguous()
    t = torch.randint(0, 100, (B,), generator=g, device=DEV)

    def nll_field():
        clamped = torch.rand(B, generator=g, device=DEV) < 0.5
        nll = torch.where(clamped, 55 + 45 * torch.rand(B, generator=g, device=DEV),
                          13.8 * torch.rand(B, generator=g, device=DEV))
        sign = torch.where(torch.rand(B, generator=g, device=DEV) < 0.5, -1., 1.)
        return (sign * torch.sqrt(2 * nll * pvar[t].double())).float()
    target, output = (torch.randn(B, D, generator=g, device=DEV) for _ in range(2))
    r = nll_field()
    q = nll_field() if qs else None
    o = torch.randn(B, generator=g, device=DEV) if os_ else None
    return dict(target=target, output=output, r=r, q=q, o=o, t=t, p2w=p2w if ps else None, pvar=pvar)


def toy_ref(a, edit=None):
    """fp64 ({name: value}, {name: bound base A}) of the seven sums and the four gradients.  edit: 'grad_through_clamp',
    'no_inv_D', 'p2_at_t_plus_1' (mutants)"""
    c_data, c_res, c_ineq, lam = TOY_COEFS
    B, D = a['output'].shape
    t = a['t']
    iv = 1 / a['pvar'].double()[t]
    if a['p2w'] is None:
        w = torch.ones(B, dtype=torch.float64, device=DEV)
    else:
        w = a['p2w'].double()[(t + 1).clamp(max=99) if edit == 'p2_at_t_plus_1' else t]
    w = w * c_data / B / (1 if edit == 'no_inv_D' else D)
    e = a['output'].double() - a['target'].double()
    v, A = {}, {}
    v['data'] = (w[:, None] * e * e).sum()
    A['data'] = v['data']
    v['g_out'] = 2 * w[:, None] * e

    def nll_term(x, c):
        x = x.double()
        nll = 0.5 * x * x * iv
        live = nll < TOY_CLAMP
        term = c / B * torch.where(live, nll, torch.tensor(TOY_CLAMP, dtype=torch.float64, device=DEV))
        grad = c / B * x * iv
        if edit != 'grad_through_clamp':
            grad = torch.where(live, grad, 0.)
        return term.sum(), term.abs().sum(), grad
    v['res'], A['res'], v['g_r'] = nll_term(a['r'], c_res)
    v['abs_r'] = a['r'].double().abs().sum() / B
    A['abs_r'] = v['abs_r']
    zero = torch.zeros((), dtype=torch.float64, device=DEV)
    if a['q'] is not None:
        v['ineq'], A['ineq'], v['g_q'] = nll_term(a['q'], c_ineq)
        v['mean_q'], A['mean_q'] = a['q'].double().sum() / B, a['q'].double().abs().sum() / B
    else:
        v['ineq'] = A['ineq'] = v['mean_q'] = A['mean_q'] = zero
    if a['o'] is not None:
        o = a['o'].double()
        v['opt'], A['opt'] = lam / B * o.sum(), lam / B * o.abs().sum()
        v['mean_o'], A['mean_o'] = o.sum() / B, o.abs().sum() / B
        v['g_o'] = torch.full((B,), lam / B, dtype=torch.float64, device=DEV)
    else:
        v['opt'] = A['opt'] = v['mean_o'] = A['mean_o'] = zero
    return v, A


SUMS = ('data', 'res', 'ineq', 'opt', 'abs_r', 'mean_q', 'mean_o')


def toy_launch(a):
    B, D = a['output'].shape
    sb, sums = guarded(7)
    gb = {k: guarded(n) for k, n in (('g_out', B * D), ('g_r', B))}
    if a['q'] is not None:
        gb['g_q'] = guarded(B)
    if a['o'] is not None:
        gb['g_o'] = guarded(B)
    g = {k: v[1] for k, v in gb.items()}
    call_sync('pidm_toy_pidm_loss', a['target'], a['output'], a['r'], a['q'], a['o'], a['t'], a['p2w'], a['pvar'],
              *TOY_COEFS, sums, g['g_out'], g['g_r'], g.get('g_q'), g.get('g_o'), B, D)
    assert guards_intact(sb) and all(guards_intact(b) for b, _ in gb.values()), 'a store landed outside an output'
    out = dict(zip(SUMS, sums))
    out.update({k: v.view(B, D) if k == 'g_out' else v for k, v in g.items()})
    return out


def toy_ratios(key, a, y, edit=None):
    v, A = toy_ref(a, edit)
    depth = toy_depth(key[0], key[1])
    q = {}
    for k in SUMS:
        q[k] = ratio((y[k].double() - v[k]).abs().view(1), ((C_TOY + depth) * U * A[k]).view(1))
    for k in ('g_out', 'g_r', 'g_q', 'g_o'):
        if k in y:
            q[k] = ratio((y[k].double() - v[k]).abs(), C_TOY * U * v[k].abs())
    return q


@pytest.mark.parametrize('key', TOY_LOSS_TABLE + TOY_SYNTH, ids=lambda k: 'B{}_D{}_q{}_o{}_p{}'.format(*k))
def test_toy_loss_replay(key):
    a = toy_inputs(key, 300 + key[0] + key[1])
    y = toy_launch(a)
    q = toy_ratios(key, a, y)
    for k, v in q.items():
        note(TAG, f'toy_loss {key} {k}', v)
    assert max(q.values()) <= 1.0, q


# ----------------------------------------------------------------------------------------------------------------------
# mutants: the predicates above reject references edited the way a subtle kernel bug would change them
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('edit', ['identity_dropped', 'a_next_at_t', 'c_from_a_t'])
def test_mutant_ddim(edit):
    tt, tn, tab, y = ddim_case(100, 129)
    assert max(ddim_ratios(tt, tn, tab, y)) <= 1.0
    assert max(ddim_ratios(tt, tn, tab, y, edit)) > 1.0, edit


def test_mutant_posterior_c1_c2_swapped():
    ops_, y = posterior_launch(4099, 57, 5)
    r, b = posterior_ref(*ops_)
    assert ratio((y.double() - r).abs(), b) <= 1.0
    r, b = posterior_ref(*ops_, edit='c1_c2_swapped')
    assert ratio((y.double() - r).abs(), b) > 1.0


@pytest.mark.parametrize('n', [4097, 4098, 4099])
def test_mutant_posterior_tail_unwritten(n):
    """the output of a kernel that ran the float4 path over n // 4 quads and skipped the n % 4 tail"""
    ops_, y = posterior_launch(n, 57, 6)
    r, b = posterior_ref(*ops_)
    assert ratio((y.double() - r).abs(), b) <= 1.0
    y = y.clone()
    y[n - n % 4:] = float('nan')
    assert ratio((y.double() - r).abs(), b) > 1.0


@pytest.mark.parametrize('edit,row', [
    ('one_step_fewer', (3, 64, 1.0, 1, 1, 5, 0, 0)),
    ('inactive_corrected', (5, 64, 1.0, 1, 3, 2, 2, 1)),
    ('batch_max_step', (3, 64, 1.0, 1, 1, 2, 0, 0)),
    ('adjoint_wrap_dropped', (3, 64, 1.0, 1, 3, 2, 0, 0)),
], ids=lambda v: v if isinstance(v, str) else '')
def test_mutant_cocogen(edit, row):
    seed = 60 + row[0] + row[5]
    assert max(cocogen_check(row, seed, note_it=False)) <= 1.0
    assert cocogen_check(row, seed, edit, note_it=False)[0] > 1.0, edit


@pytest.mark.parametrize('edit', ['grad_through_clamp', 'no_inv_D', 'p2_at_t_plus_1'])
def test_mutant_toy_loss(edit):
    key = (257, 2, 1, 1, 1)
    a = toy_inputs(key, 300 + key[0] + key[1])
    y = toy_launch(a)
    assert max(toy_ratios(key, a, y).values()) <= 1.0
    assert max(toy_ratios(key, a, y, edit).values()) > 1.0, edit


# ----------------------------------------------------------------------------------------------------------------------
# plan coverage
# ----------------------------------------------------------------------------------------------------------------------
def test_plan_coverage():
    n_sms = sms()
    Bs = [r[0] for r in DDIM_TABLE + DDIM_SYNTH]
    cases = {'ddim: one partial CTA': any(B < 128 for B in Bs), 'ddim: whole CTAs only': any(B % 128 == 0 for B in Bs),
             'ddim: a ragged last CTA after full ones': any(B > 128 and B % 128 for B in Bs),
             'ddim: B = 1': 1 in Bs, 'ddim: below the grid cap': all(grid_for(B, 128, n_sms) == -(-B // 128) for B in Bs)}
    ns = [r[0] for r in POSTERIOR_TABLE] + [_wrap(n) if isinstance(n, str) else n for n in POSTERIOR_SYNTH]
    plans = [posterior_plan(n, n_sms) for n in ns]
    cases.update({f'posterior: n % 4 = {m}': any(n % 4 == m for n in ns) for m in range(4)})
    cases.update({'posterior: n < 4': any(n < 4 for n in ns),
                  'posterior: float4 path, >= 3 passes': any(v and p >= 3 for v, p in plans),
                  'posterior: scalar path, >= 3 passes': any(not v and p >= 3 for v, p in plans)})
    cc = COCOGEN_TABLE + COCOGEN_SYNTH
    cases.update({'cocogen: more CTAs (one per sample) than SMs': any(k[0] > n_sms for k in cc),
                  'cocogen: B = 1': any(k[0] == 1 for k in cc),
                  'cocogen: both bcs': {k[4] & 2 for k in cc} == {0, 2},
                  'cocogen: both reverse_d1': {k[3] for k in cc} == {0, 1},
                  'cocogen: domain_length != 1': any(k[2] != 1.0 for k in cc),
                  'cocogen: mixed active / inactive': any(k[7] and k[0] > k[6] > 0 for k in cc)})
    for s in (0, 1, 2, 5, 200):
        cases[f'cocogen: {s} steps'] = any(k[5] == s for k in cc)
    tk = TOY_LOSS_TABLE + TOY_SYNTH
    cases.update({'toy: B < 32 (one partial warp)': any(k[0] < 32 for k in tk),
                  'toy: a partial last warp': any(k[0] % 32 for k in tk),
                  'toy: B = 256 (every thread one sample)': any(k[0] == TOY_THREADS for k in tk),
                  'toy: the loop over B wraps': any(k[0] > TOY_THREADS for k in tk),
                  'toy: D = 1, 2, 3': {k[1] for k in tk} >= {1, 2, 3},
                  'toy: every pointer combination': {k[2:] for k in tk} == {(a, b, c) for a in (0, 1) for b in (0, 1)
                                                                           for c in (0, 1)}})
    missing = [c for c, ok in cases.items() if not ok]
    assert not missing, f'rows miss {missing}'
