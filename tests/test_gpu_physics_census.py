"""Every physics-residual launch of the benchmarked steps, replayed element by element against an fp64 reference.

The Darcy residual (darcy.cu), the mechanics residual, its fused loss and the bilinear resize (mechanics.cu) choose their
grids from the batch, the SM count and the mesh size: persistent Darcy CTAs that walk the batch with a double-buffered
bulk copy, 8-row mechanics bands with a ragged last band, grid-stride resize loops.  The per-op tests in test_gpu_ops.py
compare whole tensors by a norm ratio at a few small batches, which a bug confined to one band, one BC column or the last
wave of CTAs cannot move.  Here, in the four parts of the other census files and one more:

  1. census: one eager step of every workload bench.py times is recorded at the C ABI, and the distinct keys of the
     physics entry points (entry point, integer and flag arguments, which optional pointers are set) must equal the
     tables below (`python tests/census.py --print-table` regenerates them).  The standalone sweeps of
     bench.py are fixed rows that name the function they come from;
  2. replay: every table row and synthetic row runs through the C ABI on seeded fp32-exact operands, between NaN guards,
     against the fp64 references of oracle/pidm_oracle.py, per element:
        |y - r| <= C 2^-24 A            A = the same chain evaluated on absolute values
     and for reductions (compliance, loss sums) (C + depth) 2^-24 A, depth = the fp32 accumulation chain of the kernel;
     the resize adds the error of its fp32 source coordinate (see resize_bounds);
  3. mutants: the same predicates reject the fp64 reference edited the way a subtle kernel bug would change it;
  4. plan coverage: the launch arithmetic, restated below, shows that the rows reach every grid case;
  5. completeness: every entry point the benchmarked steps call is either checked by one of the five census files (has
     a key in census.KEYS) or listed in census.LAUNCHES_NOTHING (host-side queries).
"""
import math

import pytest
import torch
import torch.nn.functional as F

from census import KEYS, LAUNCHES_NOTHING, assert_census_in_tables, assert_tables_in_census, census
from checks import P, U, call_sync, check, gen, guarded, guards_intact, resize_bounds, resize_src_index, sms
from oracle import pidm_oracle as O

pytestmark = pytest.mark.gpu
DEV = 'cuda'
TAG = 'physics census'

# Bound constants: C fp32 roundings of the absolute-value chain, each the smallest power of two that passes on an H100
# (the worst |err| / (2^-24 A) seen was 6.6 for Darcy, 4.4 for mechanics, 6.2 for the fused losses); the worst
# |err| / bound per output is recorded in DESIGN.md section 2.
C_DARCY = 8
C_MECH = 8
C_LOSS = 8
C_RESIZE = 4
CHUNK = 2048                     # samples per fp64 reference chunk on the device

# ----------------------------------------------------------------------------------------------------------------------
# the committed census tables (`python tests/census.py --print-table`)
# ----------------------------------------------------------------------------------------------------------------------
# darcy_fwd / darcy_bwd: B, P, domain_length, reverse_d1, flags
# darcy_loss: B, P, domain_length, reverse_d1, flags, model_out == x0hat, grad_x0hat set, grad_model_out set
# mech_fwd: B, nel, compliance set;  mech_bwd: B, nel, grad_residual set, grad_compliance set;  mech_loss: B, nel
# resize_fwd / resize_bwd: planes, in, out
DARCY_FWD_TABLE = [
    (16, 64, 1.0, 1, 1),  # darcy_sample_b16 darcy_sample_ddim0_b16
    (64, 64, 1.0, 1, 1),  # darcy_sample_b64
    (256, 64, 1.0, 1, 1),  # darcy_sample_b256
]
DARCY_BWD_TABLE = [
]
DARCY_LOSS_TABLE = [
    (32, 64, 1.0, 1, 1, 1, 1, 0),  # darcy_train_b32
]
MECH_FWD_TABLE = [
    (32, 64, 1),  # mech_train_b32
]
MECH_BWD_TABLE = [
    (32, 64, 1, 1),  # mech_train_b32
]
MECH_LOSS_TABLE = [
    (32, 64),  # mech_train_b32
]
RESIZE_FWD_TABLE = [
    (64, 64, 65),  # mech_train_b32
    (128, 65, 64),  # mech_train_b32
    (192, 65, 64),  # mech_train_b32
]
RESIZE_BWD_TABLE = [
    (64, 64, 65),  # mech_train_b32
]
TABLES = {'darcy_fwd': DARCY_FWD_TABLE, 'darcy_bwd': DARCY_BWD_TABLE, 'darcy_loss': DARCY_LOSS_TABLE,
          'mech_fwd': MECH_FWD_TABLE, 'mech_bwd': MECH_BWD_TABLE, 'mech_loss': MECH_LOSS_TABLE,
          'resize_fwd': RESIZE_FWD_TABLE, 'resize_bwd': RESIZE_BWD_TABLE}
# the standalone launches of bench.py, outside the recorded steps: (family, key, the bench.py function)
BENCH_ROWS = [
    ('darcy_fwd', (32768, 64, 1.0, 1, 1), 'residual_kernel_sweep'),
    ('darcy_loss', (32768, 64, 1.0, 1, 1, 1, 1, 0), 'residual_kernel_sweep'),
    ('mech_fwd', (8192, 64, 1), 'mechanics_bench'),
]


# ----------------------------------------------------------------------------------------------------------------------
# census
# ----------------------------------------------------------------------------------------------------------------------
def test_census_is_covered_by_the_table():
    assert_census_in_tables(TABLES)


def test_every_table_row_is_produced_by_the_census():
    assert_tables_in_census(TABLES)


def test_every_benchmarked_entry_point_is_checked_or_listed():
    _, names = census()
    covered = set(KEYS)
    unchecked = sorted(names - covered - set(LAUNCHES_NOTHING))
    assert not unchecked, ('entry points of the benchmarked steps that no census replays per element: add a census '
                           'family (a query that launches nothing goes in LAUNCHES_NOTHING):\n' + '\n'.join(unchecked))
    stale = sorted(set(LAUNCHES_NOTHING) - names)
    assert not stale, f'LAUNCHES_NOTHING lists entry points the benchmarked steps no longer call: {stale}'
    assert not set(LAUNCHES_NOTHING) & covered, 'an entry point is both checked and listed as launching nothing'


# ----------------------------------------------------------------------------------------------------------------------
# launch arithmetic (restated from the launches; no ABI query needed)
# ----------------------------------------------------------------------------------------------------------------------
def darcy_fwd_grid(B):          # launch_darcy_fwd: 220 KB / sizeof(DarcySmem) (64 KB) = 3 CTAs per SM, capped at B
    return min(B, 3 * sms())


def darcy_grad_grid(B):         # launch_darcy_grad: one 512-thread CTA per SM, capped at B
    return min(B, sms())


def mech_bands(nel):            # pidm_mechanics_residual_fwd / _bwd: grid (ceil((nel+1) / MECH_BAND), B), MECH_BAND = 8
    return -(-(nel + 1) // 8)


def resize_passes(planes, out):  # pidm_bilinear_resize_fwd / _bwd: 256 threads, grid min(ceil(total / 256), 8 SMs)
    total = planes * out * out
    grid = min(-(-total // 256), 8 * sms())
    return -(-total // (grid * 256))


# ----------------------------------------------------------------------------------------------------------------------
# Darcy
# ----------------------------------------------------------------------------------------------------------------------
def _bspec(spec):
    """batch of a synthetic row: an int, or (grid, kind) resolved against the SM count of this device"""
    if isinstance(spec, int):
        return spec
    which, kind = spec
    G = 3 * sms() if which == 'fwd' else sms()
    return {'-1': G - 1, '0': G, '+1': G + 1, 'ragged': 2 * G + G // 2, 'deep': 4 * G + 3}[kind]


BSPECS = [1] + [(w, k) for w in ('fwd', 'grad') for k in ('-1', '0', '+1', 'ragged', 'deep')]
GEOMS = [(L, rev, pab) for L in (1.0, 2.5) for rev in (0, 1) for pab in (0, 1)]


def _darcy_rows(table, with_geometry=True):
    """(B or spec, domain_length, reverse_d1, flags): table rows, bench rows, the synthetic batches at the default
    geometry with both bcs, and every geometry with both bcs at B = 5"""
    rows = [k[:1] + k[2:5] for k in table]
    rows += [(bs, 1.0, 1, 1 | per) for per in (0, 2) for bs in BSPECS]
    if with_geometry:
        rows += [(5, L, rev, pab | per) for per in (0, 2) for L, rev, pab in GEOMS]
    return rows


def _darcy_id(r):
    b = r[0] if isinstance(r[0], int) else f'{r[0][0]}{r[0][1]}'
    return f'B{b}_L{r[1]}_rev{r[2]}_{"periodic" if r[3] & 2 else "none"}_pab{r[3] & 1}'


def _geom(L, rev, flags):
    return dict(domain_length=L, reverse_d1=bool(rev), pixels_at_boundary=bool(flags & 1)), bool(flags & 2)


def _fields(B, seed):
    """Darcy fields [B,2,P,P] on the device, fp32 (p normal, K log-normal): exactly what the fp64 reference reads"""
    x = torch.randn(B, 2, P, P, generator=gen(seed), device=DEV)
    x[:, 1] = torch.exp(0.5 * x[:, 1])
    return x


def fs_dev():
    return O.darcy_source(P).to(DEV).contiguous()


def darcy_residual(x, per, geom, absolute=False, edit=None):
    """fp64 residual [B,P*P,3] of fp32 fields x; edit: a mutant (see test_mutant_darcy_residual)"""
    x = x.double()
    stencils, g = None, dict(geom)
    if edit == 'central_at_last_column':       # the interior stencil at column P-1 (wrapped), not the one-sided one
        stencils = O.darcy_stencils(P, per, **geom)
        central = O.darcy_stencils(P, True, **geom)
        stencils[2][-1], stencils[3][-1] = central[2][-1], central[3][-1]
    if edit == 'bc1_sign_ignores_reverse_d1':
        stencils, g['reverse_d1'] = O.darcy_stencils(P, per, **geom), True
    if edit == 'h_is_L_over_P':                # the spacing of pixels_at_boundary = False under pixels_at_boundary
        stencils = O.darcy_stencils(P, per, **{**geom, 'pixels_at_boundary': False})
    if edit == 'one_sided_row0':               # periodic: the wrap dropped at row 0
        stencils, one_sided = O.darcy_stencils(P, True, **geom), O.darcy_stencils(P, False, **geom)
        stencils[0][0], stencils[1][0] = one_sided[0][0], one_sided[1][0]
    r = O.darcy_residual_matrix(x, per, absolute, stencils, **g)
    if edit == 'fs_dropped_on_row0':
        r[:, :P, 0] += O.darcy_source(P, dtype=torch.float64).to(r.device)[0]
    if edit == 'corner_sign':
        r[:, 0, 1] = -r[:, 0, 1]
    if edit == 'last_row_zero':
        r[-1, -P:] = 0
    return r


CH_NAMES = ('eq_0', 'bc_x0', 'bc_x1')


def _fwd_launch(x, L, rev, flags):
    B = x.shape[0]
    buf, out = guarded(B * P * P * 3)
    call_sync('pidm_darcy_residual_fwd', x, fs_dev(), out, B, P, float(L), int(rev), int(flags))
    assert guards_intact(buf), 'a store landed outside the residual'
    return out.view(B, P * P, 3)


def replay_darcy_fwd(row, seed):
    B = _bspec(row[0])
    geom, per = _geom(*row[1:])
    x = _fields(B, seed)
    y = _fwd_launch(x, *row[1:])
    tag = 'periodic' if per else 'none'
    for lo in range(0, B, CHUNK):
        xs = x[lo:lo + CHUNK]
        r, A = darcy_residual(xs, per, geom), darcy_residual(xs.abs(), per, geom, absolute=True)
        for c, name in enumerate(CH_NAMES):
            check(TAG, f'darcy_fwd {tag} {name}', y[lo:lo + CHUNK, :, c], r[..., c], C_DARCY * U * A[..., c])


@pytest.mark.parametrize('row', _darcy_rows(DARCY_FWD_TABLE + [k for f, k, _ in BENCH_ROWS if f == 'darcy_fwd']),
                         ids=_darcy_id)
def test_darcy_residual_replay(row):
    replay_darcy_fwd(row, 11)


@pytest.mark.parametrize('row', _darcy_rows(DARCY_BWD_TABLE), ids=_darcy_id)
def test_darcy_vjp_replay(row):
    B = _bspec(row[0])
    geom, per = _geom(*row[1:])
    x = _fields(B, 21)
    cot = torch.randn(B, P * P, 3, generator=gen(22), device=DEV)
    buf, gx = guarded(B * 2 * P * P)
    call_sync('pidm_darcy_residual_bwd', x, fs_dev(), cot, gx, B, P, float(row[1]), int(row[2]), int(row[3]))
    assert guards_intact(buf), 'a store landed outside grad_x0hat'
    gx = gx.view(B, 2, P, P)
    for lo in range(0, B, CHUNK):
        xs, cs = x[lo:lo + CHUNK].double(), cot[lo:lo + CHUNK].double()
        ref = O.darcy_residual_vjp(xs, cs, per, **geom)
        A = O.darcy_residual_vjp(xs, cs, per, absolute=True, **geom)
        for c, name in enumerate(('dp', 'dK')):
            check(TAG, f'darcy_bwd {"periodic" if per else "none"} {name}', gx[lo:lo + CHUNK, c], ref[:, c],
                  C_DARCY * U * A[:, c])


def _tables():
    from physicsinformeddiffusionmodels_b200.denoising_utils import DenoisingDiffusion
    dd = DenoisingDiffusion(100, DEV).diff_dict
    return dd['p2_loss_weight'].float().contiguous(), dd['posterior_variance_clipped'].float().contiguous()


def darcy_loss_depth(B):
    """fp32 accumulation chain of a darcy_grad_kernel<2> sum: 4 pixels x 2 quads per thread and sample, a warp, 16
    warps, one atomic per CTA"""
    G = darcy_grad_grid(B)
    return 8 * -(-B // G) + 5 + 16 + G


def replay_darcy_loss(B, L, rev, flags, variant, seed):
    """variant: 'mean' (model_out = x0hat, grad_x0hat only), 'sample' (separate model_out, both gradients), 'loss_only'"""
    geom, per = _geom(L, rev, flags)
    p2, var = _tables()
    x = _fields(B, seed)
    tgt = torch.randn(B, 2, P, P, generator=gen(seed + 1), device=DEV)
    t = torch.randint(0, 100, (B,), generator=gen(seed + 2), device=DEV)
    m = torch.randn(B, 2, P, P, generator=gen(seed + 3), device=DEV) if variant == 'sample' else x
    bs, sums = guarded(3)
    bx, gx = guarded(B * 2 * P * P)
    bm, gm = guarded(B * 2 * P * P)
    c_data, c_res = 1.0, 1e-3
    call_sync('pidm_darcy_pidm_loss', x, m, tgt, fs_dev(), t, p2, var, c_data, c_res, sums,
              None if variant == 'loss_only' else gx, gm if variant == 'sample' else None, B, P, float(L), int(rev),
              int(flags))
    assert guards_intact(bs) and guards_intact(bx) and guards_intact(bm)
    if variant != 'sample':
        assert torch.isnan(gm).all(), 'grad_model_out was written although it was not passed'
    if variant == 'loss_only':
        assert torch.isnan(gx).all(), 'grad_x0hat was written although it was not passed'
    tag = f'darcy_loss {"periodic" if per else "none"}'
    wr_all = 0.5 * c_res / (var.double()[t] * B * P * P * 3)
    wd_all = c_data * p2.double()[t] / (B * 2 * P * P)
    rs, rA = torch.zeros(3, dtype=torch.float64, device=DEV), torch.zeros(3, dtype=torch.float64, device=DEV)
    gx, gm = gx.view(B, 2, P, P), gm.view(B, 2, P, P)
    for lo in range(0, B, CHUNK):
        sl = slice(lo, lo + CHUNK)
        xs, ms, ts = x[sl].double(), m[sl].double(), tgt[sl].double()
        wr, wd = wr_all[sl, None, None], wd_all[sl, None, None, None]
        r, Ar = darcy_residual(xs, per, geom), darcy_residual(xs.abs(), per, geom, absolute=True)
        rs += torch.stack([(wd * (ms - ts) ** 2).sum(), (wr * r ** 2).sum(), r.abs().sum() / (B * P * P * 3)])
        rA += torch.stack([(wd * (ms.abs() + ts.abs()) ** 2).sum(), (wr * Ar ** 2).sum(), Ar.sum() / (B * P * P * 3)])
        if variant == 'loss_only':
            continue
        # the fp32 cotangent 2 wr r carries the residual's own error and that of wr: the adjoint is bounded with twice
        # 2 wr Ar, which leaves C 2^-24 for each of the two
        rgx = O.darcy_residual_vjp(xs, 2 * wr * r, per, **geom)
        A_gx = O.darcy_residual_vjp(xs, 4 * wr * Ar, per, absolute=True, **geom)
        rgm, A_gm = 2 * wd * (ms - ts), 2 * wd * (ms.abs() + ts.abs())
        if variant == 'mean':                   # the data gradient folded into grad_x0hat
            check(TAG, f'{tag} grad_x0hat (mean)', gx[sl], rgx + rgm, C_LOSS * U * (A_gx + A_gm))
        else:
            check(TAG, f'{tag} grad_x0hat', gx[sl], rgx, C_LOSS * U * A_gx)
            check(TAG, f'{tag} grad_model_out', gm[sl], rgm, C_LOSS * U * A_gm)
    for i, name in enumerate(('data', 'residual', 'mean|r|')):
        check(TAG, f'{tag} sum {name}', sums[i], rs[i], (darcy_loss_depth(B) + 2 * C_LOSS) * U * rA[i])


LOSS_VARIANTS = ('mean', 'sample', 'loss_only')


def _loss_variant(k):
    same, has_gx, has_gm = k[5:8]
    return 'loss_only' if not has_gx else ('mean' if same else 'sample')


DARCY_LOSS_ROWS = ([k[:1] + k[2:5] + (_loss_variant(k),) for k in DARCY_LOSS_TABLE]
                   + [k[:1] + k[2:5] + (_loss_variant(k),) for f, k, _ in BENCH_ROWS if f == 'darcy_loss']
                   + [r + (v,) for r in _darcy_rows([], with_geometry=False) for v in LOSS_VARIANTS]
                   + [r + ('sample',) for r in _darcy_rows([])[2 * len(BSPECS):]])


@pytest.mark.parametrize('row', DARCY_LOSS_ROWS, ids=lambda r: _darcy_id(r) + '_' + r[4])
def test_darcy_loss_replay(row):
    replay_darcy_loss(_bspec(row[0]), *row[1:4], row[4], 31)


@pytest.mark.parametrize('case', ['grad_x0hat_without_grad_model_out', 'grad_model_out_without_grad_x0hat',
                                  'grad_model_out_in_mean_mode'])
def test_darcy_loss_rejects_unsupported_gradient_pointers(case):
    """pidm_darcy_pidm_loss accepts the three gradient forms pidm.h lists and refuses the others before any launch"""
    B = 3
    p2, var = _tables()
    x = _fields(B, 5)
    m = x if case == 'grad_model_out_in_mean_mode' else _fields(B, 6)
    tgt = _fields(B, 7)
    t = torch.zeros(B, dtype=torch.long, device=DEV)
    bs, sums = guarded(3)
    bx, gx = guarded(B * 2 * P * P)
    bm, gm = guarded(B * 2 * P * P)
    gx_arg = None if case == 'grad_model_out_without_grad_x0hat' else gx
    gm_arg = None if case == 'grad_x0hat_without_grad_model_out' else gm
    with pytest.raises(RuntimeError, match='darcy_pidm_loss: gradients'):
        call_sync('pidm_darcy_pidm_loss', x, m, tgt, fs_dev(), t, p2, var, 1.0, 1e-3, sums, gx_arg, gm_arg, B, P, 1.0,
                  1, 1)
    assert torch.isnan(bs).all() and torch.isnan(bx).all() and torch.isnan(bm).all(), 'a rejected call wrote'


def jacobian_max_ref(x, per, geom):
    """largest entry (signed, zeros included) of d r / d p per sample in fp64, from the stencil matrices: entry
    (pixel (i,j), p at (i',j)) = -K D2_0[i,i'] - K_0 D1_0[i,i'], likewise along columns, the two directions adding at
    the pixel itself; the BC rows hold -/+ D1_0 (rows 0 / P-1) and +/- s D1_1 (columns 0 / P-1).  Also an absolute
    bound per sample."""
    D1a, D2a, D1b, D2b = (m.to(x.device) for m in O.darcy_stencils(P, per, **geom))
    x = x.double()
    K = x[:, 1]
    K0, K1 = O.along_rows(D1a, K), O.along_cols(D1b, K)
    eye = torch.eye(P, dtype=torch.bool, device=x.device)
    off_r = ((D1a != 0) | (D2a != 0)) & ~eye
    off_c = ((D1b != 0) | (D2b != 0)) & ~eye
    er = -K[..., None] * D2a[None, :, None, :] - K0[..., None] * D1a[None, :, None, :]       # [B, i, j, i']
    ec = -K[..., None] * D2b[None, None, :, :] - K1[..., None] * D1b[None, None, :, :]      # [B, i, j, j']
    er = torch.where(off_r[None, :, None, :], er, -math.inf).amax(dim=(1, 2, 3))
    ec = torch.where(off_c[None, None, :, :], ec, -math.inf).amax(dim=(1, 2, 3))
    dg = (-K * (D2a.diagonal()[:, None] + D2b.diagonal()[None, :]) - K0 * D1a.diagonal()[:, None]
          - K1 * D1b.diagonal()[None, :]).amax(dim=(1, 2))
    s = 1.0 if geom['reverse_d1'] else -1.0
    bc = torch.cat([-D1a[0], D1a[-1], s * D1b[0], -s * D1b[-1]]).max()
    mx = torch.stack([er, ec, dg, torch.zeros_like(er) + bc.clamp_min(0)]).amax(dim=0)
    A = ((K.abs() * (D2a.abs().amax() + D2b.abs().amax()) + (K0.abs() + K1.abs()) * D1a.abs().amax()).amax(dim=(1, 2))
         + D1a.abs().amax() + D1b.abs().amax())
    return mx, A


@pytest.mark.parametrize('row', [(B, 1.0, 1, 1 | per) for per in (0, 2) for B in (1, 3, 400)]
                         + [(5, L, rev, pab | per) for per in (0, 2) for L, rev, pab in GEOMS], ids=_darcy_id)
def test_darcy_jacobian_max_replay(row):
    B = row[0]
    geom, per = _geom(*row[1:])
    x = _fields(B, 40 + B)
    if B == 3:
        x[1, 1] = -x[1, 1]                        # negative K: the maximum comes from the BC rows / zero entries
    buf, out = guarded(B)
    call_sync('pidm_darcy_jacobian_max', x, out, B, P, float(row[1]), int(row[2]), int(row[3]))
    assert guards_intact(buf)
    ref, A = torch.cat([torch.stack(jacobian_max_ref(x[lo:lo + 64], per, geom)) for lo in range(0, B, 64)], dim=1)
    check(TAG, f'darcy_jacobian_max {"periodic" if per else "none"}', out, ref, C_DARCY * U * A)
    if B <= 3 and row[1:3] == (1.0, 1) and row[3] & 1:      # the matrix form against the oracle's explicit Jacobian
        assert torch.allclose(O.jacobian_max(x.double().cpu(), periodic=per), ref.cpu(), rtol=1e-9, atol=0)


FD_MODES = ['d_d0', 'd_d1', 'd_d00', 'd_d11', 'd_d01']


@pytest.mark.parametrize('periodic', [False, True], ids=['none', 'periodic'])
@pytest.mark.parametrize('B', [1, 3, 32, 400])
@pytest.mark.parametrize('mode', FD_MODES)
def test_darcy_fd_stencil_replay(mode, B, periodic):
    from physicsinformeddiffusionmodels_b200.grad_utils import StencilGradients
    d0, d1 = O.spacing(P)
    u = _fields(B, 50 + B)[:, 0].contiguous()
    y = StencilGradients(d0=d0, d1=d1, periodic=periodic)(u, mode)
    ud = u.double()
    r = O.stencil_gradients(ud, mode, d0, d1, periodic=periodic)
    ua = ud.abs()
    D1a, D2a, D1b, D2b = (m.abs().to(DEV) for m in O.darcy_stencils(P, periodic))
    A = {'d_d0': lambda: O.along_rows(D1a, ua), 'd_d1': lambda: O.along_cols(D1b, ua),
         'd_d00': lambda: O.along_rows(D2a, ua), 'd_d11': lambda: O.along_cols(D2b, ua),
         'd_d01': lambda: O.along_rows(D1a, O.along_cols(D1b, ua))}[mode]()
    check(TAG, f'fd_stencil {"periodic" if periodic else "none"} {mode}', y, r, C_DARCY * U * A)
    buf, out = guarded(B * P * P)
    call_sync('pidm_fd_stencil', u, out, B, P, FD_MODES.index(mode) | (8 if periodic else 0), float(d0), float(d1))
    assert guards_intact(buf) and torch.equal(out.view(B, P, P), y)


# ----------------------------------------------------------------------------------------------------------------------
# mechanics
# ----------------------------------------------------------------------------------------------------------------------
NELS = [2, 7, 63, 64, 100, 256]       # one band, one exact band, eight full bands, a one-row last band, ragged, largest


def mech_operands(B, nel, seed):
    """fp32-exact u [B,2,nn,nn], rho [B,nel,nel] with exact zeros, bcs [B,4,nn,nn] with Dirichlet values 1, 0.5 and -1,
    loads on fixed dofs (which must be dropped) and at the four corner nodes"""
    g = gen(seed)
    nn = nel + 1
    u = torch.randn(B, 2, nn, nn, generator=g, device=DEV) * 0.1
    rho = torch.rand(B, nel, nel, generator=g, device=DEV)
    rho = torch.where(rho < 0.1, torch.zeros_like(rho), rho)
    bcs = torch.zeros(B, 4, nn, nn, device=DEV)
    bcs[:, 0, :, 0] = 1.
    bcs[:, 1, :, 0] = 0.5
    bcs[:, 1, -1, nn // 2:] = -1.
    loads = torch.randn(B, 2, nn, nn, generator=g, device=DEV)
    bcs[:, 2:] = torch.where(torch.rand(B, 2, nn, nn, generator=g, device=DEV) < 0.2, loads, torch.zeros_like(loads))
    bcs[:, 2, 0, 0], bcs[:, 3, 0, -1], bcs[:, 2, -1, 0], bcs[:, 3, -1, -1] = 2., -3., 1.5, -1.
    return u, rho, bcs


def ke_dev():
    return O.q4_plane_stress_stiffness().float().to(DEV).contiguous()


def mech_depth(nel):
    """fp32 accumulation chain of a compliance: 2 terms per node, nodes of a band per thread, a warp, 8 warps, one
    atomic per band"""
    nn = nel + 1
    return 2 * -(-8 * nn // 256) + 5 + 8 + mech_bands(nel)


def mech_fwd_launch(u, rho, bcs, with_compliance=True):
    B, nel = rho.shape[0], rho.shape[-1]
    nn = nel + 1
    br, r = guarded(B * 2 * nn * nn)
    bc, c = guarded(B)
    call_sync('pidm_mechanics_residual_fwd', u, rho, bcs, ke_dev(), r, c if with_compliance else None, B, nel)
    assert guards_intact(br) and guards_intact(bc)
    if not with_compliance:
        assert torch.isnan(bc).all()
    return r.view(B, -1), c


def mech_ref(u, rho, bcs, absolute=False):
    return O.mechanics_matfree(u.double(), rho.double(), bcs.double(), absolute=absolute)


def _mech_fwd_rows():
    rows = [k for k in MECH_FWD_TABLE] + [k for f, k, _ in BENCH_ROWS if f == 'mech_fwd']
    return rows + [(B, nel, 1) for nel in NELS for B in (1, 3, 32)] + [(3, 64, 0)]


@pytest.mark.parametrize('row', _mech_fwd_rows(), ids=lambda k: f'B{k[0]}_nel{k[1]}_comp{k[2]}')
def test_mechanics_residual_replay(row):
    B, nel, with_c = row
    u, rho, bcs = mech_operands(B, nel, 60 + nel)
    r, c = mech_fwd_launch(u, rho, bcs, bool(with_c))
    ch = max(1, CHUNK * 4096 // (nel * nel) // 4)
    for lo in range(0, B, ch):
        sl = slice(lo, lo + ch)
        rr, rc = mech_ref(u[sl], rho[sl], bcs[sl])
        Ar, Ac = mech_ref(u[sl], rho[sl], bcs[sl], absolute=True)
        check(TAG, 'mech_fwd residual', r[sl], rr, C_MECH * U * Ar)
        if with_c:
            check(TAG, 'mech_fwd compliance', c[sl], rc, (C_MECH + mech_depth(nel)) * U * Ac)


def mech_bwd_ref(u, rho, bcs, gr, gc, absolute=False, bcs_for_grad=None):
    """fp64 (du, drho) of sum(gr . residual) + sum(gc * compliance) by autograd; absolute: of the absolute-value form
    with |gr|, |gc|; bcs_for_grad replaces bcs (the mutant with no Dirichlet rows)"""
    # the absolute form is the signed chain on |u|, |rho|, |KE| (no |.| inside the graph: its derivative at an exact
    # zero density would be 0); the loads do not enter the gradient
    mag = (lambda v: v.double().abs()) if absolute else (lambda v: v.double())
    KE = mag(O.q4_plane_stress_stiffness())
    ud, rd = mag(u).requires_grad_(True), mag(rho).requires_grad_(True)
    b = (bcs if bcs_for_grad is None else bcs_for_grad).double()
    with torch.enable_grad():
        r, c = O.mechanics_matfree(ud, rd, b, KE)
        loss = 0
        if gr is not None:
            loss = loss + (r * mag(gr)).sum()
        if gc is not None:
            loss = loss + (c * mag(gc)).sum()
        du, drho = torch.autograd.grad(loss, (ud, rd))
    return du, drho


def mech_bwd_launch(u, rho, bcs, gr, gc):
    B, nel = rho.shape[0], rho.shape[-1]
    nn = nel + 1
    bu, du = guarded(B * 2 * nn * nn)
    bw, ws = guarded(B * 2 * nn * nn)
    bp, dp = guarded(B * nel * nel)
    call_sync('pidm_mechanics_residual_bwd', u, rho, bcs, ke_dev(), gr, gc, du, dp, ws, B, nel)
    assert guards_intact(bu) and guards_intact(bw) and guards_intact(bp)
    return du.view(B, 2, nn, nn), dp.view(B, nel, nel)


COTANGENTS = ('residual', 'compliance', 'both')


def _mech_bwd_rows():
    rows = [(k[0], k[1], {(1, 0): 'residual', (0, 1): 'compliance', (1, 1): 'both'}[k[2:4]]) for k in MECH_BWD_TABLE]
    return rows + [(B, nel, cm) for nel in NELS for B in (1, 3, 32) for cm in COTANGENTS]


@pytest.mark.parametrize('row', _mech_bwd_rows(), ids=lambda k: f'B{k[0]}_nel{k[1]}_{k[2]}')
def test_mechanics_vjp_replay(row):
    B, nel, cm = row
    nn = nel + 1
    u, rho, bcs = mech_operands(B, nel, 70 + nel)
    gr = torch.randn(B, 2 * nn * nn, generator=gen(71), device=DEV) if cm != 'compliance' else None
    gc = torch.randn(B, generator=gen(72), device=DEV) if cm != 'residual' else None
    du, drho = mech_bwd_launch(u, rho, bcs, gr, gc)
    rdu, rdrho = mech_bwd_ref(u, rho, bcs, gr, gc)
    Adu, Adrho = mech_bwd_ref(u, rho, bcs, gr, gc, absolute=True)
    check(TAG, f'mech_bwd grad_u ({cm})', du, rdu, C_MECH * U * Adu)
    check(TAG, f'mech_bwd grad_rho ({cm})', drho, rdrho, C_MECH * U * Adrho)


def mech_loss_ref(u, rho, x0, r, comp, vf, t, p2, var, c_data, c_res, c_ineq, lam, edit=None):
    """fp64 sums6 and gradients of pidm_mech_pidm_loss (the reference's mechanics loss, denoising_utils.py:669-710)
    with their bounds.  edit: 'mean_var' = mean(var) for mean(1/var); 'p2_by_b' = p2[b] for p2[t[b]]"""
    B, nel = rho.shape[0], rho.shape[-1]
    nn = nel + 1
    n, ne = nn * nn, nel * nel
    u, rho, x0, r, comp, vf = (v.double() for v in (u, rho, x0, r, comp, vf))
    p2, var = p2.double(), var.double()
    wd = c_data * (p2[:B] if edit == 'p2_by_b' else p2[t]) / (B * 3 * n)
    wr = 0.5 * c_res / (var[t] * B * 2 * n)
    rho_pad = F.pad(rho, (0, 1, 0, 1)).reshape(B, n)
    e = torch.cat([u.reshape(B, 2 * n), rho_pad], 1) - x0.reshape(B, 3 * n)
    ea = torch.cat([u.reshape(B, 2 * n).abs(), rho_pad.abs()], 1) + x0.reshape(B, 3 * n).abs()
    q = rho.reshape(B, ne).mean(1) - vf
    Aq = rho.reshape(B, ne).abs().mean(1) + vf.abs()
    mvar = (var[t].mean() if edit == 'mean_var' else (1 / var[t]).mean()) if c_ineq > 0 else torch.zeros((), dtype=u.dtype, device=u.device)
    sums = torch.stack([(wd[:, None] * e ** 2).sum(), (wr[:, None] * r ** 2).sum(), 0.5 * c_ineq * mvar * (q ** 2).sum() / B,
                        lam * comp.sum() / B, r.abs().sum() / (B * 2 * n), q.sum() / B])
    sums_A = torch.stack([(wd[:, None] * ea ** 2).sum(), (wr[:, None] * r ** 2).sum(), 0.5 * c_ineq * mvar * (Aq ** 2).sum() / B,
                          lam * comp.abs().sum() / B, r.abs().sum() / (B * 2 * n), Aq.sum() / B])
    g_u = 2 * wd[:, None] * e[:, :2 * n]
    A_gu = 2 * wd[:, None] * ea[:, :2 * n]
    g_r, A_gr = 2 * wr[:, None] * r, 2 * wr[:, None] * r.abs()
    g_c = torch.full((B,), lam / B, dtype=u.dtype, device=u.device)
    x0_rho = x0.reshape(B, 3, nn, nn)[:, 2, :nel, :nel]
    dq = c_ineq * mvar * q / (B * ne)
    g_rho = 2 * wd[:, None, None] * (rho - x0_rho) + dq[:, None, None]
    A_grho = 2 * wd[:, None, None] * (rho.abs() + x0_rho.abs())
    A_dq = (c_ineq * mvar * Aq / (B * ne))[:, None, None].expand_as(A_grho)
    return sums, sums_A, (g_u, g_rho, g_r, g_c), (A_gu, A_grho, A_dq, A_gr, g_c.abs())


def mech_loss_launch(B, nel, c_ineq, lam, t_kind, seed):
    nn = nel + 1
    n, ne = nn * nn, nel * nel
    g = gen(seed)
    u = torch.randn(B, 2 * n, generator=g, device=DEV) * 0.1
    rho = torch.rand(B, nel, nel, generator=g, device=DEV)
    x0 = torch.rand(B, 3 * n, generator=g, device=DEV)
    r = torch.randn(B, 2 * n, generator=g, device=DEV)
    comp = torch.rand(B, generator=g, device=DEV) * 10
    vf = torch.rand(B, generator=g, device=DEV)
    t = (torch.full((B,), 17, device=DEV, dtype=torch.long) if t_kind == 'repeated'
         else torch.randperm(100, generator=g, device=DEV)[:B])
    p2, var = _tables()
    bs, sums = guarded(6)
    bu, gu = guarded(B * 2 * n)
    bp, grho = guarded(B * ne)
    br, gr = guarded(B * 2 * n)
    bc, gc = guarded(B)
    call_sync('pidm_mech_pidm_loss', u, rho, x0, r, comp, vf, t, p2, var, 1.0, 1e-2, float(c_ineq), float(lam), sums,
              gu, grho, gr, gc, B, nel)
    assert all(guards_intact(b) for b in (bs, bu, bp, br, bc))
    operands = (u, rho, x0, r, comp, vf, t, p2, var, 1.0, 1e-2, c_ineq, lam)
    return operands, sums, (gu.view(B, 2 * n), grho.view(B, nel, nel), gr.view(B, 2 * n), gc)


def mech_loss_depth(B, nel):
    """fp32 chain of a mech_loss_kernel sum: strided terms per thread (2n + n), a warp, 8 warps, one atomic per
    sample; the mean of 1/var adds B more"""
    n = (nel + 1) ** 2
    return -(-2 * n // 256) + -(-n // 256) + 5 + 8 + 2 * B


def check_mech_loss(operands, sums, grads, edit=None):
    B, nel = operands[1].shape[0], operands[1].shape[-1]
    rs, rA, rg, Ag = mech_loss_ref(*operands, edit=edit)
    depth = mech_loss_depth(B, nel)
    ok = True
    for i, name in enumerate(('data', 'residual', 'inequality', 'optimisation', 'mean|r|', 'mean q')):
        bound = ((2 if i == 2 else 1) * depth + C_LOSS) * U * rA[i]
        if edit is None:
            check(TAG, f'mech_loss sum {name}', sums[i], rs[i], bound)
        ok &= bool((sums[i].double() - rs[i]).abs() <= bound)
    A_gu, A_grho, A_dq, A_gr, A_gc = Ag
    bounds = (C_LOSS * U * A_gu, C_LOSS * U * A_grho + (depth + C_LOSS) * U * A_dq, C_LOSS * U * A_gr, C_LOSS * U * A_gc)
    for name, y, r, b in zip(('grad_u', 'grad_rho', 'grad_residual', 'grad_compliance'), grads, rg, bounds):
        if edit is None:
            check(TAG, f'mech_loss {name}', y, r, b)
        ok &= bool(((y.double() - r).abs() <= b).all())
    return ok


MECH_LOSS_ROWS = ([(k[0], k[1], 0.0, 1e-3, 'distinct') for k in MECH_LOSS_TABLE]
                  + [(5, 64, ci, lam, tk) for ci in (0.0, 0.5) for lam in (0.0, 1e-3) for tk in ('repeated', 'distinct')]
                  + [(3, 7, 0.5, 1e-3, 'distinct'), (1, 2, 0.5, 1e-3, 'distinct'), (64, 64, 0.5, 1e-3, 'distinct')])


@pytest.mark.parametrize('row', MECH_LOSS_ROWS, ids=lambda k: f'B{k[0]}_nel{k[1]}_cineq{k[2]}_lam{k[3]}_{k[4]}')
def test_mech_loss_replay(row):
    operands, sums, grads = mech_loss_launch(*row, 80 + row[0])
    assert check_mech_loss(operands, sums, grads)


# ----------------------------------------------------------------------------------------------------------------------
# bilinear resize
# ----------------------------------------------------------------------------------------------------------------------
RESIZE_SHAPES = [(65, 64), (64, 65), (64, 128), (130, 64), (2, 5)]


def _planes(spec, out):
    """an int, or 'multi': enough planes that the 8 SMs x 256-thread grid cap takes at least three grid-stride passes"""
    return spec if isinstance(spec, int) else -(-3 * 8 * sms() * 256 // (out * out))


def resize_gather(x, n_out, clamp_hi=None):
    """bilinear resize from the fp64 index arithmetic (used for the mutants)"""
    n_in = x.shape[-1]
    i0, i1, w, _ = resize_src_index(n_out, n_in, clamp_hi)
    rows = x[:, i0] * (1 - w)[:, None] + x[:, i1] * w[:, None]
    return rows[:, :, i0] * (1 - w) + rows[:, :, i1] * w


@pytest.mark.parametrize('row', [k for k in RESIZE_FWD_TABLE] + [(pl, i, o) for i, o in RESIZE_SHAPES for pl in (3, 'multi')],
                         ids=lambda k: f'planes{k[0]}_{k[1]}to{k[2]}')
def test_resize_fwd_replay(row):
    planes, n_in, n_out = _planes(row[0], row[2]), row[1], row[2]
    x = torch.randn(planes, n_in, n_in, generator=gen(90 + n_in), device=DEV)
    buf, y = guarded(planes * n_out * n_out)
    call_sync('pidm_bilinear_resize_fwd', x, y, planes, n_in, n_out)
    assert guards_intact(buf)
    xd = x.double().cpu()
    r = F.interpolate(xd[:, None], size=(n_out, n_out), mode='bilinear', align_corners=False)[:, 0]
    A, coord = resize_bounds(xd, n_out)
    check(TAG, 'resize_fwd', y.view(planes, n_out, n_out).cpu(), r, C_RESIZE * U * A + coord)


def resize_bwd_bounds(dy, n_in):
    """(A, coordinate term, atomic depth) of the backward bound: A = the adjoint of |dy|; a weight error e reaches source
    rows / columns i0 - 1 .. i0 + 2; at most (out / in + 2)^2 atomics land on one element"""
    n_out = dy.shape[-1]
    A = resize_adjoint(dy.abs(), n_in)
    i0, _, _, e = resize_src_index(n_out, n_in)
    w = dy.abs() * (e[:, None] + e[None, :])
    T = torch.zeros(dy.shape[0], n_in, n_in, dtype=torch.float64)
    for dr in range(-1, 3):
        for dc in range(-1, 3):
            rr, cc = (i0 + dr).clamp(0, n_in - 1), (i0 + dc).clamp(0, n_in - 1)
            idx = (rr[:, None] * n_in + cc[None, :]).reshape(-1)
            T.view(dy.shape[0], -1).index_add_(1, idx, w.reshape(dy.shape[0], -1))
    return A, T, (math.ceil(n_out / n_in) + 2) ** 2


def resize_adjoint(dy, n_in):
    x = torch.zeros(dy.shape[0], 1, n_in, n_in, dtype=torch.float64, requires_grad=True)
    with torch.enable_grad():
        y = F.interpolate(x, size=dy.shape[-2:], mode='bilinear', align_corners=False)
        return torch.autograd.grad((y[:, 0] * dy).sum(), x)[0][:, 0]


@pytest.mark.parametrize('row', [k for k in RESIZE_BWD_TABLE] + [(pl, i, o) for i, o in RESIZE_SHAPES for pl in (3, 'multi')],
                         ids=lambda k: f'planes{k[0]}_{k[1]}to{k[2]}')
def test_resize_bwd_replay(row):
    planes, n_in, n_out = _planes(row[0], row[2]), row[1], row[2]
    dy = torch.randn(planes, n_out, n_out, generator=gen(95 + n_in), device=DEV)
    buf, dx = guarded(planes * n_in * n_in)          # NaN-filled: the entry point must zero dx itself
    call_sync('pidm_bilinear_resize_bwd', dy, dx, planes, n_in, n_out)
    assert guards_intact(buf)
    dyd = dy.double().cpu()
    r = resize_adjoint(dyd, n_in)
    A, T, depth = resize_bwd_bounds(dyd, n_in)
    check(TAG, 'resize_bwd', dx.view(planes, n_in, n_in).cpu(), r, (C_RESIZE + depth) * U * A + T)


# ----------------------------------------------------------------------------------------------------------------------
# mutants: the predicates above reject edited references
# ----------------------------------------------------------------------------------------------------------------------
def _within(y, r, bound):
    return bool(((y.double() - r).abs() <= bound).all())


DARCY_MUTANTS = {                                 # edit: the row (B, domain_length, reverse_d1, flags) that shows it
    'central_at_last_column': (32, 1.0, 1, 1),
    'bc1_sign_ignores_reverse_d1': (32, 1.0, 0, 1),
    'h_is_L_over_P': (32, 1.0, 1, 1),
    'fs_dropped_on_row0': (32, 2.5, 0, 0),
    'one_sided_row0': (32, 1.0, 1, 3),
    'corner_sign': (32, 1.0, 1, 3),
    'last_row_zero': (32, 1.0, 1, 3),
}


@pytest.mark.parametrize('edit', list(DARCY_MUTANTS))
def test_mutant_darcy_residual(edit):
    B, L, rev, flags = DARCY_MUTANTS[edit]
    geom, per = _geom(L, rev, flags)
    x = _fields(B, 42)
    y = _fwd_launch(x, L, rev, flags)
    A = darcy_residual(x.abs(), per, geom, absolute=True)
    assert _within(y, darcy_residual(x, per, geom), C_DARCY * U * A)
    assert not _within(y, darcy_residual(x, per, geom, edit=edit), C_DARCY * U * A), edit


MECH_MUTANTS = ['mask_is_eq_1', 'f_kept_on_fixed_dof', 'element_row_dropped', 'compliance_without_fixed_u2',
                'drho_from_unmasked_cotangent']


@pytest.mark.parametrize('edit', MECH_MUTANTS)
def test_mutant_mechanics(edit):
    B, nel = 3, 64
    u, rho, bcs = mech_operands(B, nel, 99)
    if edit == 'drho_from_unmasked_cotangent':
        gr = torch.randn(B, 2 * (nel + 1) ** 2, generator=gen(98), device=DEV)
        gc = torch.randn(B, generator=gen(97), device=DEV)
        _, drho = mech_bwd_launch(u, rho, bcs, gr, gc)
        bound = C_MECH * U * mech_bwd_ref(u, rho, bcs, gr, gc, absolute=True)[1]
        assert _within(drho, mech_bwd_ref(u, rho, bcs, gr, gc)[1], bound)
        free = bcs.clone()
        free[:, :2] = 0
        assert not _within(drho, mech_bwd_ref(u, rho, bcs, gr, gc, bcs_for_grad=free)[1], bound)
        return
    r, c = mech_fwd_launch(u, rho, bcs)
    rr, rc = mech_ref(u, rho, bcs)
    Ar, Ac = mech_ref(u, rho, bcs, absolute=True)
    br, bc = C_MECH * U * Ar, (C_MECH + mech_depth(nel)) * U * Ac
    assert _within(r, rr, br) and _within(c, rc, bc)
    fixed = (bcs[:, :2] != 0).double()
    flat = lambda v: v.permute(0, 2, 3, 1).reshape(B, -1)
    if edit == 'mask_is_eq_1':
        eq1 = bcs.clone()
        eq1[:, :2] = (bcs[:, :2] == 1).float()
        mr, mc = mech_ref(u, rho, eq1)
    elif edit == 'f_kept_on_fixed_dof':
        mr, mc = rr - flat(fixed * bcs[:, 2:4].double()), rc
    elif edit == 'element_row_dropped':
        cut = rho.clone()
        cut[:, -1] = 0
        mr, mc = mech_ref(u, cut, bcs)
    else:
        mr, mc = rr, rc - (fixed * u.double() ** 2).sum(dim=(1, 2, 3))
    assert not (_within(r, mr, br) and _within(c, mc, bc)), edit


@pytest.mark.parametrize('edit', ['mean_var', 'p2_by_b'])
def test_mutant_mech_loss(edit):
    operands, sums, grads = mech_loss_launch(5, 64, 0.5, 1e-3, 'distinct', 85)
    assert check_mech_loss(operands, sums, grads)
    assert not check_mech_loss(operands, sums, grads, edit=edit), edit


@pytest.mark.parametrize('edit', ['align_corners', 'clamped_one_early'])
@pytest.mark.parametrize('shape', [(65, 64), (64, 128), (2, 5)], ids=lambda s: f'{s[0]}to{s[1]}')
def test_mutant_resize(edit, shape):
    n_in, n_out = shape
    x = torch.randn(3, n_in, n_in, generator=gen(91), device=DEV)
    _, y = guarded(3 * n_out * n_out)
    call_sync('pidm_bilinear_resize_fwd', x, y, 3, n_in, n_out)
    y = y.view(3, n_out, n_out).cpu()
    xd = x.double().cpu()
    A, coord = resize_bounds(xd, n_out)
    bound = C_RESIZE * U * A + coord
    assert _within(y, F.interpolate(xd[:, None], size=(n_out, n_out), mode='bilinear', align_corners=False)[:, 0], bound)
    assert _within(y, resize_gather(xd, n_out), bound)
    if edit == 'align_corners':
        m = F.interpolate(xd[:, None], size=(n_out, n_out), mode='bilinear', align_corners=True)[:, 0]
    else:
        if n_out <= n_in:
            pytest.skip('downsampling never reaches the last source pixel as i0')
        m = resize_gather(xd, n_out, clamp_hi=n_in - 2)
    assert not _within(y, m, bound), edit


# ----------------------------------------------------------------------------------------------------------------------
# plan coverage
# ----------------------------------------------------------------------------------------------------------------------
def test_plan_coverage():
    for per in (0, 2):
        batches = {_bspec(r[0]) for r in _darcy_rows(DARCY_FWD_TABLE) if r[3] & 2 == per}
        for grid, name in ((darcy_fwd_grid, 'darcy_fwd_kernel'), (darcy_grad_grid, 'darcy_grad_kernel')):
            G = grid(10 ** 9)
            cases = {'one sample': 1 in batches, 'B = grid - 1': G - 1 in batches, 'B = grid': G in batches,
                     'B = grid + 1': G + 1 in batches,
                     'ragged last wave': any(B > G and B % G and B % G != 1 for B in batches),
                     '>= 4 samples per CTA (both mbarrier parities reused)': any(B // G >= 4 for B in batches)}
            missing = [c for c, ok in cases.items() if not ok]
            assert not missing, f'{name}, bcs {"periodic" if per else "none"}: rows miss {missing}'
    geoms = {(r[1], r[2], r[3] & 1) for r in _darcy_rows([])}
    assert {(L, rev, pab) for L, rev, pab in GEOMS} <= geoms
    for rows, name in ((_mech_fwd_rows(), 'mech fwd'), (_mech_bwd_rows(), 'mech bwd')):
        nns = {k[1] + 1 for k in rows}
        cases = {'one band (nn < 8)': any(nn < 8 for nn in nns), 'one exact band': 8 in nns,
                 'several full bands': any(nn % 8 == 0 and nn > 8 for nn in nns),
                 'a one-row last band': any(nn % 8 == 1 for nn in nns),
                 'a ragged last band': any(nn % 8 > 1 and nn > 8 for nn in nns), 'nel = 256': 257 in nns}
        missing = [c for c, ok in cases.items() if not ok]
        assert not missing, f'{name}: rows miss {missing}'
    for table in (RESIZE_FWD_TABLE, RESIZE_BWD_TABLE):
        rows = [k for k in table] + [(pl, i, o) for i, o in RESIZE_SHAPES for pl in (3, 'multi')]
        assert max(resize_passes(_planes(k[0], k[2]), k[2]) for k in rows) >= 3, 'no multi-pass resize grid'
        assert any(resize_passes(_planes(k[0], k[2]), k[2]) == 1 for k in rows)

