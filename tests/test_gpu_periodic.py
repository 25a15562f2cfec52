"""bcs='periodic' on the GPU: every periodic Darcy kernel per element against the fp64 periodic oracle, edited references
rejected by the same predicate, and the guidance branch with the periodic residual against the oracle.  The engine
against the periodic fixtures of the unmodified reference (oracle/make_golden.py periodic) runs as the 'periodic' rows
of test_gpu_e2e.py, test_gpu_parity_bench_path.py, test_gpu_cocogen.py and test_gpu_dropin.py."""
import pytest
import torch

from checks import C_BOUND, P, U, fields, guarded, guards_intact, rel, within
from oracle import pidm_oracle as O
from study import build_darcy, config, state_dict

pytestmark = pytest.mark.gpu
DEV = 'cuda'


# ---- fp64 reference (oracle.pidm_oracle.darcy_residual_matrix) and the edits the predicate has to reject -------------
def residual_op(x, absolute=False, edit=None):
    """the periodic residual in fp64 ([B,P*P,3]); absolute=True: its absolute-value operator"""
    stencils = None
    if edit == 'one_sided_row0':                 # the wrap dropped at row 0: the one-sided stencils of bcs='none' there
        stencils, one_sided = O.darcy_stencils(P, periodic=True), O.darcy_stencils(P)
        stencils[0][0], stencils[1][0] = one_sided[0][0], one_sided[1][0]
    r = O.darcy_residual_matrix(x, True, absolute, stencils)
    if edit == 'corner_sign':
        r[:, 0, 1] = -r[:, 0, 1]
    if edit == 'last_row_zero':
        r[-1, -P:] = 0
    return r


FLAGS = 1 | 2             # PIDM_DARCY_PIXELS_AT_BOUNDARY | PIDM_DARCY_PERIODIC


def fs_dev():
    return O.darcy_source(P).to(DEV).contiguous()


def launch_fwd(x):
    from physicsinformeddiffusionmodels_b200._lib import call, stream
    B = x.shape[0]
    buf, out = guarded(B * P * P * 3)
    call('pidm_darcy_residual_fwd', x.float().to(DEV).contiguous(), fs_dev(), out, B, P, 1.0, 1, FLAGS, stream())
    torch.cuda.synchronize()
    return buf, out.reshape(B, P * P, 3).cpu()


BATCHES = [1, 3, 32, 400]


@pytest.mark.parametrize('B', BATCHES)
def test_periodic_residual_per_element(B):
    x = fields(B, 10 + B)
    buf, y = launch_fwd(x)
    assert guards_intact(buf) and not torch.isnan(y).any()
    r, A = residual_op(x), residual_op(x.abs(), absolute=True)
    err = ((y.double() - r).abs() / (U * A)).max().item()
    assert within(y, r, A), err


@pytest.mark.parametrize('edit', ['one_sided_row0', 'corner_sign', 'last_row_zero'])
def test_edited_references_are_rejected(edit):
    x = fields(32, 42)
    _, y = launch_fwd(x)
    A = residual_op(x.abs(), absolute=True)
    assert within(y, residual_op(x), A)
    assert not within(y, residual_op(x, edit=edit), A), edit


@pytest.mark.parametrize('B', BATCHES)
def test_periodic_vjp_per_element(B):
    from physicsinformeddiffusionmodels_b200._lib import call, stream
    x = fields(B, 20 + B)
    cot = torch.randn(B, P * P, 3, generator=torch.Generator().manual_seed(B), dtype=torch.float64).float().double()
    buf, gx = guarded(B * 2 * P * P)
    call('pidm_darcy_residual_bwd', x.float().to(DEV).contiguous(), fs_dev(), cot.float().to(DEV).contiguous(), gx, B, P,
         1.0, 1, FLAGS, stream())
    torch.cuda.synchronize()
    assert guards_intact(buf) and not torch.isnan(gx).any()
    gx = gx.reshape(B, 2, P, P).cpu()
    ref, A = O.darcy_residual_vjp(x, cot, True), O.darcy_residual_vjp(x, cot, True, absolute=True)
    assert within(gx, ref, A), ((gx.double() - ref).abs() / (U * A)).max().item()


def _loss_reference(x, m, tgt, t, tab_p2, tab_var, c_data, c_res):
    """sums and gradients of the fused loss in fp64 with their bounds"""
    B = x.shape[0]
    r = residual_op(x)
    Ar = residual_op(x.abs(), absolute=True)
    wr = 0.5 * c_res / (tab_var[t] * B * P * P * 3)                     # per sample
    wd = c_data * tab_p2[t] / (B * 2 * P * P)
    sums = torch.stack([(wd[:, None, None, None] * (m - tgt) ** 2).sum(), (wr[:, None, None] * r ** 2).sum(),
                        r.abs().mean()])
    sums_A = torch.stack([(wd[:, None, None, None] * (m.abs() + tgt.abs()) ** 2).sum(),
                          (wr[:, None, None] * Ar ** 2).sum(), Ar.mean()])
    cot = 2 * wr[:, None, None] * r
    gx = O.darcy_residual_vjp(x, cot, True)
    # the fp32 cotangent 2 wr r carries the residual's own error (<= C_BOUND 2^-24 Ar) and that of wr: the adjoint is
    # bounded with twice 2 wr Ar, which leaves C_BOUND 2^-24 for each of the two
    A_gx = O.darcy_residual_vjp(x, 4 * wr[:, None, None] * Ar, True, absolute=True)
    gm = 2 * wd[:, None, None, None] * (m - tgt)
    A_gm = 2 * wd[:, None, None, None] * (m.abs() + tgt.abs())
    return sums, sums_A, gx, A_gx, gm, A_gm


@pytest.mark.parametrize('B', BATCHES)
@pytest.mark.parametrize('variant', ['mean', 'sample', 'loss_only'])
def test_periodic_fused_loss_per_element(B, variant):
    from physicsinformeddiffusionmodels_b200._lib import call, stream
    from physicsinformeddiffusionmodels_b200.denoising_utils import DenoisingDiffusion
    dd = DenoisingDiffusion(100, DEV).diff_dict
    p2, var = dd['p2_loss_weight'].float().contiguous(), dd['posterior_variance_clipped'].float().contiguous()
    x = fields(B, 30 + B)
    g = torch.Generator().manual_seed(300 + B)
    tgt = torch.randn(B, 2, P, P, generator=g).double()
    t = torch.randint(0, 100, (B,), generator=g)
    m = torch.randn(B, 2, P, P, generator=g).double() if variant == 'sample' else x
    xd, md = x.float().to(DEV).contiguous(), m.float().to(DEV).contiguous()
    sums = torch.zeros(3, device=DEV)
    bx, gx = guarded(B * 2 * P * P)
    bm, gm = guarded(B * 2 * P * P)
    c_data, c_res = 1.0, 1e-3
    call('pidm_darcy_pidm_loss', xd, xd if variant != 'sample' else md, tgt.float().to(DEV).contiguous(), fs_dev(),
         t.to(DEV), p2, var, c_data, c_res, sums, None if variant == 'loss_only' else gx,
         gm if variant == 'sample' else None, B, P, 1.0, 1, FLAGS, stream())
    torch.cuda.synchronize()
    rs, rA, rgx, A_gx, rgm, A_gm = _loss_reference(x, m, tgt, t, p2.double().cpu(), var.double().cpu(), c_data, c_res)
    # a sum over N terms: per-term error plus fp32 accumulation (per thread, warp, CTA, one atomic per CTA)
    depth = 4 * 2 * ((B + 131) // 132) + 5 + 16 + 132
    assert ((sums.cpu().double() - rs).abs() <= (depth + 2 * C_BOUND) * U * rA).all(), (sums.cpu(), rs)
    assert guards_intact(bx) and guards_intact(bm)
    if variant == 'loss_only':
        assert torch.isnan(gx).all() and torch.isnan(gm).all()           # NULL gradients: nothing written
        return
    gxc = gx.reshape(B, 2, P, P).cpu()
    if variant == 'mean':                                               # data gradient folded into grad_x0hat
        assert torch.isnan(gm).all()
        assert within(gxc, rgx + rgm, A_gx + A_gm)
    else:
        assert within(gxc, rgx, A_gx)
        assert within(gm.reshape(B, 2, P, P).cpu(), rgm, A_gm)


def _jacobian_max_ref(x):
    """largest entry (signed, zeros included) of d r / d p per sample in fp64, with an absolute bound per sample"""
    d0, d1 = O.spacing(P)
    D1a, _, D1b, _ = O.darcy_stencils(P, periodic=True)
    K = x[:, 1]
    K0, K1 = O.along_rows(D1a, K), O.along_cols(D1b, K)
    e = torch.stack([-K / d0 ** 2 + K0 * 0.5 / d0, -K / d0 ** 2 - K0 * 0.5 / d0,      # rows i-1, i+1
                     -K / d1 ** 2 + K1 * 0.5 / d1, -K / d1 ** 2 - K1 * 0.5 / d1,      # columns j-1, j+1
                     2 * K / d0 ** 2 + 2 * K / d1 ** 2], dim=1)                     # the pixel itself
    bc = torch.tensor(max(0.5 / abs(d0), 0.5 / abs(d1), 0.0), dtype=torch.float64)
    mx = torch.maximum(e.reshape(x.shape[0], -1).max(dim=1).values, bc)
    A = (K.abs() * (2 / d0 ** 2 + 2 / d1 ** 2) + (K0.abs() + K1.abs()) / abs(d0)).reshape(x.shape[0], -1).max(dim=1).values
    return mx, A


@pytest.mark.parametrize('B', BATCHES)
def test_periodic_jacobian_max_per_element(B):
    from physicsinformeddiffusionmodels_b200._lib import call, stream
    x = fields(B, 40 + B)
    if B == 3:
        x[1, 1] = -x[1, 1]                        # negative K: the maximum comes from the BC rows / zero entries
    buf, out = guarded(B)
    call('pidm_darcy_jacobian_max', x.float().to(DEV).contiguous(), out, B, P, 1.0, 1, FLAGS, stream())
    torch.cuda.synchronize()
    assert guards_intact(buf)
    ref, A = _jacobian_max_ref(x)
    assert within(out.cpu(), ref, A)
    if B <= 3:                                    # the closed form above against the oracle's explicit Jacobian
        assert torch.allclose(O.jacobian_max(x, periodic=True), ref, rtol=1e-9, atol=0)


@pytest.mark.parametrize('B', BATCHES)
@pytest.mark.parametrize('mode', ['d_d0', 'd_d1', 'd_d00', 'd_d11', 'd_d01'])
def test_periodic_fd_stencil_per_element(B, mode):
    from physicsinformeddiffusionmodels_b200.grad_utils import StencilGradients
    d0, d1 = O.spacing(P)
    u = fields(B, 50 + B)[:, 0]
    y = StencilGradients(d0=d0, d1=d1, periodic=True)(u.float().to(DEV), mode).cpu()
    r = O.stencil_gradients(u, mode, d0, d1, periodic=True)
    ua = u.abs()
    D1a, D2a, D1b, D2b = (m.abs() for m in O.darcy_stencils(P, periodic=True))
    A = {'d_d0': lambda: O.along_rows(D1a, ua), 'd_d1': lambda: O.along_cols(D1b, ua),
         'd_d00': lambda: O.along_rows(D2a, ua), 'd_d11': lambda: O.along_cols(D2b, ua),
         'd_d01': lambda: O.along_rows(D1a, O.along_cols(D1b, ua))}[mode]()
    assert within(y, r, A)
    from physicsinformeddiffusionmodels_b200._lib import call, stream
    buf, out = guarded(B * P * P)
    call('pidm_fd_stencil', u.float().to(DEV).contiguous(), out, B, P, ['d_d0', 'd_d1', 'd_d00', 'd_d11', 'd_d01'].index(mode)
         | 8, float(d0), float(d1), stream())
    torch.cuda.synchronize()
    assert guards_intact(buf) and torch.equal(out.reshape(B, P, P).cpu(), y)


# ---- end to end ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def ops():
    from physicsinformeddiffusionmodels_b200 import ops
    yield ops
    ops.set_precision('bf16')


def test_periodic_residual_gradient_guidance_matches_oracle(ops):
    """guidance branch (cond = d mean|r(x_t)| / d x_t with the periodic residual) through the engine vs the periodic
    oracle, fp32, with a classifier-free mask that drops one sample"""
    ops.set_precision('fp32')
    g = torch.Generator().manual_seed(77)
    B = 4
    x0 = torch.randn(B, 2, 64, 64, generator=g)
    t = torch.randint(0, 100, (B,), generator=g)
    e = torch.randn(B, 2, 64, 64, generator=g)
    mask = torch.tensor([False, True, False, False])
    sdr = {k: v.clone().requires_grad_('freqs' not in k) for k, v in state_dict().items()}
    loss_ref, _ = O.darcy_training_loss(sdr, config(), x0, t, e, O.diffusion_tables(100), guidance_null_mask=mask,
                                        periodic=True)
    loss_ref.backward()
    model, diff, res = build_darcy('periodic', residual_grad_guidance=True)
    model._null_mask_override = mask.to(DEV)
    loss, _, _, _, _ = diff.darcy_loss_from_draws(x0.to(DEV), t.to(DEV), e.to(DEV), res, 1.0, 1e-3)
    model._null_mask_override = None
    assert abs(loss.item() / loss_ref.item() - 1) < 5e-5, (loss.item(), loss_ref.item())
    loss.backward()
    named = dict(model.named_parameters())
    for k in ('emb_conv.0.weight', 'combine_conv.weight', 'final_conv.1.weight'):
        assert rel(named[k].grad, sdr[k].grad) < 2e-3, (k, rel(named[k].grad, sdr[k].grad))


def test_mechanics_periodic_equals_none():
    """ResidualsMechanics only stores the flag in the reference: 'periodic' computes exactly what 'none' computes"""
    from physicsinformeddiffusionmodels_b200.residuals_mechanics_K import ResidualsMechanics
    g = torch.Generator().manual_seed(4)
    x = torch.randn(2, 3, 64, 64, generator=g) * 0.1
    x[:, 2] = torch.sigmoid(torch.randn(2, 64, 64, generator=g))
    bcs = torch.zeros(2, 4, 65, 65)
    bcs[:, 0, :, 0] = 1.
    bcs[:, 1, :, 0] = 1.
    bcs[:, 3, 20:24, 64] = -1.
    vf = torch.tensor([0.4, 0.5])
    outs = {}
    for b in ('none', 'periodic'):
        res = ResidualsMechanics(model=None, pixels_per_dim=64, pixels_at_boundary=True, no_BC_folder='', device=DEV,
                                 bcs=b)
        assert res.periodic == (b == 'periodic')
        outs[b] = res.compute_residual((x.to(DEV), bcs.to(DEV), vf.to(DEV), None), reduce='per-batch',
                                       return_optimizer=True, return_inequality=True, pass_through=True)
    assert torch.equal(outs['none']['residual'], outs['periodic']['residual'])
    assert torch.equal(outs['none']['inequality'], outs['periodic']['inequality'])
    # compliance is a sum of fp32 atomics: equal up to their ordering
    assert rel(outs['periodic']['optimizer'], outs['none']['optimizer']) < 1e-6
