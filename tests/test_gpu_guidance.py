"""Residual-gradient guidance on the GPU: the guidance kernels per element against fp64 references (edited references
rejected by the same bounds), and the engine end to end: the optimizer update of the guidance layers, the in-graph mask
draw, the sharded draw and the guided sampler.  Graph replay against the eager step and the eager step against one
training iteration of the unmodified reference (oracle/make_golden.py guidance) are the 'guidance' rows of
test_gpu_parity_bench_path.py and test_gpu_e2e.py."""
import math

import pytest
import torch

from checks import C_BOUND, P, U, fields, guarded, guards_intact, rel, within
from oracle import pidm_oracle as O
from study import build_darcy

pytestmark = pytest.mark.gpu
DEV = 'cuda'


# ---- fp64 Darcy residual from explicit stencil matrices (oracle.pidm_oracle.darcy_residual_matrix) ------------------
def cond_reference(x, periodic, n_norm, edit=None):
    """(cond, bound A) in fp64, [B,P*P,2]: cond = J^T sign(r) / n_norm, A = |J|^T |sign(r)| / n_norm at |x|"""
    B = x.shape[0]
    cot = torch.sign(O.darcy_residual_matrix(x, periodic)) / n_norm
    if edit == 'bc_row_sign':                 # the bc_x0 seeds of row 0 with the wrong sign
        cot[:, :P, 1] = -cot[:, :P, 1]
    g = O.darcy_residual_vjp(x, cot, periodic)
    A = O.darcy_residual_vjp(x, cot, periodic, absolute=True)
    to_rows = lambda t: t.permute(0, 2, 3, 1).reshape(B, P * P, 2)      # noqa: E731
    return to_rows(g), to_rows(A)


def launch_abs_residual_grad(x, periodic, n_norm):
    from physicsinformeddiffusionmodels_b200._lib import call, stream
    B = x.shape[0]
    buf, out = guarded(B * P * P * 2)
    call('pidm_darcy_abs_residual_grad', x.float().contiguous(), O.darcy_source(P).to(DEV).contiguous(), out, B, n_norm,
         P, 1.0, 1, 1 | (2 if periodic else 0), stream())
    torch.cuda.synchronize()
    return buf, out.reshape(B, P * P, 2)


@pytest.mark.parametrize('bcs', ['none', 'periodic'])
@pytest.mark.parametrize('B', [1, 3, 32, 400])
def test_abs_residual_grad_per_element(B, bcs):
    periodic = bcs == 'periodic'
    # seeds without sign-ambiguous entries
    x = fields(B, 1008 if B == 400 else 600 + B + (7 if periodic else 0), DEV)
    # the stencil matrices restate the oracle's residual
    r = O.darcy_residual_matrix(x, periodic)
    ref_r = O.darcy_residual(x[:2].cpu(), periodic=periodic)
    assert rel(r[:2], ref_r) < 1e-12
    # no sign-ambiguous entry: every entry that is not structurally zero lies outside the residual's rounding bound
    Ar = O.darcy_residual_matrix(x, periodic, absolute=True)
    live = r != 0
    assert bool((r.abs()[live] > C_BOUND * U * Ar[live]).all())
    assert bool((r[:, :, 1:][~live[:, :, 1:]] == 0).all()) and bool(live[:, :, 0].all())
    n = B * P * P * 3
    buf, y = launch_abs_residual_grad(x, periodic, n)
    assert guards_intact(buf) and not torch.isnan(y).any()
    g, A = cond_reference(x, periodic, n)
    assert within(y, g, A), ((y.double() - g).abs() / (U * A)).max().item()


@pytest.mark.parametrize('bcs', ['none', 'periodic'])
@pytest.mark.parametrize('edit', ['local_norm', 'bc_row_sign'])
def test_abs_residual_grad_rejects_edited_references(bcs, edit):
    periodic = bcs == 'periodic'
    x = fields(32, 77, DEV)
    n = 32 * P * P * 3
    if edit == 'local_norm':              # a shard of a 2-rank global batch normalised by its local count
        _, y = launch_abs_residual_grad(x, periodic, 2 * n)
        g, A = cond_reference(x, periodic, 2 * n)
        assert within(y, g, A)
        g_bad, _ = cond_reference(x, periodic, n)
    else:
        _, y = launch_abs_residual_grad(x, periodic, n)
        g, A = cond_reference(x, periodic, n)
        assert within(y, g, A)
        g_bad, _ = cond_reference(x, periodic, n, edit='bc_row_sign')
    assert not within(y, g_bad, A), edit


# ---- guidance embedding: emb_conv[0] + GELU, and its weight gradient -------------------------------------------------
def _embed_inputs(B, seed, C=32):
    g = torch.Generator().manual_seed(seed)
    cond = (torch.randn(B, P * P, 2, generator=g) * 3e-4).to(DEV)          # the scale of d mean|r| / d x_t
    w0 = (torch.randn(C, 2, 1, 1, generator=g) * 2e3).to(DEV)
    b0 = (torch.randn(C, generator=g) * 0.5).to(DEV)
    mask = torch.zeros(B, dtype=torch.bool)
    if B > 1:
        mask[1::3] = True
    return cond, mask.to(DEV), w0, b0


def _gelu64(z, tanh=False):
    if tanh:
        return 0.5 * z * (1 + torch.tanh(math.sqrt(2 / math.pi) * (z + 0.044715 * z ** 3)))
    return 0.5 * z * (1 + torch.erf(z / math.sqrt(2)))


def _pre64(cond, mask, w0, b0, unmask=None):
    c = cond.double().clone()
    keep_masked = mask.clone()
    if unmask is not None:
        keep_masked[unmask] = False
    c[keep_masked] = 0
    W = w0.double().reshape(-1, 2)
    z = c @ W.T + b0.double()
    A = c.abs() @ W.abs().T + b0.double().abs()
    return z, A, c


def launch_embed(cond, mask, w0, b0, dtype):
    from physicsinformeddiffusionmodels_b200 import _lib
    B, C = cond.shape[0], w0.shape[0]
    buf, out = guarded(B * P * P * C, dtype)
    _lib.call('pidm_cond_embed_fwd', cond, mask, w0, b0, out, B, P * P, C, _lib.DTYPE_CODE[dtype], _lib.stream())
    torch.cuda.synchronize()
    return buf, out.reshape(B, P * P, C)


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
@pytest.mark.parametrize('B', [1, 3, 32])
def test_cond_embed_per_element(B, dtype):
    cond, mask, w0, b0 = _embed_inputs(B, 900 + B)
    buf, e = launch_embed(cond, mask, w0, b0, dtype)
    assert guards_intact(buf) and not torch.isnan(e).any()
    z, A, _ = _pre64(cond, mask, w0, b0)
    ref = _gelu64(z)
    bound = 2.0 ** -20 * A + (2.0 ** -8 * ref.abs() if dtype == torch.bfloat16 else 0)
    err = (e.double() - ref).abs()
    assert bool((err <= bound).all()), (err / bound).max().item()
    null = torch.nn.functional.gelu(b0.float()).to(dtype)
    for b in range(B):
        if mask[b]:
            assert torch.equal(e[b], null.expand(P * P, -1)), b


@pytest.mark.parametrize('edit', ['unmasked_sample', 'tanh_gelu'])
def test_cond_embed_rejects_edited_references(edit):
    cond, mask, w0, b0 = _embed_inputs(32, 950)
    _, e = launch_embed(cond, mask, w0, b0, torch.float32)
    z, A, _ = _pre64(cond, mask, w0, b0)
    assert bool(((e.double() - _gelu64(z)).abs() <= 2.0 ** -20 * A).all())
    if edit == 'unmasked_sample':
        z_bad, _, _ = _pre64(cond, mask, w0, b0, unmask=int(mask.nonzero()[0]))
        bad = _gelu64(z_bad)
    else:
        bad = _gelu64(z, tanh=True)
    assert not bool(((e.double() - bad).abs() <= 2.0 ** -20 * A).all()), edit


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
@pytest.mark.parametrize('B', [1, 3, 32])
def test_cond_embed_wgrad_per_element(B, dtype):
    from physicsinformeddiffusionmodels_b200 import _lib
    cond, mask, w0, b0 = _embed_inputs(B, 970 + B)
    C = w0.shape[0]
    g = torch.Generator().manual_seed(B)
    dg = torch.randn(B, P * P, C, generator=g).to(DEV).to(dtype)
    pre_w, pre_b = torch.full((C, 2), 0.25, device=DEV), torch.full((C,), -0.5, device=DEV)   # accumulated into
    dw, db = pre_w.clone(), pre_b.clone()
    _lib.call('pidm_cond_embed_wgrad', cond, mask, w0, b0, dg, dw, db, B, P * P, C, _lib.DTYPE_CODE[dtype], _lib.stream())
    torch.cuda.synchronize()
    z, _, c = _pre64(cond, mask, w0, b0)
    cdf, pdf = 0.5 * (1 + torch.erf(z / math.sqrt(2))), torch.exp(-0.5 * z * z) / math.sqrt(2 * math.pi)
    d = dg.double()
    dz, dz_abs = d * (cdf + z * pdf), d.abs() * (cdf + z.abs() * pdf)
    M = B * P * P
    ref_w = torch.einsum('bmo,bmk->ok', dz, c)
    ref_b = dz.sum((0, 1))
    A_w = torch.einsum('bmo,bmk->ok', dz_abs, c.abs())
    A_b = dz_abs.sum((0, 1))
    k = 16 * math.sqrt(M) * U
    assert bool(((dw.double() - pre_w.double() - ref_w).abs() <= k * A_w + U).all())
    assert bool(((db.double() - pre_b.double() - ref_b).abs() <= k * A_b + U).all())


# ---- engine ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def ops():
    from physicsinformeddiffusionmodels_b200 import ops
    yield ops
    ops.set_precision('bf16')


def _offset(eng, p):
    return eng.fp.offsets[next(i for i, q in enumerate(eng.fp.params) if q is p)]


def test_guidance_layers_take_clip_and_adam_of_the_snapshot(ops):
    from physicsinformeddiffusionmodels_b200.engine import TrainEngine
    ops.set_precision('fp32')
    model, diff, res = build_darcy('guidance')
    eng = TrainEngine(model, diff, res, use_graph=True, snapshot_grad=True)
    g = torch.Generator().manual_seed(11)
    x0 = (0.7 * torch.randn(8, 2, 64, 64, generator=g)).to(DEV)
    p0 = eng.fp.flat.clone()
    eng.step(x0)
    torch.cuda.synchronize()
    gs = eng.grad_snapshot.double()
    coef = min(eng.max_norm / (gs.norm().item() + 1e-6), 1.0)
    gc = gs * coef
    upd = eng.lr * gc / (gc.abs() + eng.eps)              # Adam step 1 with bias correction
    for name, p in model.named_parameters():
        if not name.startswith(('emb_conv.', 'combine_conv.')):
            continue
        o = _offset(eng, p)
        sl = slice(o, o + p.numel())
        assert gs[sl].abs().sum() > 0, name
        err = (eng.fp.flat[sl].double() - (p0[sl].double() - upd[sl])).abs()
        assert bool((err <= 4 * U * p0[sl].double().abs() + 1e-4 * eng.lr).all()), (name, err.max().item())


def test_in_graph_mask_is_redrawn_every_replay(ops):
    from physicsinformeddiffusionmodels_b200.engine import TrainEngine
    ops.set_precision('bf16')
    model, diff, res = build_darcy('guidance')
    eng = TrainEngine(model, diff, res, use_graph=True)
    g = torch.Generator().manual_seed(12)
    x0 = (0.7 * torch.randn(32, 2, 64, 64, generator=g)).to(DEV)
    masks = []
    for _ in range(50):
        eng.step(x0)
        masks.append(model._null_mask_last.clone())
    m = torch.stack(masks).float()
    assert sum(not torch.equal(a, b) for a, b in zip(masks[:-1], masks[1:])) >= 40
    assert 0.07 <= m.mean().item() <= 0.13, m.mean().item()


def test_sharded_cond_and_mask_are_slices_of_the_global_batch():
    from physicsinformeddiffusionmodels_b200.unet_model import draw_null_mask
    _, _, res = build_darcy('guidance')
    world, B = 4, 6
    x = fields(world * B, 31, DEV).float().permute(0, 2, 3, 1).reshape(world * B, P * P, 2).contiguous()
    full = res.residual_gradient(x)
    torch.manual_seed(9)
    mfull = draw_null_mask(world * B, 0.1, DEV)
    for rank in range(world):
        lo, hi = rank * B, (rank + 1) * B
        assert torch.equal(res.residual_gradient(x[lo:hi].contiguous(), world), full[lo:hi])
        torch.manual_seed(9)
        assert torch.equal(draw_null_mask(B, 0.1, DEV, (rank, world)), mfull[lo:hi])


def test_guidance_sample_engine_graph_equals_eager(ops, monkeypatch):
    from physicsinformeddiffusionmodels_b200.engine import SampleEngine
    ops.set_precision('fp32')
    model, diff, res = build_darcy('guidance', n_steps=6)
    model.eval()
    g = torch.Generator().manual_seed(13)
    x_T = torch.randn(2, 2, 64, 64, generator=g).to(DEV)
    zfix = torch.randn(2, 2, 64, 64, generator=g).to(DEV)
    monkeypatch.setattr(torch, 'randn_like', lambda *a, **k: zfix)
    xe = SampleEngine(model, diff, res, batch=2, use_graph=False).sample(x_init=x_T)[0].clone()
    xg = SampleEngine(model, diff, res, batch=2, use_graph=True).sample(x_init=x_T)[0].clone()
    monkeypatch.undo()
    assert torch.isfinite(xe).all()
    assert rel(xg, xe) < 1e-4, rel(xg, xe)
