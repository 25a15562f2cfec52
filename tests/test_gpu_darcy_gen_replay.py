"""Per-element checks of the Darcy data generator (csrc/darcy_gen.cu) against fp64, stage by stage, at every geometry.

pidm_darcy_gen_solve runs three stages that the `stages` mask selects, and the workspace carries the band and the
right-hand side between them (include/pidm.h), so each stage is fed chosen inputs and read back on its own.

  Tier 1, known answers, bitwise.  Dyadic operands make every operation of a stage exact (tests/test_oracle_darcy_gen.py
  checks that on the host), so any correct order of operations returns one answer:
    KLE       dyadic phi_s and z: g is exact and K must lie within 1 ulp of exp(g) in long double (CUDA's double exp
              is accurate to 1 ulp); B = 0 writes nothing; B = 65535 is the grid.y limit.
    assemble  K = k/16 and an integer source at spacing 1 (twice) and 2^-6: band and rhs equal the oracle's bit for bit,
              the pin, the zeros outside the 25 stencil offsets and those of negative column included.
    factor    band(L0 L0^T) and L0 y0 in the workspace: L0 and y0 come back bit for bit, and the band entries of negative
              column (NaN sentinels) are neither read nor written.
    post      L0 and L0^T x0: p = fl(x0 - fl(w^T x0 / w^T 1)), batch = (float) (p, K), res = fl(S / (P^2 + 4P + 1)) where
              S is exact; all eight combinations of the optional outputs.
    The three stages run as separate calls equal one call with all three.

  Tier 2, per-element bounds on realistic operands (KLE and rough log-normal K, the geometry's source and a dense random
  one) at pixels_at_boundary in {T, F} x domain_length in {1, 0.3, 2.5}; u = 2^-53, |.| the same chain on absolute
  values:
    assemble  |band - N| <= C_ASM u (|M|^T |M|),  |rhs - A^T f_s| <= C_ASM u |A|^T |f_s|; reverse_dy changes neither.
    factor    the componentwise backward error, independent of cond(N) ~ 1e14: |L L^T - N| <= C_CHOL u |L| |L|^T and
              |L y - rhs| <= C_CHOL u |L| |y| (dense fp64 products on the device; C_CHOL covers both sides' rounding).
    post      a backward error with the shift s recovered from the last unknown, which the kernel forms with one
              division: s = y_{n-1} / L_{n-1,n-1} - p_{n-1}, |error of s| <= E_s = 2u (|y_{n-1} / L_{n-1,n-1}| + |p_{n-1}|);
              |L^T (p + s) - y| <= C_POST u (|L^T| (|p| + |s|) + |y|) + |L^T| 1 E_s,  |w^T p| <= C_POST u depth w^T (|p| + |s|),
              res against the fp64 mean |M p - b| of the kernel's own p within C_POST u mean(|M| |p| + |b|).
    end to end, p and res against the host banded solve (DO.solve_banded) to 1e-5 max|p| (1e-4 at domain_length 0.3,
              where cond(N) is larger) and 1e-4.

  Edited references (a subtle kernel bug each) must be rejected by the same predicates, and the launch arithmetic of
  darcy_gen.cu is restated with the rows that reach each of its cases.  There is no census table: no benchmarked
  step calls the generator."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

from checks import (DGEN_BW, DGEN_EXACT_GEOMETRIES, GUARD, call_sync, dgen_band_to_dense, dgen_dense_to_band,
                    dgen_dyadic_factor, dgen_dyadic_K, dgen_dyadic_source, gen, guarded, guards_intact, note, ratio, sms)
from oracle import darcy_gen_oracle as DO

pytestmark = pytest.mark.gpu
DEV = 'cuda'
TAG = 'darcy_gen'
P = 64
N = P * P
BW = DGEN_BW
LD = BW + 1
U = 2.0 ** -53
ASSEMBLE, FACTOR, POST, ALL = 1, 2, 4, 7          # PIDM_DARCY_GEN_*
C_ASM = 8
C_CHOL = 32
C_POST = 4
POST_THREADS = 256
DEPTH = N // POST_THREADS + 5 + POST_THREADS // 32 + 2    # post's block sums: per thread, warp shuffle, warps, w^T 1
# end to end, |p - p_host| / max|p_host| per domain length: both solve the same normal equations backward stably (the
# stage bounds), so they differ by rounding amplified by cond(N), which grows as h shrinks (A ~ h^-2 against BC ~ h^-1)
E2E_P = {1.0: 1e-5, 2.5: 1e-5, 0.3: 1e-4}
GEOMETRIES = [dict(pixels_at_boundary=pab, reverse_dy=True, domain_length=dl)
              for pab in (True, False) for dl in (1.0, 0.3, 2.5)]
DEFAULT = GEOMETRIES[0]


def geo_id(g):
    return f"pab{int(g['pixels_at_boundary'])}_L{g['domain_length']:g}"


def bits_equal(a, b):
    it = {8: torch.int64, 4: torch.int32}[a.element_size()]
    return a.shape == b.shape and torch.equal(a.contiguous().view(it), b.contiguous().view(it))


class Workspace:
    """the solve's workspace between 0xA5 guard bytes: band [B, N, BW + 1] then rhs [B, N], fp64 (include/pidm.h)"""

    def __init__(self, B):
        from physicsinformeddiffusionmodels_b200._lib import call
        self.B = B
        self.bytes = call('pidm_darcy_gen_workspace_bytes', B, P)
        assert self.bytes == B * (N * LD + N) * 8
        g = GUARD * 8
        self.raw = torch.full((self.bytes + 2 * g,), 0xA5, dtype=torch.uint8, device=DEV)
        body = self.raw[g:g + self.bytes].view(torch.float64)
        self.band = body[:B * N * LD].view(B, N, LD)
        self.rhs = body[B * N * LD:].view(B, N)

    def intact(self):
        g = GUARD * 8
        return bool((self.raw[:g] == 0xA5).all() and (self.raw[g + self.bytes:] == 0xA5).all())


def solve(ws, K, f_s, geo, stages, p=None, res=None, batch=None):
    call_sync('pidm_darcy_gen_solve', K, f_s, p, res, batch, ws.band, ws.bytes, ws.B, P, float(geo['domain_length']),
              int(geo['reverse_dy']), int(geo['pixels_at_boundary']), stages)
    assert ws.intact()


def outputs(B):
    """NaN-guarded p [B*N] fp64, res [B] fp64, batch [B*2*N] fp32: ((buffer, view), ...)"""
    return guarded(B * N, torch.float64), guarded(B, torch.float64), guarded(B * 2 * N, torch.float32)


def dev(a):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float64, device=DEV)


@pytest.fixture(scope='module')
def kgen():
    from physicsinformeddiffusionmodels_b200.darcy_data_generation import DarcyDataGenerator
    return DarcyDataGenerator()


def realistic_K(kgen, seed):
    """[4, N]: two KLE fields of the reference's covariance and two rough log-normal fields (log-std 0.5)"""
    rough = torch.exp(0.5 * torch.randn(2, N, generator=gen(seed), device=DEV, dtype=torch.float64))
    return torch.cat([kgen.permeability(kgen.z_for_seeds([seed, seed + 1])), rough])


def sources(geo):
    """the geometry's source and a dense random one"""
    return {'source': dev(DO.source(geo['pixels_at_boundary'], geo['domain_length'])),
            'dense': torch.randn(N, generator=gen(('dense f_s', geo_id(geo))), device=DEV, dtype=torch.float64)}


# ---- fp64 references and the tier-2 predicates --------------------------------------------------------------------------
def assembly_ref(K, f_s, geo):
    """(band, |M|^T|M| band, A^T f_s, |A|^T |f_s|) on the host"""
    A, BC = DO.operators(K, **geo)
    Aa, BCa = DO.operators(K, absolute=True, **geo)
    return (DO.to_band(DO.pinned_normal(A, BC)), DO.to_band(DO.pinned_normal(Aa, BCa)), A.T @ f_s,
            Aa.T @ np.abs(f_s))


def asm_ratio(out, ref, absref):
    return ratio((out - dev(ref)).abs(), C_ASM * U * dev(absref))


def symmetric(lower):
    return lower + lower.T - torch.diag(torch.diagonal(lower))


def factor_ratios(L_band, y, N_band, rhs, N_full=None):
    """worst |L L^T - N| / (C_CHOL u |L||L|^T) and |L y - rhs| / (C_CHOL u |L||y|) for one sample"""
    L = dgen_band_to_dense(L_band)
    if N_full is None:
        N_full = symmetric(dgen_band_to_dense(N_band))
    La = L.abs()
    q_n = ratio((L @ L.T - N_full).abs(), C_CHOL * U * (La @ La.T))
    q_y = ratio((L @ y - rhs).abs(), C_CHOL * U * (La @ y.abs()))
    return q_n, q_y


def post_ratios(L_band, y, p, w):
    """worst ratios of the post stage's backward error (Lt p + s = y) and of w^T p = 0 for one sample"""
    L = dgen_band_to_dense(L_band)
    xl = y[N - 1] / L[N - 1, N - 1]
    s = xl - p[N - 1]
    Es = 2 * U * (xl.abs() + p[N - 1].abs())
    LTa = L.T.abs()
    e = L.T @ (p + s) - y
    bound = C_POST * U * (LTa @ (p.abs() + s.abs()) + y.abs()) + LTa.sum(1) * Es
    q_x = ratio(e.abs(), bound)
    q_w = ratio((w @ p).abs().reshape(1), (C_POST * U * DEPTH * (w.abs() @ (p.abs() + s.abs()))).reshape(1))
    return q_x, q_w, s


def res_ref(K, f_s, p, geo, rows=None):
    """(fp64 mean |M p - b| of the kernel's own p, mean(|M||p| + |b|)) on the host"""
    M, b = DO.system(K, f_s, **geo)
    Aa, BCa = DO.operators(K, absolute=True, **geo)
    w = DO.weights(geo['pixels_at_boundary'], geo['domain_length'])
    Ma = sp.vstack([Aa, BCa, sp.csr_matrix(np.abs(w).reshape(1, -1))]).tocsr()
    r = np.abs(M @ p - b)
    rows = rows or len(b)
    return r.sum() / rows, (Ma @ np.abs(p) + np.abs(b)).mean()


def res_ratio(res, ref, scale):
    return abs(res - ref) / (C_POST * U * scale)


# ---- tier 1: known answers ----------------------------------------------------------------------------------------------
def kle_ratio(K, g):
    """worst |K - exp(g)| / ulp, exp(g) in long double on the host"""
    assert np.finfo(np.longdouble).nmant >= 63, 'the 1-ulp check of exp needs an extended long double'
    gl = g.cpu().numpy().astype(np.longdouble)
    E = np.exp(gl)
    ulp = np.spacing(E.astype(np.float64)).astype(np.longdouble)
    return float((np.abs(K.cpu().numpy().astype(np.longdouble) - E) / ulp).max())


def dyadic_kle(q, B, key):
    g = gen(key)
    phi = torch.randint(-4, 5, (q, N), generator=g, device=DEV).double() / 16
    z = torch.randint(-4, 5, (B, q), generator=g, device=DEV).double() / 16
    return phi, z


@pytest.mark.parametrize('B', [1, 5, 300])
@pytest.mark.parametrize('q', [1, 7, 64, 4096])
def test_kle_known_answer(q, B):
    phi, z = dyadic_kle(q, B, ('kle', q, B))
    buf, K = guarded(B * N, torch.float64)
    call_sync('pidm_darcy_gen_kle', phi, z, K, B, q, P)
    assert guards_intact(buf)
    g = z @ phi                                          # exact: every partial sum is a multiple of 2^-8 below 2^9
    q_k = kle_ratio(K.view(B, N), g)
    note(TAG, f'kle q={q} B={B} K (ulp)', q_k)
    assert q_k <= 1.0
    if (q, B) == (64, 5):
        # edited references: the sum over q - 1 terms, exp in fp32
        assert kle_ratio(K.view(B, N), z[:, :-1] @ phi[:-1]) > 1
        E32 = torch.exp(g.float()).double()
        q_32 = ratio((K.view(B, N) - E32).abs(), 2 * U * K.view(B, N).abs())
        note(TAG, 'mutant kle exp in fp32', q_32)
        assert q_32 > 1


def test_kle_zero_and_grid_y_limit():
    phi, z = dyadic_kle(1, 1, 'kle B=0')
    buf, K = guarded(N, torch.float64)
    call_sync('pidm_darcy_gen_kle', phi, z, K, 0, 1, P)
    assert bool(torch.isnan(buf).all())
    B = 65535                                            # grid (N / 256, B): B is the grid.y limit
    phi, z = dyadic_kle(1, B, 'kle B=65535')
    buf, K = guarded(B * N, torch.float64)
    call_sync('pidm_darcy_gen_kle', phi, z, K, B, 1, P)
    assert guards_intact(buf)
    K = K.view(B, N)
    g = z * phi                                          # [B, N], exact; 19 distinct values
    gs, Ks = [], []
    for v in torch.unique(g):                            # every element of every sample: one K per value of g
        Kv = K[g == v]
        assert Kv.min().item() == Kv.max().item(), v
        gs.append(v)
        Ks.append(Kv[0])
    q_k = kle_ratio(torch.stack(Ks), torch.stack(gs))
    note(TAG, 'kle q=1 B=65535 K (ulp)', q_k)
    assert q_k <= 1.0
    del buf, K, g


@pytest.mark.parametrize('geo', DGEN_EXACT_GEOMETRIES, ids=geo_id)
def test_assemble_known_answer(geo):
    B = 3
    g = gen(('assemble', geo_id(geo)))
    K, f_s = dgen_dyadic_K(B, g), dgen_dyadic_source(g)
    ws = Workspace(B)
    solve(ws, K, f_s, geo, ASSEMBLE)
    r = torch.arange(N, device=DEV)[:, None]
    d = torch.arange(LD, device=DEV)[None, :]
    adx, dy = (d + 3) // P, ((d + 3) // P) * P - d
    stencil = (dy.abs() <= 3) & ((adx > 0) | (dy <= 0))   # the 25 lower offsets |dx|, |dy| <= 3
    assert int(stencil.sum()) == 25
    for b in range(B):
        band, _, rhs, _ = assembly_ref(K[b].cpu().numpy(), f_s.cpu().numpy(), geo)
        assert bits_equal(ws.band[b], dev(band)), b
        assert bits_equal(ws.rhs[b], dev(rhs)), b
        assert bool((ws.band[b][~stencil.expand(N, LD)] == 0).all() and (ws.band[b][(r - d < 0)] == 0).all())
    # the pin: N_00 is twice the unpinned sum
    A, BC = DO.operators(K[0].cpu().numpy(), **geo)
    M = sp.vstack([A, BC]).tocsr()
    assert ws.band[0, 0, 0].item() == 2 * (M.T @ M)[0, 0]
    # reverse_dy enters squared or under | |: the same band and rhs bit for bit
    ws2 = Workspace(B)
    solve(ws2, K, f_s, {**geo, 'reverse_dy': False}, ASSEMBLE)
    assert bits_equal(ws2.band, ws.band) and bits_equal(ws2.rhs, ws.rhs)


@pytest.mark.parametrize('B', [1, 3, 133])
def test_factor_known_answer(B):
    """133 CTAs of one per SM (218,656 B of shared memory each) run in a second wave past 132 SMs"""
    g = gen(('factor', B))
    L0 = dgen_dyadic_factor(B, g)                       # NaN where the column r - d is negative
    y0 = torch.randint(-8, 9, (B, N), generator=g, device=DEV).double() / 16
    ws = Workspace(B)
    for b in range(B):
        L = dgen_band_to_dense(L0[b])
        ws.band[b] = dgen_dense_to_band(L @ L.T, fill=float('nan'))
        ws.rhs[b] = L @ y0[b]
    solve(ws, None, None, DEFAULT, FACTOR)
    assert bits_equal(ws.band, L0)
    assert bits_equal(ws.rhs, y0)


def post_known_answer(geo, B, key):
    """(workspace holding L0 and y = L0^T x0, x0, K, f_s, the expected p) for the post stage"""
    g = gen(key)
    L0 = dgen_dyadic_factor(B, g)
    x0 = torch.randint(-8, 9, (B, N), generator=g, device=DEV).double() / 16
    K, f_s = dgen_dyadic_K(B, g), dgen_dyadic_source(g)
    ws = Workspace(B)
    ws.band.copy_(L0)
    for b in range(B):
        ws.rhs[b] = dgen_band_to_dense(L0[b]).T @ x0[b]                    # exact
    w = DO.weights(geo['pixels_at_boundary'], geo['domain_length'])
    p = np.empty((B, N))
    for b in range(B):
        xb = x0[b].cpu().numpy()
        p[b] = xb - np.float64(w @ xb) / np.float64(w.sum())              # w^T x0 and w^T 1 exact: one rounding each
    return ws, x0, K, f_s, dev(p)


@pytest.mark.parametrize('geo', DGEN_EXACT_GEOMETRIES[:2], ids=geo_id)
def test_post_known_answer(geo):
    B = 3
    ws, x0, K, f_s, p_exp = post_known_answer(geo, B, ('post', geo_id(geo)))
    band0, rhs0 = ws.band.clone(), ws.rhs.clone()
    full = None
    for mask in (7, 0, 1, 2, 3, 4, 5, 6):
        (pb, p), (rb, res), (bb, batch) = outputs(B)
        want = [mask & 1, mask & 2, mask & 4]
        solve(ws, K, f_s, geo, POST, p if want[0] else None, res if want[1] else None, batch if want[2] else None)
        assert bits_equal(ws.band, band0) and bits_equal(ws.rhs, rhs0)
        for (buf, _), on in zip(((pb, p), (rb, res), (bb, batch)), want):
            assert guards_intact(buf) and (on or bool(torch.isnan(buf).all()))
        if want[0]:
            assert bits_equal(p.view(B, N), p_exp)
        if want[2]:
            bt = batch.view(B, 2, N)
            assert bits_equal(bt[:, 0], p_exp.float()) and bits_equal(bt[:, 1], K.float())
        if mask == 7:
            full = res.clone()
        elif want[1]:
            assert bits_equal(res, full)
    trapezoid = geo['pixels_at_boundary']
    for b in range(B):
        Kb, fb, pb_ = K[b].cpu().numpy(), f_s.cpu().numpy(), p_exp[b].cpu().numpy()
        ref, scale = res_ref(Kb, fb, pb_, geo)
        q_r = res_ratio(full[b].item(), ref, scale)
        note(TAG, f'post known answer {geo_id(geo)} res', q_r)
        assert q_r <= 1.0
        if not trapezoid:
            # spacing 1, mean weights: p = x0 - w^T x0 is a multiple of 2^-16 and 64 A, 2 BC are integer matrices, so
            # every row of M p - b is exact and S = sum |M p - b| is an integer multiple of 2^-22 below 2^53
            A, BC = DO.operators(Kb, **geo)
            pi = np.round(pb_ * 2 ** 16).astype(np.int64)
            assert np.array_equal(pi * 2.0 ** -16, pb_)
            Ai, Bi = (A * 64).astype(np.int64), (BC * 2).astype(np.int64)
            assert (abs(Ai * (1 / 64.) - A)).max() == 0 and (abs(Bi * 0.5 - BC)).max() == 0
            S = int(np.abs(Ai @ pi - np.round(fb).astype(np.int64) * 2 ** 22).sum()) + \
                int(np.abs(Bi @ pi).sum()) * 2 ** 5
            w = DO.weights(False, geo['domain_length'])
            assert w @ pb_ == 0.0 and S < 2 ** 53
            assert full[b].item() == (S * 2.0 ** -22) / (N + 4 * P + 1), b


@pytest.mark.parametrize('geo', [DEFAULT, GEOMETRIES[5]], ids=geo_id)
def test_stage_split_equals_one_call(geo, kgen):
    K = realistic_K(kgen, 700)[:3]
    f_s = sources(geo)['source']
    runs = []
    for split in (True, False):
        ws = Workspace(3)
        (pb, p), (rb, res), (bb, batch) = outputs(3)
        for stages in ((ASSEMBLE, FACTOR, POST) if split else (ALL,)):
            solve(ws, K, f_s, geo, stages, p, res, batch)
        assert guards_intact(pb) and guards_intact(rb) and guards_intact(bb)
        runs.append((ws.band, ws.rhs, p, res, batch))
    for a, b in zip(*runs):
        assert bits_equal(a, b)


# ---- tier 2: per-element bounds at every geometry ---------------------------------------------------------------------
def run_stages(K, f_s, geo):
    """the three stages as separate calls: dict of the assembled band / rhs, L / y, p, res, batch"""
    B = K.shape[0]
    ws = Workspace(B)
    out = {}
    solve(ws, K, f_s, geo, ASSEMBLE)
    out['band'], out['rhs'] = ws.band.clone(), ws.rhs.clone()
    ws2 = Workspace(B)
    solve(ws2, K, f_s, {**geo, 'reverse_dy': not geo['reverse_dy']}, ASSEMBLE)
    assert bits_equal(ws2.band, ws.band) and bits_equal(ws2.rhs, ws.rhs)
    del ws2
    solve(ws, None, None, geo, FACTOR)
    out['L'], out['y'] = ws.band.clone(), ws.rhs.clone()
    (pb, p), (rb, res), (bb, batch) = outputs(B)
    solve(ws, K, f_s, geo, POST, p, res, batch)
    assert guards_intact(pb) and guards_intact(rb) and guards_intact(bb)
    out['p'], out['res'], out['batch'] = p.view(B, N), res, batch.view(B, 2, N)
    return out


@pytest.mark.parametrize('geo', GEOMETRIES, ids=geo_id)
def test_stages_within_bounds(geo, kgen):
    K = realistic_K(kgen, 100)
    B = K.shape[0]
    w = dev(DO.weights(geo['pixels_at_boundary'], geo['domain_length']))
    worst = {}

    def keep(k, q):
        worst[k] = max(worst.get(k, 0.), q)
    for sname, f_s in sources(geo).items():
        o = run_stages(K, f_s, geo)
        Kh, fh = K.cpu().numpy(), f_s.cpu().numpy()
        for b in range(B):
            band, band_a, rhs, rhs_a = assembly_ref(Kh[b], fh, geo)
            keep('band', asm_ratio(o['band'][b], band, band_a))
            keep('rhs', asm_ratio(o['rhs'][b], rhs, rhs_a))
            q_n, q_y = factor_ratios(o['L'][b], o['y'][b], o['band'][b], o['rhs'][b])
            keep('L', q_n)
            keep('y', q_y)
            q_x, q_w, _ = post_ratios(o['L'][b], o['y'][b], o['p'][b], w)
            keep('p', q_x)
            keep('w^T p', q_w)
            ph = o['p'][b].cpu().numpy()
            ref, scale = res_ref(Kh[b], fh, ph, geo)
            keep('res', res_ratio(o['res'][b].item(), ref, scale))
            assert bits_equal(o['batch'][b, 0], o['p'][b].float()) and bits_equal(o['batch'][b, 1], K[b].float())
            if sname == 'source' and b < 2:                 # end to end on the KLE fields
                p_or, res_or = DO.solve_banded(Kh[b], fh, **geo)
                keep('p vs host solve', np.abs(ph - p_or).max() / (E2E_P[geo['domain_length']] * np.abs(p_or).max()))
                keep('res vs host solve', abs(o['res'][b].item() - res_or) / (1e-4 * res_or))
    for k, q in worst.items():
        note(TAG, f'{geo_id(geo)} {k}', q)
    assert max(worst.values()) <= 1.0, worst


# ---- edited references ----------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def default_run(kgen):
    """sample 0 (a KLE field) at the default geometry with the dense random source (the reference's source is symmetric
    under x <-> y, so a transposed source would go unseen with it)"""
    K = realistic_K(kgen, 300)[:1]
    f_s = sources(DEFAULT)['dense']
    return K, f_s, run_stages(K, f_s, DEFAULT)


def test_edited_assembly_references_are_rejected(default_run, monkeypatch):
    K, f_s, o = default_run
    Kh, fh = K[0].cpu().numpy(), f_s.cpu().numpy()
    band, band_a, rhs, rhs_a = assembly_ref(Kh, fh, DEFAULT)
    A, BC = DO.operators(Kh, **DEFAULT)
    q = {}
    unpinned = band.copy()
    unpinned[0, 0] /= 2
    q['pin not doubled'] = asm_ratio(o['band'][0], unpinned, band_a)
    q['y = P-1 BC rows dropped'] = asm_ratio(o['band'][0], DO.to_band(DO.pinned_normal(A, BC[:3 * P])), band_a)
    q['rhs of the transposed f_s'] = asm_ratio(o['rhs'][0], A.T @ fh.reshape(P, P).T.reshape(-1), rhs_a)
    # the one-sided d1 at x = P-1 with the sign of the x = 0 end.  Flipped everywhere it is an exact symmetry of N and
    # A^T f_s (K_0 D0 and the BC rows' squares keep their sign), so the edit that changes the answer flips it where the
    # kernel forms K_0 = D0 K alone: -K_0 D0 at those rows becomes +K_0 D0
    h0, _ = DO.geometry(**DEFAULT)
    D0 = sp.kron(DO._d1(P, h0), sp.identity(P)).tocsr()
    last = (np.arange(N) // P == P - 1).astype(np.float64)
    A_flip = A + 2 * sp.diags(last * (D0 @ Kh)) @ D0
    q['d1 of K at x = P-1 with the x = 0 sign'] = asm_ratio(o['band'][0], DO.to_band(DO.pinned_normal(A_flip, BC)),
                                                            band_a)
    with monkeypatch.context() as m:
        geometry = DO.geometry
        m.setattr(DO, 'geometry', lambda pixels_at_boundary=True, reverse_dy=True, domain_length=1.:
                  geometry(False, reverse_dy, domain_length))
        q['h = L/P under pixels_at_boundary'] = asm_ratio(o['band'][0], DO.normal_band(Kh, fh, **DEFAULT)[0], band_a)
    for k, v in q.items():
        note(TAG, f'mutant {k}', v)
    assert min(q.values()) > 1, q


def test_edited_factor_and_post_references_are_rejected(default_run):
    K, f_s, o = default_run
    L = dgen_band_to_dense(o['L'][0])
    N_full = symmetric(dgen_band_to_dense(o['band'][0]))
    q = {}
    # one trailing-update term L_ik L_jk missing in the last block column (rows n-2, n-1; k outside that block)
    i, j = N - 1, N - 2
    k = int((L[i, :N - 16] * L[j, :N - 16]).abs().argmax())
    Nm = N_full.clone()
    Nm[i, j] -= L[i, k] * L[j, k]
    Nm[j, i] = Nm[i, j]
    q['trailing-update term missing'] = factor_ratios(o['L'][0], o['y'][0], None, o['rhs'][0], Nm)[0]
    # the farthest term (d = 3P+3) dropped from the back substitution
    Lm = o['L'][0].clone()
    Lm[:, BW] = 0
    w = dev(DO.weights(True, 1.))
    q['d = 3P+3 dropped from the back substitution'] = post_ratios(Lm, o['y'][0], o['p'][0], w)[0]
    # the shift taken with mean weights under the trapezoid flag
    _, _, s = post_ratios(o['L'][0], o['y'][0], o['p'][0], w)
    x = o['p'][0] + s
    q['mean-weight shift'] = post_ratios(o['L'][0], o['y'][0], x - x.mean(), w)[1]
    # res without the integral row
    ph = o['p'][0].cpu().numpy()
    ref, scale = res_ref(K[0].cpu().numpy(), f_s.cpu().numpy(), ph, DEFAULT, rows=N + 4 * P)
    q['res without the integral row'] = res_ratio(o['res'][0].item(), ref, scale)
    for k_, v in q.items():
        note(TAG, f'mutant {k_}', v)
    assert min(q.values()) > 1, q


# ---- plan coverage ----------------------------------------------------------------------------------------------------------
def test_launch_plan_coverage():
    """the launch arithmetic of darcy_gen.cu, restated: kle on grid (N / 256, B), so B = 65535 (a row above) is the
    grid.y limit; assemble on (P / 2, B) with two x-lines of 64 rows per 128-thread CTA; factor and post one CTA per
    sample, the factor with 105 resident 16 x 16 blocks, the window's right-hand side, two column buffers and two slot
    tables in shared memory: 218,656 B, more than half an SM's 228 KB, so one CTA per SM and the B = 133 row runs a
    second wave"""
    NB, WIN, NBLK = 16, 14, N // 16
    NSLOT = WIN * (WIN + 1) // 2
    smem = NSLOT * NB * NB * 8 + WIN * NB * 8 + 2 * NB * 8 + 2 * WIN * WIN * 4
    assert smem == 218656 and 2 * smem > 228 * 1024
    assert 133 > sms()
    assert N % 256 == 0 and P % 2 == 0 and (BW + NB - 1) // NB + 1 == WIN
    # the slot table of the factor, step by step: the live blocks (I, K), J <= K <= I <= J + 13, hold distinct slots;
    # over the last 14 steps no block row enters and the window drains
    T = [[-1] * WIN for _ in range(WIN)]
    s = 0
    for I in range(WIN):
        for K in range(I + 1):
            T[I][K] = s
            s += 1
    drained = 0
    for J in range(NBLK):
        live = [(I, K) for K in range(J, min(J + WIN, NBLK)) for I in range(K, min(J + WIN, NBLK))]
        slots = [T[I % WIN][K % WIN] for I, K in live]
        assert len(set(slots)) == len(slots) and all(0 <= x < NSLOT for x in slots), J
        drained += J + WIN >= NBLK
        jm = J % WIN
        Tn = [row[:] for row in T]
        for t in range(WIN):
            Tn[jm][(J + 1 + t) % WIN] = T[(J + t) % WIN][jm]
        T = Tn
    assert drained == WIN
