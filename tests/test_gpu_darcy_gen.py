"""Darcy data generation on the GPU (csrc/darcy_gen.cu, darcy_data_generation.py): the pressure solve against the
unmodified reference's output and the host oracle, the KLE product, consistency with the training residual kernel,
determinism and batch independence, guard regions, TrainEngine fed by generated batches, and the CSV round trip."""
import math

import numpy as np
import pytest
import torch

from oracle import darcy_gen_oracle as DO

pytestmark = pytest.mark.gpu
DEV = 'cuda'
P = 64
N = P * P
U = 2.0 ** -24
GUARD = 1024


@pytest.fixture(scope='module')
def fx(golden):
    return golden('darcy_gen.pt')


@pytest.fixture(scope='module')
def gen(fx):
    from physicsinformeddiffusionmodels_b200.darcy_data_generation import DarcyDataGenerator
    return DarcyDataGenerator()


def _close_p(p, p_ref, tol=1e-5):
    p, p_ref = np.asarray(p), np.asarray(p_ref)
    return np.abs(p - p_ref).max() <= tol * np.abs(p_ref).max()


def test_fixture_solve(gen, fx):
    p, res = gen.solve_pressure(fx['K'].to(DEV))
    p, res = p.cpu().numpy(), res.cpu().numpy()
    w = fx['int_cond'].numpy()
    for b in range(len(fx['seed'])):
        assert _close_p(p[b], fx['p'][b].numpy())
        assert abs(res[b] - fx['res'][b].item()) <= 1e-4 * fx['res'][b].item()
        assert abs(w @ p[b]) <= 64 * 2.0 ** -52 * (np.abs(w) @ np.abs(p[b]))


@pytest.mark.parametrize('B', [1, 3, 64, 257])
def test_fresh_fields_match_oracle(gen, B):
    K, p, res, seeds = gen.generate(range(1000 + B, 1000 + 2 * B))
    K, p, res = K.cpu().numpy(), p.cpu().numpy(), res.cpu().numpy()
    assert np.isfinite(p).all() and np.isfinite(res).all()
    check = sorted({0, B // 2, B - 1})
    for b in check:
        p_or, res_or = DO.solve_banded(K[b])
        assert _close_p(p[b], p_or), b
        assert abs(res[b] - res_or) <= 1e-4 * res_or, b
    if B == 3:
        # The normal equations square cond(M) ~ 1e7, so their rounding error reaches ~1e-5 max|p| on some fields (seed
        # 1005: 1.1e-5 on an H100; the host's banded solve of the same equations lands 1e-6 .. 3e-6 away depending on the
        # LAPACK build).  The bound is the method's, with margin; the res values agree to 1e-4.
        for b in (0, 2):
            p_ls, res_ls = DO.solve_lstsq(K[b])
            dev = np.abs(p[b] - p_ls).max() / np.abs(p_ls).max()
            assert dev <= 3e-5, (b, dev)
            assert abs(res[b] - res_ls) <= 1e-4 * res_ls, b


def test_kle(gen, fx):
    ref = fx['eigenvalues'].numpy()
    assert np.abs(gen.eigenvalues - ref).max() <= 1e-10 * np.abs(ref).max()
    z = gen.z_for_seeds([5, 6, 7, 8, 9])
    K = gen.permeability(z).cpu().numpy()
    phi_s = (np.sqrt(gen.eigenvalues)[None, :] * gen.eigenvectors)              # [N, q]
    K_ref = np.exp(z.cpu().numpy() @ phi_s.T)
    assert np.abs(K - K_ref).max() <= 1e-12 * np.abs(K_ref).max()
    # the reference's KLE_expansion on the generator's own eigenpairs
    from physicsinformeddiffusionmodels_b200.darcy_data_generation import KLE_expansion
    G, z0 = KLE_expansion(gen.eigenvalues, gen.eigenvectors, 64, N, seed=5)
    assert np.array_equal(z0, z[0].cpu().numpy())
    assert np.abs(K[0] - np.exp(G)).max() <= 1e-12 * np.abs(K[0]).max()


def test_consistent_with_training_residual(gen):
    """the fp32 batch through pidm_darcy_residual_fwd: eq_0 and the BC channels are the fp64 rows of M p - b"""
    from physicsinformeddiffusionmodels_b200.residuals_darcy import ResidualsDarcy
    from physicsinformeddiffusionmodels_b200._lib import call, stream
    B = 6
    K, p, _, _ = gen.generate(range(300, 300 + B))
    batch = next(gen.batches(B, seed0=300))
    assert torch.equal(batch[:, 0].reshape(B, -1), p.float())
    assert torch.equal(batch[:, 1].reshape(B, -1), K.float())
    rd = ResidualsDarcy(model=None, fd_acc=2, pixels_per_dim=P, pixels_at_boundary=True, reverse_d1=True, device=DEV)
    r = torch.empty(B, N, 3, device=DEV)
    call('pidm_darcy_residual_fwd', batch, rd.f_s_flat, r, B, P, 1.0, 1, 1, stream())
    r = r.double().cpu().numpy()
    K, p = K.cpu().numpy(), p.cpu().numpy()
    idx = np.arange(N).reshape(P, P)
    worst = 0.
    for b in range(B):
        A, BC = DO.operators(K[b])
        Aabs, _ = DO.operators(K[b], absolute=True)
        eq0 = A @ p[b] - DO.source()
        bound = 16 * U * (Aabs @ np.abs(p[b]) + np.abs(DO.source())) + 1e-30
        worst = max(worst, (np.abs(r[b, :, 0] - eq0) / bound).max())
        bc = BC @ p[b]
        bc_bound = 16 * U * (abs(BC) @ np.abs(p[b])) + 1e-30
        # BC rows of M in order: x = 0, x = P-1 (channel 1), y = 0, y = P-1 (channel 2)
        for k, (ch, rows) in enumerate(((1, idx[0, :]), (1, idx[-1, :]), (2, idx[:, 0]), (2, idx[:, -1]))):
            sl = slice(k * P, (k + 1) * P)
            worst = max(worst, (np.abs(r[b, rows, ch] - bc[sl]) / bc_bound[sl]).max())
    assert worst <= 1.0, worst


def test_deterministic_and_batch_independent(gen):
    seeds = list(range(5000, 5064))
    K1, p1, r1, _ = gen.generate(seeds)
    K2, p2, r2, _ = gen.generate(seeds)
    assert torch.equal(K1, K2) and torch.equal(p1, p2) and torch.equal(r1, r2)
    for i in (0, 17, 63):
        Ka, pa, ra, _ = gen.generate([seeds[i]])
        assert torch.equal(Ka[0], K1[i]) and torch.equal(pa[0], p1[i]) and torch.equal(ra[0], r1[i])


def test_guards(gen):
    from physicsinformeddiffusionmodels_b200._lib import call, stream
    B = 3
    K = gen.permeability(gen.z_for_seeds([1, 2, 3]))

    def guarded(n, dtype):
        buf = torch.full((n + 2 * GUARD,), float('nan'), device=DEV, dtype=dtype)
        return buf, buf[GUARD:GUARD + n]
    need = call('pidm_darcy_gen_workspace_bytes', B, P)
    ws = torch.full((need + 2 * GUARD * 8,), 0xA5, dtype=torch.uint8, device=DEV)
    pb, p = guarded(B * N, torch.float64)
    rb, res = guarded(B, torch.float64)
    bb, batch = guarded(B * 2 * N, torch.float32)
    kb, Kg = guarded(B * N, torch.float64)
    call('pidm_darcy_gen_kle', gen.phi_s, gen.z_for_seeds([1, 2, 3]), Kg, B, 64, P, stream())
    call('pidm_darcy_gen_solve', K, gen.f_s, p, res, batch, ws[GUARD * 8:], need, B, P, 1.0, 1, 1, 7, stream())
    torch.cuda.synchronize()
    for buf in (pb, rb, bb, kb):
        assert bool(torch.isnan(buf[:GUARD]).all() and torch.isnan(buf[-GUARD:]).all())
    assert bool((ws[:GUARD * 8] == 0xA5).all() and (ws[GUARD * 8 + need:] == 0xA5).all())
    assert torch.equal(Kg, K.reshape(-1))
    p_ref, r_ref = gen.solve_pressure(K)
    assert torch.equal(p.reshape(B, N), p_ref) and torch.equal(res, r_ref)


def test_train_engine_on_generated_batches(gen):
    from physicsinformeddiffusionmodels_b200 import ops
    from physicsinformeddiffusionmodels_b200.engine import TrainEngine
    from study import build_darcy
    ops.set_precision('bf16')
    model, diff, rd = build_darcy()
    eng = TrainEngine(model, diff, rd, use_graph=True)
    it = gen.batches(32, seed0=10)
    r_gen = []
    for _ in range(5):
        x0 = next(it)
        loss, _, _ = eng.step(x0)
        assert math.isfinite(loss.item())
        r_gen.append(rd.compute_residual(x0, pass_through=True)['residual'].abs().mean().item())
    torch.cuda.synchronize()
    assert eng._graph is not None
    r_randn = rd.compute_residual(torch.randn(32, 2, P, P, device=DEV), pass_through=True)['residual'].abs().mean()
    assert max(r_gen) < 1e-2 and r_randn.item() > 1e2, (r_gen, r_randn.item())


def test_csv_round_trip(gen, tmp_path):
    from physicsinformeddiffusionmodels_b200.data_utils import Dataset
    K, p, res, seeds = gen.write_csv(tmp_path, 5, seed0=40, batch_size=2)
    ds = Dataset((tmp_path / 'p_data.csv', tmp_path / 'K_data.csv'), use_double=True)
    assert ds.data.shape == (5, 2, P, P)
    # the files hold the shortest round-trip decimal of every value; pandas' default parser (which Dataset uses) is not
    # correctly rounded and lands within about an ulp of 1 in absolute terms, the round-trip parser is exact
    for got, ref in ((ds.data[:, 0].reshape(5, -1), p.cpu()), (ds.data[:, 1].reshape(5, -1), K.cpu())):
        assert (got - ref).abs().max() <= 4e-16 * max(1., ref.abs().max().item())
    import pandas as pd

    def exact(name):
        return pd.read_csv(tmp_path / name, header=None, float_precision='round_trip').to_numpy()
    assert np.array_equal(exact('seeds.csv')[:, 0], np.arange(40, 45))
    assert np.array_equal(exact('res_data.csv')[:, 0], res.cpu().numpy())
    assert np.array_equal(exact('p_data.csv'), p.cpu().numpy()) and np.array_equal(exact('K_data.csv'), K.cpu().numpy())


# ---- a second geometry: pixel centres, h = L / P, the plain mean, reverse_dy = False -----------------------------------
@pytest.fixture(scope='module')
def fxg(golden):
    return {k[len('geometry_'):]: v for k, v in golden('darcy_gen.pt').items() if k.startswith('geometry_')}


def _geometry(fxg):
    return dict(pixels_at_boundary=bool(fxg['pixels_at_boundary']), reverse_dy=bool(fxg['reverse_dy']),
                domain_length=float(fxg['domain_length']))


def test_fixture_solve_at_another_geometry(gen, fxg):
    from physicsinformeddiffusionmodels_b200.darcy_data_generation import DarcyDataGenerator
    geo = _geometry(fxg)
    g = DarcyDataGenerator(eigenpairs=(gen.eigenvalues, gen.eigenvectors), **geo)
    assert np.array_equal(g.f_s_np, fxg['f_s'].numpy())
    assert np.array_equal(g.int_cond.reshape(-1), fxg['int_cond'].numpy())
    p, res = g.solve_pressure(fxg['K'].to(DEV))
    p, res = p.cpu().numpy(), res.cpu().numpy()
    for b in range(len(fxg['seed'])):
        assert _close_p(p[b], fxg['p'][b].numpy())
        assert abs(res[b] - fxg['res'][b].item()) <= 1e-4 * fxg['res'][b].item()


@pytest.mark.parametrize('pab, dl', [(False, 2.), (True, 0.3)])
def test_generate_sample_infers_the_geometry(gen, pab, dl):
    """the reference's argument tuple carries the geometry as d0 and the shape of int_cond: generate_sample must solve
    at the geometry that tuple describes, bit for bit what DarcyDataGenerator at that geometry computes"""
    from physicsinformeddiffusionmodels_b200 import darcy_data_generation as G
    shape, q = (P, P), gen.q
    d0 = dl / (P - 1) if pab else dl / P
    grid = G.uniform_points_pixelwise(P, dl, pab)
    f_s = G.create_f_s(grid[:, 0], grid[:, 1])
    int_cond = G.create_int_cond(pab, shape, d0)
    args = (17, gen.eigenvalues, gen.eigenvectors, q, P, shape, 2, d0, d0, f_s, int_cond, *G.create_boundary_idcs(shape),
            False)
    K, p, res, seed = G.generate_sample(args)
    g = G.DarcyDataGenerator(domain_length=dl, reverse_dy=False, pixels_at_boundary=pab,
                             eigenpairs=(gen.eigenvalues, gen.eigenvectors))
    K_ref, p_ref, res_ref, seeds = g.generate([17])
    assert seed == 17 == int(seeds[0])
    assert np.array_equal(K, K_ref[0].cpu().numpy()) and np.array_equal(p, p_ref[0].cpu().numpy())
    assert res == res_ref[0].item()
    # and not the default geometry's answer
    assert not np.array_equal(p, gen.solve_pressure(K_ref)[0][0].cpu().numpy())
