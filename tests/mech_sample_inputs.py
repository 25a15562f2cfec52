"""Inputs of tests/golden/mechanics_sample_loop.pt, rebuilt rather than stored so that the fixture stays small.  TEST
INFRASTRUCTURE ONLY; plain torch on the CPU, imported both by the mech_sample recipe of oracle/make_golden.py (which runs
the reference) and by the tests.

* `conditioning_batch()`: the B = 2 conditioning fields, boundary conditions and data densities of the fixture.
* `replay_draws(gd, mode)`: the reference loop's draws regenerated from the fixture's seed on the CPU generator, checked
  against the fixture's per-draw checksums, so a generator mismatch is reported as such and not as a parity failure.
* `binarised_designs(B, seed)`: binarised densities under four support / load cases, the systems the evaluation solve
  is checked on."""
import torch

B = 2
SAMPLE = 4096            # elements kept of each large output (oracle.pidm_oracle.golden_sample)


def conditioning_batch():
    """(conditioning [B,3,65,65], bcs [B,4,65,65], rho_simp [B,64,64]): a clamped left edge for both samples, a downward
    load on the right edge (sample 0), rollers on the bottom edge and a horizontal load on the top edge (sample 1)."""
    i64 = torch.arange(64, dtype=torch.float32) / 63
    Xe, Ye = torch.meshgrid(i64, i64, indexing='ij')
    rho = torch.stack([(0.55 + 0.45 * torch.sin(3.1 * Xe + 0.4) * torch.cos(2.3 * Ye)).clamp(0.05, 1.0),
                       (0.5 + 0.5 * torch.cos(2.0 * Xe - 0.3) * torch.sin(3.7 * Ye + 0.2)).clamp(0.05, 1.0)])
    bcs = torch.zeros(B, 4, 65, 65)
    bcs[:, 0, :, 0] = 1.
    bcs[:, 1, :, 0] = 1.
    bcs[0, 3, 30:34, 64] = -0.25
    bcs[1, 1, 64, :] = 1.
    bcs[1, 2, 0, 40:44] = 0.25
    g = torch.Generator().manual_seed(31)
    cond = torch.rand(B, 3, 65, 65, generator=g)
    cond[:, 0] = torch.tensor([0.45, 0.5])[:, None, None]   # volume-fraction plane
    return cond, bcs, rho


def draws(seed, n_steps, mode):
    """The reference loop's draws after torch.manual_seed(seed): x_T [B,3,65,65], then per step, in 'sample' mode, the
    DDIM walk's [B,3,64,64] draw before the posterior's z [B,3,65,65].  Returns (x_T, z [n,B,3,65,65], ddim [n,...] or
    None)."""
    torch.manual_seed(seed)
    x_T = torch.randn(B, 3, 65, 65)
    zs, ddim = [], []
    for _ in range(n_steps):
        if mode == 'sample':
            ddim.append(torch.randn(B, 3, 64, 64))
        zs.append(torch.randn(B, 3, 65, 65))
    return x_T, torch.stack(zs), (torch.stack(ddim) if ddim else None)


def checksums(x_T, zs, ddim):
    parts = [x_T[None], zs] + ([] if ddim is None else [ddim])
    return torch.cat([p.double().sum(dim=tuple(range(1, p.ndim))) for p in parts])


def replay_draws(gd, mode):
    x_T, zs, ddim = draws(int(gd['seed']), int(gd['n_steps']), mode)
    assert torch.equal(checksums(x_T, zs, ddim), gd[f'{mode}_noise_checksum']), \
        'CPU generator does not reproduce the draws of the golden run (torch version mismatch?)'
    return x_T, zs, ddim


def inputs(gd):
    """(conditioning, bcs, solution) of the fixture; the rebuilt inputs are checked against the stored checksums"""
    cond, bcs, rho = conditioning_batch()
    assert torch.equal(torch.stack([cond.double().sum(), bcs.double().sum(), rho.double().sum()]), gd['input_checksum'])
    assert torch.equal(gd['solution'][:, 2, :-1, :-1], rho)
    return cond, bcs, gd['solution']


def binarised_designs(B, seed):
    """B designs with rho in {1e-3, 1} (smooth random fields thresholded) under different supports and loads"""
    g = torch.Generator().manual_seed(seed)
    i = torch.arange(64, dtype=torch.float32) / 63
    X, Y = torch.meshgrid(i, i, indexing='ij')
    rho = torch.empty(B, 64, 64)
    bcs = torch.zeros(B, 4, 65, 65)
    for b in range(B):
        f = torch.zeros(64, 64)
        for _ in range(5):
            a, kx, ky, ph = torch.randn(1, generator=g), *torch.randint(1, 5, (2,), generator=g), torch.rand(1, generator=g) * 6
            f += a * torch.sin(3.1 * kx * X + ph) * torch.cos(3.1 * ky * Y + 0.5 * ph)
        thr = torch.quantile(f.reshape(-1), 0.3 + 0.3 * torch.rand(1, generator=g).item())
        rho[b] = torch.where(f > thr, torch.ones_like(f), torch.full_like(f, 1e-3))
        case = b % 4
        if case in (0, 1):                                # cantilever: clamped left edge
            bcs[b, 0, :, 0] = 1.
            bcs[b, 1, :, 0] = 1.
        else:                                             # bridge: pinned bottom corners
            bcs[b, :2, 64, :3] = 1.
            bcs[b, 1, 64, 62:] = 1.
        row = int(torch.randint(8, 56, (1,), generator=g))
        if case == 0:
            bcs[b, 3, row:row + 3, 64] = -1. / 3
        elif case == 1:
            bcs[b, 2, 0, 20 + row // 2] = 0.5
            bcs[b, 3, 64, 60] = -0.5
        else:
            bcs[b, 3, 0, row - 4:row + 4] = -1. / 8
    return rho, bcs
