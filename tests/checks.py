"""Helpers shared by the tests: relative error, NaN-guarded output buffers and the per-element bound predicate of the
fp32 Darcy kernels against their fp64 references."""
import torch

P = 64
U = 2.0 ** -24
C_BOUND = 16            # |y - r| <= C_BOUND * 2^-24 * A: a handful of fp32 roundings along each stencil / product chain
GUARD = 1024            # NaN guard elements on each side of every output


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def guarded(n, dtype=torch.float32):
    """(buffer, its middle n elements) on the GPU, every element NaN"""
    buf = torch.full((n + 2 * GUARD,), float('nan'), device='cuda', dtype=dtype)
    return buf, buf[GUARD:GUARD + n]


def guards_intact(buf):
    return bool(torch.isnan(buf[:GUARD]).all() and torch.isnan(buf[-GUARD:]).all())


def within(y, r, A, c=C_BOUND):
    return bool(((y.double() - r).abs() <= c * U * A).all())


def fields(B, seed, device='cpu'):
    """fp64 Darcy fields [B,2,P,P] (p normal, K log-normal) that fp32 represents exactly"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 2, P, P, generator=g, dtype=torch.float64)
    x[:, 1] = torch.exp(0.5 * x[:, 1])
    return x.float().double().to(device)
