"""Helpers shared by the tests: relative error, NaN-guarded output buffers, the per-element bound predicate of the fp32
Darcy kernels against their fp64 references, the seeding, launch, dtype and |err| / bound helpers of the census files,
and the fp64 reference of the implicit-GEMM convolution contract that both convolution census files replay."""
import math
import zlib

import torch
import torch.nn.functional as F

P = 64
U = 2.0 ** -24
C_BOUND = 16            # |y - r| <= C_BOUND * 2^-24 * A: a handful of fp32 roundings along each stencil / product chain
GUARD = 1024            # NaN guard elements on each side of every output

DTYPES = [torch.bfloat16, torch.float32]
CODE = {torch.float32: 0, torch.bfloat16: 1}                      # the dtype code of the C ABI
DTYPE = {c: t for t, c in CODE.items()}
NAME = {torch.bfloat16: 'bf16', torch.float32: 'fp32'}
RND = {torch.bfloat16: 2.0 ** -8, torch.float32: 2.0 ** -24}      # one rounding to the type, relative


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


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def gen(key):
    """a device generator: an int is the seed, anything else seeds by the crc32 of its repr"""
    seed = key if isinstance(key, int) else zlib.crc32(repr(key).encode())
    return torch.Generator(device='cuda').manual_seed(seed)


def call_sync(name, *a):
    """one C-ABI call on the package's stream, synchronized"""
    from physicsinformeddiffusionmodels_b200._lib import call, stream
    call(name, *a, stream())
    torch.cuda.synchronize()


def ratio(err, bound):
    """worst |err| / bound; a non-finite error (an unwritten NaN sentinel) counts as infinitely bad"""
    q = err / bound.clamp_min(1e-300)
    q = torch.where(torch.isfinite(q), q, torch.full_like(q, math.inf))
    return q.max().item() if q.numel() else 0.0


def ratios(out, r, b, sl=slice(None)):
    """worst |out - r| / bound of every output in the reference (an unwritten NaN counts as inf)"""
    return {k: ratio((out[k][sl].double() - r[k]).abs(), b[k]) for k in r}


def rounded(r, dtype, act):
    """a reference as a correct kernel would return it: the outputs in `act` rounded to the activation type, the rest to
    fp32"""
    return {k: v.to(dtype if k in act else torch.float32) for k, v in r.items()}


def note(tag, what, q):
    """prints one worst |err| / bound, prefixed by the census tag"""
    print(f'[{tag}] {what} |err|/bound {q:.4g}')


def note_all(tag, what, rs):
    for k, q in rs.items():
        note(tag, f'{what} {k}', q)


def assert_ok(rs, where):
    assert max(rs.values()) <= 1.0, f'{where}: worst |err| / bound = {rs}'


def check(tag, what, y, r, bound):
    """notes and asserts the worst |y - r| / bound (y on the device, r and bound fp64)"""
    q = ratio((y.double() - r).abs(), bound)
    note(tag, what, q)
    assert q <= 1.0, f'{what}: worst |err| / bound = {q:.4g}'


def conv_ref(x, wp, bias, res, k):
    """fp64 y of the implicit-GEMM convolution contract of include/pidm.h (pidm_conv2d_simt, pidm_conv2d_tc_general):
    y = sum A(m,k) Wp[n,k] (+ bias) (+ residual), NHWC, for k = (B, H, W, Cin, Ho, Wo, Cout, KH, KW, stride, pad,
    transposed, ...)"""
    B, H, W, Cin, Ho, Wo, Cout, KH, KW, s, p, tr = k[:12]
    w4 = wp.view(Cout, KH, KW, Cin)
    xn = x.permute(0, 3, 1, 2)
    if not tr:
        y = F.conv2d(xn, w4.permute(0, 3, 1, 2), stride=s, padding=p)
    else:                           # gather at ((oh + p - r) / s, ...) == ConvTranspose with w[c][n][r][q] = Wp[n][r][q][c]
        op = Ho - ((H - 1) * s - 2 * p + KH)
        y = F.conv_transpose2d(xn, w4.permute(3, 0, 1, 2), stride=s, padding=p, output_padding=op)
    y = y.permute(0, 2, 3, 1)
    if bias is not None:
        y = y + bias
    if res is not None:
        y = y + res
    return y


# ---- bilinear resize (align_corners=False, no antialias), shared by the physics and mechanics-evaluation census files ---
def resize_src_index(n_out, n_in, clamp_hi=None):
    """bil_src in fp64: source rows i0, i1, the weight of i1 and the error of bil_src's fp32 source coordinate
    s = (o + 0.5) * fl(in / out) - 0.5: each of fl(in / out), the product and the subtraction rounds once, so
    |s32 - s| <= 2^-24 (3 (o + 0.5) in / out + 1).  clamp_hi: the largest i0 (the mutant clamps one pixel early)."""
    o = torch.arange(n_out, dtype=torch.float64)
    s = ((o + 0.5) * (n_in / n_out) - 0.5).clamp_min(0)
    i0 = s.floor().clamp_max(n_in - 1 if clamp_hi is None else clamp_hi).long()
    i1 = torch.where(i0 < n_in - 1, i0 + 1, i0)
    return i0, i1, s - i0, U * (3 * (o + 0.5) * n_in / n_out + 1)


def resize_bounds(x, n_out):
    """(C-free part A, coordinate term) of the forward bound: |y - r| <= C u A + (e_h + e_w) D, D = twice the largest
    |x| on source rows / columns i0 - 1 .. i0 + 1 (a coordinate error e moves y by at most e times the largest
    neighbour difference, also when it moves s across a pixel boundary)"""
    n_in = x.shape[-1]
    A = F.interpolate(x.abs()[:, None], size=(n_out, n_out), mode='bilinear', align_corners=False)[:, 0]
    i0, _, _, e = resize_src_index(n_out, n_in)
    M = F.max_pool2d(x.abs()[:, None], 3, stride=1, padding=1)[:, 0]
    D = 2 * M[:, i0][:, :, i0]
    return A, (e[:, None] + e[None, :]) * D


# ---- known-answer operands of the Darcy data generator (tests/test_gpu_darcy_gen_replay.py; their exactness is
# checked on the host in tests/test_oracle_darcy_gen.py) ----------------------------------------------------------------
DGEN_BW = 3 * P + 3                 # half-bandwidth of the normal equations; the row-band layout holds d = 0 .. DGEN_BW
# spacing exactly 1 (twice) and 2^-6: every A coefficient, N = M^T M entry and A^T f_s of the dyadic operands below is
# exact in fp64, so the kernel's assembly must equal the oracle's bit for bit
DGEN_EXACT_GEOMETRIES = [dict(pixels_at_boundary=True, reverse_dy=True, domain_length=63.),
                         dict(pixels_at_boundary=False, reverse_dy=True, domain_length=64.),
                         dict(pixels_at_boundary=False, reverse_dy=True, domain_length=1.)]


def dgen_dyadic_K(B, g, device='cuda'):
    """K = k / 16, k in [16, 256): [B, P*P] fp64"""
    return torch.randint(16, 256, (B, P * P), generator=g, device=device).double() / 16


def dgen_dyadic_source(g, device='cuda'):
    """a dense integer source in [-8, 8]: [P*P] fp64"""
    return torch.randint(-8, 9, (P * P,), generator=g, device=device).double()


def dgen_dyadic_factor(B, g, device='cuda', fill=float('nan')):
    """L0 in row-band layout [B, P*P, DGEN_BW + 1]: diagonal 4, the other band entries in {-2..2} / 256 and `fill` where
    the column r - d is negative.  L0 L0^T is exact in fp64 and diagonally dominant, so its Cholesky factor is L0 in
    any order of operations"""
    n = P * P
    L = torch.randint(-2, 3, (B, n, DGEN_BW + 1), generator=g, device=device).double() / 256
    L[:, :, 0] = 4.
    r = torch.arange(n, device=device)[:, None]
    d = torch.arange(DGEN_BW + 1, device=device)[None, :]
    L[:, (r - d < 0)] = fill
    return L


def dgen_band_to_dense(band):
    """lower-triangular dense [P*P, P*P] from one row-band matrix [P*P, DGEN_BW + 1] (entries of negative column
    ignored)"""
    n = band.shape[0]
    r = torch.arange(n, device=band.device)[:, None].expand(n, DGEN_BW + 1)
    c = r - torch.arange(DGEN_BW + 1, device=band.device)[None, :]
    ok = c >= 0
    dense = torch.zeros(n, n, dtype=band.dtype, device=band.device)
    dense[r[ok], c[ok]] = band[ok]
    return dense


def dgen_dense_to_band(dense, fill=0.):
    """row-band layout of the lower triangle of dense [P*P, P*P]: band[r, d] = dense[r, r - d], `fill` where r < d"""
    n = dense.shape[0]
    r = torch.arange(n, device=dense.device)[:, None]
    c = r - torch.arange(DGEN_BW + 1, device=dense.device)[None, :]
    band = dense[r, c.clamp_min(0)]
    return torch.where(c >= 0, band, torch.full_like(band, fill))
