"""Darcy training data on the GPU (reference src/darcy_data_generation.py).

`DarcyDataGenerator` draws log-normal permeability fields K = exp(G) from the Karhunen-Loeve expansion of the
exponential covariance exp(-|x - x'| / l) and solves the reference's least-squares Darcy problem for the pressure p:
the operator A = -K D00 - K_0 D0 - K D11 - K_1 D1 with the source f_s, 4P Neumann rows and the integral condition
w^T p = 0 (reference :123-165).  The eigenpairs are set-up (fp64 eigensolver on the host, once per instance); the KLE
product, the banded normal-equation assembly, the banded fp64 Cholesky solve, the constant shift and the residual are
the libpidm kernels of csrc/darcy_gen.cu.  There is no CPU path.

Seeds: the z of a sample is `numpy.random.RandomState(seed).standard_normal(q)`, which is what the reference's
`np.random.seed(seed); norm.rvs(size=q)` draws, so z[i] depends on seeds[i] alone.  The eigenvector basis of the
repeated eigenvalues (the grid is symmetric under x <-> y) depends on the eigensolver, so the K drawn for a given seed is
not the reference's; the eigenvalues and the solve for a given K are."""
import itertools
import os

import numpy as np
import torch

from ._lib import call, stream

_FLAG_PIXELS_AT_BOUNDARY = 1      # PIDM_DARCY_PIXELS_AT_BOUNDARY
_ALL_STAGES = 7                   # PIDM_DARCY_GEN_ALL


def uniform_points_pixelwise(n, domain_length, boundary=False, dim=2):
    """[n**dim, dim] grid points, point index i*n + j with axis 0 first (reference :12-29)."""
    pixel_size = domain_length / n
    start, end = (0., domain_length) if boundary else (pixel_size / 2, domain_length - pixel_size / 2)
    xi = [np.linspace(start, end, num=n) for _ in range(dim)]
    return np.array(list(itertools.product(*xi)))


def create_f_s(x, y, w=0.125, r=10.):
    """source term: +r on the lower-left w x w corner, -r on the upper-right one (reference :31-39)"""
    result = np.zeros_like(x)
    result[np.logical_and(np.abs(x - 0.5 * w) <= 0.5 * w, np.abs(y - 0.5 * w) <= 0.5 * w)] = r
    result[np.logical_and(np.abs(x - 1 + 0.5 * w) <= 0.5 * w, np.abs(y - 1 + 0.5 * w) <= 0.5 * w)] = -r
    return result


def complete_covariance_matrix(grid, l):
    """exp(-|x - x'| / l) on the grid points (reference :41-50)"""
    dx = grid[:, None, 0] - grid[None, :, 0]
    dy = grid[:, None, 1] - grid[None, :, 1]
    return np.exp(-np.sqrt(dx ** 2 + dy ** 2) / l)


def compute_eigenpairs(cov_matrix, q):
    """the q largest eigenpairs in descending order (reference :52-61); only those q are computed"""
    from scipy.linalg import eigh
    n = cov_matrix.shape[0]
    w, v = eigh(cov_matrix, subset_by_index=[n - q, n - 1])
    return w[::-1].copy(), v[:, ::-1].copy()


def create_int_cond(use_trapezoid, shape, d0):
    """integral-condition weights: trapezoid {1, 2, 4} d0^2 / 4, or the plain mean (reference :99-121)"""
    if use_trapezoid:
        w = np.full(shape, 4.)
        w[0, :] = w[-1, :] = w[:, 0] = w[:, -1] = 2.
        w[0, 0] = w[0, -1] = w[-1, 0] = w[-1, -1] = 1.
        return w * (d0 ** 2 / 4.)
    return np.ones(shape).reshape(-1, 1) / (shape[0] ** 2)


def create_boundary_idcs(shape):
    """boolean masks of the flattened grid: rows 0 and -1 (axis 0), columns 0 and -1 (reference :80-97)"""
    masks = []
    for sl in ((0, slice(None)), (-1, slice(None)), (slice(None), 0), (slice(None), -1)):
        m = np.zeros(shape, dtype=np.bool_)
        m[sl] = True
        masks.append(m.reshape(-1))
    return tuple(masks)


def z_from_seed(seed, q):
    """the reference's np.random.seed(seed); norm.rvs(size=q)"""
    return np.random.RandomState(seed).standard_normal(q)


def KLE_expansion(eigenvalues, eigenvectors, q, grid_points, seed=None):
    """(G, z): log-permeability sum_k sqrt(lambda_k) z_k phi_k of one sample on the host (reference :63-78).  The
    batched product is DarcyDataGenerator.permeability."""
    z = z_from_seed(seed, q) if seed is not None else np.random.standard_normal(q)
    G = np.zeros(grid_points)
    for k in range(q):
        G += np.sqrt(eigenvalues[k]) * z[k] * eigenvectors[:, k]
    return G, z


class DarcyDataGenerator:
    """Reference defaults: P = 64, domain 1, length scale 0.1, q = 64 KLE terms, second-order FD, reverse_dy.
    eigenpairs: (eigenvalues [>= q], eigenvectors [P*P, >= q]) in descending order to use instead of computing them."""

    def __init__(self, pixels_per_dim=64, domain_length=1., length_scale=0.1, q=64, acc=2, reverse_dy=True,
                 pixels_at_boundary=True, device='cuda', eigenpairs=None):
        if acc != 2:
            raise NotImplementedError('only second-order finite differences (acc=2) are implemented')
        if pixels_per_dim != 64:
            raise ValueError(f'pixels_per_dim must be 64, got {pixels_per_dim}')
        if not 1 <= q <= pixels_per_dim ** 2:
            raise ValueError(f'q must be in [1, {pixels_per_dim ** 2}], got {q}')
        self.device = torch.device(device)
        if self.device.type != 'cuda':
            raise ValueError(f'DarcyDataGenerator runs on a CUDA device only, got {device!r}')
        self.pixels_per_dim = P = pixels_per_dim
        self.domain_length = float(domain_length)
        self.length_scale = length_scale
        self.q = q
        self.reverse_dy = bool(reverse_dy)
        self.pixels_at_boundary = bool(pixels_at_boundary)
        self.shape = (P, P)
        grid = uniform_points_pixelwise(P, domain_length, pixels_at_boundary)
        d0 = domain_length / (P - 1) if pixels_at_boundary else domain_length / P
        if eigenpairs is None:
            eigenpairs = compute_eigenpairs(complete_covariance_matrix(grid, length_scale), q)
        self.eigenvalues = np.asarray(eigenpairs[0], dtype=np.float64)[:q]
        self.eigenvectors = np.asarray(eigenpairs[1], dtype=np.float64)[:, :q]
        self.f_s_np = create_f_s(grid[:, 0], grid[:, 1])
        self.int_cond = create_int_cond(self.pixels_at_boundary, self.shape, d0)
        phi_s = (np.sqrt(self.eigenvalues)[None, :] * self.eigenvectors).T          # [q, P*P]
        self.phi_s = torch.tensor(np.ascontiguousarray(phi_s), dtype=torch.float64, device=self.device)
        self.f_s = torch.tensor(self.f_s_np, dtype=torch.float64, device=self.device)
        self._flags = _FLAG_PIXELS_AT_BOUNDARY if self.pixels_at_boundary else 0
        self._ws = None

    # ---- building blocks ------------------------------------------------------------------------------------------
    def _check(self, t, name, cols):
        if not (isinstance(t, torch.Tensor) and t.device.type == 'cuda'):
            raise ValueError(f'{name} must be a CUDA tensor')
        if t.dim() != 2 or t.shape[1] != cols:
            raise ValueError(f'{name} must have shape [B, {cols}], got {tuple(t.shape)}')
        return t.to(self.device, torch.float64).contiguous()

    def z_for_seeds(self, seeds):
        """[B, q] fp64 device tensor of the KLE coefficients of each seed"""
        z = np.stack([z_from_seed(int(s), self.q) for s in seeds]) if len(seeds) else np.zeros((0, self.q))
        return torch.tensor(z, dtype=torch.float64).to(self.device)

    def permeability(self, z):
        """K [B, P*P] fp64 = exp(sum_k sqrt(lambda_k) z_k phi_k) for z [B, q]"""
        z = self._check(z, 'z', self.q)
        K = torch.empty(z.shape[0], self.pixels_per_dim ** 2, dtype=torch.float64, device=self.device)
        call('pidm_darcy_gen_kle', self.phi_s, z, K, z.shape[0], self.q, self.pixels_per_dim, stream())
        return K

    def _workspace(self, B):
        need = call('pidm_darcy_gen_workspace_bytes', B, self.pixels_per_dim)
        if self._ws is None or self._ws.numel() < need:
            self._ws = None
            self._ws = torch.empty(need, dtype=torch.uint8, device=self.device)
        return self._ws

    def _solve(self, K, p, res, batch):
        B = K.shape[0]
        ws = self._workspace(B)
        call('pidm_darcy_gen_solve', K, self.f_s, p, res, batch, ws, ws.numel(), B, self.pixels_per_dim,
             self.domain_length, int(self.reverse_dy), self._flags, _ALL_STAGES, stream())

    def solve_pressure(self, K):
        """(p [B, P*P] fp64, res [B] fp64) for K [B, P*P]: the reference's lstsq solution and mean |M p - b|"""
        K = self._check(K, 'K', self.pixels_per_dim ** 2)
        p = torch.empty_like(K)
        res = torch.empty(K.shape[0], dtype=torch.float64, device=self.device)
        self._solve(K, p, res, None)
        return p, res

    # ---- data sets ---------------------------------------------------------------------------------------------------
    def generate(self, seeds, chunk=256):
        """(K, p, res, seeds) for the given seeds: K, p [n, P*P] fp64, res [n] fp64, seeds [n] int64, all on the device.
        Solved `chunk` samples at a time (about 6.5 MB of workspace per sample)."""
        seeds = [int(s) for s in seeds]
        Ks, ps, rs = [], [], []
        for i in range(0, len(seeds), chunk):
            K = self.permeability(self.z_for_seeds(seeds[i:i + chunk]))
            p, r = self.solve_pressure(K)
            Ks.append(K)
            ps.append(p)
            rs.append(r)
        n2 = self.pixels_per_dim ** 2
        cat = (lambda xs, *s: torch.cat(xs) if xs else torch.zeros(0, *s, dtype=torch.float64, device=self.device))
        return cat(Ks, n2), cat(ps, n2), cat(rs), torch.tensor(seeds, dtype=torch.int64, device=self.device)

    def batches(self, batch_size, seed0=0):
        """endless iterator of fp32 [B, 2, P, P] (p, K) device batches, the layout TrainEngine.step takes; batch k holds
        the samples of seeds seed0 + k*B .. seed0 + k*B + B - 1"""
        P = self.pixels_per_dim
        k = 0
        while True:
            seeds = range(seed0 + k * batch_size, seed0 + (k + 1) * batch_size)
            K = self.permeability(self.z_for_seeds(seeds))
            out = torch.empty(batch_size, 2, P, P, dtype=torch.float32, device=self.device)
            self._solve(K, None, None, out)
            yield out
            k += 1

    def write_csv(self, directory, n, seed0=0, batch_size=256):
        """the reference's seeds.csv, K_data.csv, p_data.csv, res_data.csv (no header, one sample per row, fp64 text)
        for seeds seed0 .. seed0 + n - 1; data_utils.Dataset((dir/'p_data.csv', dir/'K_data.csv')) reads them back"""
        import pandas as pd
        os.makedirs(directory, exist_ok=True)
        K, p, res, seeds = self.generate(range(seed0, seed0 + n), chunk=batch_size)
        for name, t in (('seeds.csv', seeds), ('K_data.csv', K), ('p_data.csv', p), ('res_data.csv', res)):
            pd.DataFrame(t.cpu().numpy()).to_csv(os.path.join(directory, name), index=False, header=False)
        return K, p, res, seeds


_GENERATORS = {}


def generate_sample(args):
    """(K, p, res, seed) of one sample for the reference's argument tuple (reference :123-165), solved on the GPU.
    The seed is the sample index i of the tuple, where the reference takes pid * time (see main)."""
    (i, eigenvalues, eigenvectors, q, pixels_per_dim, shape, acc, d0, d1, f_s, int_cond, xmin_bd, xmax_bd, ymin_bd,
     ymax_bd, reverse_dy) = args
    pab = np.asarray(int_cond).shape == tuple(shape)           # trapezoid weights are [P, P], the mean is [P*P, 1]
    domain_length = d0 * (pixels_per_dim - 1) if pab else d0 * pixels_per_dim
    key = (id(eigenvalues), id(eigenvectors), q, pixels_per_dim, acc, domain_length, bool(reverse_dy), pab)
    gen = _GENERATORS.get(key)
    if gen is None:
        gen = _GENERATORS[key] = DarcyDataGenerator(pixels_per_dim, domain_length, q=q, acc=acc, reverse_dy=reverse_dy,
                                                    pixels_at_boundary=pab, eigenpairs=(eigenvalues, eigenvectors))
    K, p, res, seed = gen.generate([i])
    return K[0].cpu().numpy(), p[0].cpu().numpy(), float(res[0]), int(seed[0])


def main(n_samples=10, seed0=0, save_dir='./data/darcy/', batch_size=256):
    """The reference's data set (reference :167-236): seeds.csv, K_data.csv, p_data.csv and res_data.csv in save_dir.
    One deliberate difference: sample i takes the seed seed0 + i, where the reference takes pid * time in milliseconds
    mod 2^32.  The files are then reproducible, and the seeds are unique by construction."""
    import time
    start_time = time.time()
    gen = DarcyDataGenerator(pixels_per_dim=64, domain_length=1., length_scale=0.1, q=64, acc=2, reverse_dy=True,
                             pixels_at_boundary=True)
    print(f'Time elapsed for the eigenpairs: {time.time() - start_time}')
    mid_time = time.time()
    gen.write_csv(save_dir, n_samples, seed0=seed0, batch_size=batch_size)
    print(f'Time elapsed for data generation and storing: {time.time() - mid_time}')
    print('Data generation finished.')
