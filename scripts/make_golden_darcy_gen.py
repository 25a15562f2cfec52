"""Golden vectors for the Darcy data generator.  TEST INFRASTRUCTURE ONLY; runs on the CPU.

Runs the UNMODIFIED reference src/darcy_data_generation.py (checkout in PIDM_REFERENCE, imported through oracle/ref_shims/
exactly as oracle/make_golden.py does) and writes tests/golden/darcy_gen.pt in fp64:
    eigenvalues [64]   the q = 64 largest covariance eigenvalues (compute_eigenpairs on complete_covariance_matrix)
    f_s [4096], int_cond [4096]   create_f_s and the trapezoid weights of create_int_cond
    seed [4], z [4, 64], K [4, 4096], p [4, 4096], res [4]   generate_sample on four argument tuples

generate_sample draws its seed from os.getpid() * time.time(); the recipe replaces the module's `os` and `time` names by
stand-ins (pid = seed, clock = 1 ms), so that unique_seed = seed.  The reference file itself is not touched.

The generator calls findiff's operator API (FinDiff(...)(array), .matrix(shape), Coef(array) * FinDiff, sums and
differences), which the findiff shim of oracle/ref_shims/ does not provide: it is added here, on the shim module, from
the same acc = 2 tables (the shim's `_tab1d`), for this process only.

    PIDM_REFERENCE=<checkout of the original project> python scripts/make_golden_darcy_gen.py
"""
import importlib.util
import os
import types

import numpy as np
import scipy.sparse as sp
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
_spec = importlib.util.spec_from_file_location('make_golden', os.path.join(ROOT, 'oracle', 'make_golden.py'))
MG = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(MG)

SEEDS = (1, 20231, 777, 4242424)


def _install_operator_api(fd):
    """FinDiff operator algebra on the shim: one-dimensional acc = 2 matrices (C in the interior, L / H at the ends),
    Kronecker products over the axes, Coef(c) * op = diag(c) op, sums and differences of operators."""
    def mat1d(n, h, order):
        tab = fd._tab1d(order, h)
        D = sp.lil_matrix((n, n))
        for i in range(n):
            key = 'L' if i == 0 else ('H' if i == n - 1 else 'C')
            for o, c in tab[key].items():
                D[i, i + o] = c
        return D.tocsr()

    class Op:
        def __init__(self, build):
            self.build = build            # shape -> scipy.sparse matrix

        def matrix(self, shape):
            return self.build(tuple(shape))

        def __call__(self, u):
            return (self.matrix(u.shape) @ u.reshape(-1)).reshape(u.shape)

        def __add__(self, other):
            return Op(lambda s: self.matrix(s) + other.matrix(s))

        def __sub__(self, other):
            return Op(lambda s: self.matrix(s) - other.matrix(s))

    def findiff_matrix(self, shape):
        M = None
        for (axis, h, order) in self.terms:
            mats = [mat1d(n, h, order) if ax == axis else sp.identity(n, format='csr') for ax, n in enumerate(shape)]
            K = mats[0]
            for m in mats[1:]:
                K = sp.kron(K, m, format='csr')
            M = K if M is None else M @ K
        return M.tocsr()

    class Coef:
        def __init__(self, c):
            self.c = np.asarray(c)

        def __mul__(self, op):
            return Op(lambda s: (sp.diags(self.c.reshape(-1)) @ op.matrix(s)).tocsr())

    fd.FinDiff.matrix = findiff_matrix
    fd.FinDiff.__call__ = Op.__call__
    fd.FinDiff.__add__ = Op.__add__
    fd.FinDiff.__sub__ = Op.__sub__
    fd.Coef = Coef


def main():
    import findiff
    assert os.path.abspath(findiff.__file__).startswith(os.path.join(ROOT, 'oracle', 'ref_shims')), findiff.__file__
    _install_operator_api(findiff)
    import src.darcy_data_generation as G
    assert os.path.abspath(G.__file__).startswith(os.path.abspath(MG.REF)), G.__file__

    P, dl, l, q, acc = 64, 1., 0.1, 64, 2
    shape = (P, P)
    pts = G.uniform_points_pixelwise(P, dl, True)
    d0 = dl / (P - 1)
    d1 = -d0
    eigenvalues, eigenvectors = G.compute_eigenpairs(G.complete_covariance_matrix(pts, l), q)
    f_s = G.create_f_s(pts[:, 0], pts[:, 1])
    xmin_bd, xmax_bd, ymin_bd, ymax_bd = G.create_boundary_idcs(shape)
    int_cond = G.create_int_cond(True, shape, d0)

    out = dict(seed=[], z=[], K=[], p=[], res=[])
    for s in SEEDS:
        G.os = types.SimpleNamespace(getpid=lambda s=s: s)
        G.time = types.SimpleNamespace(time=lambda: 0.001)
        args = (0, eigenvalues, eigenvectors, q, P, shape, acc, d0, d1, f_s, int_cond, xmin_bd, xmax_bd, ymin_bd,
                ymax_bd, True)
        K, p, res, seed = G.generate_sample(args)
        assert seed == s, (seed, s)
        np.random.seed(s)
        z = G.norm.rvs(size=q)
        out['seed'].append(seed)
        out['z'].append(z)
        out['K'].append(K)
        out['p'].append(p)
        out['res'].append(res)
        print(f'seed {s}: res {res:.6e}  max|p| {np.abs(p).max():.4f}')
    t = lambda a: torch.tensor(np.asarray(a), dtype=torch.float64)  # noqa: E731
    MG.save('darcy_gen.pt', dict(eigenvalues=t(eigenvalues), f_s=t(f_s), int_cond=t(int_cond).reshape(-1),
                                 seed=torch.tensor(out['seed'], dtype=torch.int64), z=t(out['z']), K=t(out['K']),
                                 p=t(out['p']), res=t(out['res'])))


if __name__ == '__main__':
    main()
