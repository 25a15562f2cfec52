"""Import shim (test infrastructure): findiff for acc=2, covering both uses the reference makes of it.
  * FinDiff(...).stencil(shape).data, at reference grad_utils.py:154-159 (init time only).
  * The operator API of reference darcy_data_generation.py: FinDiff(...)(array), .matrix(shape), Coef(array) * FinDiff,
    sums and differences of operators.  One-dimensional matrices hold the C rows inside and the L / H rows at the
    ends; an operator over several axes is the Kronecker product, Coef(c) * op = diag(c) op.
Closed-form second-order tables:
  d/dx    C: {-1:-1/2h, +1:+1/2h}      L: {0:-3/2h, 1:2/h, 2:-1/2h}     H: {0:3/2h, -1:-2/h, -2:1/2h}
  d2/dx2  C: {-1:1, 0:-2, 1:1}/h^2     L: {0:2, 1:-5, 2:4, 3:-1}/h^2    H: {0:2, -1:-5, -2:4, -3:-1}/h^2
Mixed derivatives are tensor products.  findiff itself is not installed here: parity of these
tables against findiff>=0.10 is pinned analytically only (exactness on quadratics), see DESIGN.md."""
import itertools

import numpy as np


def _tab1d(order, h):
    if order == 1:
        return {'C': {-1: -0.5 / h, 1: 0.5 / h},
                'L': {0: -1.5 / h, 1: 2.0 / h, 2: -0.5 / h},
                'H': {0: 1.5 / h, -1: -2.0 / h, -2: 0.5 / h}}
    if order == 2:
        h2 = h * h
        return {'C': {-1: 1.0 / h2, 0: -2.0 / h2, 1: 1.0 / h2},
                'L': {0: 2.0 / h2, 1: -5.0 / h2, 2: 4.0 / h2, 3: -1.0 / h2},
                'H': {0: 2.0 / h2, -1: -5.0 / h2, -2: 4.0 / h2, -3: -1.0 / h2}}
    raise NotImplementedError(order)


def _mat1d(n, h, order):
    import scipy.sparse as sp
    tab = _tab1d(order, h)
    D = sp.lil_matrix((n, n))
    for i in range(n):
        key = 'L' if i == 0 else ('H' if i == n - 1 else 'C')
        for o, c in tab[key].items():
            D[i, i + o] = c
    return D.tocsr()


class _StencilSet:
    def __init__(self, data):
        self.data = data


class _Operator:
    """a linear operator on arrays of a given shape, defined by its scipy.sparse matrix"""
    def __init__(self, build):
        self.build = build            # shape -> scipy.sparse matrix

    def matrix(self, shape):
        return self.build(tuple(shape))

    def __call__(self, u):
        return (self.matrix(u.shape) @ u.reshape(-1)).reshape(u.shape)

    def __add__(self, other):
        return _Operator(lambda s: self.matrix(s) + other.matrix(s))

    def __sub__(self, other):
        return _Operator(lambda s: self.matrix(s) - other.matrix(s))


class FinDiff(_Operator):
    def __init__(self, *args, acc=2):
        if acc != 2:
            raise NotImplementedError('shim supports acc=2 only (model.yaml: fd_acc: 2)')
        if isinstance(args[0], (tuple, list)):
            self.terms = [tuple(a) for a in args]
        else:
            self.terms = [tuple(args)]

    def matrix(self, shape):
        import scipy.sparse as sp
        M = None
        for (axis, h, order) in self.terms:
            mats = [_mat1d(n, h, order) if ax == axis else sp.identity(n, format='csr') for ax, n in enumerate(shape)]
            K = mats[0]
            for m in mats[1:]:
                K = sp.kron(K, m, format='csr')
            M = K if M is None else M @ K
        return M.tocsr()

    def stencil(self, shape):
        ndim = len(shape)
        data = {}
        for key in itertools.product('LCH', repeat=ndim):
            # product over the partial derivatives (one per listed axis)
            st = {tuple([0] * ndim): 1.0}
            for (axis, h, order) in self.terms:
                tab = _tab1d(order, h)[key[axis]]
                new = {}
                for off, c in st.items():
                    for o, c1 in tab.items():
                        off2 = list(off)
                        off2[axis] += o
                        new[tuple(off2)] = new.get(tuple(off2), 0.0) + c * c1
                st = new
            data[key] = st
        return _StencilSet(data)


class Coef:
    def __init__(self, c):
        self.c = np.asarray(c)

    def __mul__(self, op):
        import scipy.sparse as sp
        return _Operator(lambda s: (sp.diags(self.c.reshape(-1)) @ op.matrix(s)).tocsr())
