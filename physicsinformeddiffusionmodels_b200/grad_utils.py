"""Finite-difference helpers with the reference's names (reference src/grad_utils.py:9-184).

The training / sampling path never calls these one derivative at a time: `ResidualsDarcy` evaluates all six
derivatives, the PDE residual, the boundary terms and (in training) the loss inside ONE kernel (csrc/darcy.cu).
`GradientsHelper.stencil_gradients` is kept for callers that want a single derivative field; it is one libpidm
launch (second-order central stencil in the interior, one-sided 3/4-point stencils on the boundary -- the net
effect of the reference's 9 conv2d + 9 slice assignments, grad_utils.py:64-146; with periodic=True the central stencil
with wrapped neighbours at every pixel, grad_utils.py:76-81).  Forward only."""
import numpy as np
import torch


def generalized_image_to_b_xy_c(tensor):
    """[B, c0, c1, ..., X, Y] -> [B, X*Y, c0, c1, ...]"""
    nd = tensor.dim()
    perm = (0, nd - 2, nd - 1) + tuple(range(1, nd - 2))
    t = tensor.permute(*perm)
    return t.reshape(t.shape[0], t.shape[1] * t.shape[2], *t.shape[3:])


def generalized_b_xy_c_to_image(tensor, pixels_x=None, pixels_y=None):
    """[B, X*Y, c0, c1, ...] -> [B, c0, c1, ..., X, Y]"""
    if pixels_x is None or pixels_y is None:
        pixels_x = pixels_y = int(np.sqrt(tensor.shape[1]))
    t = tensor.reshape(tensor.shape[0], pixels_x, pixels_y, *tensor.shape[2:])
    nd = t.dim()
    perm = (0,) + tuple(range(3, nd)) + (1, 2)
    return t.permute(*perm)


_MODES = {'d_d0': 0, 'd_d1': 1, 'd_d00': 2, 'd_d11': 3, 'd_d01': 4}
_FD_PERIODIC = 8                         # PIDM_FD_PERIODIC (pidm.h)


class StencilGradients(torch.nn.Module):
    def __init__(self, d0=1, d1=1, fd_acc=2, periodic=False, device='cpu'):
        super().__init__()
        if fd_acc != 2:
            raise NotImplementedError('only fd_acc = 2 is built (model.yaml: "keep at 2")')
        self.d0, self.d1 = float(d0), float(d1)
        self.periodic = bool(periodic)          # wrapped central stencil at every pixel (grad_utils.py:76-81)

    def forward(self, x, mode):
        from ._lib import call, stream
        if mode == 'all':
            return tuple(self.forward(x, m) for m in ('d_d0', 'd_d1', 'd_d00', 'd_d11', 'd_d01'))
        if mode not in _MODES:
            raise NotImplementedError(mode)
        if not x.is_cuda:
            raise RuntimeError('stencil_gradients needs a CUDA tensor (no CPU fallback on the product path)')
        shp = x.shape
        P = shp[-1]
        xf = x.detach().contiguous().float().reshape(-1, P, P)
        out = torch.empty_like(xf)
        mode_bits = _MODES[mode] | (_FD_PERIODIC if self.periodic else 0)
        call('pidm_fd_stencil', xf, out, xf.shape[0], P, mode_bits, self.d0, self.d1, stream())
        return out.reshape(shp)


class GradientsHelper:
    def __init__(self, d0, d1, fd_acc, periodic=False, device='cpu', eps=1e-6):
        self.eps = eps
        self.stencil_gradients = StencilGradients(d0=d0, d1=d1, fd_acc=fd_acc, periodic=periodic, device=device)
