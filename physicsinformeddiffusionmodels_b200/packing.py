"""Device-side tables that let ONE kernel launch service every layer of the U-Net:

* WeightPacker  -- fp32 master weights (framework layout, owned by nn.Parameters) -> packed GEMM operands
                   Wp[n][tap*Cin + c] in the activation dtype, forward and dgrad variants, for every
                   convolution / linear layer, refreshed by a single pidm_pack_weights launch.
* MlpTable      -- pointers of all ResnetBlock time-MLPs for pidm_block_mlps_{fwd,bwd}.
"""
import numpy as np
import torch

from . import _lib
from ._lib import call, stream

_PACK_DT = np.dtype([('src', '<u8'), ('dst', '<u8'), ('s_n', '<i8'), ('s_c', '<i8'), ('N', '<i4'), ('C', '<i4'),
                     ('Cpad', '<i4'), ('taps', '<i4'), ('flip', '<i4'), ('pad_', '<i4')])
_PAIR_DT = np.dtype([('src', '<u8'), ('dst_f', '<u8'), ('dst_d', '<u8'), ('s_co', '<i8'), ('s_ci', '<i8'), ('Cout', '<i4'),
                     ('Cin', '<i4'), ('taps', '<i4'), ('flip', '<i4'), ('tile0', '<i4'), ('pad_', '<i4')])
_MLP_DT = np.dtype([('W', '<u8'), ('b', '<u8'), ('dW', '<u8'), ('db', '<u8'), ('out', '<u8'), ('dout', '<u8'),
                    ('n', '<i4'), ('pad_', '<i4')])


def _to_device_bytes(arr, device):
    """Upload a small structured numpy table (through pinned memory, stream-ordered)."""
    host = torch.from_numpy(arr.view(np.uint8).copy()).pin_memory()
    dev = torch.empty(host.numel(), dtype=torch.uint8, device=device)
    dev.copy_(host, non_blocking=True)
    return dev, host


class ConvSpec:
    """Geometry + packed-operand views of one convolution-like layer.

    kind 'conv'  : weight [Cout, Cin, (1,) kh, kw]   (nn.Conv3d/Conv2d/Linear layout)
    kind 'convT' : weight [Cin, Cout, (1,) kh, kw]   (nn.ConvTranspose3d layout), forward = transposed gather

    circular=True: the layer pads periodically (padding_mode='circular').  It then runs on a copy of its input with a
    wrapped halo of `halo` pixels: a valid convolution for 'conv', the transposed gather with pad + 2 for 'convT'.
    `dgrad_halo` is the halo its input gradient needs on dy.  A layer without padding is never circular.
    """

    def __init__(self, weight, kind, kh, kw, stride, pad, cin_pad=None, need_dgrad=True, circular=False):
        self.weight = weight
        self.kind = kind
        self.kh, self.kw, self.stride, self.pad = kh, kw, stride, pad
        self.taps = kh * kw
        self.transposed = kind == 'convT'
        self.circular = bool(circular) and pad > 0
        self.halo = self.dgrad_halo = 0
        if self.circular:
            if kh != kw or not ((stride == 1 and kh == 2 * pad + 1) or (stride == 2 and kh == 2 * pad + 2)):
                raise ValueError(f'circular padding needs a "same" stride-1 or a k = 2 pad + 2 stride-2 layer '
                                 f'(got {kh}x{kw}, stride {stride}, pad {pad})')
            self.halo = 1 if self.transposed else pad
            self.dgrad_halo = pad if stride == 1 else 1
        if kind == 'conv':
            self.cout, self.cin_real = weight.shape[0], weight.shape[1]
            self.w_stride_n, self.w_stride_c = self.cin_real * self.taps, self.taps
        else:
            self.cin_real, self.cout = weight.shape[0], weight.shape[1]
            self.w_stride_n, self.w_stride_c = self.taps, self.cout * self.taps
        self.cin = cin_pad or self.cin_real
        self.need_dgrad = need_dgrad
        self.wp_fwd = None
        self.wp_dgrad = None

    def out_hw(self, H, W):
        if self.transposed:
            return (H - 1) * self.stride - 2 * self.pad + self.kh, (W - 1) * self.stride - 2 * self.pad + self.kw
        return (H + 2 * self.pad - self.kh) // self.stride + 1, (W + 2 * self.pad - self.kw) // self.stride + 1

    def fwd_elems(self):
        return self.cout * self.taps * self.cin

    def dgrad_elems(self):
        return self.cin * self.taps * self.cout if self.need_dgrad else 0


class WeightPacker:
    def __init__(self):
        self.specs = []
        self._key = None
        self._table = None
        self._buf = None
        self._n = 0
        self._n_pairs = 0
        self._packed_for = None

    def add(self, spec):
        self.specs.append(spec)
        return spec

    def _build(self, device, dtype):
        total = sum(s.fwd_elems() + s.dgrad_elems() for s in self.specs)
        # every packed matrix starts on a 128-element boundary (TMA needs 16-byte aligned bases; 256 B is safer)
        total += 128 * 2 * len(self.specs)
        self._buf = torch.zeros(total, device=device, dtype=dtype)
        rows, off = [], 0

        def take(n):
            nonlocal off
            v = self._buf[off:off + n]
            off += (n + 127) // 128 * 128
            return v
        pairs, tile_map = [], []
        self._tiles_before_spec = []           # number of pair tiles owned by the specs in front of spec i
        for s in self.specs:
            self._tiles_before_spec.append(len(tile_map))
            s.wp_fwd = take(s.fwd_elems())
            if s.need_dgrad:
                s.wp_dgrad = take(s.dgrad_elems())
            flip = 1 if (s.stride == 1 and not s.transposed) else 0
            # layers with whole 32-channel blocks and <= 16 taps: both operands from one read (pidm_pack_weights_pairs);
            # the rest (channel-padded 7x7 stem) through the generic strided kernel
            if (s.cin == s.cin_real and s.cin % 32 == 0 and s.cout % 32 == 0 and s.taps <= 16
                    and s.taps in (s.w_stride_n, s.w_stride_c)):
                pairs.append((s.weight.data_ptr(), s.wp_fwd.data_ptr(), s.wp_dgrad.data_ptr() if s.need_dgrad else 0,
                              s.w_stride_n, s.w_stride_c, s.cout, s.cin, s.taps, flip, len(tile_map), 0))
                tile_map += [len(pairs) - 1] * ((s.cout // 32) * (s.cin // 32))
                continue
            rows.append((s.weight.data_ptr(), s.wp_fwd.data_ptr(), s.w_stride_n, s.w_stride_c, s.cout, s.cin_real,
                         s.cin, s.taps, 0, 0))
            if s.need_dgrad:
                rows.append((s.weight.data_ptr(), s.wp_dgrad.data_ptr(), s.w_stride_c, s.w_stride_n, s.cin, s.cout,
                             s.cout, s.taps, flip, 0))
        self._n = len(rows)
        self._table = self._host = None
        if rows:
            arr = np.array(rows, dtype=_PACK_DT)
            assert arr.dtype.itemsize == call('pidm_pack_entry_size')
            self._table, self._host = _to_device_bytes(arr, device)
        self._n_pairs = len(pairs)
        self._pair_table = self._pair_host = None
        if pairs:
            arr = np.array(pairs, dtype=_PAIR_DT)
            assert arr.dtype.itemsize == call('pidm_pack_pair_entry_size')
            self._pair_table, self._pair_host = _to_device_bytes(arr, device)
            self._pair_map, self._pair_map_host = _to_device_bytes(np.array(tile_map, dtype=np.int32), device)
            self._pair_tiles = len(tile_map)
            self._pair_taps = int(max(r[7] for r in pairs))

    def _versions(self, dtype):
        return (tuple(s.weight.data_ptr() for s in self.specs), tuple(s.weight._version for s in self.specs), dtype)

    def invalidate(self):
        """Parameters were changed behind autograd's back (flat-buffer optimizer kernel): the packed copy is stale."""
        self._packed_for = None

    def stale(self, dtype):
        return self._packed_for != self._versions(dtype)

    def refresh_if_stale(self, dtype):
        if self.specs and self.stale(dtype):
            self.refresh(dtype)

    def refresh(self, dtype, early_specs=0):
        """Re-pack all weights.  Rebuilds the tables if parameters moved (e.g. .to(device)).
        early_specs > 0: the operands of the first `early_specs` layers (registration order = execution order) are packed by
        a first launch and a CUDA event recorded behind it is returned, so a consumer can start on them while the second
        launch packs the rest; otherwise returns None."""
        if not self.specs:
            return None
        w0 = self.specs[0].weight
        key = (tuple(s.weight.data_ptr() for s in self.specs), dtype)
        if key != self._key:
            self._build(w0.device, dtype)
            self._key = key
        code, event = _lib.DTYPE_CODE[dtype], None
        if self._n:
            call('pidm_pack_weights', self._table, self._n, code, stream())
        if self._n_pairs:
            first = self._tiles_before_spec[early_specs] if 0 < early_specs < len(self.specs) else 0
            if first > 0:
                call('pidm_pack_weights_pairs', self._pair_table, self._pair_map, 0, first, self._pair_taps, code, stream())
                event = torch.cuda.Event()
                event.record(torch.cuda.current_stream())
            call('pidm_pack_weights_pairs', self._pair_table, self._pair_map, first, self._pair_tiles - first, self._pair_taps,
                 code, stream())
        self._packed_for = self._versions(dtype)
        return event


class MlpTable:
    """All ResnetBlock `mlp.1` Linear layers; entry i writes its own [B, n_i] output tensor."""

    def __init__(self, linears):
        self.linears = list(linears)           # objects with .weight [n, td], .bias [n]
        self.n = len(self.linears)
        self.rows = [l.weight.shape[0] for l in self.linears]
        self.max_rows = max(self.rows) if self.rows else 0
        self._cache = {}
        self._keep = []

    @property
    def params(self):
        out = []
        for l in self.linears:
            out += [l.weight, l.bias]
        return out

    def device_table(self, outs, douts=None, grad_bufs=None):
        ptr = lambda t: 0 if t is None else t.data_ptr()
        rows = []
        for i, l in enumerate(self.linears):
            rows.append((l.weight.data_ptr(), l.bias.data_ptr(),
                         ptr(grad_bufs[2 * i]) if grad_bufs else 0, ptr(grad_bufs[2 * i + 1]) if grad_bufs else 0,
                         ptr(outs[i]) if outs else 0, ptr(douts[i]) if douts else 0, self.rows[i], 0))
        key = tuple(rows)
        hit = self._cache.get(key)
        if hit is None:
            arr = np.array(rows, dtype=_MLP_DT)
            assert arr.dtype.itemsize == call('pidm_mlp_entry_size')
            hit = _to_device_bytes(arr, self.linears[0].weight.device)
            if torch.cuda.is_current_stream_capturing():
                self._keep.append(hit)        # the captured copy node re-reads this pinned block at every replay
            elif len(self._cache) > 32:
                self._cache.clear()
            self._cache[key] = hit
        return hit[0]
