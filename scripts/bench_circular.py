"""Unet3D(padding_mode='zeros') against padding_mode='circular', timed alternately in one process on one GPU.

Per round and per setting (bf16 activations, CUDA graphs, same weights and inputs):
  - the graph-replayed Darcy TrainEngine step at batch 32;
  - a 100-step SampleEngine loop at batch 16;
  - the mechanics TrainEngine step, Unet3D(dim=128, channels=10, out_dim=3), batch 32 (bench.py's configuration).
Both padding modes run the Darcy residual with bcs='periodic' (the setting a circular model is meant for), so the
ratios measure the halo copies alone.  Once: the halo kernel (pidm_wrap_pad_nhwc) at a large standalone size in GB/s
(bytes read + written), and the halo bytes and launches per Darcy step computed from the layer shapes.  Prints the card name and power limit first
(read-only query), one JSON line per round and setting, then a summary.

    python scripts/bench_circular.py [--rounds 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def timed(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def halo_census(model, B, P, esize=2):
    """halo'd copies per training step from the layer shapes: (forward operands, backward dy, bytes written)"""
    fwd = bwd = nbytes = 0
    H = {}
    res = P
    # spatial size at each layer (registration order = execution order): down-sampling halves, up-sampling doubles
    for s in model._packer.specs:
        H[id(s)] = res
        if s.kind == 'conv' and s.stride == 2:
            res //= 2
        elif s.kind == 'convT':
            res *= 2
    for s in model._packer.specs:
        if not s.circular:
            continue
        hin = H[id(s)]
        fwd += 1
        nbytes += B * (hin + 2 * s.halo) ** 2 * s.cin * esize
        if s.need_dgrad:
            ho = s.out_hw(hin, hin)[0]
            bwd += 1
            nbytes += B * (ho + 2 * s.dgrad_halo) ** 2 * s.cout * esize
    return fwd, bwd, nbytes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'needs a CUDA device'
    from physicsinformeddiffusionmodels_b200 import ops
    from physicsinformeddiffusionmodels_b200._lib import call, stream
    from physicsinformeddiffusionmodels_b200.denoising_utils import DenoisingDiffusion
    from physicsinformeddiffusionmodels_b200.engine import SampleEngine, TrainEngine
    from physicsinformeddiffusionmodels_b200.residuals_darcy import ResidualsDarcy
    from physicsinformeddiffusionmodels_b200.residuals_mechanics_K import ResidualsMechanics
    from physicsinformeddiffusionmodels_b200.unet_model import Unet3D
    print(json.dumps({'card': card()}), flush=True)
    dev = torch.device('cuda')
    ops.set_precision('bf16')
    modes = ('zeros', 'circular')

    # ---- halo kernel standalone: 64 x [64, 64, 256] bf16 -> halo 1 (about 0.55 GB moved per call)
    xs = torch.randn(64, 64, 64, 256, device=dev).bfloat16()
    ys = torch.empty(64, 66, 66, 256, device=dev, dtype=torch.bfloat16)
    halo_fn = lambda: call('pidm_wrap_pad_nhwc', xs, ys, 64, 64, 64, 256, 1, 1, stream())   # noqa: E731
    for _ in range(3):
        halo_fn()
    halo_bytes = xs.numel() * 2 + ys.numel() * 2

    torch.manual_seed(0)
    sd = Unet3D(dim=32, channels=2).state_dict()
    torch.manual_seed(0)
    sd_m = Unet3D(dim=128, channels=10, out_dim=3, sigmoid_last_channel=True).state_dict()

    def circ(d, pm):
        if pm == 'zeros':
            return d
        out = {}
        for k, v in d.items():
            parts = k.split('.')
            if parts[0] == 'ups' and parts[2] == '3':
                k = '.'.join(parts[:3] + ['conv_transpose'] + parts[3:])
            out[k] = v
        return out
    g = torch.Generator().manual_seed(1234)
    x0 = torch.randn(32, 2, 64, 64, generator=g).to(dev)
    x_T = torch.randn(16, 2, 64, 64, generator=g).to(dev)
    cond = torch.rand(32, 3, 65, 65, generator=g)
    cond[:, 0] = (0.3 + 0.4 * torch.rand(32, generator=g))[:, None, None]
    xm = torch.cat((0.2 * torch.randn(32, 2, 65, 65, generator=g), torch.rand(32, 1, 65, 65, generator=g).clamp(1e-3, 1.)), 1)
    bcs = torch.zeros(32, 4, 65, 65)
    bcs[:, 0, :, 0] = 1.
    bcs[:, 1, :, 0] = 1.
    bcs[:, 3, 32, 64] = -1.
    inp_m = torch.cat((cond, xm, bcs), dim=1).to(dev)
    eng, census = {}, {}
    for pm in modes:
        model = Unet3D(dim=32, channels=2, padding_mode=pm).to(dev)
        model.load_state_dict(circ(sd, pm))
        census[pm] = halo_census(model, 32, 64)
        res = ResidualsDarcy(model=model, fd_acc=2, pixels_per_dim=64, pixels_at_boundary=True, reverse_d1=True,
                             device=dev, bcs='periodic', domain_length=1.)
        te = TrainEngine(model, DenoisingDiffusion(100, dev), res, use_graph=True)
        smodel = Unet3D(dim=32, channels=2, padding_mode=pm).to(dev)
        smodel.load_state_dict(circ(sd, pm))
        smodel.eval()
        sres = ResidualsDarcy(model=smodel, fd_acc=2, pixels_per_dim=64, pixels_at_boundary=True, reverse_d1=True,
                              device=dev, bcs='periodic', domain_length=1.)
        se = SampleEngine(smodel, DenoisingDiffusion(100, dev), sres, batch=16, use_graph=True)
        mm = Unet3D(dim=128, channels=10, out_dim=3, sigmoid_last_channel=True, padding_mode=pm).to(dev)
        mm.load_state_dict(circ(sd_m, pm))
        mres = ResidualsMechanics(model=mm, pixels_per_dim=64, pixels_at_boundary=True, no_BC_folder='', device=dev)
        me = TrainEngine(mm, DenoisingDiffusion(100, dev), mres, lr=1e-4, max_norm=1.0, ema_mu=0.99, c_data=1.0,
                         c_residual=1e-2, c_ineq=0., lambda_opt=1e-3, use_graph=True)
        for _ in range(5):                     # capture + warm-up
            te.step(x0)
            me.step(inp_m)
        se.sample(x_init=x_T)
        torch.cuda.synchronize()
        eng[pm] = (te, se, me)

    rows = {pm: [] for pm in modes}
    halo = []
    for rnd in range(args.rounds):
        ms = timed(halo_fn, 20)
        halo.append(halo_bytes / ms / 1e6)
        for pm in modes:
            te, se, me = eng[pm]
            row = {'round': rnd, 'padding_mode': pm,
                   'darcy_train_step_ms': timed(lambda: te.step(x0), 20),
                   'sample_100_ms': timed(lambda: se.sample(x_init=x_T), 1),
                   'mechanics_train_step_ms': timed(lambda: me.step(inp_m), 10)}
            rows[pm].append(row)
            print(json.dumps(row), flush=True)
    keys = ('darcy_train_step_ms', 'sample_100_ms', 'mechanics_train_step_ms')
    summary = {'halo_kernel_gbs': dict(mean=statistics.mean(halo), min=min(halo), max=max(halo),
                                       shape='[64,64,64,256] bf16, halo 1')}
    for pm, rs in rows.items():
        for k in keys:
            v = [rw[k] for rw in rs]
            summary[f'{pm}.{k}'] = dict(mean=statistics.mean(v), min=min(v), max=max(v))
    for k in keys:
        summary['circular/zeros.' + k] = summary[f'circular.{k}']['mean'] / summary[f'zeros.{k}']['mean']
    fwd, bwd, nbytes = census['circular']
    summary['darcy_step_halo'] = dict(forward_copies=fwd, backward_dy_copies=bwd, launches=fwd + bwd,
                                      bytes_written=nbytes, batch=32)
    print(json.dumps({'summary': summary}), flush=True)


if __name__ == '__main__':
    main()
