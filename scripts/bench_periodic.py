"""bcs='none' against bcs='periodic', timed alternately in one process on one GPU.

Per round and per setting:
  - the residual kernel (pidm_darcy_residual_fwd) and the fused loss + gradient kernel (pidm_darcy_pidm_loss) at
    B = 32768, in GB/s over the algorithmic bytes bench.py uses (read x0_hat, write the residual; read x0_hat + target,
    write the gradient);
  - the CUDA-graph-replayed Darcy TrainEngine step at batch 32 (bf16);
  - a 100-step SampleEngine loop at batch 16 (bf16, CUDA graph).
Prints the card name and power limit first (read-only query), one JSON line per round and setting, then a summary.

    python scripts/bench_periodic.py [--rounds 5]
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

FLAGS = {'none': 1, 'periodic': 3}        # PIDM_DARCY_PIXELS_AT_BOUNDARY (| PIDM_DARCY_PERIODIC)


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
    from physicsinformeddiffusionmodels_b200.unet_model import Unet3D
    print(json.dumps({'card': card()}), flush=True)
    dev = torch.device('cuda')
    ops.set_precision('bf16')

    # ---- standalone kernels at B = 32768 (2.7 GB working set, far beyond L2)
    Bs = 32768
    x = torch.randn(Bs, 2, 64, 64, device=dev)
    fs = torch.zeros(4096, device=dev)
    fs[:8 * 64].view(8, 64)[:, :8] = 10.0
    r = torch.empty(Bs, 4096, 3, device=dev)
    tgt = torch.randn_like(x)
    t = torch.randint(0, 100, (Bs,), device=dev)
    tab = torch.rand(100, device=dev) + 0.1
    sums = torch.zeros(3, device=dev)
    gx = torch.empty_like(x)
    kern = {}
    for b, f in FLAGS.items():
        kern[b] = {'fwd': (lambda f=f: call('pidm_darcy_residual_fwd', x, fs, r, Bs, 64, 1.0, 1, f, stream()), Bs * 81920),
                   'loss': (lambda f=f: call('pidm_darcy_pidm_loss', x, x, tgt, fs, t, tab, tab, 1.0, 1e-3, sums, gx, None,
                                             Bs, 64, 1.0, 1, f, stream()), Bs * (2 * 4096 * 4 * 3))}

    # ---- engines, one per setting (same weights, same batch)
    torch.manual_seed(0)
    sd = Unet3D(dim=32, channels=2).state_dict()
    g = torch.Generator().manual_seed(1234)
    x0 = torch.randn(32, 2, 64, 64, generator=g).to(dev)
    x_T = torch.randn(16, 2, 64, 64, generator=g).to(dev)
    eng = {}
    for b in FLAGS:
        model = Unet3D(dim=32, channels=2).to(dev)
        model.load_state_dict(sd)
        diff = DenoisingDiffusion(100, dev)
        res = ResidualsDarcy(model=model, fd_acc=2, pixels_per_dim=64, pixels_at_boundary=True, reverse_d1=True,
                             device=dev, bcs=b, domain_length=1.)
        te = TrainEngine(model, diff, res, use_graph=True)
        smodel = Unet3D(dim=32, channels=2).to(dev)
        smodel.load_state_dict(sd)
        smodel.eval()
        sres = ResidualsDarcy(model=smodel, fd_acc=2, pixels_per_dim=64, pixels_at_boundary=True, reverse_d1=True,
                              device=dev, bcs=b, domain_length=1.)
        se = SampleEngine(smodel, DenoisingDiffusion(100, dev), sres, batch=16, use_graph=True)
        for _ in range(5):                     # capture + warm-up
            te.step(x0)
        se.sample(x_init=x_T)
        for fn, _ in kern[b].values():
            for _ in range(3):
                fn()
        torch.cuda.synchronize()
        eng[b] = (te, se)

    rows = {b: [] for b in FLAGS}
    for rnd in range(args.rounds):
        for b in FLAGS:
            row = {'round': rnd, 'bcs': b}
            for k, (fn, nbytes) in kern[b].items():
                ms = timed(fn, 10)
                row[k + '_ms'] = ms
                row[k + '_gbs'] = nbytes / ms / 1e6
            te, se = eng[b]
            row['train_step_ms'] = timed(lambda: te.step(x0), 20)
            row['sample_100_ms'] = timed(lambda: se.sample(x_init=x_T), 1)
            rows[b].append(row)
            print(json.dumps(row), flush=True)
    summary = {}
    for b, rs in rows.items():
        for k in ('fwd_gbs', 'loss_gbs', 'train_step_ms', 'sample_100_ms'):
            v = [rw[k] for rw in rs]
            summary[f'{b}.{k}'] = dict(mean=statistics.mean(v), min=min(v), max=max(v))
    for k in ('fwd_gbs', 'loss_gbs', 'train_step_ms', 'sample_100_ms'):
        summary['periodic/none.' + k] = summary[f'periodic.{k}']['mean'] / summary[f'none.{k}']['mean']
    print(json.dumps({'summary': summary}), flush=True)


if __name__ == '__main__':
    main()
