"""Topology-optimisation sampling and its evaluation solve, timed in alternating rounds in one process on one GPU (bf16).

  - sampling: per-step time of the eager drop-in `DenoisingDiffusion.p_sample_loop` (conditioning input,
    eval_residuals / return_optimizer / return_inequality as sample.py runs it) against `SampleEngine` (CUDA graph,
    10 steps per graph) for the reference's model, Unet3D(dim=128, channels=10, out_dim=3, sigmoid_last_channel), over
    100 steps at batch 5 (sample.py) and 32; the evaluation metrics are off in both arms;
  - solver: `fem_solve` (torch ops, a host check every 50 iterations) against `fem_solve_fused` (one launch) on
    binarised designs (rho in {1e-3, 1}) at B = 5, 32, 132 and 256, with the fused solve's iteration counts and the
    largest relative difference between the two compliances.
Prints the card name and power limit first (read-only query), one JSON line per measurement, then a summary (min /
median / max over the rounds).

    python scripts/bench_mech_sample.py [--rounds 5] [--solver-rounds 3] [--out results.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, out


def conditioning(B, seed, dev):
    g = torch.Generator().manual_seed(seed)
    cond = torch.rand(B, 3, 65, 65, generator=g)
    cond[:, 0] = (0.3 + 0.4 * torch.rand(B, generator=g))[:, None, None]
    bcs = torch.zeros(B, 4, 65, 65)
    bcs[:, 0, :, 0] = 1.
    bcs[:, 1, :, 0] = 1.
    bcs[:, 3, 32, 64] = -1.
    return cond.to(dev), bcs.to(dev)


def designs(B, seed, dev):
    """binarised smooth random fields under a clamped left edge and a load at a random height of the right edge"""
    g = torch.Generator().manual_seed(seed)
    i = torch.arange(64, dtype=torch.float32) / 63
    X, Y = torch.meshgrid(i, i, indexing='ij')
    k = torch.randint(1, 5, (B, 5, 2), generator=g).float()
    a, ph = torch.randn(B, 5, 1, 1, generator=g), 6 * torch.rand(B, 5, 1, 1, generator=g)
    f = (a * torch.sin(3.1 * k[..., 0, None, None] * X + ph) * torch.cos(3.1 * k[..., 1, None, None] * Y)).sum(1)
    thr = f.reshape(B, -1).quantile(0.45, dim=1)[:, None, None]
    rho = torch.where(f > thr, torch.ones_like(f), torch.full_like(f, 1e-3))
    bcs = torch.zeros(B, 4, 65, 65)
    bcs[:, 0, :, 0] = 1.
    bcs[:, 1, :, 0] = 1.
    rows = torch.randint(4, 60, (B,), generator=g)
    bcs[torch.arange(B), 3, rows, 64] = -1.
    return rho.to(dev), bcs.to(dev)


def summary(xs):
    return {'min': min(xs), 'median': statistics.median(xs), 'max': max(xs)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--solver-rounds', type=int, default=3)
    ap.add_argument('--steps', type=int, default=100)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'needs a CUDA device'
    from physicsinformeddiffusionmodels_b200 import ops
    from physicsinformeddiffusionmodels_b200.denoising_utils import DenoisingDiffusion
    from physicsinformeddiffusionmodels_b200.engine import SampleEngine
    from physicsinformeddiffusionmodels_b200.residuals_mechanics_K import ResidualsMechanics
    from physicsinformeddiffusionmodels_b200.unet_model import Unet3D
    results = {'card': card()}
    print(json.dumps(results), flush=True)
    dev = torch.device('cuda')
    ops.set_precision('bf16')
    torch.manual_seed(0)
    model = Unet3D(dim=128, channels=10, out_dim=3, sigmoid_last_channel=True).to(dev).eval()
    diff = DenoisingDiffusion(args.steps, dev)
    res = ResidualsMechanics(model=model, pixels_per_dim=64, pixels_at_boundary=True, no_BC_folder='', device=dev)

    # ---- sampling ------------------------------------------------------------------------------------------------
    samp = {}
    for B in (5, 32):
        cond, bcs = conditioning(B, B, dev)
        eng = SampleEngine(model, diff, res, batch=B, image_shape=(3, 65, 65), use_graph=True, steps_per_graph=10)
        eager = lambda: diff.p_sample_loop((cond, bcs, None), (B, 3, 65, 65), surpress_noise=True, residual_func=res,
                                           eval_residuals=True, return_optimizer=True, return_inequality=True)
        engine = lambda: eng.sample(conditioning_input=(cond, bcs, None))
        eager()
        engine()                                            # capture + warm-up
        t_e, t_g = [], []
        for r in range(args.rounds):
            t_e.append(wall(eager)[0] / args.steps)
            t_g.append(wall(engine)[0] / args.steps)
            print(json.dumps({'sampling': B, 'round': r, 'eager_ms_per_step': t_e[-1], 'engine_ms_per_step': t_g[-1]}),
                  flush=True)
        samp[B] = {'eager_ms_per_step': summary(t_e), 'engine_ms_per_step': summary(t_g)}
        del eng
    results['sampling'] = samp

    # ---- evaluation solve ----------------------------------------------------------------------------------------
    solv = {}
    for B in (5, 32, 132, 256):
        rho, bcs = designs(B, 100 + B, dev)
        f = bcs[:, 2:4] * (bcs[:, :2] == 0)
        res.fem_solve_fused(rho, bcs)
        t_t, t_f = [], []
        for r in range(args.solver_rounds):
            tt, u_t = wall(lambda: res.fem_solve(rho, bcs))
            tf, (u_f, iters, relres) = wall(lambda: res.fem_solve_fused(rho, bcs))
            t_t.append(tt)
            t_f.append(tf)
            c_t, c_f = (u_t * f).sum(dim=(1, 2, 3)), (u_f * f).sum(dim=(1, 2, 3))
            it = iters.cpu().tolist()
            line = {'solver': B, 'round': r, 'fem_solve_ms': tt, 'fused_ms': tf, 'iters_min': min(it),
                    'iters_median': statistics.median(it), 'iters_max': max(it),
                    'all_converged': bool((relres < 1e-6).all()),
                    'max_rel_compliance_diff': ((c_f - c_t).abs() / c_t.abs()).max().item()}
            print(json.dumps(line), flush=True)
        solv[B] = {'fem_solve_ms': summary(t_t), 'fused_ms': summary(t_f), 'iters_min': line['iters_min'],
                   'iters_median': line['iters_median'], 'iters_max': line['iters_max']}
    results['solver'] = solv
    print(json.dumps(results, indent=1), flush=True)
    if args.out:
        with open(args.out, 'w') as fh:
            json.dump(results, fh, indent=1)


if __name__ == '__main__':
    main()
