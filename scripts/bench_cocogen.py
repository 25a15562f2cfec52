"""CoCoGen residual corrections, timed in alternating rounds in one process on one GPU.

  (a) corrections alone on fields of batch B = 16 and 64, M = 1, 100 and 1000 corrections:
      - kernel:   one `pidm_darcy_cocogen` launch with steps = M;
      - graph:    M copies of the multi-launch correction `ResidualsDarcy.residual_correction` used to be (residual,
                  2r, adjoint, Jacobian maximum, clamp, divide, update, residual), captured in one CUDA graph;
      - dropin:   what `DenoisingDiffusion.p_sample_loop` does after the loop, M `residual_correction` calls with their
                  layout copies, eager;
      - dropin_old: the same loop with the multi-launch correction, eager (the post-loop path before this kernel).
  (b) the 100-step Darcy sampling loop at batch 16, Unet3D(dim=32), bf16: `SampleEngine` without corrections,
      `SampleEngine` with N_correction=10, M_correction=100, 'xt', and the drop-in `p_sample_loop` with the same settings.
Times are CUDA-event times of whole calls (ms).  Prints the card name and power limit first (read-only query), one JSON
line per measurement, then a summary (min / median / max over the rounds).

    python scripts/bench_cocogen.py [--rounds 5] [--out results.json]
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
P = 64


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def timed(fn, reps=1):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def summary(xs):
    return {'min': min(xs), 'median': statistics.median(xs), 'max': max(xs)}


def fields(B, seed, dev):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 2, P, P, generator=g)
    x[:, 1] = (0.5 * x[:, 1]).exp()
    return x.to(dev)


def old_correction(res, x0_pred_in):
    """the multi-launch residual_correction this kernel replaced, on a [B, P*P, 2] tensor (updated in place)"""
    from physicsinformeddiffusionmodels_b200 import ops
    from physicsinformeddiffusionmodels_b200._lib import call, stream
    from physicsinformeddiffusionmodels_b200.grad_utils import generalized_b_xy_c_to_image
    img = generalized_b_xy_c_to_image(x0_pred_in).contiguous().float()
    B = img.shape[0]
    r = ops.darcy_residual(img, res.f_s_flat, *res.geometry)
    gx = torch.empty_like(img)
    call('pidm_darcy_residual_bwd', img, res.f_s_flat, (2.0 * r).contiguous(), gx, B, P, *res._abi_geometry(), stream())
    mx = torch.empty(B, device=img.device, dtype=torch.float32)
    call('pidm_darcy_jacobian_max', img, mx, B, P, *res._abi_geometry(), stream())
    eps = 1.e-6 / torch.clamp(mx, max=1e12)
    x0_pred_in[:, :, 0] -= eps.unsqueeze(1) * gx[:, 0].reshape(B, -1)
    return x0_pred_in, ops.darcy_residual(generalized_b_xy_c_to_image(x0_pred_in).contiguous().float(), res.f_s_flat,
                                          *res.geometry)


def post_loop(res, cur_x, M, correction):
    """p_sample_loop's post-loop corrections (denoising_utils.py), with the given correction function"""
    from physicsinformeddiffusionmodels_b200.grad_utils import generalized_b_xy_c_to_image, generalized_image_to_b_xy_c
    for _ in range(M):
        cm, _ = correction(generalized_image_to_b_xy_c(cur_x.clone()))
        cur_x = generalized_b_xy_c_to_image(cm).contiguous()
    return cur_x


def corrections_alone(res, rounds, dev):
    out = {}
    for B in (16, 64):
        x0 = fields(B, B, dev)
        for M in (1, 100, 1000):
            xk, rk = x0.clone(), torch.empty(B, P * P, 3, device=dev)
            kernel = lambda: res.cocogen(xk, rk, M)
            xg = x0.clone().permute(0, 2, 3, 1).reshape(B, P * P, 2)      # a b_xy_c view of an image buffer
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                old_correction(res, xg)
            torch.cuda.current_stream().wait_stream(s)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                for _ in range(M):
                    old_correction(res, xg)
            # one-time correctness check of the timed arms on the same input
            xa = x0.clone()
            res.cocogen(xa, rk, M)
            xb = post_loop(res, x0.clone(), M, lambda v: old_correction(res, v))
            d, db = (xa - x0)[:, 0], (xb - x0)[:, 0]
            check = ((d - db).norm() / db.norm().clamp_min(1e-30)).item()
            arms = {'kernel': kernel, 'graph': graph.replay,
                    'dropin': lambda: post_loop(res, x0, M, res.residual_correction),
                    'dropin_old': lambda: post_loop(res, x0, M, lambda v: old_correction(res, v))}
            reps = {'kernel': max(1, 200 // M), 'graph': max(1, 20 // M), 'dropin': 1, 'dropin_old': 1}
            for name, fn in arms.items():
                fn()                                                    # warm-up
            ts = {name: [] for name in arms}
            for r in range(rounds):
                for name, fn in arms.items():
                    ts[name].append(timed(fn, reps[name]))
                print(json.dumps({'corrections': {'B': B, 'M': M}, 'round': r, **{k + '_ms': v[-1] for k, v in ts.items()}}),
                      flush=True)
            out[f'B{B}_M{M}'] = {**{k + '_ms': summary(v) for k, v in ts.items()}, 'delta_rel_diff_kernel_vs_old': check}
            del graph
    return out


def sampling_loop(rounds, dev, n_steps=100, B=16):
    from physicsinformeddiffusionmodels_b200 import ops
    from physicsinformeddiffusionmodels_b200.denoising_utils import DenoisingDiffusion
    from physicsinformeddiffusionmodels_b200.engine import SampleEngine
    from physicsinformeddiffusionmodels_b200.residuals_darcy import ResidualsDarcy
    from physicsinformeddiffusionmodels_b200.unet_model import Unet3D
    ops.set_precision('bf16')
    torch.manual_seed(0)
    model = Unet3D(dim=32, channels=2).to(dev).eval()
    diff = DenoisingDiffusion(n_steps, dev)
    res = ResidualsDarcy(model=model, fd_acc=2, pixels_per_dim=P, pixels_at_boundary=True, reverse_d1=True, device=dev,
                         bcs='none', domain_length=1.)
    kw = dict(N_correction=10, M_correction=100, correction_mode='xt')
    plain = SampleEngine(model, diff, res, batch=B)
    corr = SampleEngine(model, diff, res, batch=B, **kw)
    arms = {'engine_plain': plain.sample, 'engine_cocogen': corr.sample,
            'dropin_cocogen': lambda: diff.p_sample_loop(None, (B, 2, P, P), surpress_noise=True, residual_func=res,
                                                         eval_residuals=True, **kw)}
    for fn in arms.values():
        fn()                                                            # capture + warm-up
    ts = {name: [] for name in arms}
    for r in range(rounds):
        for name, fn in arms.items():
            ts[name].append(timed(fn))
        print(json.dumps({'sampling': {'B': B, 'steps': n_steps}, 'round': r, **{k + '_ms': v[-1] for k, v in ts.items()}}),
              flush=True)
    return {k + '_ms': summary(v) for k, v in ts.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'needs a CUDA device'
    from physicsinformeddiffusionmodels_b200.residuals_darcy import ResidualsDarcy
    results = {'card': card()}
    print(json.dumps(results), flush=True)
    dev = torch.device('cuda')
    res = ResidualsDarcy(model=None, fd_acc=2, pixels_per_dim=P, pixels_at_boundary=True, reverse_d1=True, device=dev,
                         bcs='none', domain_length=1.)
    with torch.no_grad():
        results['corrections'] = corrections_alone(res, args.rounds, dev)
        results['sampling'] = sampling_loop(args.rounds, dev)
    print(json.dumps(results, indent=1), flush=True)
    if args.out:
        with open(args.out, 'w') as fh:
            json.dump(results, fh, indent=1)


if __name__ == '__main__':
    main()
