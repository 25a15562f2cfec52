"""Residual-gradient guidance, timed in alternating rounds in one process on one GPU (bf16).

Per round:
  - the CUDA-graph-replayed Darcy TrainEngine step at batch 32 without guidance, and the same step with guidance;
  - the eager guidance iteration as the reference's main.py runs it (drop-in loss, backward, torch clip_grad_norm_,
    torch Adam, the per-tensor EMA) at batch 32;
  - a 100-step guidance SampleEngine loop at batch 16 (CUDA graph; two network passes per step);
  - the guidance kernels standalone at B = 32 and B = 4096, in GB/s over algorithmic bytes from shapes:
    pidm_darcy_abs_residual_grad reads x_t (32 KiB / sample) and writes cond (32 KiB), pidm_cond_embed_fwd reads cond
    (32 KiB) and writes the bf16 activation (256 KiB at 32 channels).
Prints the card name and power limit first (read-only query), one JSON line per round, then a summary.

    python scripts/bench_guidance.py [--rounds 5]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'needs a CUDA device'
    from physicsinformeddiffusionmodels_b200 import _lib, ops
    from physicsinformeddiffusionmodels_b200.denoising_utils import EMA, DenoisingDiffusion
    from physicsinformeddiffusionmodels_b200.engine import SampleEngine, TrainEngine
    from physicsinformeddiffusionmodels_b200.residuals_darcy import ResidualsDarcy
    from physicsinformeddiffusionmodels_b200.unet_model import Unet3D
    print(json.dumps({'card': card()}), flush=True)
    dev = torch.device('cuda')
    ops.set_precision('bf16')
    torch.manual_seed(0)
    sd = Unet3D(dim=32, channels=2).state_dict()
    g = torch.Generator().manual_seed(1234)
    x0 = torch.randn(32, 2, 64, 64, generator=g).to(dev)
    x_T = torch.randn(16, 2, 64, 64, generator=g).to(dev)

    def darcy(guidance, eval_mode=False):
        model = Unet3D(dim=32, channels=2).to(dev)
        model.load_state_dict(sd)
        if eval_mode:
            model.eval()
        res = ResidualsDarcy(model=model, fd_acc=2, pixels_per_dim=64, pixels_at_boundary=True, reverse_d1=True,
                             device=dev, bcs='none', domain_length=1., residual_grad_guidance=guidance)
        return model, DenoisingDiffusion(100, dev, residual_grad_guidance=guidance), res

    work = {}
    for name, guidance in (('train_step_ms', False), ('train_step_guidance_ms', True)):
        te = TrainEngine(*darcy(guidance), use_graph=True)
        work[name] = (lambda te=te: te.step(x0), 20)

    # the reference's loop body (main.py:158-179) on the drop-in modules: loss, backward, clip, torch Adam, EMA
    model_e, diff_e, res_e = darcy(True)
    opt = torch.optim.Adam(model_e.parameters(), lr=1e-4)
    ema = EMA(0.99)
    ema.register(model_e)

    def eager_iteration():
        loss, _, _, _, _ = diff_e.model_estimation_loss(x0, residual_func=res_e, c_data=1., c_residual=1e-3, c_ineq=0.,
                                                        lambda_opt=0., sync_scalars=False)
        opt.zero_grad()
        loss.backward()
        torch.nn.utils.clip_grad_norm_(model_e.parameters(), 1.0)
        opt.step()
        ema.update(model_e)
    work['eager_guidance_iteration_ms'] = (eager_iteration, 5)

    se = SampleEngine(*darcy(True, eval_mode=True), batch=16, use_graph=True)
    work['sample_100_guidance_ms'] = (lambda: se.sample(x_init=x_T), 1)

    _, _, res_k = darcy(True)
    for B in (32, 4096):
        xt = torch.randn(B, 4096, 2, device=dev)
        xi = xt.reshape(B, 64, 64, 2).permute(0, 3, 1, 2).contiguous()
        cond = torch.empty(B, 4096, 2, device=dev)
        act = torch.empty(B, 4096, 32, device=dev, dtype=torch.bfloat16)
        mask = torch.rand(B, device=dev) < 0.1
        w0, b0 = torch.randn(32, 2, device=dev), torch.randn(32, device=dev)
        dl, rev, fl = res_k._abi_geometry()
        work[f'abs_residual_grad_B{B}'] = (
            lambda xi=xi, cond=cond, B=B: _lib.call('pidm_darcy_abs_residual_grad', xi, res_k.f_s_flat, cond, B,
                                                    B * 4096 * 3, 64, dl, rev, fl, _lib.stream()), 20, B * 65536)
        work[f'cond_embed_fwd_B{B}'] = (
            lambda cond=cond, act=act, mask=mask, B=B: _lib.call('pidm_cond_embed_fwd', cond, mask, w0, b0, act, B, 4096,
                                                                 32, 1, _lib.stream()), 20, B * (32768 + 262144))
    for k, v in work.items():                  # capture + warm-up
        for _ in range(3):
            v[0]()
        torch.cuda.synchronize()
        print(f'warmed up {k}', file=sys.stderr, flush=True)

    rows = []
    for rnd in range(args.rounds):
        row = {'round': rnd}
        for k, v in work.items():
            ms = timed(v[0], v[1])
            if len(v) == 3:
                row[k + '_gbs'] = v[2] / ms / 1e6
            else:
                row[k] = ms
        rows.append(row)
        print(json.dumps(row), flush=True)
    summary = {k: dict(mean=statistics.mean(r[k] for r in rows), min=min(r[k] for r in rows),
                       max=max(r[k] for r in rows)) for k in rows[0] if k != 'round'}
    summary['guidance/plain train step'] = (summary['train_step_guidance_ms']['mean'] /
                                            summary['train_step_ms']['mean'])
    summary['eager/engine guidance iteration'] = (summary['eager_guidance_iteration_ms']['mean'] /
                                                  summary['train_step_guidance_ms']['mean'])
    print(json.dumps({'summary': summary}), flush=True)


if __name__ == '__main__':
    main()
