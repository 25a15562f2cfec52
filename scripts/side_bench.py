"""Side measurements of the study options, one family each, in one process on one GPU.

    python scripts/side_bench.py [--rounds 5] [--out FILE] FAMILY [FAMILY ...]

Builds the library, prints the card's name, power limit and maximum SM clock (a read-only query), then for each family
one JSON line per timed round and the family's results; --out also writes all results to FILE.  The arms of a family are
warmed by one untimed round (which also captures their CUDA graphs) and then timed in turn, round after round, so that
drifting clocks and neighbours on the host reach every arm alike.  A summary is {min, median, max, mean} over the rounds.
The figures in DESIGN.md §7 and README.md come from these families.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DEV = torch.device('cuda')
P = 64
PIX = P * P
STEPS = 100                                                    # diffusion steps of every model and sampling loop

# algorithmic bytes per sample of the standalone kernels: fp32 planes of P x P unless noted
DARCY_BYTES = {'fwd': (2 + 3) * PIX * 4,                       # read x0_hat, write the 3-plane residual
               'loss': (2 + 2 + 2) * PIX * 4}                  # read x0_hat and the target, write the gradient
GUIDANCE_BYTES = {'abs_residual_grad': (2 + 2) * PIX * 4,      # read x_t, write cond
                  'cond_embed_fwd': 2 * PIX * 4 + 32 * PIX * 2}  # read cond, write the bf16 activation at 32 channels
# the Darcy generator's banded Cholesky: n = 4096 unknowns, half-bandwidth b = 195
N_PTS, BW = 4096, 195
FACTOR_FLOP = N_PTS * BW * (BW + 3) + 2 * N_PTS * BW          # Cholesky + forward substitution, per sample
FACTOR_BYTES = 2 * N_PTS * (BW + 1) * 8                        # read the band of N, write the band of L
PEAK_FP64, PEAK_FP64_TC, PEAK_BW = 34e12, 67e12, 3.35e12       # H100 SXM data sheet

MECH_CFG = dict(dim=128, channels=10, out_dim=3, sigmoid_last_channel=True)   # the topology-optimisation U-Net


# ---- shared measurement helpers --------------------------------------------------------------------------------------

def card():
    """the card's name, power limit and maximum SM clock (a read-only query), else torch's device name"""
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30)
        if q.returncode == 0 and q.stdout.strip():
            return q.stdout.strip().splitlines()[0]
    except (OSError, subprocess.TimeoutExpired):
        pass
    return torch.cuda.get_device_name()


def event_ms(fn, reps=1):
    """CUDA-event ms per call over `reps` back-to-back calls, started on an idle device"""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def wall(fn):
    """(host ms, result) of one call between two device synchronisations, for calls that synchronise on the host"""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, out


def spread(xs):
    return {'min': min(xs), 'median': statistics.median(xs), 'max': max(xs), 'mean': statistics.mean(xs)}


def alternate(arms, rounds, tag, timer=event_ms):
    """Time arms = {key: (fn, reps)} or {key: (fn, reps, bytes per call)} in turn for `rounds` rounds after one untimed
    round.  timer(fn, reps) gives the ms per call kept under `key`; an arm with a byte count also gives GB/s under `key`
    with its '_ms' suffix replaced by '_gbs'.  Prints one JSON line per round, led by `tag`; returns {key: spread}."""
    for fn, reps, *_ in arms.values():
        timer(fn, reps)
    ts = {}
    for r in range(rounds):
        row = {}
        for k, (fn, reps, *nbytes) in arms.items():
            row[k] = ms = timer(fn, reps)
            if nbytes:
                row[k.removesuffix('_ms') + '_gbs'] = nbytes[0] / ms / 1e6
        print(json.dumps({**tag, 'round': r, **row}), flush=True)
        for k, v in row.items():
            ts.setdefault(k, []).append(v)
    return {k: spread(v) for k, v in ts.items()}


# ---- shared inputs ---------------------------------------------------------------------------------------------------

def darcy_state_dict():
    """the weights of every Darcy arm: Unet3D(dim=32, channels=2) initialised under torch.manual_seed(0)"""
    from physicsinformeddiffusionmodels_b200.unet_model import Unet3D
    torch.manual_seed(0)
    return Unet3D(dim=32, channels=2).state_dict()


def darcy(sd, bcs='none', padding_mode='zeros', guidance=False, eval_mode=False):
    """(model, diffusion, residuals) of the Darcy study with the weights `sd`"""
    from physicsinformeddiffusionmodels_b200.denoising_utils import DenoisingDiffusion
    from physicsinformeddiffusionmodels_b200.residuals_darcy import ResidualsDarcy
    from physicsinformeddiffusionmodels_b200.unet_model import Unet3D
    model = Unet3D(dim=32, channels=2, padding_mode=padding_mode).to(DEV)
    model.load_state_dict(sd)
    if eval_mode:
        model.eval()
    res = ResidualsDarcy(model=model, fd_acc=2, pixels_per_dim=P, pixels_at_boundary=True, reverse_d1=True, device=DEV,
                         bcs=bcs, domain_length=1., residual_grad_guidance=guidance)
    return model, DenoisingDiffusion(STEPS, DEV, residual_grad_guidance=guidance), res


def darcy_inputs():
    """the seeded Darcy training batch x0 [32, 2, P, P] and sampling start x_T [16, 2, P, P]"""
    g = torch.Generator().manual_seed(1234)
    return torch.randn(32, 2, P, P, generator=g).to(DEV), torch.randn(16, 2, P, P, generator=g).to(DEV)


def mech_conditioning(B, seed):
    """(conditioning [B, 3, 65, 65], bcs [B, 4, 65, 65]) of the topology-optimisation study: a random volume fraction,
    the left edge clamped and a unit load at the middle of the right edge"""
    g = torch.Generator().manual_seed(seed)
    cond = torch.rand(B, 3, 65, 65, generator=g)
    cond[:, 0] = (0.3 + 0.4 * torch.rand(B, generator=g))[:, None, None]
    bcs = torch.zeros(B, 4, 65, 65)
    bcs[:, 0, :, 0] = 1.
    bcs[:, 1, :, 0] = 1.
    bcs[:, 3, 32, 64] = -1.
    return cond.to(DEV), bcs.to(DEV)


def mechanics_residuals(model):
    from physicsinformeddiffusionmodels_b200.residuals_mechanics_K import ResidualsMechanics
    return ResidualsMechanics(model=model, pixels_per_dim=P, pixels_at_boundary=True, no_BC_folder='', device=DEV)


# ---- the families ----------------------------------------------------------------------------------------------------

def periodic(rounds):
    """bcs='none' against bcs='periodic', per setting:
      - the residual kernel (pidm_darcy_residual_fwd) and the fused loss + gradient kernel (pidm_darcy_pidm_loss) at
        B = 32768, in GB/s over the algorithmic bytes bench.py uses (DARCY_BYTES);
      - the CUDA-graph-replayed Darcy TrainEngine step at batch 32 (bf16);
      - a 100-step SampleEngine loop at batch 16 (bf16, CUDA graph)."""
    from physicsinformeddiffusionmodels_b200._lib import call, stream
    from physicsinformeddiffusionmodels_b200.engine import SampleEngine, TrainEngine
    B = 32768                                  # 2.7 GB working set, far beyond L2
    x = torch.randn(B, 2, P, P, device=DEV)
    fs = torch.zeros(PIX, device=DEV)
    fs[:8 * P].view(8, P)[:, :8] = 10.0
    r = torch.empty(B, PIX, 3, device=DEV)
    tgt = torch.randn_like(x)
    t = torch.randint(0, 100, (B,), device=DEV)
    tab = torch.rand(100, device=DEV) + 0.1
    sums = torch.zeros(3, device=DEV)
    gx = torch.empty_like(x)
    sd = darcy_state_dict()
    x0, x_T = darcy_inputs()
    arms = {}
    for bcs, f in (('none', 1), ('periodic', 3)):     # PIDM_DARCY_PIXELS_AT_BOUNDARY (| PIDM_DARCY_PERIODIC)
        te = TrainEngine(*darcy(sd, bcs), use_graph=True)
        se = SampleEngine(*darcy(sd, bcs, eval_mode=True), batch=16, use_graph=True)
        arms[f'{bcs}.fwd_ms'] = (lambda f=f: call('pidm_darcy_residual_fwd', x, fs, r, B, P, 1.0, 1, f, stream()), 10,
                                 B * DARCY_BYTES['fwd'])
        arms[f'{bcs}.loss_ms'] = (lambda f=f: call('pidm_darcy_pidm_loss', x, x, tgt, fs, t, tab, tab, 1.0, 1e-3, sums, gx,
                                                   None, B, P, 1.0, 1, f, stream()), 10, B * DARCY_BYTES['loss'])
        arms[f'{bcs}.train_step_ms'] = (lambda te=te: te.step(x0), 20)
        arms[f'{bcs}.sample_100_ms'] = (lambda se=se: se.sample(x_init=x_T), 1)
    s = alternate(arms, rounds, {'family': 'periodic'})
    for k in ('fwd_gbs', 'loss_gbs', 'train_step_ms', 'sample_100_ms'):
        s['periodic/none.' + k] = s[f'periodic.{k}']['mean'] / s[f'none.{k}']['mean']
    return s


def circular_keys(sd):
    """a zeros-padded Unet3D state dict keyed for padding_mode='circular' (up-sampling convolutions in `conv_transpose`)"""
    out = {}
    for k, v in sd.items():
        parts = k.split('.')
        if parts[0] == 'ups' and parts[2] == '3':
            k = '.'.join(parts[:3] + ['conv_transpose'] + parts[3:])
        out[k] = v
    return out


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


def circular(rounds):
    """Unet3D(padding_mode='zeros') against padding_mode='circular' (bf16 activations, CUDA graphs, same weights and
    inputs), per setting:
      - the graph-replayed Darcy TrainEngine step at batch 32;
      - a 100-step SampleEngine loop at batch 16;
      - the mechanics TrainEngine step, Unet3D(dim=128, channels=10, out_dim=3), batch 32 (bench.py's configuration).
    Both padding modes run the Darcy residual with bcs='periodic' (the setting a circular model is meant for), so the
    ratios measure the halo copies alone.  Also the halo kernel (pidm_wrap_pad_nhwc) at a large standalone size in GB/s
    (bytes read + written), and the halo bytes and launches per Darcy step computed from the layer shapes."""
    from physicsinformeddiffusionmodels_b200._lib import call, stream
    from physicsinformeddiffusionmodels_b200.denoising_utils import DenoisingDiffusion
    from physicsinformeddiffusionmodels_b200.engine import SampleEngine, TrainEngine
    from physicsinformeddiffusionmodels_b200.unet_model import Unet3D
    # 64 x [64, 64, 256] bf16 -> halo 1: about 0.55 GB moved per call
    xs = torch.randn(64, 64, 64, 256, device=DEV).bfloat16()
    ys = torch.empty(64, 66, 66, 256, device=DEV, dtype=torch.bfloat16)
    arms = {'halo_kernel_ms': (lambda: call('pidm_wrap_pad_nhwc', xs, ys, 64, 64, 64, 256, 1, 1, stream()), 20,
                               (xs.numel() + ys.numel()) * 2)}
    sd = darcy_state_dict()
    torch.manual_seed(0)
    sd_m = Unet3D(**MECH_CFG).state_dict()
    x0, x_T = darcy_inputs()
    cond, bcs = mech_conditioning(32, seed=32)
    g = torch.Generator().manual_seed(33)
    xm = torch.cat((0.2 * torch.randn(32, 2, 65, 65, generator=g),
                    torch.rand(32, 1, 65, 65, generator=g).clamp(1e-3, 1.)), 1).to(DEV)
    inp_m = torch.cat((cond, xm, bcs), dim=1)
    for pm in ('zeros', 'circular'):
        sd_pm, sd_m_pm = (sd, sd_m) if pm == 'zeros' else (circular_keys(sd), circular_keys(sd_m))
        model, diff, res = darcy(sd_pm, 'periodic', pm)
        if pm == 'circular':
            census = halo_census(model, 32, P)
        te = TrainEngine(model, diff, res, use_graph=True)
        se = SampleEngine(*darcy(sd_pm, 'periodic', pm, eval_mode=True), batch=16, use_graph=True)
        mm = Unet3D(**MECH_CFG, padding_mode=pm).to(DEV)
        mm.load_state_dict(sd_m_pm)
        me = TrainEngine(mm, DenoisingDiffusion(STEPS, DEV), mechanics_residuals(mm), lr=1e-4, max_norm=1.0, ema_mu=0.99,
                         c_data=1.0, c_residual=1e-2, c_ineq=0., lambda_opt=1e-3, use_graph=True)
        arms[f'{pm}.darcy_train_step_ms'] = (lambda te=te: te.step(x0), 20)
        arms[f'{pm}.sample_100_ms'] = (lambda se=se: se.sample(x_init=x_T), 1)
        arms[f'{pm}.mechanics_train_step_ms'] = (lambda me=me: me.step(inp_m), 10)
    s = alternate(arms, rounds, {'family': 'circular'})
    s['halo_kernel_gbs']['shape'] = '[64,64,64,256] bf16, halo 1'
    for k in ('darcy_train_step_ms', 'sample_100_ms', 'mechanics_train_step_ms'):
        s['circular/zeros.' + k] = s[f'circular.{k}']['mean'] / s[f'zeros.{k}']['mean']
    fwd, bwd, nbytes = census
    s['darcy_step_halo'] = dict(forward_copies=fwd, backward_dy_copies=bwd, launches=fwd + bwd, bytes_written=nbytes,
                                batch=32)
    return s


def guidance(rounds):
    """Residual-gradient guidance (bf16):
      - the CUDA-graph-replayed Darcy TrainEngine step at batch 32 without guidance, and the same step with guidance;
      - the eager guidance iteration as the reference's main.py runs it (drop-in loss, backward, torch clip_grad_norm_,
        torch Adam, the per-tensor EMA) at batch 32;
      - a 100-step guidance SampleEngine loop at batch 16 (CUDA graph; two network passes per step);
      - the guidance kernels standalone at B = 32 and B = 4096, in GB/s over algorithmic bytes from shapes
        (GUIDANCE_BYTES): pidm_darcy_abs_residual_grad reads x_t and writes cond, pidm_cond_embed_fwd reads cond and
        writes the bf16 activation at 32 channels."""
    from physicsinformeddiffusionmodels_b200 import _lib
    from physicsinformeddiffusionmodels_b200.denoising_utils import EMA
    from physicsinformeddiffusionmodels_b200.engine import SampleEngine, TrainEngine
    sd = darcy_state_dict()
    x0, x_T = darcy_inputs()
    arms = {}
    for key, g in (('train_step_ms', False), ('train_step_guidance_ms', True)):
        te = TrainEngine(*darcy(sd, guidance=g), use_graph=True)
        arms[key] = (lambda te=te: te.step(x0), 20)

    # the reference's loop body (main.py:158-179) on the drop-in modules: loss, backward, clip, torch Adam, EMA
    model_e, diff_e, res_e = darcy(sd, guidance=True)
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
    arms['eager_guidance_iteration_ms'] = (eager_iteration, 5)

    se = SampleEngine(*darcy(sd, guidance=True, eval_mode=True), batch=16, use_graph=True)
    arms['sample_100_guidance_ms'] = (lambda: se.sample(x_init=x_T), 1)

    dl, rev, fl = res_e._abi_geometry()
    for B in (32, 4096):
        xt = torch.randn(B, PIX, 2, device=DEV)
        xi = xt.reshape(B, P, P, 2).permute(0, 3, 1, 2).contiguous()
        cond = torch.empty(B, PIX, 2, device=DEV)
        act = torch.empty(B, PIX, 32, device=DEV, dtype=torch.bfloat16)
        mask = torch.rand(B, device=DEV) < 0.1
        w0, b0 = torch.randn(32, 2, device=DEV), torch.randn(32, device=DEV)
        arms[f'abs_residual_grad_B{B}_ms'] = (
            lambda xi=xi, cond=cond, B=B: _lib.call('pidm_darcy_abs_residual_grad', xi, res_e.f_s_flat, cond, B,
                                                    B * PIX * 3, P, dl, rev, fl, _lib.stream()),
            20, B * GUIDANCE_BYTES['abs_residual_grad'])
        arms[f'cond_embed_fwd_B{B}_ms'] = (
            lambda cond=cond, act=act, mask=mask, w0=w0, b0=b0, B=B: _lib.call(
                'pidm_cond_embed_fwd', cond, mask, w0, b0, act, B, PIX, 32, 1, _lib.stream()),
            20, B * GUIDANCE_BYTES['cond_embed_fwd'])
    s = alternate(arms, rounds, {'family': 'guidance'})
    s['guidance/plain train step'] = s['train_step_guidance_ms']['mean'] / s['train_step_ms']['mean']
    s['eager/engine guidance iteration'] = s['eager_guidance_iteration_ms']['mean'] / s['train_step_guidance_ms']['mean']
    return s


def fields(B, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 2, P, P, generator=g)
    x[:, 1] = (0.5 * x[:, 1]).exp()
    return x.to(DEV)


def old_correction(res, x0_pred_in):
    """the multi-launch residual_correction that pidm_darcy_cocogen replaced, on a [B, P*P, 2] tensor (updated in
    place)"""
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


def cocogen(rounds):
    """CoCoGen residual corrections, CUDA-event times of whole calls (ms):
      (a) corrections alone on fields of batch B = 16 and 64, M = 1, 100 and 1000 corrections:
          - kernel:   one `pidm_darcy_cocogen` launch with steps = M;
          - graph:    M copies of the multi-launch correction `ResidualsDarcy.residual_correction` used to be
                      (residual, 2r, adjoint, Jacobian maximum, clamp, divide, update, residual), captured in one CUDA
                      graph;
          - dropin:   what `DenoisingDiffusion.p_sample_loop` does after the loop, M `residual_correction` calls with
                      their layout copies, eager;
          - dropin_old: the same loop with the multi-launch correction, eager (the post-loop path before this kernel);
          and the relative difference of the accumulated change of p between the kernel and the old correction.
      (b) the 100-step Darcy sampling loop at batch 16, Unet3D(dim=32), bf16: `SampleEngine` without corrections,
          `SampleEngine` with N_correction=10, M_correction=100, 'xt', and the drop-in `p_sample_loop` with the same
          settings."""
    from physicsinformeddiffusionmodels_b200.engine import SampleEngine
    model, diff, res = darcy(darcy_state_dict(), eval_mode=True)
    out = {'corrections': {}}
    with torch.no_grad():
        for B in (16, 64):
            x0 = fields(B, B)
            for M in (1, 100, 1000):
                xk, rk = x0.clone(), torch.empty(B, PIX, 3, device=DEV)
                xg = x0.clone().permute(0, 2, 3, 1).reshape(B, PIX, 2)      # a b_xy_c view of an image buffer
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
                arms = {'kernel_ms': (lambda: res.cocogen(xk, rk, M), max(1, 200 // M)),
                        'graph_ms': (graph.replay, max(1, 20 // M)),
                        'dropin_ms': (lambda: post_loop(res, x0, M, res.residual_correction), 1),
                        'dropin_old_ms': (lambda: post_loop(res, x0, M, lambda v: old_correction(res, v)), 1)}
                out['corrections'][f'B{B}_M{M}'] = {**alternate(arms, rounds, {'corrections': {'B': B, 'M': M}}),
                                                    'delta_rel_diff_kernel_vs_old': check}
                del graph

        kw = dict(N_correction=10, M_correction=100, correction_mode='xt')
        plain = SampleEngine(model, diff, res, batch=16)
        corr = SampleEngine(model, diff, res, batch=16, **kw)
        arms = {'engine_plain_ms': (plain.sample, 1), 'engine_cocogen_ms': (corr.sample, 1),
                'dropin_cocogen_ms': (lambda: diff.p_sample_loop(None, (16, 2, P, P), surpress_noise=True, residual_func=res,
                                                                 eval_residuals=True, **kw), 1)}
        out['sampling'] = alternate(arms, rounds, {'sampling': {'B': 16, 'steps': STEPS}})
    return out


def designs(B, seed):
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
    return rho.to(DEV), bcs.to(DEV)


def mech_sample(rounds):
    """Topology-optimisation sampling and its evaluation solve (bf16):
      - sampling: per-step host time of the eager drop-in `DenoisingDiffusion.p_sample_loop` (conditioning input,
        eval_residuals / return_optimizer / return_inequality as sample.py runs it) against `SampleEngine` (CUDA graph,
        10 steps per graph) for the reference's model, Unet3D(dim=128, channels=10, out_dim=3, sigmoid_last_channel),
        over 100 steps at batch 5 (sample.py) and 32; the evaluation metrics are off in both arms;
      - solver: `fem_solve` (torch ops, a host check every 50 iterations) against `fem_solve_fused` (one launch) on
        binarised designs (rho in {1e-3, 1}) at B = 5, 32, 132 and 256, three rounds, with the fused solve's iteration
        counts and the largest relative difference between the two compliances."""
    from physicsinformeddiffusionmodels_b200.denoising_utils import DenoisingDiffusion
    from physicsinformeddiffusionmodels_b200.engine import SampleEngine
    from physicsinformeddiffusionmodels_b200.unet_model import Unet3D
    torch.manual_seed(0)
    model = Unet3D(**MECH_CFG).to(DEV).eval()
    diff = DenoisingDiffusion(STEPS, DEV)
    res = mechanics_residuals(model)

    samp = {}
    for B in (5, 32):
        cond, bcs = mech_conditioning(B, seed=B)
        eng = SampleEngine(model, diff, res, batch=B, image_shape=(3, 65, 65), use_graph=True, steps_per_graph=10)
        arms = {'eager_ms_per_step': (lambda: diff.p_sample_loop((cond, bcs, None), (B, 3, 65, 65), surpress_noise=True,
                                                                 residual_func=res, eval_residuals=True,
                                                                 return_optimizer=True, return_inequality=True), 1),
                'engine_ms_per_step': (lambda: eng.sample(conditioning_input=(cond, bcs, None)), 1)}
        samp[B] = alternate(arms, rounds, {'sampling': B}, timer=lambda fn, reps: wall(fn)[0] / STEPS)
        del eng

    solv = {}
    for B in (5, 32, 132, 256):
        rho, bcs = designs(B, 100 + B)
        f = bcs[:, 2:4] * (bcs[:, :2] == 0)
        res.fem_solve_fused(rho, bcs)
        t_t, t_f = [], []
        for r in range(3):
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
        solv[B] = {'fem_solve_ms': spread(t_t), 'fused_ms': spread(t_f), 'iters_min': line['iters_min'],
                   'iters_median': line['iters_median'], 'iters_max': line['iters_max']}
    return {'sampling': samp, 'solver': solv}


def darcy_gen(rounds):
    """Throughput of the GPU Darcy data generator (csrc/darcy_gen.cu) against two baselines, measured once:
      - samples/s of DarcyDataGenerator.generate (z draw on the host, KLE, assembly, Cholesky, post) at 256, 1024 and
        4096 samples;
      - CUDA-event times per kernel at B = 256 (KLE, assembly, factorisation, post-processing; mean of 5);
      - the factorisation's fp64 rate from the algorithmic count n*b*(b+3) flop per sample (banded Cholesky, n = 4096,
        b = 195, plus the forward substitution it carries) and the bytes it must move (read N, write L: 2 * n * (b+1) * 8),
        against the H100 SXM data sheet (34 TFLOP/s fp64, 67 with the tensor cores, 3.35 TB/s);
      - stock PyTorch on the same GPU: batched dense fp64 torch.linalg.cholesky + cholesky_solve of N (B = 8);
      - the reference algorithm (dense scipy lstsq of the 4353 x 4096 system) on the host cores, one sample."""
    from scipy.sparse import vstack

    from oracle import darcy_gen_oracle as DO
    from physicsinformeddiffusionmodels_b200._lib import call, stream
    from physicsinformeddiffusionmodels_b200.darcy_data_generation import DarcyDataGenerator
    out = {}
    ms, gen = wall(DarcyDataGenerator)
    out['eigenpairs_s'] = ms * 1e-3

    gen.generate(range(256))
    out['samples_per_s'] = {n: n / (wall(lambda: gen.generate(range(10_000, 10_000 + n)))[0] * 1e-3)
                            for n in (256, 1024, 4096)}

    # ---- per kernel at B = 256 ----
    B = 256
    z = gen.z_for_seeds(range(B))
    K = torch.empty(B, N_PTS, dtype=torch.float64, device=DEV)
    p = torch.empty_like(K)
    res = torch.empty(B, dtype=torch.float64, device=DEV)
    need = call('pidm_darcy_gen_workspace_bytes', B, 64)
    ws = torch.empty(need, dtype=torch.uint8, device=DEV)

    def kle():
        call('pidm_darcy_gen_kle', gen.phi_s, z, K, B, gen.q, 64, stream())

    def stage(mask):
        return lambda: call('pidm_darcy_gen_solve', K, gen.f_s, p, res, None, ws, need, B, 64, 1.0, 1, 1, mask, stream())

    def factor():                    # the factorisation overwrites the band: re-assemble before each timed one
        stage(1)()
        return event_ms(stage(2))
    kle()
    stage(7)()
    kern = {'kle': event_ms(kle, 5) * 1e-3, 'assemble': event_ms(stage(1), 5) * 1e-3}
    factor()
    kern['factor'] = statistics.mean(factor() for _ in range(5)) * 1e-3
    kern['post'] = event_ms(stage(4), 5) * 1e-3
    out['kernel_s_at_B256'] = kern
    out['kernel_us_per_sample'] = {k: v / B * 1e6 for k, v in kern.items()}
    tflops = FACTOR_FLOP * B / kern['factor']
    tbs = FACTOR_BYTES * B / kern['factor']
    t_min_flop, t_min_bytes = FACTOR_FLOP * B / PEAK_FP64_TC, FACTOR_BYTES * B / PEAK_BW
    out['factor'] = dict(flop_per_sample=FACTOR_FLOP, bytes_per_sample=FACTOR_BYTES, fp64_tflops=tflops / 1e12,
                         share_of_fp64_34=tflops / PEAK_FP64, share_of_fp64_tc_67=tflops / PEAK_FP64_TC,
                         hbm_tb_per_s=tbs / 1e12, bound='bytes' if t_min_bytes > t_min_flop else 'compute',
                         share_of_bound=max(t_min_flop, t_min_bytes) / kern['factor'])

    # ---- baseline 1: stock PyTorch dense fp64 Cholesky on the same GPU ----
    Kh = K[:2].cpu().numpy()
    Ns, rhs = [], []
    for b in range(2):
        A, BC = DO.operators(Kh[b])
        MA = vstack([A, BC]).tocsr()
        Nm = (MA.T @ MA).toarray()
        Nm[0, 0] *= 2.
        Ns.append(Nm)
        rhs.append(A.T @ DO.source())
    Bt = 8
    Nd = torch.tensor(np.stack([Ns[i % 2] for i in range(Bt)]), device=DEV)
    rd = torch.tensor(np.stack([rhs[i % 2] for i in range(Bt)]), device=DEV).unsqueeze(-1)

    def torch_chol():
        L = torch.linalg.cholesky(Nd)
        return torch.cholesky_solve(rd, L)
    torch_chol()
    t = event_ms(torch_chol, 3) * 1e-3
    pt = torch_chol()[:2, :, 0].cpu().numpy()
    w = DO.weights()
    pt = pt - (pt @ w)[:, None] / w.sum()
    out['torch_dense_cholesky'] = dict(batch=Bt, s=t, samples_per_s=Bt / t,
                                       max_abs_diff_vs_generator=float(np.abs(pt - p[:2].cpu().numpy()).max()))

    # ---- baseline 2: the reference algorithm on the host ----
    th = wall(lambda: DO.solve_lstsq(Kh[0]))[0] * 1e-3
    out['host_lstsq'] = dict(cores=os.cpu_count(), s_per_sample=th, samples_per_s=1 / th)
    return out


def ema_eval(rounds):
    """Validation on the EMA weights (reference main.py:181-198), Darcy U-Net, bf16, batch 32:
      - the EMA swap in and out of TrainEngine.ema_weights() (two pidm_swap_f32 over the flat buffers), in GB/s over
        its algorithmic bytes (each of the two buffers read and written once per swap: 16 bytes per element);
      - TrainEngine.validate() replayed from its CUDA graph, and eager;
      - the whole evaluation as a training loop pays it: swap in, the repack of the bf16 operands the swap made stale,
        validate() replayed from its graph, swap out;
      - the drop-in evaluation as main.py runs it on a second model: ema.ema, model_estimation_loss (which reads the
        tracked scalars on the host), ema.restore."""
    from physicsinformeddiffusionmodels_b200.denoising_utils import EMA
    from physicsinformeddiffusionmodels_b200.engine import TrainEngine
    sd = darcy_state_dict()
    xv, _ = darcy_inputs()
    te = TrainEngine(*darcy(sd), use_graph=True)
    te_eager = TrainEngine(*darcy(sd), use_graph=False)
    model_d, diff_d, res_d = darcy(sd)
    ema = EMA(0.99)
    ema.register(model_d)

    def swap_in_out():
        te._swap_ema()
        te._swap_ema()

    def dropin():
        ema.ema(model_d)
        diff_d.model_estimation_loss(xv, residual_func=res_d, c_data=1., c_residual=1e-3, c_ineq=0., lambda_opt=0.)
        ema.restore(model_d)
    def ema_validate():
        with te.ema_weights():
            te.validate(xv)
    arms = {'swap_in_out_ms': (swap_in_out, 20, 2 * 16 * te.fp.total),
            'validate_graph_ms': (lambda: te.validate(xv), 20),
            'ema_validate_graph_ms': (ema_validate, 20),
            'validate_eager_ms': (lambda: te_eager.validate(xv), 5),
            'dropin_eval_ms': (dropin, 5)}
    s = alternate(arms, rounds, {'family': 'ema_eval'})
    s['flat_elements'] = te.fp.total
    s['dropin/engine eval'] = s['dropin_eval_ms']['mean'] / s['ema_validate_graph_ms']['mean']
    return s


FAMILIES = {'periodic': periodic, 'circular': circular, 'guidance': guidance, 'cocogen': cocogen,
            'mech_sample': mech_sample, 'darcy_gen': darcy_gen, 'ema_eval': ema_eval}


def main(argv=None):
    ap = argparse.ArgumentParser(description='Side measurements of the study options on one GPU.')
    ap.add_argument('--rounds', type=int, default=5, help='timed rounds of each alternation (default: 5)')
    ap.add_argument('--out', default=None, help='also write the JSON results to this file')
    ap.add_argument('families', nargs='+', choices=list(FAMILIES), metavar='FAMILY',
                    help=f'families to measure: {", ".join(FAMILIES)}')
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit('side_bench.py measures on the GPU: no CUDA device')
    import __graft_entry__
    __graft_entry__.build()
    from physicsinformeddiffusionmodels_b200 import ops
    ops.set_precision('bf16')
    results = {'card': card()}
    print(json.dumps(results), flush=True)
    for name in args.families:
        results[name] = FAMILIES[name](args.rounds)
        print(json.dumps({name: results[name]}, indent=1), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(results, f, indent=1)


if __name__ == '__main__':
    main()
