"""Device time of the linear-attention block at the 32-channel levels, old composition against the block op.

    python scripts/bench_linattn_block.py [--rounds 5] [--reps 20]

old = pidm_linattn_fused_* plus the to_out 1x1 convolution (forward with bias and residual, dgrad, weight gradient) and
the bias column sum; new = pidm_linattn_block_* plus the bias column sum.  Each phase -- forward, main-stream backward
(everything that produces dxn), weight-gradient-stream work -- is captured `reps` times into a CUDA graph and timed by
replay with CUDA events; the two compositions alternate for `rounds` rounds.  Shapes: batch 32 at 64x64 and 32x32, the
Darcy training step's.  Prints one line per (shape, phase) and a JSON summary."""
import argparse
import json
import math
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from physicsinformeddiffusionmodels_b200 import packing  # noqa: E402
from physicsinformeddiffusionmodels_b200._lib import call  # noqa: E402


def setup(B, H):
    dev = 'cuda'
    N = H * H
    g = torch.Generator(device=dev).manual_seed(B * 1000 + H)
    r = lambda *s, scale=1.0: torch.randn(*s, generator=g, device=dev) * scale
    wq = torch.nn.Parameter(r(768, 32, 1, 1, 1, scale=1.5 / math.sqrt(32)))
    wo = torch.nn.Parameter(r(32, 256, 1, 1, 1, scale=1 / 16))
    sq, so = packing.ConvSpec(wq, 'conv', 1, 1, 1, 0), packing.ConvSpec(wo, 'conv', 1, 1, 1, 0)
    pk = packing.WeightPacker()
    pk.add(sq)
    pk.add(so)
    pk.refresh(torch.bfloat16)
    bf = lambda *s: r(*s).bfloat16()
    t = dict(B=B, H=H, N=N, sq=sq, so=so, pk=pk, xn=bf(B, N, 32), x=bf(B, N, 32), dy=bf(B, N, 32), bo=r(32),
             out=bf(B, N, 256), dout=bf(B, N, 256), y=bf(B, N, 32), dxn=bf(B, N, 32),
             ctx=r(B, 8, 32, 32), dctx=r(B, 8, 32, 32), kmax=r(B, 8, 32), kzinv=r(B, 8, 32),
             ws=r(call('pidm_linattn_fused_workspace_floats', B, N)), gq=r(768, 32), go=r(32, 256), gb=r(32))
    return t


def phases(t, s):
    """{phase: {'old': fn, 'new': fn}} -- each fn enqueues one instance of the phase on stream handle s"""
    B, H, N, sq, so = t['B'], t['H'], t['N'], t['sq'], t['so']

    def old_fwd():
        call('pidm_linattn_fused_fwd', t['xn'], sq.wp_fwd, t['out'], t['ctx'], t['kmax'], t['kzinv'], t['ws'], B, N, s)
        call('pidm_conv2d_tc_general', t['out'], so.wp_fwd, t['bo'], t['x'], t['y'], B, H, H, 256, H, H, 32, 1, 1, 1, 0,
             0, None, 0, 0, s)

    def new_fwd():
        call('pidm_linattn_block_fwd', t['xn'], sq.wp_fwd, so.wp_fwd, t['bo'], t['x'], t['y'], t['ctx'], t['kmax'],
             t['kzinv'], t['ws'], B, N, s)

    def old_bwd():
        call('pidm_conv2d_tc_general', t['dy'], so.wp_dgrad, None, None, t['dout'], B, H, H, 32, H, H, 256, 1, 1, 1, 0,
             0, None, 0, 0, s)
        call('pidm_linattn_fused_bwd', t['xn'], sq.wp_fwd, t['dout'], t['ctx'], t['kmax'], t['kzinv'], t['dxn'],
             t['dctx'], B, N, s)

    def new_bwd():
        call('pidm_linattn_block_bwd', t['xn'], sq.wp_fwd, so.wp_fwd, t['dy'], t['ctx'], t['kmax'], t['kzinv'],
             t['dxn'], t['dctx'], B, N, s)

    def old_wgrad():
        call('pidm_conv2d_wgrad_tc', t['out'], t['dy'], t['go'], B, H, H, 256, 256, H, H, 32, 1, 1, 1, 0,
             so.w_stride_c, so.w_stride_n, s)
        call('pidm_colsum', t['dy'], t['gb'], B * N, 32, 1, s)
        call('pidm_linattn_fused_wgrad', t['xn'], sq.wp_fwd, t['dout'], t['ctx'], t['dctx'], t['kmax'], t['kzinv'],
             t['gq'], B, N, sq.w_stride_n, sq.w_stride_c, s)

    def new_wgrad():
        call('pidm_linattn_block_wgrad', t['xn'], sq.wp_fwd, so.wp_fwd, t['dy'], t['ctx'], t['dctx'], t['kmax'],
             t['kzinv'], t['gq'], sq.w_stride_n, sq.w_stride_c, t['go'], so.w_stride_n, so.w_stride_c, B, N, s)
        call('pidm_colsum', t['dy'], t['gb'], B * N, 32, 1, s)

    return {'forward': {'old': old_fwd, 'new': new_fwd}, 'backward (main stream)': {'old': old_bwd, 'new': new_bwd},
            'weight gradient (side stream)': {'old': old_wgrad, 'new': new_wgrad}}


def graph_of(fn, st, reps):
    with torch.cuda.stream(st):
        fn()
        fn()
    st.synchronize()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr, stream=st):
        for _ in range(reps):
            fn()
    with torch.cuda.stream(st):
        gr.replay()
    st.synchronize()
    return gr


def time_graph(gr, st, reps, replays=5):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(st):                # replay() launches on the current stream
        e0.record(st)
        for _ in range(replays):
            gr.replay()
        e1.record(st)
    st.synchronize()
    return e0.elapsed_time(e1) * 1000.0 / (replays * reps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--reps', type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_linattn_block: needs a CUDA device')
    st = torch.cuda.Stream()
    s = st.cuda_stream
    summary = {'device': torch.cuda.get_device_name(0), 'rounds': a.rounds, 'unit': 'us per call', 'shapes': {}}
    for B, H in ((32, 64), (32, 32)):
        t = setup(B, H)
        ph = phases(t, s)
        graphs = {(p, v): graph_of(fn, st, a.reps) for p, d in ph.items() for v, fn in d.items()}
        times = {k: [] for k in graphs}
        for _ in range(a.rounds):
            for p in ph:
                for v in ('old', 'new'):
                    times[(p, v)].append(time_graph(graphs[(p, v)], st, a.reps))
        res = {}
        for p in ph:
            o, n = times[(p, 'old')], times[(p, 'new')]
            res[p] = {'old_mean': statistics.mean(o), 'new_mean': statistics.mean(n), 'old_min': min(o), 'old_max': max(o),
                      'new_min': min(n), 'new_max': max(n)}
            print(f'B={B} {H}x{H} {p:30s} old {statistics.mean(o):8.2f} us [{min(o):.2f}, {max(o):.2f}]   '
                  f'new {statistics.mean(n):8.2f} us [{min(n):.2f}, {max(n):.2f}]')
        summary['shapes'][f'{B}x{H}x{H}'] = res
        del graphs
    print(json.dumps(summary))


if __name__ == '__main__':
    main()
