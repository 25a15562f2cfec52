"""Throughput of the GPU Darcy data generator (csrc/darcy_gen.cu) against two baselines on the same machine.

    python scripts/bench_darcy_gen.py [--out results.json] [--sizes 256,1024,4096]

Prints the results as JSON; --out also writes them to a file.

Reports, with the card's name and power limit read in the same run:
  * samples/s of DarcyDataGenerator.generate (z draw on the host, KLE, assembly, Cholesky, post) at each size,
  * CUDA-event times per kernel at B = 256 (KLE, assembly, factorisation, post-processing; mean of 5 after a warm-up),
  * the factorisation's fp64 rate from the algorithmic count n*b*(b+3) flop per sample (banded Cholesky, n = 4096,
    b = 195, plus the forward substitution it carries) and the bytes it must move (read N, write L: 2 * n * (b+1) * 8),
    against the H100 SXM data sheet (34 TFLOP/s fp64, 67 with the tensor cores, 3.35 TB/s),
  * stock PyTorch on the same GPU: batched dense fp64 torch.linalg.cholesky + cholesky_solve of N (B = 8),
  * the reference algorithm (dense scipy lstsq of the 4353 x 4096 system) on the host cores, one sample.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N_PTS, BW = 4096, 195
FACTOR_FLOP = N_PTS * BW * (BW + 3) + 2 * N_PTS * BW          # Cholesky + forward substitution, per sample
FACTOR_BYTES = 2 * N_PTS * (BW + 1) * 8                        # read the band of N, write the band of L
PEAK_FP64, PEAK_FP64_TC, PEAK_BW = 34e12, 67e12, 3.35e12


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'],
                            capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:          # noqa: BLE001
        pl = f'unavailable ({e})'
    return name, pl


def event_time(fn, reps=5):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) * 1e-3)
    return float(np.mean(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None, help='also write the JSON results to this file')
    ap.add_argument('--sizes', default='256,1024,4096')
    ap.add_argument('--skip-host', action='store_true')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_darcy_gen.py measures the GPU generator: no CUDA device')
    import __graft_entry__
    __graft_entry__.build()
    from physicsinformeddiffusionmodels_b200._lib import call, stream
    from physicsinformeddiffusionmodels_b200.darcy_data_generation import DarcyDataGenerator
    from oracle import darcy_gen_oracle as DO

    out = {}
    out['card'], out['power_limit_and_max_sm_clock'] = card()
    t0 = time.time()
    gen = DarcyDataGenerator()
    out['eigenpairs_s'] = time.time() - t0

    # ---- end-to-end samples/s ----
    gen.generate(range(256))
    torch.cuda.synchronize()
    out['samples_per_s'] = {}
    for n in [int(s) for s in args.sizes.split(',')]:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        gen.generate(range(10_000, 10_000 + n))
        torch.cuda.synchronize()
        out['samples_per_s'][n] = n / (time.perf_counter() - t0)

    # ---- per kernel at B = 256 ----
    B = 256
    z = gen.z_for_seeds(range(B))
    K = torch.empty(B, N_PTS, dtype=torch.float64, device='cuda')
    p = torch.empty_like(K)
    res = torch.empty(B, dtype=torch.float64, device='cuda')
    need = call('pidm_darcy_gen_workspace_bytes', B, 64)
    ws = torch.empty(need, dtype=torch.uint8, device='cuda')

    def kle():
        call('pidm_darcy_gen_kle', gen.phi_s, z, K, B, gen.q, 64, stream())

    def stage(mask):
        return lambda: call('pidm_darcy_gen_solve', K, gen.f_s, p, res, None, ws, need, B, 64, 1.0, 1, 1, mask, stream())
    kle()
    stage(7)()
    kern = {'kle': event_time(kle), 'assemble': event_time(stage(1))}
    # the factorisation overwrites the band: re-assemble before each timed factorisation
    tf = []
    for _ in range(6):
        stage(1)()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        stage(2)()
        b.record()
        b.synchronize()
        tf.append(a.elapsed_time(b) * 1e-3)
    kern['factor'] = float(np.mean(tf[1:]))
    kern['post'] = event_time(stage(4))
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
        MA = __import__('scipy.sparse', fromlist=['vstack']).vstack([A, BC]).tocsr()
        Nm = (MA.T @ MA).toarray()
        Nm[0, 0] *= 2.
        Ns.append(Nm)
        rhs.append(A.T @ DO.source())
    Bt = 8
    Nd = torch.tensor(np.stack([Ns[i % 2] for i in range(Bt)]), device='cuda')
    rd = torch.tensor(np.stack([rhs[i % 2] for i in range(Bt)]), device='cuda').unsqueeze(-1)

    def torch_chol():
        L = torch.linalg.cholesky(Nd)
        return torch.cholesky_solve(rd, L)
    t = event_time(torch_chol, reps=3)
    pt = torch_chol()[:2, :, 0].cpu().numpy()
    w = DO.weights()
    pt = pt - (pt @ w)[:, None] / w.sum()
    out['torch_dense_cholesky'] = dict(batch=Bt, s=t, samples_per_s=Bt / t,
                                       max_abs_diff_vs_generator=float(np.abs(pt - p[:2].cpu().numpy()).max()))

    # ---- baseline 2: the reference algorithm on the host ----
    if not args.skip_host:
        t0 = time.perf_counter()
        DO.solve_lstsq(Kh[0])
        th = time.perf_counter() - t0
        out['host_lstsq'] = dict(cores=os.cpu_count(), s_per_sample=th, samples_per_s=1 / th)

    print(json.dumps(out, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
