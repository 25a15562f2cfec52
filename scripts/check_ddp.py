"""Multi-GPU consistency checks of the data-parallel training step (run with torchrun on >= 2 GPUs):

  torchrun --nnodes=1 --nproc-per-node=2 --master-addr 127.0.0.1 scripts/check_ddp.py [--guidance] [--validate]

--guidance runs every check with residual-gradient guidance: the classifier-free mask is drawn for the global batch
and sliced, and the guidance gradient is normalised by the global count, so part 1 holds with guidance too.

 1. the 2-rank step on row shards of a global batch, with t / eps drawn for the global batch and sliced, produces the
    same (all-reduced, averaged) flat gradient as the ONE-process step on the whole batch             (fp32, 1e-4)
 2. the bucketed / overlapped gradient exchange equals the single all-reduce: flat gradient after the exchange (5e-5)
    and bitwise-identical parameters on all ranks, eager and CUDA graph
 3. the process group is destroyed and the process exits normally (no os._exit) with captured NCCL graphs alive before.
 4. (--validate) TrainEngine.validate() inside ema_weights() on row shards, t / eps drawn for the global batch: every rank
    reports the same five values, those of the ONE-process validation of the global batch        (fp32, 1e-5), eager and
    CUDA graph (the all-reduce of the five values is captured in the graph).
"""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from physicsinformeddiffusionmodels_b200 import ops  # noqa: E402
from physicsinformeddiffusionmodels_b200.denoising_utils import DenoisingDiffusion  # noqa: E402
from physicsinformeddiffusionmodels_b200.engine import TrainEngine  # noqa: E402
from physicsinformeddiffusionmodels_b200.residuals_darcy import ResidualsDarcy  # noqa: E402
from physicsinformeddiffusionmodels_b200.unet_model import Unet3D  # noqa: E402

rank, local, world = int(os.environ['RANK']), int(os.environ['LOCAL_RANK']), int(os.environ['WORLD_SIZE'])
torch.cuda.set_device(local)
dev = torch.device('cuda', local)
dist.init_process_group('nccl', device_id=dev)
ops.set_precision(os.environ.get('PIDM_CHECK_PRECISION', 'fp32'))
PER = 8
GUIDANCE = '--guidance' in sys.argv[1:]
VALIDATE = '--validate' in sys.argv[1:]


def rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()


def build(world_, rank_, use_graph, bucketed, global_draws=True):
    torch.manual_seed(0)
    model = Unet3D(dim=32, channels=2).to(dev)
    diff = DenoisingDiffusion(100, dev, residual_grad_guidance=GUIDANCE)
    res = ResidualsDarcy(model=model, fd_acc=2, pixels_per_dim=64, pixels_at_boundary=True, reverse_d1=True, device=dev,
                         residual_grad_guidance=GUIDANCE)
    return model, TrainEngine(model, diff, res, use_graph=use_graph, world=world_, rank=rank_, bucketed_allreduce=bucketed,
                              global_draws=global_draws, snapshot_grad=True)


g = torch.Generator().manual_seed(7)
X = (0.7 * torch.randn(world * PER, 2, 64, 64, generator=g)).to(dev)       # identical on every rank
ok = True

# ---- 1. data parallel == one process on the global batch
model, eng = build(world, rank, False, False)
torch.cuda.manual_seed(4321)                                              # identical generator state on every rank
eng.step(X[rank * PER:(rank + 1) * PER])
g_ddp = eng.grad_snapshot.clone() / world
names = {id(p): n for n, p in model.named_parameters()}
lay_ddp = {names[id(p)]: o for p, o in zip(eng.fp.params, eng.fp.offsets)}
model1, eng1 = build(1, 0, False, False)
torch.cuda.manual_seed(4321)
eng1.step(X)
g_one = eng1.grad_snapshot
r1 = rel(g_ddp, g_one)
tail = eng.grad_snapshot[eng.fp.live_total:].abs().max().item()
if rank == 0:
    print(f'[1] (guidance={GUIDANCE}) {world}-rank step vs one process on the global batch of {world * PER}: rel diff of the flat gradient {r1:.3e}; '
          f'unused-parameter tail max |g| = {tail:.1e} ({eng.fp.total - eng.fp.live_total} elements not exchanged)', flush=True)
ok = ok and r1 < 1e-4 and tail == 0.0
eng.close(); eng1.close()
del eng, eng1, model, model1

# ---- 2. bucketed exchange == single all-reduce
for use_graph in (False, True):
    outs = {}
    for bucketed in (False, True):
        model, eng = build(world, rank, use_graph, bucketed)
        torch.cuda.manual_seed(99)
        for _ in range(3):
            eng.step(X[rank * PER:(rank + 1) * PER])
        torch.cuda.synchronize()
        names = {id(p): n for n, p in model.named_parameters()}
        grads = {names[id(p)]: eng.grad_snapshot[o:o + p.numel()].clone() for p, o in zip(eng.fp.params, eng.fp.offsets)}
        flat = torch.cat([p.detach().reshape(-1) for _, p in sorted(model.named_parameters())])
        ref = flat.clone()
        dist.broadcast(ref, 0)
        dmax = torch.tensor([(flat - ref).abs().max().item()], device=dev)
        dist.all_reduce(dmax, op=dist.ReduceOp.MAX)                      # worst rank (rank 0 compares with itself)
        outs[bucketed] = (grads, dmax.item(), sorted(getattr(eng, '_reduced', [])))
        eng.close()
        del eng, model
    worst = max(rel(outs[True][0][n], outs[False][0][n]) for n in outs[False][0] if outs[False][0][n].abs().max() > 0)
    if rank == 0:
        print(f'[2] graph={use_graph}: bucketed vs single all-reduce, worst per-tensor rel diff of the exchanged gradient '
              f'{worst:.3e}; max |rank diff| of the parameters {outs[True][1]:.1e} / {outs[False][1]:.1e}; groups reduced '
              f'early {outs[True][2]}', flush=True)
    ok = ok and worst < 5e-5 and outs[True][1] == 0.0 and outs[False][1] == 0.0      # fp32 atomics: order-dependent at 1e-5

# ---- 4. validation loss of the global batch on every rank
if VALIDATE:
    for use_graph in (False, True):
        model, eng = build(world, rank, use_graph, False)
        model1, eng1 = build(1, 0, False, False)
        vals = []
        for e, x in ((eng, X[rank * PER:(rank + 1) * PER]), (eng1, X)):
            torch.cuda.manual_seed(55)
            with e.ema_weights():
                vals.append(torch.stack(e.validate(x)).clone())
        v_ddp, v_one = vals
        ref = v_ddp.clone()
        dist.broadcast(ref, 0)
        same = torch.tensor([float(torch.equal(ref, v_ddp))], device=dev)
        dist.all_reduce(same, op=dist.ReduceOp.MIN)
        r4 = rel(v_ddp, v_one)
        if rank == 0:
            print(f'[4] graph={use_graph}: {world}-rank validation vs one process on the global batch: rel diff {r4:.3e}; '
                  f'ranks identical {bool(same.item())}; values {v_ddp.tolist()}', flush=True)
        ok = ok and r4 < 1e-5 and same.item() == 1.0
        eng.close(); eng1.close()
        del eng, eng1, model, model1

# ---- 3. clean teardown (every engine was close()d: no captured NCCL kernel is alive any more)
import threading
watchdog = threading.Timer(60.0, lambda: (print('TEARDOWN_HUNG', flush=True), os._exit(3)))
watchdog.daemon = True
watchdog.start()
torch.cuda.synchronize()
dist.barrier()
dist.destroy_process_group()
watchdog.cancel()
if rank == 0:
    print('DDP_CHECK_OK' if ok else 'DDP_CHECK_MISMATCH', flush=True)
sys.exit(0 if (ok or rank != 0) else 1)      # rank 0 holds the verdict (the comparisons of part 1 run there)
