"""Training-step engine: the body of the reference's loop (main.py:157-183) as a H100-native step.

    q_sample -> U-Net -> x0_hat -> Darcy residual + loss (fused) -> backward -> [NCCL all-reduce of ONE flat
    fp32 gradient buffer] -> global-norm clip + Adam + EMA (one fused kernel over the flat buffers)

* Flat buffers: parameters, gradients, Adam moments and the EMA shadow live in five flat fp32 buffers; every
  nn.Parameter is a view, and every wgrad-type kernel accumulates straight into the flat gradient
  (`_pidm_grad`, see ops._grad_buffer), so there are no per-tensor copies, no 3,303 `copy_` calls per step.
* CUDA graph: the whole step (RNG draws included) is captured once and replayed; the Adam step count lives on
  the device.  Tracked scalars stay on the device (no `.item()` syncs in the loop).
* Data parallel: one process per GPU; rank r owns rows [r*B, (r+1)*B) of the global batch; a single
  `all_reduce(SUM)` of the flat gradient per step, averaged inside the Adam kernel (grad_scale = 1/world).
"""
import contextlib

import torch
import torch.distributed as dist

from . import ops
from ._lib import call, stream

_ALIGN = 64     # elements: every parameter starts on a 256-byte boundary (float4 / TMA friendly)


class FlatParams:
    """Re-homes the trainable parameters of `model` into one flat fp32 buffer (plus grad / moment / EMA twins)."""

    def __init__(self, model, with_optimizer_state=True, group_of=None, guidance=False):
        """group_of(name) -> int (optional): parameters are laid out group by group (stable within a group), and
        `group_bounds[g] = (lo, hi)` is the flat range of group g -- the engine all-reduces ranges separately.
        Parameters the forward pass never uses (model.unused_parameter_names(), 1.46 M elements for the Darcy U-Net)
        are laid out LAST: `live_total` is the length of the prefix that can carry a gradient, and only that prefix
        is exchanged between the ranks (their gradient is identically zero on every rank).  guidance: the model runs the
        residual-gradient guidance branch, whose layers (emb_conv, combine_conv) are then live."""
        named = [(n, p) for n, p in model.named_parameters() if p.requires_grad]
        dead = set(model.unused_parameter_names(guidance=guidance)) if hasattr(model, 'unused_parameter_names') else set()
        order = {n: i for i, (n, _) in enumerate(named)}
        named.sort(key=lambda np_: (np_[0] in dead, group_of(np_[0]) if group_of is not None else 0, order[np_[0]]))
        params = [p for _, p in named]
        dev = params[0].device
        offs, total = [], 0
        self.group_bounds = {}
        self.live_total = None
        for n, p in named:
            if n in dead and self.live_total is None:
                self.live_total = total
            offs.append(total)
            if group_of is not None and n not in dead:
                g = group_of(n)
                lo, _ = self.group_bounds.get(g, (total, total))
                self.group_bounds[g] = (lo, total + (p.numel() + _ALIGN - 1) // _ALIGN * _ALIGN)
            total += (p.numel() + _ALIGN - 1) // _ALIGN * _ALIGN
        if self.live_total is None:
            self.live_total = total
        self.total = total
        self.params, self.offsets = params, offs
        self.flat = torch.zeros(total, device=dev, dtype=torch.float32)
        self.grad = torch.zeros(total, device=dev, dtype=torch.float32)
        for p, o in zip(params, offs):
            view = self.flat[o:o + p.numel()].view(p.shape)
            view.copy_(p.data)
            p.data = view
            p._pidm_grad = self.grad[o:o + p.numel()].view(p.shape)
        if with_optimizer_state:
            self.exp_avg = torch.zeros_like(self.flat)
            self.exp_avg_sq = torch.zeros_like(self.flat)
            self.ema = self.flat.clone()
        self.step_dev = torch.zeros(1, device=dev, dtype=torch.int32)
        self.gnorm_sq = torch.zeros(1, device=dev, dtype=torch.float32)
        self.gnorm_ws = torch.zeros(1 + 148 * 8, device=dev, dtype=torch.float32)      # pidm_sumsq partials + ticket

    def release(self):
        for p in self.params:
            if hasattr(p, '_pidm_grad'):
                del p._pidm_grad


def shard_rows(global_batch, rank, world):
    """Rows [lo, hi) of the global batch owned by `rank` (equal shards; the loss is a mean over equal shards)."""
    assert global_batch % world == 0, 'global batch must divide evenly over the ranks'
    per = global_batch // world
    return rank * per, (rank + 1) * per


def allreduce_flat_grad(flat_grad, world, live=None):
    """The single exchange step of the data-parallel path: sum of the flat gradient over all ranks.  `live`: length of
    the prefix that can be non-zero (FlatParams.live_total); the tail belongs to parameters the forward never uses."""
    if world > 1:
        dist.all_reduce(flat_grad if live is None else flat_grad[:live], op=dist.ReduceOp.SUM)
    return flat_grad


def allreduce_validation(vals, world):
    """vals [5]: this rank's validation values (means over its equal shard) -> their mean over the ranks, in place: the
    values of the global batch (one all-reduce; the mechanics inequality term, a product of two batch means, gets the
    shard mean, as its gradient does in the training step)."""
    if world > 1:
        dist.all_reduce(vals, op=dist.ReduceOp.SUM)
        vals.div_(world)
    return vals


def _unet_grad_group(name):
    """Gradient-readiness groups of Unet3D parameters (backward runs final -> ups -> mid -> downs -> stem; the time-MLP
    branches of every block finish last because they collect contributions from all blocks):
    2 = ups + final_conv (complete once backward has left the up path), 1 = mid + the two deepest down levels,
    0 = everything else (stem, shallow down levels, all time-conditioning MLPs, parameters without gradient)."""
    if name.startswith('time_mlp.') or '.mlp.' in name:
        return 0
    if name.startswith('ups.') or name.startswith('final_conv.'):
        return 2
    if name.startswith(('mid_block1.', 'mid_block2.', 'mid_spatial_attn.', 'downs.2.', 'downs.3.')):
        return 1
    return 0


class TrainEngine:
    def __init__(self, model, diffusion, residuals, lr=1e-4, betas=(0.9, 0.999), eps=1e-8, max_norm=1.0, ema_mu=0.99,
                 c_data=1.0, c_residual=1e-3, use_graph=True, world=1, bucketed_allreduce=None, ema_start=-1,
                 c_ineq=0., lambda_opt=0., rank=0, global_draws=False, snapshot_grad=False):
        """ema_start: the EMA shadow is updated when the 0-based iteration index exceeds it (reference main.py:52,178
        uses 1000); -1 = from the first step on.  The comparison runs on the device against the step counter, so it is
        CUDA-graph safe.  global_draws (world > 1): t and eps are drawn for the GLOBAL batch from a generator that is
        identical on every rank and sliced to this rank's rows (SURVEY 8e: seed parity with the one-process run).
        snapshot_grad: keep a copy of the (all-reduced, unclipped) flat gradient of the last step in `grad_snapshot`
        (parity tests; the Adam kernel zeroes the live buffer).
        Residual-gradient guidance (residuals.residual_grad_guidance): the guidance front end runs inside the step, the
        classifier-free mask is drawn inside the captured graph (a fresh draw every replay; the last one is left in
        model._null_mask_last) and, with global_draws, drawn for the global batch and normalised by the global count."""
        self.guidance = bool(getattr(residuals, 'residual_grad_guidance', False))
        self.model, self.diffusion, self.residuals = model, diffusion, residuals
        self.lr, self.betas, self.eps, self.max_norm, self.ema_mu = lr, betas, eps, max_norm, ema_mu
        self.c_data, self.c_residual, self.c_ineq, self.lambda_opt = c_data, c_residual, c_ineq, lambda_opt
        self.world, self.rank = world, rank
        self.ema_first_step = int(ema_start) + 2
        self.global_draws = bool(global_draws) and world > 1
        # Overlap of the gradient exchange with backward (default for world > 1; bucketed_allreduce=False selects the
        # single all-reduce behind the last weight gradient): the flat gradient is laid out in three readiness groups
        # and a group is all-reduced on its own stream as soon as backward has crossed the matching boundary of the U-Net.
        # scripts/check_ddp.py (2 GPUs): ranks stay bitwise identical, exchanged gradient equal to the single all-reduce
        # to 2e-5 (fp32 atomics), eager and CUDA graph.
        if bucketed_allreduce is None:
            bucketed_allreduce = world > 1
        self.bucketed = bool(bucketed_allreduce) and hasattr(model, '_boundary_cb')
        self.fp = FlatParams(model, group_of=_unet_grad_group if self.bucketed else None, guidance=self.guidance)
        self._ar_stream = None
        self._reduced = set()
        if self.bucketed:
            model._boundary_cb = self._on_boundary
        self.grad_snapshot = torch.empty_like(self.fp.grad) if snapshot_grad else None
        self.use_graph = use_graph
        self._graph = None
        self._static_x0 = None
        self._static_out = None
        self.steps_done = 0
        self._ema_active = False
        self._val_graphs = {}           # (input shape, injected draws) -> (graph, static inputs, outputs)
        self._val_masks = {}            # batch -> classifier-free mask tensor of the validation forward (guidance)

    # ---- one step, eager (also the body that gets captured) -------------------------------------------------
    def _step_body(self, x0):
        fp = self.fp
        shard = (self.rank, self.world) if self.global_draws else None
        loss, data_l, rabs, _, _ = self.diffusion.model_estimation_loss(
            x0, residual_func=self.residuals, c_data=self.c_data, c_residual=self.c_residual, c_ineq=self.c_ineq,
            lambda_opt=self.lambda_opt, sync_scalars=False, draw_shard=shard)
        ops.side_stream_begin()                 # weight-gradient kernels overlap the dgrad chain (joined below)
        self._reduced = set()
        try:
            loss.backward()
        finally:
            ops.side_stream_join()
        if self.bucketed and self.world > 1:
            for g in sorted(fp.group_bounds, reverse=True):          # the groups backward did not hand over early
                if g not in self._reduced:
                    lo, hi = fp.group_bounds[g]
                    dist.all_reduce(fp.grad[lo:hi], op=dist.ReduceOp.SUM)
            if self._ar_stream is not None:
                torch.cuda.current_stream().wait_stream(self._ar_stream)
        else:
            allreduce_flat_grad(fp.grad, self.world, fp.live_total)
        if self.grad_snapshot is not None:
            self.grad_snapshot.copy_(fp.grad)
        fp.gnorm_sq.zero_()
        call('pidm_sumsq', fp.grad, fp.total, fp.gnorm_sq, fp.gnorm_ws, stream())
        call('pidm_adam_ema_step', fp.flat, fp.grad, fp.exp_avg, fp.exp_avg_sq, fp.ema, fp.total, self.lr,
             self.betas[0], self.betas[1], self.eps, 0, fp.step_dev, fp.gnorm_sq, 1.0 / self.world, self.max_norm,
             self.ema_mu, self.ema_first_step, 1, stream())
        return loss.detach(), data_l, rabs

    def _on_boundary(self, group):
        """Called (from a tensor hook inside backward) when every kernel that writes the gradients of `group` has been
        launched: all-reduce that flat range on the exchange stream, behind the main and the weight-gradient streams."""
        if self.world <= 1 or group in self._reduced or group not in self.fp.group_bounds:
            return
        if self._ar_stream is None:
            self._ar_stream = torch.cuda.Stream()
        ar = self._ar_stream
        ar.wait_stream(torch.cuda.current_stream())
        if ops._SIDE['active']:
            ar.wait_stream(ops._SIDE['stream'])
        lo, hi = self.fp.group_bounds[group]
        with torch.cuda.stream(ar):
            dist.all_reduce(self.fp.grad[lo:hi], op=dist.ReduceOp.SUM)
        self._reduced.add(group)

    def step(self, x0):
        """x0: [B, 2, 64, 64] fp32 on the device.  Returns (loss, data_loss, mean|r|) as device tensors."""
        if self._ema_active:
            raise RuntimeError('TrainEngine.step() inside ema_weights(): the model holds the EMA weights, and an optimizer '
                               'step would train them; leave the context first')
        try:
            if not self.use_graph:
                out = self._step_body(x0)
                self.steps_done += 1
                return out
            if self._graph is None:
                self._capture(x0)
            if x0.shape != self._static_x0.shape:
                raise ValueError(f'TrainEngine was captured for batches of shape {tuple(self._static_x0.shape)}, got '
                                 f'{tuple(x0.shape)}: build a second engine (or use_graph=False) for another batch size')
            self._static_x0.copy_(x0, non_blocking=True)
            self._graph.replay()
            self.steps_done += 1
            return self._static_out
        finally:
            packer = getattr(self.model, '_packer', None)
            if packer is not None:
                packer.invalidate()              # the optimizer kernel rewrote the weights behind autograd's back

    def _capture(self, x0):
        self._static_x0 = x0.clone()
        fp = self.fp
        # The warm-up below (allocator, lazy module state, table uploads; on a side stream as capture requires) runs real
        # steps: snapshot every piece of training state first and put it back afterwards, so that the first batch gets
        # exactly ONE optimizer update and the RNG stream continues where the caller left it.
        keep = [t.clone() for t in (fp.flat, fp.exp_avg, fp.exp_avg_sq, fp.ema, fp.step_dev)]
        rng = torch.cuda.get_rng_state(fp.flat.device)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):
                self._step_body(self._static_x0)
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        for t, k in zip((fp.flat, fp.exp_avg, fp.exp_avg_sq, fp.ema, fp.step_dev), keep):
            t.copy_(k)
        fp.grad.zero_()
        torch.cuda.set_rng_state(rng, fp.flat.device)
        torch.cuda.synchronize()
        self._graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self._graph):
            self._static_out = self._step_body(self._static_x0)

    # ---- the EMA weights in the model, and the validation loss (reference main.py:181-198) ------------------------
    def _swap_ema(self):
        fp = self.fp
        call('pidm_swap_f32', fp.flat, fp.ema, fp.total, stream())
        packer = getattr(self.model, '_packer', None)
        if packer is not None:
            packer.invalidate()             # the swap rewrote the weights without bumping their version counters

    @contextlib.contextmanager
    def ema_weights(self):
        """Inside the block the model's parameters hold the EMA shadow (reference main.py:183 `ema.ema(model)`, undone by
        `ema.restore(model)` at :316): the flat weight buffer and the shadow are exchanged in place by one launch on the
        current stream, and exchanged back on exit, also when the block raises, which restores every bit of both.  No
        pointer moves, so the captured training graph, SampleEngine graphs built on the same model and every packing
        table stay valid; before iteration ema_start + 1 the shadow still holds the initial weights, as in the
        reference.  step() raises inside the block and the block does not nest."""
        if self._ema_active:
            raise RuntimeError('TrainEngine.ema_weights() is already active (the contexts do not nest)')
        self._swap_ema()
        self._ema_active = True
        try:
            yield self
        finally:
            self._swap_ema()
            self._ema_active = False

    def _validate_body(self, x0, t=None, noise=None):
        shard = (self.rank, self.world) if self.global_draws else None
        model = self.model
        # the guided forward writes its classifier-free mask into model._null_mask_last, whose storage the captured
        # training step holds: validation keeps a mask tensor of its own per batch size
        train_mask = getattr(model, '_null_mask_last', None)
        model._null_mask_last = self._val_masks.get(x0.shape[0])
        try:
            with torch.no_grad():
                if t is None:
                    out = self.diffusion.model_estimation_loss(
                        x0, residual_func=self.residuals, c_data=self.c_data, c_residual=self.c_residual,
                        c_ineq=self.c_ineq, lambda_opt=self.lambda_opt, sync_scalars=False, draw_shard=shard)
                elif getattr(self.residuals, 'gov_eqs', 'darcy') == 'mechanics':
                    out = self.residuals.training_loss(self.diffusion, x0, t, self.c_data, self.c_residual, self.c_ineq,
                                                       self.lambda_opt, sync_scalars=False, draw_shard=shard, noise=noise)
                else:
                    out = self.diffusion.darcy_loss_from_draws(x0, t, noise, self.residuals, self.c_data, self.c_residual,
                                                               sync_scalars=False, draw_shard=shard)
                vals = torch.stack([v.detach().float().reshape(()) if isinstance(v, torch.Tensor)
                                    else torch.full((), float(v), device=x0.device) for v in out])
                allreduce_validation(vals, self.world)
        finally:
            self._val_masks[x0.shape[0]] = model._null_mask_last
            model._null_mask_last = train_mask
        return tuple(vals.unbind(0))

    def _capture_validate(self, x0, t, noise):
        static = [None if v is None else v.clone() for v in (x0, t, noise)]
        dev = self.fp.flat.device
        # warm-up as in _capture: it reads the weights and writes nothing the training step owns, and the RNG stream
        # continues where the caller left it
        rng = torch.cuda.get_rng_state(dev)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):
                self._validate_body(*static)
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        torch.cuda.set_rng_state(rng, dev)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = self._validate_body(*static)
        return graph, static, out

    def validate(self, x0, t=None, noise=None):
        """The reference's validation loss (main.py:185-198: model_estimation_loss on a validation batch), forward only, on
        whatever weights the model holds -- inside ema_weights() the EMA weights.  Returns (loss, data_loss, mean|r|,
        inequality, optimisation) as 0-d device tensors (zero where a term does not apply) without synchronising with
        the host; under world > 1 they are the mean over the ranks' equal shards, i.e. the values of the global batch
        (except the mechanics inequality loss term, a product of two batch means: see allreduce_validation).
        The draws come from the default CUDA generator in the reference's order (t, eps, then the classifier-free mask
        under guidance) and leave it where the eager model_estimation_loss would; `t` and `noise` inject them instead.
        use_graph: one CUDA graph per input shape, captured on first use (the last batch of an epoch may be smaller);
        its outputs are static tensors, overwritten by the next validate() of that shape."""
        if (t is None) != (noise is None):
            raise ValueError('validate(): give both t and noise, or neither')
        packer = getattr(self.model, '_packer', None)
        if packer is not None:
            packer.refresh_if_stale(ops.act_dtype())       # outside the graph, as in SampleEngine.sample
        if not self.use_graph:
            return self._validate_body(x0, t, noise)
        key = (tuple(x0.shape), t is not None)
        if key not in self._val_graphs:
            self._val_graphs[key] = self._capture_validate(x0, t, noise)
        graph, static, out = self._val_graphs[key]
        for dst, src in zip(static, (x0, t, noise)):
            if dst is not None:
                dst.copy_(src, non_blocking=True)
        graph.replay()
        return out

    def close(self):
        """Release everything that pins NCCL / CUDA-graph resources: the captured graph (it holds NCCL kernels when
        world > 1, and ncclCommDestroy waits for it), the static tensors, and the model -> engine back reference of the
        bucketed exchange (a reference cycle that would keep the graph alive past `del engine`).  Call before
        torch.distributed.destroy_process_group()."""
        import gc
        torch.cuda.synchronize()
        self._graph = None
        self._static_x0 = None
        self._static_out = None
        self._val_graphs = {}
        if getattr(self.model, '_boundary_cb', None) is not None:
            self.model._boundary_cb = None
        gc.collect()
        torch.cuda.synchronize()

    def ema_state_dict(self):
        """EMA weights keyed like model.state_dict() (what the reference checkpoints hold, main.py:314), also inside
        ema_weights(), where the reference saves its checkpoint and the shadow sits in the weight buffer."""
        sd = {k: v.clone() for k, v in self.model.state_dict().items()}
        name_of = {id(p): n for n, p in self.model.named_parameters()}
        shadow = self.fp.flat if self._ema_active else self.fp.ema
        for p, o in zip(self.fp.params, self.fp.offsets):
            sd[name_of[id(p)]] = shadow[o:o + p.numel()].view(p.shape).clone()
        return sd


class SampleEngine:
    """H100-native ancestral sampling loop (reference denoising_utils.py:388-545 p_sample / p_sample_loop, called from
    sample.py:145): the same per-step work as DenoisingDiffusion.p_sample -- x0 estimate through the residual object
    (network call, or the DDIM walk when use_ddim_x0), Darcy residual, posterior step with sigma_t = sqrt(beta_t) --
    but with the time index and the posterior coefficients living on the DEVICE, so that a captured CUDA graph of
    `steps_per_graph` consecutive steps is replayed n_steps / steps_per_graph times and nothing is decided on the host
    inside the loop.  The packed bf16 weights are produced once per loop, not once per step (they only change when an
    optimizer has run).  `DenoisingDiffusion.p_sample_loop` remains the drop-in API (host-side step index, CPU
    trajectory); this is the throughput path.

    external_noise=True: the per-step noise z is read from a static buffer that `sample(noises=...)` refreshes before
    every replay (parity tests inject the reference's draws); otherwise z is drawn by torch's Philox inside the graph.

    Topology optimisation (residuals.gov_eqs == 'mechanics', image_shape=(3, 65, 65); reference sample.py:136-150,
    244-342): `sample(conditioning_input=(conditioning, bcs, solution))` copies the resized conditioning and boundary
    conditions into a static buffer, so a new test batch needs no recapture.  A step is the input kernel
    (pidm_mech_sample_input) -> U-Net (or the DDIM walk) -> the posterior kernel (pidm_mech_posterior_step).  The
    residual, compliance and inequality are needed at t = 0 only and are evaluated once, on the last step's x0
    prediction; with residuals.topopt_eval and a solution the evaluation metrics use the fused solver.  A batch
    smaller than `batch` is padded with copies of its last sample and the results are sliced.

    CoCoGen residual corrections (Darcy; N_correction, M_correction, correction_mode as in p_sample_loop, reference
    denoising_utils.py:433-459,517-540): while t < N_correction a step corrects the x0 estimate before the posterior
    step ('x0') or the new sample after it ('xt'), and the step's residual is the corrected one.  Every step launches
    `pidm_darcy_cocogen` with the device-side time index and n_active = N_correction, so one captured graph serves the
    whole loop.  After the loop, M_correction corrections of x run in one launch and the residual returned is the one
    after the last of them.  With trajectory=True those M corrections add ONE entry, the final corrected state
    (p_sample_loop records each of them).  N_correction = M_correction = 0 launches nothing extra."""

    def __init__(self, model, diffusion, residuals, batch, image_shape=(2, 64, 64), surpress_noise=True, use_graph=True,
                 steps_per_graph=None, external_noise=False, N_correction=0, M_correction=0, correction_mode='none'):
        from .denoising_utils import _axpby, image_to_b_xy_c, generalized_b_xy_c_to_image
        self._axpby, self._to_rows, self._to_img = _axpby, image_to_b_xy_c, generalized_b_xy_c_to_image
        self.model, self.diffusion, self.residuals = model, diffusion, residuals
        self.use_graph, self.surpress_noise = use_graph, surpress_noise
        dd = diffusion.diff_dict
        dev = dd['alphas'].device
        self.n_steps = diffusion.n_steps
        if steps_per_graph is None:
            steps_per_graph = next(k for k in (10, 5, 4, 2, 1) if self.n_steps % k == 0)
        assert self.n_steps % steps_per_graph == 0, 'steps_per_graph must divide n_steps'
        self.k = steps_per_graph if use_graph else 1
        self.external_noise = external_noise
        self.mechanics = getattr(residuals, 'gov_eqs', 'darcy') == 'mechanics'
        self.N_correction, self.M_correction = int(N_correction), int(M_correction)
        if self.N_correction < 0 or self.M_correction < 0:
            raise ValueError(f'N_correction = {N_correction} and M_correction = {M_correction} must not be negative')
        if self.N_correction and correction_mode not in ('x0', 'xt'):
            raise ValueError(f"correction_mode must be 'x0' or 'xt' with N_correction > 0 (got {correction_mode!r})")
        if (self.N_correction or self.M_correction) and self.mechanics:
            raise ValueError('CoCoGen correction is only implemented for the Darcy flow study (reference main.py:37-38).')
        self.correction_mode = correction_mode
        if self.mechanics:
            assert tuple(image_shape) == (3, 65, 65), 'the topology-optimisation model samples [B, 3, 65, 65]'
            self.batch = batch
            self.planes = torch.zeros(batch, 7, 64, 64, device=dev)      # resized conditioning (3) and bcs (4)
            self.net_in = torch.zeros(batch, 10, 64, 64, device=dev)
            self.x0_pred = None
        self.x = torch.zeros(batch, *image_shape, device=dev)
        self.z = torch.zeros(self.k, batch, *image_shape, device=dev) if external_noise else None
        self.t = torch.zeros(batch, device=dev, dtype=torch.long)
        self.residual = None
        self.c1 = dd['posterior_mean_coef1'].float().contiguous()
        self.c2 = dd['posterior_mean_coef2'].float().contiguous()
        sig = dd['betas'].float().sqrt().contiguous()
        if surpress_noise:
            sig = sig.clone()
            sig[0] = 0.
        self.sigma = sig
        self._graph = None

    def _step_body(self, j=0):
        if self.mechanics:
            return self._mech_step_body(j)
        with torch.no_grad():
            x, t = self.x, self.t
            out = self.residuals.compute_residual(((self._to_rows(x), t),), reduce='per-batch', return_model_out=True,
                                                  sample=True, ddim_func=self.diffusion.ddim_sample_x0)
            model_out = out['model_out']
            if model_out.dim() == 3:
                model_out = self._to_img(model_out)
            if self.residual is None:
                self.residual = torch.empty_like(out['residual'])
            self.residual.copy_(out['residual'])
            correct = self.N_correction > 0
            if correct and self.correction_mode == 'x0':   # the corrected x0 estimate feeds the posterior step
                model_out = model_out.float().clone(memory_format=torch.contiguous_format)
                self.residuals.cocogen(model_out, self.residual, 1, t, self.N_correction)
            z = self.z[j] if self.external_noise else torch.randn_like(x)   # drawn at every step, t == 0 included
            new_x = self._axpby(self.c1[t].contiguous(), model_out.float(), self.c2[t].contiguous(), x,
                                self.sigma[t].contiguous(), z)
            self.x.copy_(new_x)
            if correct and self.correction_mode == 'xt':
                self.residuals.cocogen(self.x, self.residual, 1, t, self.N_correction)
            self.t.sub_(1)

    def _mech_step_body(self, j=0):
        with torch.no_grad():
            x, t = self.x, self.t
            ops.mech_sample_input(x, self.planes, self.net_in)
            res = self.residuals
            if res.use_ddim_x0:
                x0_pred, y = self.diffusion.ddim_sample_x0(self.net_in, t, res.model, x.shape, res.ddim_steps, 0.,
                                                           gov_eqs='mechanics')
            else:
                x0_pred = y = res.model(self.net_in, t)
            z = self.z[j] if self.external_noise else torch.randn_like(x)   # drawn at every step, t == 0 included
            ops.mech_posterior_step(y.float().contiguous(), x, z, t, self.c1, self.c2, self.sigma, x)
            self.x0_pred = x0_pred                  # the last step's tensor: after the loop it holds the x0 of t = 0
            self.t.sub_(1)

    def _mech_condition(self, conditioning_input):
        """Resize the conditioning and boundary conditions into the static planes (padded to `batch` rows)."""
        from .residuals_mechanics_K import resize_image
        conditioning, bcs, _ = conditioning_input
        n = conditioning.shape[0]
        assert 0 < n <= self.batch and bcs.shape[0] == n, f'conditioning of {n} samples for an engine of batch {self.batch}'
        planes = torch.cat((resize_image(conditioning, 64), resize_image(bcs, 64)), dim=1)
        self.planes[:n].copy_(planes)
        if n < self.batch:
            self.planes[n:].copy_(planes[n - 1:n].expand(self.batch - n, -1, -1, -1))
        return n

    def _mech_aux(self, conditioning_input, n):
        """Residual, compliance and inequality of the last x0 prediction (reference aux keys), and the evaluation metrics
        (fused solver) when residuals.topopt_eval is set and a solution is given; device tensors, no host sync."""
        from .residuals_mechanics_K import _MechResidual, resize_image
        conditioning, bcs, solution = conditioning_input
        res = self.residuals
        bcs = bcs.contiguous().float()
        x0 = self.x0_pred[:n].float()
        u = resize_image(x0[:, :-1], x0.shape[-1] + 1)
        rho = x0[:, -1].contiguous()
        residual, compliance = _MechResidual.apply(u, rho, bcs, res.KE)
        vf = conditioning[:, 0, 0, 0]
        aux = {'residual': residual, 'optimized_quant': compliance, 'inequality_quant': rho.reshape(n, -1).mean(1) - vf}
        if res.topopt_eval and solution is not None:
            aux.update(res.topopt_metrics(rho, bcs, vf, solution, solver='fused'))
        return aux

    def _capture(self):
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):
                self.t.fill_(self.n_steps - 1)
                self._step_body()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        self.t.fill_(self.n_steps - 1)
        self._graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self._graph):
            for j in range(self.k):
                self._step_body(j)

    def sample(self, x_init=None, trajectory=False, noises=None, conditioning_input=None):
        """Runs the whole loop; returns (x_0 [B,C,P,P], residual of the last step [B,P*P,3]) as device tensors and,
        if asked, the trajectory [n_steps+1,B,C,P,P] (device; recorded per replay, so it needs steps_per_graph=1).
        noises [n_steps,B,C,P,P]: the z of every step (external_noise engines only).
        Topology optimisation: conditioning_input=(conditioning [n,3,65,65], bcs [n,4,65,65], solution or None) with
        n <= batch is required, x_init / noises have n rows, and the second value returned is the dict of the
        reference's aux keys (residual, optimized_quant, inequality_quant and, with topopt_eval and a solution,
        rel_CE_error_full_batch, vf_error_full_batch, fm_error_full_batch)."""
        assert (noises is not None) == self.external_noise, 'noises= goes with external_noise=True'
        assert not (trajectory and self.k != 1), 'trajectory=True needs steps_per_graph=1'
        assert (conditioning_input is not None) == self.mechanics, 'conditioning_input= goes with the mechanics study'
        n = self._mech_condition(conditioning_input) if self.mechanics else self.x.shape[0]
        packer = getattr(self.model, '_packer', None)
        if packer is not None:
            packer.refresh_if_stale(ops.act_dtype())       # the captured steps do not re-pack the weights
        if self.use_graph and self._graph is None:
            self._capture()
        if x_init is None:
            x_init = torch.randn_like(self.x[:n])
        self.x[:n].copy_(x_init)
        if n < self.x.shape[0]:
            self.x[n:].copy_(x_init[n - 1:n].expand(self.x.shape[0] - n, *x_init.shape[1:]))
        self.t.fill_(self.n_steps - 1)
        traj = [self.x[:n].clone()] if trajectory else None
        for it in range(self.n_steps // self.k):
            if self.external_noise:
                self.z[:, :n].copy_(noises[it * self.k:(it + 1) * self.k])
            if self.use_graph:
                self._graph.replay()
            else:
                self._step_body()
            if trajectory:
                traj.append(self.x[:n].clone())
        if self.M_correction:
            self.residuals.cocogen(self.x, self.residual, self.M_correction)
            if trajectory:
                traj.append(self.x[:n].clone())
        traj = torch.stack(traj) if trajectory else None
        if self.mechanics:
            return self.x[:n], self._mech_aux(conditioning_input, n), traj
        return self.x, self.residual, traj
