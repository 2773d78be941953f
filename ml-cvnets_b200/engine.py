"""The reference's training iteration (engine/training_engine.py:236-312) for the hot-path models, as ONE replayable CUDA graph:

    forward -> cross entropy (label smoothing) -> backward (weight gradients written straight into a flat buffer)
            -> [data parallel: bucketed all-reduce of that buffer over NCCL, overlapped with the rest of the backward]
            -> GradScaler unscale + inf check + clip_grad_norm_ + AdamW or SGD (+ EMA) + GradScaler update   (two launches)

``TrainStep`` is host code only -- every kernel it launches is one of the library's (include/cvnets_b200.h); there is no ATen kernel
inside the step (zero-fills are memset nodes, the loss is cvb_ce_*).  Semantics follow the reference: per-GPU BatchNorm statistics
(``batch_norm``, not ``sync_batch_norm``), DDP's gradient mean over ranks and per-step buffer broadcast from rank 0
(main_train.py:90-96), the two AdamW parameter groups of cvnets/misc/common.py:122-176, max-norm clipping at
``common.grad_clip`` (10.0 in the recipe, config/classification/imagenet/mobilevit_v2.yaml:9), EMA as averaging_utils.py:43-55.

    step = TrainStep(model, lr=2e-3, weight_decay=0.05, max_norm=10.0, label_smoothing=0.1)
    step.capture(x_example, y_example)        # optional: whole step as one CUDA graph (inputs are copied into static buffers)
    for x, y in loader:
        step.set_lr(scheduler_lr)             # device scalar: schedulers keep working under replay
        loss = step(x, y)                     # device tensor; no host sync

A variable-batch sampler draws a (crop, batch) pair per iteration; ``capture_shapes`` captures one graph per pair in the same TrainStep
(``variable_batch_pairs`` gives the reference sampler's table):

    pairs = variable_batch_pairs(224, 224, 256, max_scales=5, check_scale=32, min_w=128, max_w=320, min_h=128, max_h=320)
    step.capture_shapes([(torch.randn(b, 3, h, w, device="cuda"), torch.zeros(b, dtype=torch.long, device="cuda")) for h, w, b in pairs])

Gradient accumulation (the reference's ``common.accum_freq``): every call is one micro-batch, and every ``accum_freq``-th call applies the
update to the summed gradients; ``updated`` says whether the last call did (advance the scheduler and the iteration count then):

    step = TrainStep(model, optimizer="sgd", lr=0.1, weight_decay=4e-5, max_norm=None, accum_freq=2)
    for epoch in range(epochs):
        step.zero_grad()                      # the reference's per-epoch _zero_grad(): drops a window left open by the last epoch
        for x, y in loader:
            loss = step(x, y)
            if step.updated:
                iteration += 1
"""
from __future__ import annotations

import gc
import math
from types import SimpleNamespace
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import functional as Fn
from . import ops
from .optim import FlatAdamW, FlatSGD
from .workspace import StepWorkspace


def cross_entropy(logits: torch.Tensor, target: torch.Tensor, label_smoothing: float = 0.0, ignore_index: int = -1,
                  _cfg: Optional[SimpleNamespace] = None) -> torch.Tensor:
    """F.cross_entropy(logits, target, ignore_index=..., label_smoothing=...) with mean reduction (the reference's classification loss,
    loss_fn/classification/cross_entropy.py:74-95) on the library's kernels; returns a 0-dim fp32 tensor."""
    if not logits.is_cuda:
        raise RuntimeError("cross_entropy: ml-cvnets_b200 runs on CUDA only (no CPU fallback)")
    cfg = _cfg if _cfg is not None else SimpleNamespace(label_smoothing=float(label_smoothing), ignore_index=int(ignore_index), scale=None)
    return Fn.CrossEntropyFn.apply(logits, target, cfg)


class TrainStep:
    def __init__(self, model: torch.nn.Module, *, lr: float = 2e-3, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 0.05,
                 no_decay_bn_filter_bias: bool = True, max_norm: float = 10.0, label_smoothing: float = 0.1, ignore_index: int = -1,
                 ema_momentum: Optional[float] = None, init_scale: float = 65536.0, growth_interval: int = 2000,
                 process_group=None, data_parallel: Optional[bool] = None, n_buckets: int = 3, broadcast_buffers: bool = True,
                 forward_loss=None, optimizer: str = "adamw", momentum: float = 0.9, nesterov: bool = True,
                 aug_loss: Optional["NeuralAugmentationLoss"] = None, ce_weight: float = 1.0, ema_buffers: bool = False, accum_freq: int = 1):
        """``forward_loss(model, *inputs, cfg) -> loss`` replaces the default ``cross_entropy(model(x), y)`` (e.g. CLIP's contrastive step);
        ``cfg.scale`` is the device-resident loss scale the loss's backward must multiply by, ``cfg.world / rank / group`` the process group.
        ``optimizer="sgd"`` swaps AdamW for SGD with ``momentum`` / ``nesterov`` (optim.FlatSGD; ``betas`` / ``eps`` are then unused and
        ``max_norm`` None / 0 means no clipping).  A model with a RangeAugment augmentor returns ``{"augmented_tensor", "logits"}``; the cross
        entropy reads ``logits``, and with ``aug_loss`` the step minimises ``ce_weight * CE + aug_loss.weight * L_na`` (the RangeAugment recipes'
        composite_loss); ``loss_parts`` (device fp32 [2]) then holds (CE, L_na) of the last step.  A ``forward_loss`` of such a model returns
        ``(loss, augmented_tensor)``; with ``aug_loss`` the step then minimises ``ce_weight * loss + aug_loss.weight * L_na`` and ``loss_parts``
        holds (loss, L_na).  ``loss`` must apply ``cfg.scale`` in its backward, as the built-in losses do; the composite hands it its weighted
        gradient unscaled (the CLIP recipe's step: INTEGRATION.md).

        ``ema_buffers=True`` (needs ``ema_momentum``) extends the EMA to the whole state, as the reference's EMA averages the whole
        state_dict (averaging_utils.py:43-55): the model's floating-point buffers (BatchNorm running statistics) become views of one flat fp32
        tensor, a second one holds their EMA (initialised from the buffers), and every step launches ``cvb_ema_update`` after its forward
        has updated the statistics.  Data parallel: each rank averages its own post-forward statistics.  ``ema_model()`` is the evaluable
        EMA twin.

        ``accum_freq`` > 1 accumulates gradients over that many calls (micro-batches) per optimizer update, as the reference's
        ``common.accum_freq`` does (engine/training_engine.py:286-312): each call runs forward, loss, backward and the data-parallel exchange
        into the workspace's gradient buffer and adds it into one flat fp32 accumulator (``grad_acc``; ``p.grad`` become views of it), so the
        gradients are summed, not averaged.  Every ``accum_freq``-th call then runs the optimizer tail over the accumulator, the buffer EMA,
        and zeroes the accumulator: loss scale, step count and EMA change only there, and an inf / nan in any micro-batch skips that window's
        update and backs the scale off once.  BatchNorm statistics update on every micro-batch.  ``updated`` is True after a call that
        applied the update; ``zero_grad()`` discards an open window.  ``accum_freq`` 1 (the default) is the plain step, with no accumulator."""
        import torch.distributed as dist
        if optimizer not in ("adamw", "sgd"):
            raise ValueError(f"optimizer must be 'adamw' or 'sgd', got {optimizer!r}")
        if isinstance(accum_freq, bool) or int(accum_freq) != accum_freq or accum_freq < 1:
            raise ValueError(f"accum_freq must be an integer >= 1, got {accum_freq!r}")
        self.model = model
        self.ws = StepWorkspace(model)
        self.accum_freq = int(accum_freq)
        self.grad_acc = None
        if self.accum_freq > 1:
            self.grad_acc = torch.zeros_like(self.ws.flat_g)
            for p in self.ws.params:
                o, k = self.ws.offsets[id(p)]
                p.grad = self.grad_acc[o:o + k].view_as(p)
        self._window = 0        # micro-batches accumulated in the open window
        self.updated = False    # whether the last call applied the optimizer update
        common = dict(lr=lr, weight_decay=weight_decay, no_decay_bn_filter_bias=no_decay_bn_filter_bias, max_norm=max_norm, init_scale=init_scale,
                      growth_interval=growth_interval, ema_momentum=ema_momentum, grads=self.grad_acc)
        if optimizer == "adamw":
            self.opt = FlatAdamW(model, self.ws, betas=betas, eps=eps, **common)
        else:
            self.opt = FlatSGD(model, self.ws, momentum=momentum, nesterov=nesterov, **common)
        if data_parallel is None:
            data_parallel = dist.is_available() and dist.is_initialized() and dist.get_world_size(process_group) > 1
        self.world = 1
        self.broadcast_buffers = broadcast_buffers
        if data_parallel:
            self.ws.enable_ddp(process_group, n_buckets)
            self.world = self.ws.world
            # DDP's constructor broadcasts rank 0's parameters and buffers (torch DistributedDataParallel._sync_module_states)
            dist.broadcast(self.opt.flat_p, src=0, group=process_group)
            if self.opt.ema is not None:
                self.opt.ema.copy_(self.opt.flat_p)
            self.ws.broadcast_buffers()
        self.loss_cfg = SimpleNamespace(label_smoothing=float(label_smoothing), ignore_index=int(ignore_index), scale=self.opt.loss_scale(),
                                        mix=self.ws.mix)
        self.forward_loss = forward_loss
        if aug_loss is None and ce_weight != 1.0:
            raise ValueError("ce_weight weighs the cross entropy against aug_loss; without aug_loss the loss is the cross entropy")
        self.aug_loss, self.ce_weight = aug_loss, float(ce_weight)
        self.loss_parts = torch.zeros(2, device=self.ws.device, dtype=torch.float32) if aug_loss is not None else None
        self.loss_cfg.group = process_group
        self.loss_cfg.world, self.loss_cfg.rank = self.world, (dist.get_rank(process_group) if data_parallel else 0)
        if ema_buffers and ema_momentum is None:
            raise ValueError("ema_buffers=True averages the buffers alongside the weights: it needs ema_momentum")
        # after the data-parallel set-up: the EMA starts from rank 0's buffers, as the reference's deepcopy of the synchronised model does
        flat_buf = self.ws.flat_buffers() if ema_buffers else None
        self.ema_buffers = flat_buf.clone() if flat_buf is not None else None
        self._ema_buffers_on = bool(ema_buffers)
        self._ema_model = None
        self._one = torch.ones((), device=self.ws.device, dtype=torch.float32)
        self._graphs: Dict[tuple, tuple] = {}  # input signature -> (CUDA graph, static inputs, static loss), in capture order
        self._update_graph = None  # accum_freq > 1: the shape-independent update (optimizer tail, buffer EMA, accumulator clear)
        self.launches_per_update: Optional[int] = None
        self._pool = None
        self.eager_steps = 0

    # ---- scheduler / checkpoint hooks
    def set_lr(self, lr: float) -> None:
        self.opt.set_lr(lr)

    def set_epoch(self, epoch: int) -> None:
        """Curriculum position of ``aug_loss`` for the NEXT steps (the epoch, or the iteration when the scheduler is iteration based); a device
        scalar, so a captured step follows it."""
        if self.aug_loss is None:
            raise RuntimeError("set_epoch: this TrainStep has no aug_loss")
        self.aug_loss.set_epoch(epoch)

    def set_mix(self, kind: Optional[str] = None, lam: float = 1.0, box=(0, 0, 0, 0)) -> None:
        """Batch mixing for the NEXT steps (SURVEY.md 8f row 3; reference: apply_mixing_transforms, engine/training_engine.py:236-238).
        kind None = off; "mixup": x = lam*x + (1-lam)*x.roll(1, 0); "cutmix": the box (x1, y1, x2, y2) is pasted from x.roll(1, 0) and
        ``lam`` must be 1 - box_area / image_area (image_torch.py:338).  Targets become lam*onehot(y) + (1-lam)*onehot(y.roll(1)).  Both
        are applied inside the stem's gather kernel and the loss kernels: no mixed image or soft-target tensor exists.  The values live in
        a device buffer, so a captured step follows per-iteration changes."""
        mode = {None: 0.0, "mixup": 1.0, "cutmix": 2.0}[kind]
        # a fresh pinned buffer per call: the copy queued by an earlier call may not have run yet (replayed graphs let the host run ahead)
        # and must still read its own values (the host allocator keeps the buffer until the copy is done)
        h = torch.tensor([mode, float(lam)] + [float(v) for v in box], dtype=torch.float32).pin_memory()
        self.ws.mix.copy_(h, non_blocking=True)

    def state_dict(self):
        sd = self.opt.state_dict()
        if self.ema_buffers is not None:
            sd["ema_buffers"] = self.ema_buffers.clone()
        return sd

    def load_state_dict(self, sd):
        self.opt.load_state_dict(sd)
        if self.ema_buffers is not None:
            self.ema_buffers.copy_(sd["ema_buffers"])
        ops.invalidate_prepared_weights()  # the EMA weights were written behind the twin's parameters (no Tensor._version bump there)

    def ema_model(self) -> torch.nn.Module:
        """The EMA model (the reference's ``EMA.ema_model``) as an eval-mode twin of ``model`` that owns no copy of the state: its parameters
        are views of the optimizer's flat EMA, its floating-point buffers views of the buffer EMA (``ema_buffers=True``), so it always shows
        the latest step.  It has no gradients, and kernel-layout weight caches of its own.  Its ``state_dict()`` has the reference EMA
        model's keys and values, except ``num_batches_tracked``: integer buffers are not averaged and the twin reports the live counter
        (DESIGN.md).  Evaluate it with ``EvalStep(step.ema_model())``."""
        if self.opt.ema is None:
            raise RuntimeError("ema_model: this TrainStep keeps no EMA (ema_momentum=None)")
        if self._ema_model is not None:
            return self._ema_model
        live_bufs = [b for b in self.model.buffers() if b.is_floating_point()]
        if live_bufs and not self._ema_buffers_on:
            raise RuntimeError("ema_model: the model has BatchNorm running statistics; construct the TrainStep with ema_buffers=True so the "
                               "EMA model averages them as the reference's EMA does")
        import copy
        twin = copy.deepcopy(self.model)  # the workspace does not travel (StepWorkspace.__deepcopy__); the parameters are re-pointed below
        live_params = dict(self.model.named_parameters())
        for name, p in twin.named_parameters():
            lp = live_params[name]
            if id(lp) in self.ws.offsets:
                o, k = self.ws.offsets[id(lp)]
                p.data = self.opt.ema[o:o + k].view_as(p)
            p.requires_grad_(False)
            p.grad = None
        live_named = dict(self.model.named_buffers())
        o = 0
        for name, b in twin.named_buffers():
            lb = live_named[name]
            if b.is_floating_point():
                k = b.numel()
                b.data = self.ema_buffers[o:o + k].view_as(b)
                o += k
            else:
                b.data = lb.data  # num_batches_tracked: the live counter
        self._ema_model = twin.eval()
        return self._ema_model

    def zero_grad(self) -> None:
        """Discard the open accumulation window: zero the accumulator and restart the count (the reference's ``_zero_grad()`` at the start of
        every epoch, which drops a partial window left by the previous one).  Nothing to discard with ``accum_freq`` 1."""
        if self.grad_acc is not None:
            self._clear_acc()
        self._window = 0

    def _clear_acc(self) -> None:
        ops._lib().cvb_memset_zero(self.grad_acc.data_ptr(), self.grad_acc.numel() * 4, ops._stream())  # a memset node under capture

    # ---- one iteration, eager launches
    def _step(self, *inputs: torch.Tensor) -> torch.Tensor:
        """One call's launches: the whole step, or with accum_freq > 1 one micro-batch up to and including its accumulate."""
        loss = self._forward_backward(*inputs)
        if self.grad_acc is None:
            self._update()
        else:
            ops.grad_accumulate(self.grad_acc, self.ws.flat_g)
        return loss

    def _update(self) -> None:
        self.opt.step(grad_div=float(self.world))
        if self.ema_buffers is not None:
            ops.ema_update(self.ema_buffers, self.ws.flat_buffers(), self.opt.ema_momentum)
        if self.grad_acc is not None:
            self._clear_acc()

    def _end_window(self) -> bool:
        """Count the call just made into the window; True when it completes the window (always with accum_freq 1)."""
        self._window += 1
        if self._window < self.accum_freq:
            return False
        self._window = 0
        return True

    def _forward_backward(self, *inputs: torch.Tensor) -> torch.Tensor:
        ws = self.ws
        ws.begin_step()
        if self.world > 1 and self.broadcast_buffers:
            ws.broadcast_buffers()
        ws.active = True
        try:
            if self.forward_loss is None:
                x, y = inputs
                out = self.model(x)
                if isinstance(out, dict):  # a model with a RangeAugment augmentor (base_image_encoder.py:282-298)
                    loss = cross_entropy(out["logits"], y, _cfg=self.loss_cfg)
                    if self.aug_loss is not None:
                        loss = self.aug_loss.composite(out["augmented_tensor"], loss, self.ce_weight, self.loss_cfg.scale, self.loss_parts)
                elif self.aug_loss is not None:
                    raise ValueError("TrainStep(aug_loss=...) needs a model with a RangeAugment augmentor (model.learn_augmentation.mode: "
                                     "distribution); this model returned plain logits")
                else:
                    loss = cross_entropy(out, y, _cfg=self.loss_cfg)
            else:
                loss = self.forward_loss(self.model, *inputs, self.loss_cfg)
                if isinstance(loss, tuple):  # (loss, augmented_tensor): a model with a RangeAugment augmentor, e.g. CLIP
                    if self.aug_loss is None:
                        raise ValueError("forward_loss returned (loss, augmented_tensor) but this TrainStep has no aug_loss: pass "
                                         "aug_loss=NeuralAugmentationLoss(...) or return the loss alone")
                    loss, x_aug = loss
                    loss = self.aug_loss.composite(x_aug, loss, self.ce_weight, self.loss_cfg.scale, self.loss_parts)
            torch.autograd.backward(loss, grad_tensors=self._one)
        finally:
            ws.active = False
        ws.finish_reduce()
        return loss

    def step(self, *inputs: torch.Tensor) -> torch.Tensor:
        """One training step on ``inputs`` (with accum_freq > 1, one micro-batch; ``updated`` tells whether it applied the update).  Before
        capture it runs eagerly; after capture it replays the graph captured for the inputs' shapes (``ValueError`` for a shape that was not
        captured), and the update graph when the call completes a window.  The returned loss is this micro-batch's, a static tensor of the
        graph: read or clone it before the next step."""
        if not self._graphs:
            self.eager_steps += 1
            loss = self._step(*inputs)
            self.updated = self._end_window()
            if self.updated and self.grad_acc is not None:
                self._update()
            return loss
        graph, statics, sloss = self._graph_for(inputs)
        for s_in, t in zip(statics, inputs):
            if t is not s_in:
                s_in.copy_(t, non_blocking=True)
        graph.replay()
        self.updated = self._end_window()
        if self.updated and self._update_graph is not None:
            self._update_graph.replay()
        if self.updated:
            ops.invalidate_prepared_weights()
        return sloss

    __call__ = step

    def _graph_for(self, inputs) -> tuple:
        entry = self._graphs.get(_signature(inputs))
        if entry is None:  # same shapes, other dtypes: the copy into the static buffers converts them (as a single-shape capture always did)
            shapes = _shapes(inputs)
            entry = next((e for sig, e in self._graphs.items() if tuple(s for s, _ in sig) == shapes), None)
        if entry is None:
            # no eager fall-back: an eager step at a new shape could re-plan the step arena under the captured graphs
            raise ValueError(f"TrainStep.step: no CUDA graph was captured for input shapes {list(_shapes(inputs))}; captured: "
                             f"{[list(s) for s in self.captured_shapes]} (capture every shape the sampler draws with capture_shapes)")
        return entry

    # ---- whole step as one CUDA graph per input shape
    def capture(self, *inputs: torch.Tensor, warmup: int = 3):
        """Warm up eagerly (workspace planning needs two steps), then capture fwd + loss + bwd (+ all-reduce) + optimizer tail: the
        one-shape case of ``capture_shapes``."""
        return self.capture_shapes([inputs], warmup=warmup)

    def capture_shapes(self, examples: Sequence[Sequence[torch.Tensor]], warmup: int = 3):
        """Capture one CUDA graph per distinct input signature (shapes and dtypes) of ``examples``: ``(x, y)`` tuples, or the inputs of
        ``forward_loss`` (e.g. ``(images, text_tokens)``).  ``step()`` then replays the graph of its inputs' shapes.  With accum_freq > 1
        these are micro-step graphs (up to and including the accumulate), and ONE more graph, captured last into the same pool, holds the
        shape-independent update that ``step()`` replays at the end of every window.

        Warm-up: ``max(warmup, 3)`` passes over the distinct examples in the order given, each step a real eager training step on that
        example (with one shape, eager steps already taken count toward the passes, as ``capture`` always did).  The first pass raises every
        arena key's record to its maximum over all shapes, the next re-plans the step arena once at that size and caches each shape's
        descriptor tables at their final addresses.  The arena is then frozen: every graph bakes in its addresses, and a step that would
        re-plan it raises.

        The graphs are captured most demanding first (largest inputs) into ONE memory pool, so K shapes reserve about what the largest
        needs: a graph's temporaries may reuse blocks another graph freed at the end of its capture, which is safe because the graphs replay
        one at a time on one stream, and whatever outlives a capture (the static loss, per-shape caches such as the contrastive loss's
        labels) stays allocated.  The static inputs of all shapes are views into one buffer per input position, sized for the largest.
        Everything else is shared by all graphs because it already lives on the device: the flat parameters, gradients and optimizer
        state, the learning rate, the mix buffer, the dropout generator, the RangeAugment curriculum position and the BatchNorm running
        statistics; replaying shapes in any order follows the trajectory of eager steps in that order.

        Data parallel: the bucket plan covers the flat gradient buffer, whose layout does not depend on the shape, so one plan serves every
        graph; all ranks must replay the same shape at the same step (the variable-batch sampler draws the same (crop, batch) on every
        rank), and a forward_loss that all-gathers features (CLIP) needs the same per-rank batch on every rank, as the reference's does.

        ``launches_per_shape`` maps each captured tuple of input shapes to its launch count; ``launches_per_step`` is the largest of them
        (the one count of a single-shape capture).  ``launches_per_update`` counts the update graph's launches (None with accum_freq 1)."""
        assert not self._graphs, "already captured"
        by_sig: Dict[tuple, tuple] = {}
        for ex in examples:
            ex = tuple(ex)
            by_sig.setdefault(_signature(ex), ex)
        if not by_sig:
            raise ValueError("capture_shapes: no examples")
        if len({len(ex) for ex in by_sig.values()}) != 1:
            raise ValueError("capture_shapes: every example must have the same number of inputs")
        dev = self.ws.device
        statics = _static_buffers(list(by_sig.items()), dev)
        passes = max(warmup, 3) - (self.eager_steps if len(by_sig) == 1 else 0)
        torch.cuda.synchronize(dev)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(max(0, passes)):
                for sig, st in statics.items():
                    for s_in, t in zip(st, by_sig[sig]):
                        s_in.copy_(t)
                    self.step(*st)  # real eager calls: with accum_freq > 1 they advance the window and update at its end
            self._first = next(iter(by_sig))
            for s_in, t in zip(statics[self._first], by_sig[self._first]):  # static_inputs hold the first example, as they always have
                s_in.copy_(t)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize(dev)
        self.ws.freeze()
        gc.collect()  # no autograd graph of an eager step (leaf accumulators are bound to the stream they were created on) may survive into capture
        self._pool = torch.cuda.graph_pool_handle()
        order = sorted(statics, key=lambda sig: -sum(math.prod(s) * d.itemsize for s, d in sig))  # stable: ties keep the given order
        self.launches_per_shape: Dict[tuple, int] = {}
        for sig in order:
            graph = torch.cuda.CUDAGraph()
            n0 = ops.launch_count
            with torch.cuda.graph(graph, pool=self._pool):
                # detached: the loss's autograd graph (and the activations its nodes hold) dies here, so the next capture can reuse them
                sloss = self._step(*statics[sig]).detach()
            gc.collect()
            self.launches_per_shape[tuple(s for s, _ in sig)] = ops.launch_count - n0
            self._graphs[sig] = (graph, statics[sig], sloss)
        self.launches_per_step = max(self.launches_per_shape.values())
        if self.grad_acc is not None:
            graph = torch.cuda.CUDAGraph()
            n0 = ops.launch_count
            with torch.cuda.graph(graph, pool=self._pool):
                self._update()
            self.launches_per_update = ops.launch_count - n0
            self._update_graph = graph
        return self

    @property
    def static_inputs(self):
        """The static input buffers that ``step()`` copies into, those of the first example given to ``capture_shapes`` (with one shape they
        hold the example until the next step with other inputs; with several, all shapes' buffers share memory)."""
        return None if not self._graphs else self._graphs[self._first][1]

    @property
    def captured_shapes(self) -> List[tuple]:
        """The captured tuples of input shapes, in capture order."""
        return [tuple(s for s, _ in sig) for sig in self._graphs]

    def graph_pool_bytes(self) -> int:
        """Device memory the captured graphs' shared pool holds (0 before capture)."""
        return _pool_bytes(self._pool)


def _pool_bytes(pool_handle) -> int:
    if pool_handle is None:
        return 0
    segs = torch.cuda.memory_snapshot(mempool_id=pool_handle, include_traces=False)
    pool = tuple(pool_handle)
    return sum(s["total_size"] for s in segs if tuple(s.get("segment_pool_id", pool)) == pool)


def _shapes(inputs) -> tuple:
    return tuple(tuple(t.shape) for t in inputs)


def _signature(inputs) -> tuple:
    return tuple((tuple(t.shape), t.dtype) for t in inputs)


def _static_buffers(examples: List[Tuple[tuple, tuple]], dev) -> Dict[tuple, tuple]:
    """Per signature, static input buffers for its example: views into ONE buffer per input position, sized for the largest shape, with
    the strides ``clone`` would give the example (channels-last stays channels-last).  The shapes share memory: a step copies its batch in."""
    n_in = len(examples[0][1])
    nbytes = [max(ex[i].numel() * ex[i].element_size() for _, ex in examples) for i in range(n_in)]
    bufs = [torch.empty(max(n, 16), device=dev, dtype=torch.uint8) for n in nbytes]
    out = {}
    for sig, ex in examples:
        views = []
        for buf, t in zip(bufs, ex):
            flat = buf[:t.numel() * t.element_size()].view(t.dtype)
            views.append(flat.as_strided(t.shape, torch.empty_like(t, device="meta").stride()))
        out[sig] = tuple(views)
    return out


def variable_batch_pairs(crop_w: int, crop_h: int, batch: int, max_scales: int = 5, check_scale: int = 32, min_w: int = 160, max_w: int = 320,
                         min_h: int = 160, max_h: int = 320) -> List[Tuple[int, int, int]]:
    """The sorted (h, w, batch) table the reference's variable-batch sampler draws from (``sampler.vbs``: crop_size_width / _height,
    train_batch_size0, max_n_scales, check_scale, min/max_crop_size_width / _height).  Per axis, ``max_scales`` evenly spaced sizes from min
    to max plus the base crop (exact duplicates merged), each rounded to the nearest multiple of ``check_scale`` (never below it, and one step
    up where rounding lost more than 10 %), sorted.  The i-th height pairs with the i-th width, and each pair's batch keeps crop_h * crop_w *
    batch pixels: max(1, int(round(pixels / (h * w), 2))).  Duplicate pairs are merged."""
    def sizes(base, lo, hi):
        vals = {float(v) for v in _linspace(lo, hi, max_scales)}
        vals.add(base)
        return sorted(_round_to(v, check_scale) for v in vals)
    pixels = crop_w * crop_h * batch
    pairs = {(h, w, max(1, int(round(pixels / (h * w), 2)))) for h, w in zip(sizes(crop_h, min_h, max_h), sizes(crop_w, min_w, max_w))}
    return sorted(pairs)


def _linspace(lo: float, hi: float, n: int) -> List[float]:
    import numpy as np
    return [float(v) for v in np.linspace(lo, hi, int(n))]


def _round_to(v: float, d: int) -> int:
    r = max(d, int(v + d / 2) // d * d)
    return r + d if r < 0.9 * v else r


def linear_curriculum(start: float, end: float, period: int) -> torch.Tensor:
    """loss_fn/neural_augmentation.py:linear_curriculum: period + 1 points from start to end."""
    return torch.linspace(start=start, end=end, steps=period + 1, dtype=torch.float)


def cosine_curriculum(start: float, end: float, period: int) -> torch.Tensor:
    """loss_fn/neural_augmentation.py:cosine_curriculum."""
    import math
    return torch.tensor([end + 0.5 * (start - end) * (1 + math.cos(math.pi * i / (period + 1))) for i in range(period + 1)], dtype=torch.float)


def psnr_to_mse(psnr: float) -> float:
    """PSNR = 20 log10(255) - 10 log10(MSE) (neural_augmentation.py:69)."""
    import math
    return 10.0 ** ((20.0 * math.log10(255.0) - psnr) / 10.0)


class NeuralAugmentationLoss:
    """The RangeAugment loss with the PSNR metric (loss_fn/neural_augmentation.py:NeuralAugmentation): a smooth-L1 loss between each augmented
    image's MSE against its (mixed) input, in 0..255 units, and a target MSE, times alpha / 65025.  ``target_value`` is a PSNR or a
    (start, end) pair followed over ``period`` (= scheduler.max_epochs, or max_iterations when iteration based) steps by the ``linear`` or
    ``cosine`` curriculum; past the end the last entry holds.  The table and the position (``set_epoch``) live on the device.  ``weight`` is
    the term's weight in the composite loss.  The loss reads the squared errors the augmentor kernels computed (``augmented_tensor`` must come
    from ``DistributionNeuralAugmentor``)."""

    def __init__(self, target_value=(40, 10), curriculum_method: str = "cosine", alpha: float = 100.0, period: Optional[int] = None,
                 weight: float = 1.0):
        if isinstance(target_value, (int, float)):
            self.table = torch.tensor([psnr_to_mse(float(target_value))], dtype=torch.float)
        elif isinstance(target_value, (list, tuple)) and len(target_value) == 2:
            if period is None:
                raise ValueError("a (start, end) target needs period (scheduler.max_epochs or scheduler.max_iterations)")
            fn = {"linear": linear_curriculum, "cosine": cosine_curriculum}.get(curriculum_method)
            if fn is None:
                raise NotImplementedError(f"curriculum_method {curriculum_method!r}: 'linear' or 'cosine'")
            self.table = fn(start=psnr_to_mse(float(target_value[0])), end=psnr_to_mse(float(target_value[1])), period=int(period))
        else:
            raise NotImplementedError(f"target_value {target_value!r}: a PSNR or a (start, end) pair")
        self.alpha, self.weight = float(alpha), float(weight)
        self.epoch = 0
        self._target = self._step = None

    def _device(self, device):
        if self._target is None or self._target.device != device:
            self._target = self.table.to(device)
            self._step = torch.tensor([self.epoch], dtype=torch.int64, device=device)
        return self._target, self._step

    def set_epoch(self, epoch: int) -> None:
        self.epoch = int(epoch)
        if self._step is not None:
            # a fresh pinned buffer per call: the copy queued by an earlier call may not have run yet and must still read its own value
            # (the host allocator keeps the buffer until the copy is done)
            self._step.copy_(torch.tensor([self.epoch], dtype=torch.int64).pin_memory(), non_blocking=True)

    def _apply(self, x_aug: torch.Tensor, ce, w_na: float, ce_weight: float, scale, parts):
        sq = getattr(x_aug, "_cvb_sq", None)
        if sq is None:
            raise ValueError("NeuralAugmentationLoss needs the augmented_tensor of a DistributionNeuralAugmentor (model output in training mode)")
        target, step = self._device(sq.device)
        cfg = SimpleNamespace(target=target, step=step, alpha=self.alpha, w_na=w_na, w_ce=float(ce_weight), H=x_aug.shape[2], W=x_aug.shape[3],
                              scale=scale, parts=parts)
        return Fn.NeuralAugLossFn.apply(sq, ce, cfg)

    def __call__(self, input_sample, prediction) -> torch.Tensor:
        """L_na of ``prediction["augmented_tensor"]`` (the reference's call signature; the input is the image the augmentor was given)."""
        return self._apply(prediction["augmented_tensor"], None, 1.0, 1.0, None, None)

    def composite(self, x_aug: torch.Tensor, ce: torch.Tensor, ce_weight: float = 1.0, scale=None, parts=None) -> torch.Tensor:
        """ce_weight * ce + weight * L_na in one launch; ``parts`` (device fp32 [2]) receives (ce, L_na)."""
        return self._apply(x_aug, ce, self.weight, ce_weight, scale, parts)


class MixingSampler:
    """Host-side sampling of the mixing parameters exactly as the reference's transforms draw them (data/transforms/image_torch.py:124-137,
    :315-338; selection between the two as apply_mixing_transforms :446-470): lambda ~ Beta(alpha, alpha) via torch._sample_dirichlet, the
    cutmix box from two randint draws.  ``sample(H, W)`` returns the arguments of ``TrainStep.set_mix``."""

    def __init__(self, mixup_alpha: Optional[float] = 0.2, mixup_p: float = 1.0, cutmix_alpha: Optional[float] = 1.0, cutmix_p: float = 1.0):
        self.mixup = (float(mixup_alpha), float(mixup_p)) if mixup_alpha else None
        self.cutmix = (float(cutmix_alpha), float(cutmix_p)) if cutmix_alpha else None

    def sample(self, H: int, W: int):
        import math
        import random
        choices = [c for c in (("mixup",) + self.mixup if self.mixup else None, ("cutmix",) + self.cutmix if self.cutmix else None) if c]
        if not choices:
            return None, 1.0, (0, 0, 0, 0)
        kind, alpha, p = random.choice(choices)
        if torch.rand(1).item() >= p:
            return None, 1.0, (0, 0, 0, 0)
        lam = float(torch._sample_dirichlet(torch.tensor([alpha, alpha]))[0])
        if kind == "mixup":
            return "mixup", lam, (0, 0, 0, 0)
        r_x, r_y = int(torch.randint(W, (1,))), int(torch.randint(H, (1,)))
        r = 0.5 * math.sqrt(1.0 - lam)
        rw, rh = int(r * W), int(r * H)
        x1, y1, x2, y2 = max(r_x - rw, 0), max(r_y - rh, 0), min(r_x + rw, W), min(r_y + rh, H)
        return "cutmix", float(1.0 - (x2 - x1) * (y2 - y1) / (W * H)), (x1, y1, x2, y2)


class ZeroShotAccuracy:
    """Zero-shot top-1 / top-5 accuracy of a CLIP model over an evaluation set (the recipe's ``top1.zero_shot_image_logits``: clip.py:184-202,
    metrics/topk_accuracy.py).  The class table is built once, from the prompts [B, Cl, M, L], when the metric is created; the model must
    be in eval mode.  ``update`` scores one image batch and counts its hits on the device (no host sync); ``compute`` syncs once and
    returns percentages.

        acc = ZeroShotAccuracy(model.eval(), prompts)
        for images, labels in loader:
            acc.update(images, labels)
        acc.compute()                         # {"top1": ..., "top5": ...}
    """

    def __init__(self, model: torch.nn.Module, class_tokens: torch.Tensor):
        self.model = model
        self.table = model.zero_shot_table(class_tokens)
        self.hits = torch.zeros(2, device=self.table.device, dtype=torch.int64)
        self.count = 0

    def update(self, images: torch.Tensor, targets: torch.Tensor) -> None:
        targets = targets.to(device=self.table.device, dtype=torch.int64).contiguous()
        self.model.zero_shot_logits(images, self.table, targets=targets, hits=self.hits)
        self.count += int(targets.shape[0])

    def compute(self) -> dict:
        top1, top5 = self.hits.tolist()
        n = max(self.count, 1)
        return {"top1": 100.0 * top1 / n, "top5": 100.0 * top5 / n}


class EvalStep:
    """The reference's ``val_epoch`` (engine/training_engine.py:608-640) for a classifier: the eval-mode forward and the recipes'
    ``stats.val: [loss, top1, top5]``, counted on the device (``cvb_cls_metrics``), optionally one CUDA graph per crop.

        ev = EvalStep(step.ema_model())          # or EvalStep(model): the live model, switched to eval for each pass and restored after
        ev.capture(batch=100, crop=(256, 256))   # optional, one graph per crop; eager without it
        for x, y in val_loader:
            ev.update(x, y)                      # no host sync
        metrics = ev.compute()                   # {"loss", "top1", "top5"}: one sync; summed over the process group
        ev.reset()

    ``loss`` is the cross entropy without label smoothing (the reference's loss in eval mode; RangeAugment's augmentation term is 0 there),
    summed over the rows and divided by their number N at ``compute``; ``topk`` = 100 * hits / N.  A row is a top-k hit iff fewer than k
    classes have a logit strictly greater than the target's, compared on the classifier's bf16 logits (ties count for the target; torch.topk
    leaves tie order unspecified).  Rows whose target is ``ignore_index`` are not counted.

    Captured: ``update`` copies a batch into the static buffers of its crop's graph; a smaller batch (the ragged last one) fills the first
    rows and the rest get target ``ignore_index``, so it needs no graph of its own.  A batch larger than the captured one, or a crop that was
    not captured, raises.  All graphs share one memory pool.

    Weight refresh: the forward reads kernel-layout (bf16) copies of the weights, which an eval-mode forward refreshes only when a weight
    changed -- a decision taken on the host, which a captured graph would freeze.  So before the first pass after any weight change (a
    ``_WEIGHTS_GENERATION`` bump, which every TrainStep step or replay and every optimizer step makes, or a parameter's version moving)
    ``update`` refreshes every kernel-layout copy of the evaluated model once, eagerly; the captured graphs contain no refresh and always read
    current weights.

    Data parallel: each rank counts its own shard; ``compute`` sums ``[loss_sum, top1, top5, n]`` over ``process_group`` with one
    all-reduce."""

    def __init__(self, model: torch.nn.Module, *, ignore_index: int = -1, process_group=None):
        import torch.distributed as dist
        self.model = model
        self.device = next(model.parameters()).device
        self.ignore_index = int(ignore_index)
        self.group = process_group
        self.world = dist.get_world_size(process_group) if dist.is_available() and dist.is_initialized() else 1
        self.loss_sum = torch.zeros(1, device=self.device, dtype=torch.float64)
        self.counts = torch.zeros(3, device=self.device, dtype=torch.int64)  # top-1 hits, top-5 hits, rows
        self._ticket = torch.zeros(1, device=self.device, dtype=torch.int32)
        self._row_loss = torch.zeros(0, device=self.device, dtype=torch.float32)
        self._graphs: Dict[tuple, tuple] = {}  # (C, H, W) -> (CUDA graph, static images, static targets, static logits)
        self._pool = None
        self._weights_seen = None
        self.logits: Optional[torch.Tensor] = None  # bf16 logits of the last batch (captured: the graph's static output; all its rows)
        self.launches_per_crop: Dict[tuple, int] = {}  # (C, H, W) -> kernel launches of its captured pass

    # ---- weights
    def _prepared(self) -> list:
        """Every kernel-layout weight cache of the model (the ``prep`` of each module's kernel configuration)."""
        out, seen = [], set()
        for m in self.model.modules():
            for v in vars(m).values():
                prep = getattr(v, "prep", None) if isinstance(v, SimpleNamespace) else None
                if isinstance(prep, ops.PreparedWeights) and id(prep) not in seen:
                    seen.add(id(prep))
                    out.append(prep)
        return out

    def _refresh(self, force: bool = False) -> None:
        key = (ops._WEIGHTS_GENERATION[0], sum(p._version for p in self.model.parameters()))
        if force or key != self._weights_seen:
            for prep in self._prepared():
                prep.refresh()
            self._weights_seen = key

    # ---- one pass
    def _scratch(self, B: int) -> torch.Tensor:
        if self._row_loss.numel() < B:
            if self._graphs:
                raise ValueError(f"EvalStep: batch {B} exceeds the captured batch {self._row_loss.numel()}")
            self._row_loss = torch.zeros(B, device=self.device, dtype=torch.float32)
        return self._row_loss

    def _pass(self, x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
        training = self.model.training
        if training:
            self.model.eval()
        try:
            out = self.model(x)
        finally:
            if training:
                self.model.train(True)
        logits = out["logits"] if isinstance(out, dict) else out  # a RangeAugment model: {"augmented_tensor": None, "logits"} in eval
        ops.cls_metrics(logits, y, self.loss_sum, self.counts, self._scratch(y.shape[0]), self._ticket, self.ignore_index)
        return logits

    def update(self, images: torch.Tensor, targets: torch.Tensor) -> None:
        """Count one validation batch (no host sync)."""
        targets = targets.to(device=self.device, dtype=torch.int64)
        self._refresh()
        with torch.no_grad():
            if not self._graphs:
                self.logits = self._pass(images.to(self.device), targets.contiguous())
                return
            key = tuple(images.shape[1:])
            entry = self._graphs.get(key)
            if entry is None:
                raise ValueError(f"EvalStep.update: no CUDA graph was captured for images of shape [*, {', '.join(map(str, key))}]; captured: "
                                 f"{[list(k) for k in self._graphs]}")
            graph, sx, sy, logits = entry
            b = images.shape[0]
            if b > sx.shape[0]:
                raise ValueError(f"EvalStep.update: batch {b} exceeds the captured batch {sx.shape[0]}")
            sx[:b].copy_(images, non_blocking=True)
            sy[:b].copy_(targets, non_blocking=True)
            if b < sy.shape[0]:
                sy[b:].fill_(self.ignore_index)
            graph.replay()
            self.logits = logits

    # ---- capture
    def capture(self, batch: int, crop: Tuple[int, int], channels: int = 3, warmup: int = 2) -> "EvalStep":
        """Capture the eval pass of ``batch`` images of size ``crop`` (H, W) as one CUDA graph (call once per crop; the first capture fixes the
        largest batch).  Warm-up passes run eagerly on rows that all carry ``ignore_index``, so they count nothing."""
        H, W = int(crop[0]), int(crop[1])
        key = (int(channels), H, W)
        if key in self._graphs:
            raise ValueError(f"EvalStep.capture: crop {crop} was already captured")
        dev = self.device
        sx = torch.zeros((batch,) + key, device=dev, dtype=torch.float32)
        sy = torch.full((batch,), self.ignore_index, device=dev, dtype=torch.int64)
        self._scratch(batch)
        torch.cuda.synchronize(dev)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side), torch.no_grad():
            self._refresh()
            for _ in range(max(1, warmup)):
                self._pass(sx, sy)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize(dev)
        self._refresh(force=True)  # caches the warm-up created included: the graph's forward then skips every refresh
        torch.cuda.synchronize(dev)
        gc.collect()
        if self._pool is None:
            self._pool = torch.cuda.graph_pool_handle()
        graph = torch.cuda.CUDAGraph()
        n0 = ops.launch_count
        with torch.cuda.graph(graph, pool=self._pool), torch.no_grad():
            logits = self._pass(sx, sy)
        self.launches_per_crop[key] = ops.launch_count - n0
        self._graphs[key] = (graph, sx, sy, logits)
        return self

    def graph_pool_bytes(self) -> int:
        """Device memory the captured eval graphs' shared pool holds (0 before capture)."""
        return _pool_bytes(self._pool)

    # ---- results
    def compute(self) -> Dict[str, float]:
        """{"loss", "top1", "top5"} over every row counted since the last ``reset`` (summed over the process group): one host sync."""
        acc = torch.cat([self.loss_sum, self.counts.to(torch.float64)])
        if self.world > 1:
            import torch.distributed as dist
            dist.all_reduce(acc, op=dist.ReduceOp.SUM, group=self.group)
        loss, top1, top5, n = acc.tolist()
        if n == 0:
            return {"loss": float("nan"), "top1": float("nan"), "top5": float("nan")}
        return {"loss": loss / n, "top1": 100.0 * top1 / n, "top5": 100.0 * top5 / n}

    def reset(self) -> None:
        self.loss_sum.zero_()
        self.counts.zero_()
