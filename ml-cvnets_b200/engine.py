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
"""
from __future__ import annotations

import gc
from types import SimpleNamespace
from typing import Optional

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
                 aug_loss: Optional["NeuralAugmentationLoss"] = None, ce_weight: float = 1.0):
        """``forward_loss(model, *inputs, cfg) -> loss`` replaces the default ``cross_entropy(model(x), y)`` (e.g. CLIP's contrastive step);
        ``cfg.scale`` is the device-resident loss scale the loss's backward must multiply by, ``cfg.world / rank / group`` the process group.
        ``optimizer="sgd"`` swaps AdamW for SGD with ``momentum`` / ``nesterov`` (optim.FlatSGD; ``betas`` / ``eps`` are then unused and
        ``max_norm`` None / 0 means no clipping).  A model with a RangeAugment augmentor returns ``{"augmented_tensor", "logits"}``; the cross
        entropy reads ``logits``, and with ``aug_loss`` the step minimises ``ce_weight * CE + aug_loss.weight * L_na`` (the RangeAugment recipes'
        composite_loss); ``loss_parts`` (device fp32 [2]) then holds (CE, L_na) of the last step."""
        import torch.distributed as dist
        if optimizer not in ("adamw", "sgd"):
            raise ValueError(f"optimizer must be 'adamw' or 'sgd', got {optimizer!r}")
        self.model = model
        self.ws = StepWorkspace(model)
        common = dict(lr=lr, weight_decay=weight_decay, no_decay_bn_filter_bias=no_decay_bn_filter_bias, max_norm=max_norm, init_scale=init_scale,
                      growth_interval=growth_interval, ema_momentum=ema_momentum)
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
        self._mix_host = torch.tensor([0.0, 1.0, 0.0, 0.0, 0.0, 0.0]).pin_memory()
        self.forward_loss = forward_loss
        if aug_loss is None and ce_weight != 1.0:
            raise ValueError("ce_weight weighs the cross entropy against aug_loss; without aug_loss the loss is the cross entropy")
        self.aug_loss, self.ce_weight = aug_loss, float(ce_weight)
        self.loss_parts = torch.zeros(2, device=self.ws.device, dtype=torch.float32) if aug_loss is not None else None
        self.loss_cfg.group = process_group
        self.loss_cfg.world, self.loss_cfg.rank = self.world, (dist.get_rank(process_group) if data_parallel else 0)
        self._one = torch.ones((), device=self.ws.device, dtype=torch.float32)
        self._graph = None
        self._static = None
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
        h = self._mix_host
        h[0], h[1] = mode, float(lam)
        h[2], h[3], h[4], h[5] = [float(v) for v in box]
        self.ws.mix.copy_(h, non_blocking=True)

    def state_dict(self):
        return self.opt.state_dict()

    def load_state_dict(self, sd):
        self.opt.load_state_dict(sd)

    # ---- one iteration, eager launches
    def _step(self, *inputs: torch.Tensor) -> torch.Tensor:
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
            torch.autograd.backward(loss, grad_tensors=self._one)
        finally:
            ws.active = False
        ws.finish_reduce()
        self.opt.step(grad_div=float(self.world))
        return loss

    def step(self, *inputs: torch.Tensor) -> torch.Tensor:
        if self._graph is None:
            self.eager_steps += 1
            return self._step(*inputs)
        *statics, sloss = self._static
        for s_in, t in zip(statics, inputs):
            if t is not s_in:
                s_in.copy_(t, non_blocking=True)
        self._graph.replay()
        ops.invalidate_prepared_weights()
        return sloss

    __call__ = step

    # ---- whole step as one CUDA graph
    def capture(self, *inputs: torch.Tensor, warmup: int = 3):
        """Warm up eagerly (workspace planning needs two steps), then capture fwd + loss + bwd (+ all-reduce) + optimizer tail."""
        assert self._graph is None, "already captured"
        dev = self.ws.device
        statics = [t.to(dev).clone() for t in inputs]
        torch.cuda.synchronize(dev)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(max(0, max(warmup, 3) - self.eager_steps)):
                self._step(*statics)
                self.eager_steps += 1
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize(dev)
        gc.collect()  # no autograd graph of an eager step (leaf accumulators are bound to the stream they were created on) may survive into capture
        graph = torch.cuda.CUDAGraph()
        n0 = ops.launch_count
        with torch.cuda.graph(graph):
            sloss = self._step(*statics)
        self.launches_per_step = ops.launch_count - n0
        self._graph, self._static = graph, (*statics, sloss)
        return self

    @property
    def static_inputs(self):
        return None if self._static is None else self._static[:-1]


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
