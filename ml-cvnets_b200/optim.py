"""Fused per-step tail of the reference's training loop (engine/training_engine.py:289-312) on ONE flat fp32 buffer per quantity:
GradScaler unscale + inf check, ``clip_grad_norm_``, AdamW with the reference's two parameter groups (cvnets/misc/common.py:122-176),
GradScaler update and -- optionally -- the EMA of the weights (cvnets/misc/averaging_utils.py:43-55): two kernel launches, all state on
the device, so the step stays one CUDA graph.  ``FlatSGD`` is the same step around SGD with (Nesterov) momentum.

    ws   = StepWorkspace(model)                 # p.grad become views of ws.flat_g (workspace.py)
    tail = FlatAdamW(model, ws, lr=2e-3, weight_decay=0.05, max_norm=10.0)
    ...backward...;  tail.step()                # cvb_grad_norm + cvb_adamw_step over the flat buffers

The learning rate lives in a DEVICE scalar (``set_lr``), so a per-iteration scheduler (scheduler.update_lr, training_engine.py:246-249)
keeps working under graph replay; ``state_dict`` / ``load_state_dict`` carry the moments, step count and loss-scale state for
checkpoint / resume (the reference checkpoints optimizer + gradient-scaler state: utils/checkpoint_utils.py).
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

from .ops import _count, _lib, _stream, invalidate_prepared_weights
from .workspace import StepWorkspace


class _FlatStep:
    """Flat parameter / gradient / weight-decay buffers, loss-scale state, device learning rate and EMA shared by the optimizer steps; a
    subclass owns its per-element state (``_moments``) and launches its step kernel in ``_update``."""

    _moments = ()

    def __init__(self, model: torch.nn.Module, ws: Optional[StepWorkspace], lr: float, weight_decay: float, no_decay_bn_filter_bias: bool,
                 max_norm: Optional[float], init_scale: float, growth_factor: float, backoff_factor: float, growth_interval: int,
                 ema_momentum: Optional[float], grads: Optional[torch.Tensor] = None):
        self.ws = ws if ws is not None else StepWorkspace(model)
        ws = self.ws
        self.params = ws.params
        dev, n = ws.device, ws.n
        self.n = n
        self.flat_p = torch.zeros(n, device=dev, dtype=torch.float32)
        self.flat_g = ws.flat_g if grads is None else grads  # the gradient buffer the step reads (TrainStep's accumulator with accum_freq > 1)
        assert self.flat_g.shape == ws.flat_g.shape and self.flat_g.dtype == torch.float32 and self.flat_g.is_contiguous()
        for name in self._moments:
            setattr(self, name, torch.zeros(n, device=dev, dtype=torch.float32))
        self.wd = torch.zeros(n, device=dev, dtype=torch.float32)
        for p in self.params:
            o, k = ws.offsets[id(p)]
            assert p.dtype == torch.float32 and p.is_contiguous()
            self.flat_p[o:o + k].copy_(p.data.view(-1))
            p.data = self.flat_p[o:o + k].view_as(p)  # parameters become views of the flat buffer (state_dict / modules see no change)
            decay = weight_decay if not (no_decay_bn_filter_bias and p.dim() == 1) else 0.0
            self.wd[o:o + k].fill_(decay)
        self.ema = self.flat_p.clone() if ema_momentum is not None else None
        self.ema_momentum = float(ema_momentum) if ema_momentum is not None else 0.0
        self.stats = torch.zeros(4, device=dev, dtype=torch.float32)
        self.partials = torch.zeros(2 * int(_lib().cvb_grad_norm_blocks(n)), device=dev, dtype=torch.float32)
        self.scale = torch.tensor([init_scale, 0.0], device=dev, dtype=torch.float32)
        self.step_count = torch.zeros(1, device=dev, dtype=torch.float32)
        self.hp = torch.tensor([float(lr)], device=dev, dtype=torch.float32)
        self._hp_host = torch.tensor([float(lr)], dtype=torch.float32).pin_memory()
        self.max_norm = float(max_norm) if max_norm else 0.0
        self.gs = (float(growth_factor), float(backoff_factor), int(growth_interval))
        # the reference optimizer interface schedulers poke at (optim/scheduler/base_scheduler.py: param_group['lr'] = ...)
        self.param_groups = [{"lr": float(lr), "weight_decay": float(weight_decay)}]

    # ---- scheduler hook: host value -> device scalar (a tiny async copy outside the captured step)
    def set_lr(self, lr: float) -> None:
        self.param_groups[0]["lr"] = float(lr)
        self._hp_host[0] = float(lr)
        self.hp.copy_(self._hp_host, non_blocking=True)

    def loss_scale(self) -> torch.Tensor:
        return self.scale[0:1]

    def step(self, grad_div: float = 1.0) -> None:
        """Gradients are read from ``flat_g``: the workspace's flat buffer or the buffer given as ``grads`` (already summed over ranks when data
        parallel; grad_div = world size)."""
        lr_now = self.param_groups[0]["lr"]
        if lr_now != float(self._hp_host[0]) and not torch.cuda.is_current_stream_capturing():
            self.set_lr(lr_now)
        _lib().cvb_grad_norm(self.flat_g.data_ptr(), self.n, self.scale.data_ptr(), float(grad_div), self.stats.data_ptr(),
                             self.partials.data_ptr(), _stream())
        _count()
        self._update()
        _count()
        invalidate_prepared_weights()  # raw-pointer update: eval-mode weight caches must refresh (Tensor._version did not move)

    def _update(self) -> None:
        raise NotImplementedError

    def _tail_args(self):
        gf, bf, gi = self.gs
        return (self.stats.data_ptr(), self.scale.data_ptr(), self.step_count.data_ptr(), gf, bf, gi,
                self.ema.data_ptr() if self.ema is not None else None, self.ema_momentum, self.partials.data_ptr(), _stream())

    # ---- EMA weights as a state_dict-shaped mapping (what EMA.ema_model.state_dict() holds for the parameters)
    def ema_parameters(self, model: torch.nn.Module) -> Dict[str, torch.Tensor]:
        assert self.ema is not None, "EMA is off (ema_momentum=None)"
        out = {}
        for name, p in model.named_parameters():
            if id(p) in self.ws.offsets:
                o, k = self.ws.offsets[id(p)]
                out[name] = self.ema[o:o + k].view_as(p)
        return out

    # ---- checkpoint / resume
    def state_dict(self) -> Dict[str, torch.Tensor]:
        sd = {name: getattr(self, name).clone() for name in self._moments}
        sd.update({"step": self.step_count.clone(), "scale": self.scale.clone(), "lr": self.hp.clone()})
        if self.ema is not None:
            sd["ema"] = self.ema.clone()
        return sd

    def load_state_dict(self, sd: Dict[str, torch.Tensor]) -> None:
        for name in self._moments:
            getattr(self, name).copy_(sd[name])
        self.step_count.copy_(sd["step"])
        self.scale.copy_(sd["scale"])
        self.set_lr(float(sd["lr"][0]))
        if self.ema is not None and "ema" in sd:
            self.ema.copy_(sd["ema"])


class FlatAdamW(_FlatStep):
    _moments = ("exp_avg", "exp_avg_sq")

    def __init__(self, model: torch.nn.Module, ws: Optional[StepWorkspace] = None, lr: float = 2e-3, betas=(0.9, 0.999), eps: float = 1e-8,
                 weight_decay: float = 0.05, no_decay_bn_filter_bias: bool = True, max_norm: float = 10.0, init_scale: float = 65536.0,
                 growth_factor: float = 2.0, backoff_factor: float = 0.5, growth_interval: int = 2000, ema_momentum: Optional[float] = None,
                 grads: Optional[torch.Tensor] = None):
        super().__init__(model, ws, lr, weight_decay, no_decay_bn_filter_bias, max_norm, init_scale, growth_factor, backoff_factor, growth_interval,
                         ema_momentum, grads)
        self.consts = (float(betas[0]), float(betas[1]), float(eps))

    def _update(self) -> None:
        b1, b2, eps = self.consts
        _lib().cvb_adamw_step(self.flat_p.data_ptr(), self.flat_g.data_ptr(), self.exp_avg.data_ptr(), self.exp_avg_sq.data_ptr(),
                              self.wd.data_ptr(), self.n, self.hp.data_ptr(), b1, b2, eps, self.max_norm, *self._tail_args())


class FlatSGD(_FlatStep):
    """torch.optim.SGD(momentum, nesterov, weight_decay) with the reference's two parameter groups (optim/sgd.py; the EfficientNet and MobileNet
    recipes: momentum 0.9, Nesterov, weight decay 4e-5, no_decay_bn_filter_bias).  ``max_norm`` None / 0 = no clipping (those recipes set no
    grad_clip).  ``state_dict`` carries ``momentum_buffer`` in place of AdamW's moments."""
    _moments = ("momentum_buffer",)

    def __init__(self, model: torch.nn.Module, ws: Optional[StepWorkspace] = None, lr: float = 0.1, momentum: float = 0.9, nesterov: bool = True,
                 weight_decay: float = 4e-5, no_decay_bn_filter_bias: bool = True, max_norm: Optional[float] = None, init_scale: float = 65536.0,
                 growth_factor: float = 2.0, backoff_factor: float = 0.5, growth_interval: int = 2000, ema_momentum: Optional[float] = None,
                 grads: Optional[torch.Tensor] = None):
        if nesterov and momentum <= 0.0:
            raise ValueError("Nesterov momentum requires momentum > 0 (torch.optim.SGD)")
        super().__init__(model, ws, lr, weight_decay, no_decay_bn_filter_bias, max_norm, init_scale, growth_factor, backoff_factor, growth_interval,
                         ema_momentum, grads)
        self.momentum, self.nesterov = float(momentum), bool(nesterov)

    def _update(self) -> None:
        _lib().cvb_sgd_step(self.flat_p.data_ptr(), self.flat_g.data_ptr(), self.momentum_buffer.data_ptr(), self.wd.data_ptr(), self.n,
                            self.hp.data_ptr(), self.momentum, int(self.nesterov), self.max_norm, *self._tail_args())
