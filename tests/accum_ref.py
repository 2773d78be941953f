"""fp32 restatement of the reference's training loop with gradient accumulation (engine/training_engine.py:221-312, ``common.accum_freq``),
built on the EfficientNet restatement (tests/efficientnet_ref.py) and pinned to tests/golden/accum_fp32.pt (make_golden_accum.py):

  * every micro-batch: forward in training mode (BatchNorm running statistics and ``num_batches_tracked`` move), the label-smoothed cross
    entropy, backward into ``.grad`` -- gradients are SUMMED over the window, the loss is not divided by ``accum_freq``;
  * every ``accum_freq``-th micro-batch: ``torch.optim.SGD`` (momentum, Nesterov, weight decay on the parameters of more than one dimension:
    the reference's ``no_decay_bn_filter_bias`` groups), zero the gradients, and one EMA update of the whole state (eval_ref.ema_state).

``flat_sample`` is the fixture's snapshot format: the tensors' fixed samples (golden_sample.py, at most 32 elements each) as one fp32 vector."""
from typing import Dict, List, Sequence

import torch
import torch.nn.functional as F
from torch import Tensor

import efficientnet_ref as E
import eval_ref
from golden_sample import sample_positions

SAMPLE = 32


def flat_sample(tensors: Sequence[Tensor]) -> Tensor:
    out = []
    for t in tensors:
        t = t.detach().reshape(-1)
        out.append(t[sample_positions(t.numel(), min(t.numel(), SAMPLE), t.device)].float())
    return torch.cat(out).cpu()


def train_windows(P: Dict[str, Tensor], xs: List[Tensor], ys: List[Tensor], *, accum_freq: int, lr: float, momentum: float,
                  weight_decay: float, label_smoothing: float, ema_momentum: float, mode: str = "b0"):
    """Train ``P`` (oracle parameters: weights require grad, buffers in place) on the micro-batches in order.  Returns (losses, the state
    after every micro-batch, the (state, optimizer, EMA) after every window) with ``P`` itself, so the caller samples what it needs."""
    weights = [v for v in P.values() if v.requires_grad]
    opt = torch.optim.SGD([{"params": [p for p in weights if p.dim() > 1], "weight_decay": weight_decay},
                           {"params": [p for p in weights if p.dim() == 1], "weight_decay": 0.0}], lr=lr, momentum=momentum, nesterov=True)
    ema = {k: v.detach().clone() for k, v in P.items()}
    nbt = [k for k in P if k.endswith("num_batches_tracked")]
    opt.zero_grad()
    losses, micro, windows = [], [], []
    for batch_id, (x, y) in enumerate(zip(xs, ys)):
        loss = F.cross_entropy(E.efficientnet_forward(P, x, mode=mode, training=True), y, label_smoothing=label_smoothing)
        loss.backward()
        with torch.no_grad():
            for k in nbt:
                P[k] += 1
        losses.append(float(loss.detach()))
        micro.append({k: v.detach().clone() for k, v in P.items()})
        if (batch_id + 1) % accum_freq == 0:
            opt.step()
            opt.zero_grad()
            ema = eval_ref.ema_state(ema, {k: v.detach() for k, v in P.items()}, ema_momentum)
            windows.append(({k: v.detach().clone() for k, v in P.items()}, {k: opt.state[P[k]]["momentum_buffer"].clone()
                                                                            for k in P if P[k].requires_grad}, ema))
    return losses, micro, windows
