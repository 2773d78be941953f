"""fp32 / fp64 restatements of classification validation, pinned to tests/golden/eval_fp32.pt (make_golden_eval.py):

  * ``ema_state``: one update of the reference's EMA of the whole state_dict (cvnets/misc/averaging_utils.py:55,
    ``ema * (1 - m) + m * v`` in the tensor's dtype; an integer buffer gets the fp32 average truncated back to its dtype, as ``copy_`` does);
  * ``cls_metrics``: the validation statistics of one batch in fp64 -- the summed cross entropy without label smoothing, and top-1 / top-5
    hits by the rank rule of cvb_cls_metrics (a hit iff fewer than k classes have a logit strictly greater than the target's; rows with
    ``ignore_index`` skipped)."""
from typing import Dict

import torch
from torch import Tensor


def ema_state(ema: Dict[str, Tensor], live: Dict[str, Tensor], momentum: float) -> Dict[str, Tensor]:
    out = {}
    for k, e in ema.items():
        v = live[k]
        out[k] = (e * (1.0 - momentum) + momentum * v).to(e.dtype)
    return out


def ema_flat(ema: Tensor, src: Tensor, momentum: float) -> Tensor:
    """The same update on flat fp32 buffers (cvb_ema_update's operation order)."""
    return ema * (1.0 - momentum) + momentum * src


def cls_metrics(logits: Tensor, target: Tensor, ignore_index: int = -1) -> Dict[str, float]:
    """{"loss_sum", "top1", "top5", "n"} of one batch; logits [B, C] in any float dtype (compared as given, summed in fp64)."""
    keep = target != ignore_index
    lg, t = logits[keep], target[keep].long()
    if lg.shape[0] == 0:
        return {"loss_sum": 0.0, "top1": 0, "top5": 0, "n": 0}
    ce = torch.logsumexp(lg.double(), dim=1) - lg.double().gather(1, t[:, None])[:, 0]
    rank = (lg > lg.gather(1, t[:, None])).sum(1)
    return {"loss_sum": float(ce.sum()), "top1": int((rank < 1).sum()), "top5": int((rank < 5).sum()), "n": int(lg.shape[0])}


def summarize(parts) -> Dict[str, float]:
    """EvalStep.compute's numbers from per-batch ``cls_metrics``: loss = sum CE / N, topk = 100 * hits / N."""
    n = sum(p["n"] for p in parts)
    return {"loss": sum(p["loss_sum"] for p in parts) / n, "top1": 100.0 * sum(p["top1"] for p in parts) / n,
            "top5": 100.0 * sum(p["top5"] for p in parts) / n}
