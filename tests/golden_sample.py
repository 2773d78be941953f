"""Large reference tensors in tests/golden are stored as a fixed sample of their elements (keeps every fixture file under 1 MB):
``{"shape": [...], "val": values}`` at the evenly strided flat positions ``i * numel // len(val)``.  The comparisons reduce our
tensor to the same positions; small tensors are stored whole and pass through unchanged."""
import math

import torch


def sample_positions(numel, n, device=None):
    return torch.arange(n, device=device, dtype=torch.int64) * numel // n


def sample_large(t, limit=8192, n=4096):
    """Fixture side: `t` itself, or `n` of its elements when it has more than `limit`."""
    if not torch.is_tensor(t) or t.numel() <= limit:
        return t
    return {"shape": list(t.shape), "val": t.detach().flatten()[sample_positions(t.numel(), n)].clone()}


def at_sample(ours, ref):
    """(ours, reference) restricted to the stored positions when the reference is a sample."""
    if not isinstance(ref, dict):
        return ours, ref
    assert list(ours.shape) == ref["shape"], (list(ours.shape), ref["shape"])
    return ours.flatten()[sample_positions(ours.numel(), ref["val"].numel(), ours.device)], ref["val"].to(ours.device)


def ref_shape(ref):
    return tuple(ref["shape"]) if isinstance(ref, dict) else tuple(ref.shape)


def ref_norm(ref):
    """L2 norm of the reference tensor (estimated from the sample for a sampled one)."""
    if not isinstance(ref, dict):
        return float(ref.float().norm())
    return float(ref["val"].float().norm()) * math.sqrt(math.prod(ref["shape"]) / ref["val"].numel())
