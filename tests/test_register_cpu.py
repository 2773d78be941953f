"""register._make_shell without a reference checkout: each classifier register_with_cvnets() registers, wrapped in a shell around a
stand-in for the reference's BaseImageEncoder (a plain nn.Module taking opts)."""
import pytest
import torch
from torch import nn

import ml_cvnets_b200 as m
from ml_cvnets_b200.register import _KEEP_REFERENCE, _make_shell

OURS = ("forward", "forward_classifier", "extract_features", "reset_parameters")


class StandInBase(nn.Module):
    def __init__(self, opts, *args, **kwargs) -> None:
        super().__init__()


MODELS = {
    "mobilevit_v2": (m.MobileViTv2, lambda: m.default_opts(0.5, n_classes=10)),
    "mobilevit": (m.MobileViT, lambda: m.default_mit_opts("xx_small", n_classes=10)),
    "vit": (m.VisionTransformer, lambda: m.default_vit_opts("tiny", n_classes=10)),
    "efficientnet": (m.EfficientNet, lambda: m.default_effnet_opts("b0", n_classes=10)),
}


@pytest.mark.parametrize("kind", list(MODELS))
def test_shell_runs_this_package_and_holds_the_same_model(kind):
    cls, opts = MODELS[kind]
    shell_cls = _make_shell(cls, StandInBase, cls.__name__ + "B200")
    assert issubclass(shell_cls, StandInBase)
    for name in OURS:  # inherited ones (ImageEncoder.forward) included
        assert getattr(shell_cls, name) is getattr(cls, name), name
    for name in _KEEP_REFERENCE:
        assert name not in shell_cls.__dict__, name
    torch.manual_seed(0)
    shell = shell_cls(opts())
    torch.manual_seed(0)
    plain = cls(opts())
    ours, ref = shell.state_dict(), plain.state_dict()
    assert list(ours) == list(ref)
    for k in ref:
        assert torch.equal(ours[k], ref[k]), k
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        shell(torch.zeros(1, 3, 64, 64))
