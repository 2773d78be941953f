"""Injection into an importable apple/ml-cvnets checkout (SURVEY.md 8b): the reference has no operator/FFI boundary, its
plug-in mechanism is ``MODEL_REGISTRY`` plus the import namespaces ``cvnets.modules`` / ``cvnets.layers``.

    import ml_cvnets_b200.register as r; r.register_with_cvnets()
    opts.model.classification.name = "mobilevit_v2_b200"   # or keep "mobilevit_v2" after rebind_modules()
    model = cvnets.get_model(opts)                          # engine/training_engine.py consumes it unchanged

Nothing here is needed (or importable) on the GPU box, where the reference does not exist; the product is standalone.
"""
from __future__ import annotations


def rebind_modules() -> None:
    """Injection point 1: replace the block classes in the namespaces the reference's model files import from
    (``from cvnets.modules import InvertedResidual, MobileViTBlockv2`` at mobilevit_v2.py:15-16).  Must run before the
    first ``MODEL_REGISTRY`` lookup (which lazily imports cvnets/models/**)."""
    import cvnets.modules as cm
    from . import modules as ours
    cm.InvertedResidual = ours.InvertedResidual
    cm.InvertedResidualSE = ours.InvertedResidualSE  # mobilenetv3.py / efficientnet.py import it from cvnets.modules
    cm.EfficientNetBlock = ours.EfficientNetBlock  # models/classification/efficientnet.py
    cm.SqueezeExcitation = ours.SqueezeExcitation
    cm.MobileViTBlockv2 = ours.MobileViTBlockv2
    cm.TransformerEncoder = ours.TransformerEncoder  # used by vit.py:29, mobilevit_block.py (v1), text_encoders/transformer.py:20


# reference plumbing the shells keep from BaseImageEncoder / BaseAnyNNModel (optimizer groups, freezing, logging, CLI, fine-tuning hooks)
_KEEP_REFERENCE = {"get_trainable_parameters", "freeze_norm_layers", "info", "update_classifier", "dummy_input_and_label", "build_model",
                   "add_arguments", "get_activation_checkpoint_submodule_class", "get_fsdp_wrap_policy", "set_gradient_checkpointing"}


def _make_shell(ours_cls, base_cls, shell_name: str):
    """A ``base_cls`` (the reference's own base encoder: utils/registry.py:111-167 only accepts BaseAnyNNModel subclasses) whose children,
    parameters, buffers and private state are those of this package's model, and whose forward / feature-extraction methods are this package's."""
    import types

    def __init__(self, opts, *args, **kwargs) -> None:
        base_cls.__init__(self, opts, *args, **kwargs)
        inner = ours_cls(opts, *args, **kwargs)
        for k, m in inner.named_children():
            setattr(self, k, m)
        for k, prm in inner._parameters.items():
            self.register_parameter(k, prm)
        for k, buf in inner._buffers.items():
            self.register_buffer(k, buf)
        skip = {"_parameters", "_buffers", "_modules", "training"}
        for k, v in inner.__dict__.items():  # plain attributes: kernel-layout caches, module chains, configuration
            if k not in skip and not (k.startswith("_") and "hook" in k) and k not in self._modules:
                self.__dict__[k] = v

    ns = {"__init__": __init__, "__doc__": f"Reference-side shell around ml_cvnets_b200.{ours_cls.__name__}; forward goes straight to the CUDA path."}
    for k, v in ours_cls.__dict__.items():
        if isinstance(v, types.FunctionType) and not (k.startswith("__") and k.endswith("__")) and k not in _KEEP_REFERENCE:
            ns[k] = v
    return type(shell_name, (base_cls,), ns)


def register_with_cvnets(name: str = "mobilevit_v2_b200"):
    """Injection point 2: register this package's assemblers under new model names: ``mobilevit_v2_b200`` (or ``name``), ``mobilevit_b200``, ``vit_b200``,
    ``efficientnet_b200``.  Returns the MobileViTv2 shell class."""
    from cvnets.models import MODEL_REGISTRY
    from cvnets.models.classification.base_image_encoder import BaseImageEncoder
    from .models import MobileViTv2
    from .models_effnet import EfficientNet
    from .models_mit import MobileViT
    from .models_vit import VisionTransformer

    out = None
    for reg_name, cls in ((name, MobileViTv2), ("mobilevit_b200", MobileViT), ("vit_b200", VisionTransformer), ("efficientnet_b200", EfficientNet)):
        key = f"classification:{reg_name}"
        registry = getattr(MODEL_REGISTRY, "registry", {})
        if key in registry:
            shell = registry[key]
        else:
            shell = _make_shell(cls, BaseImageEncoder, cls.__name__ + "B200")
            MODEL_REGISTRY.register(name=reg_name, type="classification")(shell)
        out = out or shell
    return out
