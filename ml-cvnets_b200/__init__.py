"""ml-cvnets_b200: the apple/ml-cvnets vision-backbone hot path (MobileViTv2: InvertedResidual, MobileViTBlockv2,
LinearSelfAttention, LinearAttnFFN, conv+BN+SiLU; plus the ViT-style MultiHeadAttention / TransformerEncoder / LayerNorm) as hand-written sm_90a CUDA kernels behind a C ABI
(include/cvnets_b200.h) with drop-in ``nn.Module``s on top.  Import name: ``ml_cvnets_b200`` (alias package at the repo root).
"""
from . import _lib  # noqa: F401
from .layers import (GELU, BatchNorm2d, ConvLayer2d, Dropout, GlobalPool, Identity, LayerNorm, LayerNorm2D_NCHW, LayerNormFP32,  # noqa: F401
                     LinearLayer, LinearSelfAttention, MultiHeadAttention, Swish)
from .models import MobileViTv2, default_opts, get_configuration  # noqa: F401
from .models_effnet import EfficientNet, default_effnet_opts, get_effnet_configuration  # noqa: F401
from .models_clip import CLIP, SimpleImageProjectionHead, TextTransformer, clip_contrastive_loss, default_clip_opts  # noqa: F401
from .models_mit import MobileViT, default_mit_opts, get_mit_configuration  # noqa: F401
from .models_vit import VisionTransformer, default_vit_opts, get_vit_configuration  # noqa: F401
from .modules import EfficientNetBlock, InvertedResidual, InvertedResidualSE, SqueezeExcitation, LinearAttnFFN, MobileViTBlock, MobileViTBlockv2, TransformerEncoder  # noqa: F401
from .engine import EvalStep, NeuralAugmentationLoss, TrainStep, ZeroShotAccuracy, cross_entropy, variable_batch_pairs  # noqa: F401
from .neural_aug import Clip, DistributionNeuralAugmentor, UniformSampler, build_neural_augmentor  # noqa: F401
from .optim import FlatAdamW, FlatSGD  # noqa: F401
from .workspace import StepWorkspace  # noqa: F401

__all__ = ["InvertedResidualSE", "SqueezeExcitation", "MobileViTv2", "default_opts", "get_configuration", "InvertedResidual", "LinearAttnFFN", "MobileViTBlockv2",
           "ConvLayer2d", "LinearSelfAttention", "BatchNorm2d", "LayerNorm2D_NCHW", "GlobalPool", "LinearLayer", "Swish",
           "Dropout", "Identity", "TransformerEncoder", "MultiHeadAttention", "LayerNorm", "GELU", "TrainStep", "cross_entropy", "FlatAdamW",
           "StepWorkspace", "LayerNormFP32", "VisionTransformer", "default_vit_opts", "get_vit_configuration", "MobileViT", "default_mit_opts", "get_mit_configuration", "MobileViTBlock", "CLIP", "TextTransformer", "SimpleImageProjectionHead", "clip_contrastive_loss", "default_clip_opts", "ZeroShotAccuracy",
           "EfficientNetBlock", "EfficientNet", "default_effnet_opts", "get_effnet_configuration", "FlatSGD", "NeuralAugmentationLoss",
           "DistributionNeuralAugmentor", "UniformSampler", "Clip", "build_neural_augmentor", "variable_batch_pairs", "EvalStep"]
