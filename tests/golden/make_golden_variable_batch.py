"""Golden fixture FROM THE REAL REFERENCE for engine.variable_batch_pairs: the (h, w, batch) table of every ``sampler.vbs`` block in the
recipes this library trains, as the reference's variable-batch sampler builds it (data/sampler/utils.py:image_batch_pairs, called by
VariableBatchSampler / VariableBatchSamplerDDP with the recipe's crop sizes, train_batch_size0, max_n_scales and check_scale).

data/sampler/utils.py is loaded on its own: importing the ``data`` package pulls in video decoding (``av``), which the table does not need.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_variable_batch.py
"""
import importlib.util
import json
import os
import sys

import yaml

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference"
RECIPES = (
    "examples/range_augment/classification/efficientnet_b0.yaml",
    "examples/range_augment/classification/efficientnet_b1.yaml",
    "examples/range_augment/classification/efficientnet_b2.yaml",
    "examples/range_augment/classification/efficientnet_b3.yaml",
    "examples/vit/classification/vit_base.yaml",
    "config/classification/imagenet/vit.yaml",
    "examples/range_augment/clip/clip_vit_base.yaml",
    "examples/range_augment/clip/clip_vit_huge.yaml",
    "examples/range_augment/clip_finetune_imagenet/clip_vit_base.yaml",
    "examples/range_augment/clip_finetune_imagenet/clip_vit_huge.yaml",
    "config/multi_modal_img_text/clip_vit.yaml",
)


def load_sampler_utils():
    sys.path.insert(0, REF)  # for utils.math_utils
    spec = importlib.util.spec_from_file_location("ref_sampler_utils", os.path.join(REF, "data/sampler/utils.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    U = load_sampler_utils()
    out = []
    for path in RECIPES:
        with open(os.path.join(REF, path)) as f:
            cfg = yaml.safe_load(f)
        assert cfg["sampler"]["name"] == "variable_batch_sampler", path
        v = cfg["sampler"]["vbs"]
        args = dict(crop_w=v["crop_size_width"], crop_h=v["crop_size_height"], batch=int(cfg["dataset"]["train_batch_size0"]),
                    max_scales=v["max_n_scales"], check_scale=v["check_scale"], min_w=v["min_crop_size_width"], max_w=v["max_crop_size_width"],
                    min_h=v["min_crop_size_height"], max_h=v["max_crop_size_height"])
        pairs = U.image_batch_pairs(crop_size_w=args["crop_w"], crop_size_h=args["crop_h"], batch_size_gpu0=args["batch"],
                                    max_scales=args["max_scales"], check_scale_div_factor=args["check_scale"], min_crop_size_w=args["min_w"],
                                    max_crop_size_w=args["max_w"], min_crop_size_h=args["min_h"], max_crop_size_h=args["max_h"])
        out.append({"recipe": path, "args": args, "pairs": [[int(h), int(w), int(b)] for h, w, b in pairs]})
        print(path, [tuple(p) for p in out[-1]["pairs"]])
    with open(os.path.join(HERE, "variable_batch_pairs.json"), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
