"""Golden fixture FROM THE REAL REFERENCE for SURVEY.md 8f row 4: MobileViTv2 as a segmentation backbone.

``get_model(opts, category="classification", output_stride=8)`` is how the reference's segmentation models build their encoder
(cvnets/models/segmentation/enc_dec.py:120-129): layer_4 / layer_5 keep the 1/8 resolution and their depthwise convs dilate by 2 / 4
(base_image_encoder.py:38-47, mobilevit_v2.py:176-191).  Saved: out_l3 / out_l4 / out_l5 of ``extract_end_points_all`` in train mode
(width 0.5, batch 4 at 128x128), and the gradients of sum(gy4 * out_l4) + sum(gy5 * out_l5) for every parameter tensor <= 5k elements.
The same for output_stride=16 (forward end points only).

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_dilated.py
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from golden_sample import sample_large  # noqa: E402
from make_golden import O, get_model, load_seeded, make_opts, torch  # noqa: E402


def main():
    torch.manual_seed(0)
    width, res, B, seed = 0.5, 128, 4, 81
    fx = dict(width=width, res=res, batch=B, seed=seed, x_seed=381)
    for os_ in (8, 16):
        model = get_model(make_opts(width), category="classification", output_stride=os_)
        P = O.mobilevit_v2_shapes(width)
        load_seeded(model, P, seed)
        model.train()
        x = O.seeded_input((B, 3, res, res), 381)
        ends = model.extract_end_points_all(x, use_l5=True, use_l5_exp=False)
        rec = {"ends": {k: sample_large(v.detach().clone()) for k, v in ends.items() if k in ("out_l3", "out_l4", "out_l5")},
               "dilations": {n: list(m.dilation) for n, m in model.named_modules() if isinstance(m, torch.nn.Conv2d) and m.dilation != (1, 1)}}
        if os_ == 8:
            gy4, gy5 = O.seeded_input(tuple(ends["out_l4"].shape), 481), O.seeded_input(tuple(ends["out_l5"].shape), 482)
            ((ends["out_l4"] * gy4).sum() + (ends["out_l5"] * gy5).sum()).backward()
            grads = {k: p.grad for k, p in model.named_parameters() if p.grad is not None}
            rec.update(gy_seeds=(481, 482), grad_norms={k: float(g.norm()) for k, g in grads.items()},
                       grads={k: sample_large(g.clone()) for k, g in grads.items() if g.numel() <= 5000})
        fx[f"os{os_}"] = rec
        print(os_, {k: tuple(v.shape) for k, v in ends.items()}, rec["dilations"])
    torch.save(fx, os.path.join(HERE, "mobilevit_v2_dilated_fp32.pt"))
    print(os.path.getsize(os.path.join(HERE, "mobilevit_v2_dilated_fp32.pt")), "bytes")


if __name__ == "__main__":
    main()
