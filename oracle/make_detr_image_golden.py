"""Writes ``tests/golden/detr_image.npz``: outputs of the UNMODIFIED reference DETR run from images (oracle/ref_detr_image.py).

TEST INFRASTRUCTURE ONLY.  Run in the build container (needs ``/root/reference``)::

    python -m oracle.make_detr_image_golden

Inputs: two N(0, 1) images of different sizes (3x96x160, 3x128x96), padded to one batch as nested_tensor_from_tensor_list
does, so that the mask is True at some feature positions.  Weights: not stored - ``weights.model`` / ``weights.seed`` name
the seeded oracle initialiser (oracle/detr_backbone_oracle.py, ResNet-50 + the 64-wide transformer), as the large fixtures
do (tests/util.py load_golden).  Contents:
  images.{0,1}, tq                 the inputs and the target query of each image
  mask, pos, src                   DETR.forward's mask, pos and input_proj(src) for the padded batch (detr.py:63-69)
  pred_logits, pred_boxes          DETR.forward on the padded batch
  single.{b}.src / .pos            input_proj(src) and pos of image b alone (the Generator runs one image at a time)
  R.{b}.n{0,1}s{0,1}               Generator.generate_ours(image b, tq[b], use_lrp=False) for the flag sets
  base.{b}.{raw_attn,rollout,attn_gradcam}   the reference Generator's baselines on image b
  ref.state_dict_keys              the reference module's state_dict() key set
"""
from __future__ import annotations

import os

import numpy as np
import torch

from . import detr_backbone_oracle as bo
from . import ref_detr_image as rdi

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
SEED = 3
FLAGS = ((1, 1), (0, 1), (1, 0))     # (normalize_self_attention, apply_self_in_rule_10)


def images(seed: int = 11):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(3, 96, 160, generator=g), torch.randn(3, 128, 96, generator=g)]


def main():
    cfg = bo.DETR_IMAGE
    sd = bo.init_state_dict(cfg, SEED)
    m = rdi.build(cfg, sd)
    imgs = images()
    tq = [1, 4]
    out = {"weights.model": np.array("detr_backbone_oracle.DETR_IMAGE"), "weights.seed": np.array(SEED),
           "tq": np.array(tq, dtype=np.int64), "ref.state_dict_keys": np.array(sorted(m.state_dict()))}
    for b, t in enumerate(imgs):
        out[f"images.{b}"] = t.numpy()
    mask, pos, src = rdi.front_end(m, imgs)
    out["mask"], out["pos"], out["src"] = mask.numpy(), pos.numpy(), src.numpy()
    o = rdi.forward(m, imgs)
    out["pred_logits"], out["pred_boxes"] = o["pred_logits"].numpy(), o["pred_boxes"].numpy()
    for b, t in enumerate(imgs):
        _, p1, s1 = rdi.front_end(m, [t])
        out[f"single.{b}.src"], out[f"single.{b}.pos"] = s1.numpy(), p1.numpy()
        for norm, s10 in FLAGS:
            out[f"R.{b}.n{norm}s{s10}"] = rdi.generator_maps(m, t, tq[b], normalize_self_attention=bool(norm),
                                                            apply_self_in_rule_10=bool(s10)).numpy()
        for method in ("raw_attn", "rollout", "attn_gradcam"):
            out[f"base.{b}.{method}"] = rdi.generator_maps(m, t, tq[b], method).numpy()
    np.savez_compressed(os.path.join(OUT, "detr_image.npz"), **out)
    print("wrote detr_image", {k: v.shape for k, v in out.items() if k.startswith(("src", "R.0"))})


if __name__ == "__main__":
    main()
