"""Writes ``tests/golden/detr_dc5.npz``: outputs of the UNMODIFIED reference DETR built with the DC5 (dilated layer4)
backbone, run from images (oracle/detr_dc5_oracle.py ``build_reference``).

TEST INFRASTRUCTURE ONLY.  Run in the build container (needs ``/root/reference``)::

    python -m oracle.make_detr_dc5_golden

Weights: the seeded ``DETR_IMAGE`` state dict of ``detr_image.npz`` (dilation changes no shape), stored by name and seed
(tests/util.py load_golden).  Images: stored by seed as well (``detr_dc5_oracle.pair_images`` / ``long_image``).
Contents:
  tq, long.tq                      the target query of each image of the pair, of the long image
  mask, pos, src                   DETR.forward's mask, pos and input_proj(src) for the padded pair (detr.py:63-69)
  pred_logits, pred_boxes          DETR.forward on the padded pair
  R.{b}.n{0,1}s{0,1}               Generator.generate_ours(image b, tq[b], use_lrp=False) for the flag sets
  base.{b}.{raw_attn,rollout,attn_gradcam}   the reference Generator's baselines on image b
  long.R.n{0,1}s{0,1}              generate_ours on the 3x520x540 image: 33x34 = 1122 tokens, past the single-pass kernels
  ref.state_dict_keys              the DC5 module's state_dict() key set
"""
from __future__ import annotations

import os

import numpy as np
import torch

from . import detr_backbone_oracle as bo
from . import detr_dc5_oracle as dc5
from . import ref_detr_image as rdi
from .make_detr_image_golden import FLAGS, SEED

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def main():
    cfg = bo.DETR_IMAGE
    sd = bo.init_state_dict(cfg, SEED)
    m = dc5.build_reference(cfg, sd)
    imgs = dc5.pair_images()
    big = dc5.long_image()
    tq, long_tq = [1, 4], 2
    out = {"weights.model": np.array("detr_backbone_oracle.DETR_IMAGE"), "weights.seed": np.array(SEED),
           "images.seed": np.array(dc5.PAIR_SEED), "long.seed": np.array(dc5.LONG_SEED),
           "tq": np.array(tq, dtype=np.int64), "long.tq": np.array(long_tq, dtype=np.int64),
           "ref.state_dict_keys": np.array(sorted(m.state_dict()))}
    mask, pos, src = rdi.front_end(m, imgs)
    out["mask"], out["pos"], out["src"] = mask.numpy(), pos.numpy(), src.numpy()
    o = rdi.forward(m, imgs)
    out["pred_logits"], out["pred_boxes"] = o["pred_logits"].numpy(), o["pred_boxes"].numpy()
    for b, t in enumerate(imgs):
        for norm, s10 in FLAGS:
            out[f"R.{b}.n{norm}s{s10}"] = rdi.generator_maps(m, t, tq[b], normalize_self_attention=bool(norm),
                                                            apply_self_in_rule_10=bool(s10)).numpy()
        for method in ("raw_attn", "rollout", "attn_gradcam"):
            out[f"base.{b}.{method}"] = rdi.generator_maps(m, t, tq[b], method).numpy()
    for norm, s10 in FLAGS:
        out[f"long.R.n{norm}s{s10}"] = rdi.generator_maps(m, big, long_tq, normalize_self_attention=bool(norm),
                                                         apply_self_in_rule_10=bool(s10)).numpy()
    np.savez_compressed(os.path.join(OUT, "detr_dc5.npz"), **out)
    print("wrote detr_dc5", {k: v.shape for k, v in out.items() if k.startswith(("src", "R.0", "long.R"))})


if __name__ == "__main__":
    main()
