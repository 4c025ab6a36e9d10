"""Writes ``tests/golden/detr_panoptic.npz``: the UNMODIFIED reference segmentation driver step (oracle/ref_detr_panoptic.py)
- ``MaskGenerator.get_panoptic``, ``PostProcess`` and ``PostProcessSegm`` - on two images run alone.

TEST INFRASTRUCTURE ONLY.  Run in the build container (needs ``/root/reference``)::

    python -m oracle.make_detr_panoptic_golden

Weights: not stored - ``weights.model`` / ``weights.seed`` name the seeded initialiser (tests/util.py load_golden), and
``weights.class_scale`` the factor class_embed (weight and bias) is multiplied by so that each image keeps 2 - 6 queries.
The factor is chosen so that no query's score lies within 1e-3 of the 0.5 keep threshold.  Images: stored by seed.
Contents, for image b (run alone, ``size`` = its own size, ``orig_size`` != size):
  {b}.size, {b}.orig_size                  target["size"], target["orig_size"] (int64 [2])
  {b}.src, {b}.pos                         input_proj(src) and pos of the image (detr.py:63-69)
  {b}.pred_logits, {b}.pred_boxes, {b}.keep   get_panoptic's forward and keep rule (the same for every method)
  {b}.scores, {b}.labels, {b}.boxes        PostProcess (independent of the method)
  {b}.{method}.cams                        the reference Generator's maps of the kept queries [K, h*w]
  {b}.{method}.pred_masks                  get_panoptic's pred_masks [1, 100, h, w]
  {b}.{method}.masks                       PostProcessSegm's uint8 masks [100, 1, oh, ow]
and a synthetic two-image PostProcessSegm batch (N(0, 3) logits with exact zeros, power-of-two bilinear ratios so that
torch's CPU and CUDA arithmetic agree): syn.pred_masks [2, 5, 6, 8], syn.size, syn.orig_size, syn.masks.{0,1}.
"""
from __future__ import annotations

import os

import numpy as np
import torch

from . import ref_detr_image as rdi
from . import ref_detr_panoptic as rp

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
SEED = 57
IMAGES_SEED = 21
SYN_SEED = 5
SIZES = ((256, 320), (224, 288))
ORIG_SIZES = ((300, 383), (150, 201))       # one larger, one smaller than the input
MARGIN = 1e-3


def images(seed: int = IMAGES_SEED):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(3, h, w, generator=g) for h, w in SIZES]


def synthetic(seed: int = SYN_SEED):
    g = torch.Generator().manual_seed(seed)
    x = 3.0 * torch.randn(2, 5, 6, 8, generator=g)
    x[torch.rand(x.shape, generator=g) < 0.15] = 0.0
    return x, torch.tensor([[24, 32], [20, 28]]), torch.tensor([[37, 45], [12, 50]])


def pick_scale(m, imgs):
    """The smallest class_scale on a 0.01 grid for which every image keeps 2 - 6 queries and no score is within MARGIN of
    0.5.  Scaling class_embed's weight and bias scales the logits exactly as much, so one forward per image suffices."""
    logits = [rdi.forward(m, [t])["pred_logits"][0].double() for t in imgs]
    for s in np.arange(1.0, 30.0, 0.01):
        ok = True
        for lg in logits:
            p = (s * lg).softmax(-1)[:, :-1].max(-1).values
            k = int((p > 0.5).sum())
            ok &= 2 <= k <= 6 and bool(((p - 0.5).abs() > MARGIN).all())
        if ok:
            return float(s)
    raise RuntimeError("no class_scale keeps 2 - 6 queries per image")


def main():
    cfg = rp.DETR_PANOPTIC
    sd = rp.init_state_dict(cfg, SEED)
    imgs = images()
    scale = float(np.float32(pick_scale(rdi.build(cfg, sd), imgs)))      # the value stored, as the tests apply it
    m = rdi.build(cfg, rp.scaled(sd, scale))
    out = {"weights.model": np.array("ref_detr_panoptic.DETR_PANOPTIC"), "weights.seed": np.array(SEED),
           "weights.class_scale": np.array(scale, dtype=np.float32), "images.seed": np.array(IMAGES_SEED)}
    for b, t in enumerate(imgs):
        size, orig = torch.tensor([list(SIZES[b])]), torch.tensor([list(ORIG_SIZES[b])])
        out[f"{b}.size"], out[f"{b}.orig_size"] = size[0].numpy(), orig[0].numpy()
        _, pos, src = rdi.front_end(m, [t])
        out[f"{b}.src"], out[f"{b}.pos"] = src.numpy(), pos.numpy()
        for method in rp.METHODS:
            o = rp.get_panoptic(m, t, method)
            keep = o["pred_logits"].softmax(-1)[0, :, :-1].max(-1).values > 0.5     # mask_generator.py:50-51
            p = o["pred_logits"].softmax(-1)[0, :, :-1].max(-1).values
            assert (p - 0.5).abs().min() > MARGIN and 2 <= int(keep.sum()) <= 6, (b, method)
            res = rp.postprocess(o, orig, size)
            out[f"{b}.pred_logits"], out[f"{b}.pred_boxes"] = o["pred_logits"].numpy(), o["pred_boxes"].numpy()
            out[f"{b}.keep"] = keep.numpy()
            out[f"{b}.scores"], out[f"{b}.labels"] = res[0]["scores"].numpy(), res[0]["labels"].numpy()
            out[f"{b}.boxes"] = res[0]["boxes"].numpy()
            out[f"{b}.{method}.cams"] = rp.cams(m, t, keep.nonzero().flatten().tolist(), method).numpy()
            out[f"{b}.{method}.pred_masks"] = o["pred_masks"].numpy()
            out[f"{b}.{method}.masks"] = res[0]["masks"].numpy()
    x, size, orig = synthetic()
    res = rp.postprocess({"pred_logits": torch.zeros(2, 5, 6), "pred_boxes": torch.zeros(2, 5, 4), "pred_masks": x}, orig, size)
    out["syn.pred_masks"], out["syn.size"], out["syn.orig_size"] = x.numpy(), size.numpy(), orig.numpy()
    for i in range(2):
        out[f"syn.masks.{i}"] = res[i]["masks"].numpy()
    np.savez_compressed(os.path.join(OUT, "detr_panoptic.npz"), **out)
    print("wrote detr_panoptic: class_scale", scale, {k: int(v.sum()) for k, v in out.items() if k.endswith(".keep")})


if __name__ == "__main__":
    main()
