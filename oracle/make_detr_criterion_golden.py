"""Writes ``tests/golden/detr_criterion.npz``: the UNMODIFIED reference criterion (oracle/ref_detr_criterion.py) -
HungarianMatcher + SetCriterion with aux_outputs and masks - and scipy's linear_sum_assignment on tied and edge-case
matrices.

TEST INFRASTRUCTURE ONLY.  Run in the build container (needs ``/root/reference``)::

    python -m oracle.make_detr_criterion_golden

Weights: not stored - ``weights.model`` / ``weights.seed`` / ``weights.class_scale`` as in detr_panoptic.npz
(DETR_PANOPTIC, 6 decoder layers); images by seed.  Contents:
  {b}.pred_logits, {b}.pred_boxes, {b}.pred_masks, {b}.aux.{i}.pred_logits / pred_boxes
                                 the reference get_panoptic (method raw_attn) of image b, aux_outputs included
  {b}.labels, {b}.boxes, {b}.masks      seeded targets of image b (int64, cxcywh fp32, uint8 at the image size)
  batch.pred_logits / pred_boxes / aux.{i}.* / pred_masks   DETR.forward on the two images as one padded batch, with
                                 seeded get_panoptic-like pred_masks (-1 rows, {0, 255} planes)
  {run}.loss.{key} (fp32 0-d) and {run}.keys (the dict's key order), {run}.idx.{layer}.{b}.i / .j (layer 0 = the final
  output) for run in {0, 1, batch}; eos_coef, num_classes, weight_dict (JSON)
  empty.error                    what the reference raises for an image whose target list is empty (with masks)
  empty.loss.{key}               its losses without masks
  lsa.{name}.cost and .i / .j or .error   scipy on tied / edge-case / random matrices
Every stored image-level assignment survives 20 seeded perturbations of 1e-4 max|C| (PERTURB), so that the 1e-5
differences allowed between the device forward and the reference cannot flip a match.
"""
from __future__ import annotations

import json
import os

import numpy as np
import torch
from scipy.optimize import linear_sum_assignment

from . import detr_criterion_oracle as co
from . import make_detr_panoptic_golden as mp
from . import ref_detr_criterion as rc
from . import ref_detr_panoptic as rp

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
TARGET_SEED = 3
MASK_SEED = 9
LSA_SEED = 11
EOS = 0.1
COUNTS = (3, 5)
PERTURB = 1e-4
RANDOM_T = (0, 1, 7, 20, 63, 100, 120)


def targets(sizes, counts, classes, seed):
    g = torch.Generator().manual_seed(seed)
    out = []
    for (H, W), n in zip(sizes, counts):
        c = 0.2 + 0.6 * torch.rand(n, 2, generator=g)
        wh = 0.05 + 0.35 * torch.rand(n, 2, generator=g)
        out.append({"labels": torch.randint(0, classes, (n,), generator=g), "boxes": torch.cat([c, wh], 1),
                    "masks": (torch.rand(n, H, W, generator=g) < 0.3).to(torch.uint8)})
    return out


def stable(outputs, tgts) -> bool:
    """every layer's image-level assignment is unchanged under PERTURB-sized seeded perturbations of its cost"""
    g = np.random.default_rng(0)
    for o in [outputs] + list(outputs.get("aux_outputs", [])):
        for c in co.cost_blocks({k: v.double() for k, v in o.items() if k != "aux_outputs"},
                                [{k: v.double() if v.is_floating_point() else v for k, v in t.items()} for t in tgts]):
            c = c.numpy()
            if c.size == 0:
                continue
            base = linear_sum_assignment(c)
            for _ in range(20):
                p = linear_sum_assignment(c + PERTURB * np.abs(c).max() * g.uniform(-1, 1, c.shape))
                if not (np.array_equal(base[0], p[0]) and np.array_equal(base[1], p[1])):
                    return False
    return True


def lsa_cases(seed=LSA_SEED):
    g = np.random.default_rng(seed)
    cases = {"int_3x3": g.integers(0, 3, (3, 3)).astype(float), "ones_4x4": np.ones((4, 4)),
             "one": np.array([[2.5]]), "wide_3x6": g.integers(0, 2, (3, 6)).astype(float),
             "tall_6x3": g.integers(0, 2, (6, 3)).astype(float), "empty_100x0": np.zeros((100, 0)),
             "nan": np.array([[1.0, np.nan], [0.0, 1.0]]), "neg_inf": np.array([[1.0, -np.inf], [0.0, 1.0]]),
             "infeasible": np.array([[np.inf, np.inf], [1.0, np.inf]]), "pos_inf_ok": np.array([[np.inf, 1.0], [2.0, np.inf]])}
    d = g.integers(0, 4, (5, 7)).astype(float)
    d[3] = d[1]
    d[:, 6] = d[:, 2]
    cases["dup_rows_cols_5x7"] = d
    cases["dup_rows_cols_7x5"] = d.T.copy()
    for k in range(20):                       # small-integer ties at the matcher's shape
        r, c = 100, int(g.integers(1, 30))
        cases[f"tie_100x{c}_{k}"] = g.integers(0, 3, (r, c)).astype(float)
    for T in RANDOM_T:
        cases[f"rand_100x{T}"] = g.standard_normal((100, T)).astype(np.float32).astype(float)
    return cases


def main():
    cfg = rp.DETR_PANOPTIC
    sd = rp.init_state_dict(cfg, mp.SEED)
    imgs = mp.images()
    g0 = np.load(os.path.join(OUT, "detr_panoptic.npz"))
    scale = float(g0["weights.class_scale"])
    m = rc.build(cfg, rp.scaled(sd, scale))
    out = {"weights.model": np.array("ref_detr_panoptic.DETR_PANOPTIC"), "weights.seed": np.array(mp.SEED),
           "weights.class_scale": np.array(scale, dtype=np.float32), "images.seed": np.array(mp.IMAGES_SEED),
           "eos_coef": np.array(EOS), "num_classes": np.array(cfg.classes)}
    crit = rc.criterion(cfg.classes, EOS, rc.LOSSES, cfg.dec_layers)
    out["weight_dict"] = np.array(json.dumps(crit.weight_dict))
    outs = [rc.get_panoptic(m, t, "raw_attn") for t in imgs]
    assert all(list(o) == ["pred_logits", "pred_boxes", "aux_outputs", "pred_masks"] for o in outs)
    batch = rc.forward(m, imgs)
    gm = torch.Generator().manual_seed(MASK_SEED)
    fh, fw = outs[0]["pred_masks"].shape[-2:]
    pm = torch.where(torch.rand(2, cfg.queries, fh, fw, generator=gm) < 0.4, 255.0, 0.0)
    pm[torch.rand(2, cfg.queries, generator=gm) < 0.8] = -1.0
    batch["pred_masks"] = pm
    seed = TARGET_SEED
    while True:
        tg = targets(mp.SIZES, COUNTS, cfg.classes, seed)
        if all(stable(o, [t]) for o, t in zip(outs, tg)) and stable(batch, tg):
            break
        seed += 1
    out["targets.seed"] = np.array(seed)

    def put(prefix, o):
        for k in ("pred_logits", "pred_boxes", "pred_masks"):
            out[f"{prefix}.{k}"] = o[k].numpy()
        for i, a in enumerate(o["aux_outputs"]):
            out[f"{prefix}.aux.{i}.pred_logits"], out[f"{prefix}.aux.{i}.pred_boxes"] = a["pred_logits"].numpy(), a["pred_boxes"].numpy()

    for b, (o, t) in enumerate(zip(outs, tg)):
        put(str(b), o)
        for k in ("labels", "boxes", "masks"):
            out[f"{b}.{k}"] = t[k].numpy()
    put("batch", batch)
    for run, o, t in (("0", outs[0], tg[:1]), ("1", outs[1], tg[1:]), ("batch", batch, tg)):
        losses, idx = rc.run(crit, o, t)
        out[f"{run}.keys"] = np.array(list(losses))
        for k, v in losses.items():
            out[f"{run}.loss.{k}"] = v.numpy()
        for l, ind in enumerate(idx):
            for b, (i, j) in enumerate(ind):
                out[f"{run}.idx.{l}.{b}.i"], out[f"{run}.idx.{l}.{b}.j"] = i.numpy(), j.numpy()
    empty = [{k: v[:0] for k, v in tg[0].items()}]
    losses, _ = rc.run(rc.criterion(cfg.classes, EOS, rc.LOSSES[:3], cfg.dec_layers), outs[0], empty)
    for k, v in losses.items():
        out[f"empty.loss.{k}"] = v.numpy()
    try:
        rc.run(crit, outs[0], empty)
        out["empty.error"] = np.array("")
    except Exception as e:                                  # noqa: BLE001 - recorded, whatever it is
        out["empty.error"] = np.array(type(e).__name__)
    for name, c in lsa_cases().items():
        out[f"lsa.{name}.cost"] = c
        try:
            i, j = linear_sum_assignment(c)
            out[f"lsa.{name}.i"], out[f"lsa.{name}.j"] = i.astype(np.int64), j.astype(np.int64)
        except ValueError as e:
            out[f"lsa.{name}.error"] = np.array(str(e))
    np.savez_compressed(os.path.join(OUT, "detr_criterion.npz"), **out)
    print("wrote detr_criterion: targets seed", seed, "empty:", out["empty.error"],
          {k[:-5]: float(v) for k, v in out.items() if k.startswith("batch.loss.") and "_" not in k[11:]})


if __name__ == "__main__":
    main()
