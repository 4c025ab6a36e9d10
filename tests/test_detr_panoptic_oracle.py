"""CPU: the DETR segmentation golden (oracle/make_detr_panoptic_golden.py, the unmodified reference get_panoptic /
PostProcess / PostProcessSegm) against itself and the plain-PyTorch restatement of the two post-processors
(oracle/detr_postprocess_oracle.py)."""
import numpy as np
import torch

from oracle import detr_postprocess_oracle as po
from util import load_golden

METHODS = ("ours_no_lrp", "raw_attn", "rollout")


def test_key_set(golden_dir):
    g = load_golden(golden_dir, "detr_panoptic.npz")
    per_image = {"size", "orig_size", "src", "pos", "pred_logits", "pred_boxes", "keep", "scores", "labels", "boxes"}
    want = {"weights.model", "weights.seed", "weights.class_scale", "images.seed", "syn.pred_masks", "syn.size",
            "syn.orig_size", "syn.masks.0", "syn.masks.1"}
    for b in (0, 1):
        want |= {f"{b}.{k}" for k in per_image}
        want |= {f"{b}.{m}.{k}" for m in METHODS for k in ("cams", "pred_masks", "masks")}
    assert {k for k in g.files if not k.startswith("sd.")} == want


def test_pred_masks_rows(golden_dir):
    """-1 exactly on the dropped queries, the {0, 255} Otsu mask on the kept ones (2 - 6 per image), one cam per kept query;
    the keep rule is softmax(pred_logits)[0, :, :-1].max(-1) > 0.5 with every score away from 0.5."""
    g = load_golden(golden_dir, "detr_panoptic.npz")
    for b in (0, 1):
        keep = g[f"{b}.keep"]
        p = torch.from_numpy(g[f"{b}.pred_logits"]).softmax(-1)[0, :, :-1].max(-1).values
        assert np.array_equal((p > 0.5).numpy(), keep) and 2 <= keep.sum() <= 6
        assert (p - 0.5).abs().min() > 1e-3
        for m in METHODS:
            pm = g[f"{b}.{m}.pred_masks"][0]
            assert pm.shape[0] == 100
            assert (pm[~keep] == -1).all()
            assert np.isin(pm[keep], (0.0, 255.0)).all()
            assert g[f"{b}.{m}.cams"].shape == (keep.sum(), pm.shape[1] * pm.shape[2])


def test_restatement_reproduces_postprocessors(golden_dir):
    g = load_golden(golden_dir, "detr_panoptic.npz")
    for b in (0, 1):
        size, orig = torch.from_numpy(g[f"{b}.size"])[None], torch.from_numpy(g[f"{b}.orig_size"])[None]
        scores, labels, boxes = po.postprocess(torch.from_numpy(g[f"{b}.pred_logits"]), torch.from_numpy(g[f"{b}.pred_boxes"]), orig)
        assert torch.equal(scores[0], torch.from_numpy(g[f"{b}.scores"]))
        assert torch.equal(labels[0], torch.from_numpy(g[f"{b}.labels"]))
        assert torch.equal(boxes[0], torch.from_numpy(g[f"{b}.boxes"]))
        for m in METHODS:
            masks = po.postprocess_segm(torch.from_numpy(g[f"{b}.{m}.pred_masks"]), size, orig)[0]
            assert masks.dtype == torch.uint8 and tuple(masks.shape) == (100, 1, *g[f"{b}.orig_size"])
            assert np.array_equal(masks.numpy(), g[f"{b}.{m}.masks"])
    syn = po.postprocess_segm(torch.from_numpy(g["syn.pred_masks"]), torch.from_numpy(g["syn.size"]),
                              torch.from_numpy(g["syn.orig_size"]))
    for i in (0, 1):
        assert np.array_equal(syn[i].numpy(), g[f"syn.masks.{i}"])
