"""Runs the UNMODIFIED reference ``SetCriterion`` / ``HungarianMatcher`` (DETR/models/detr.py:103-275,
DETR/models/matcher.py, DETR/models/segmentation.py:172-215) and ``MaskGenerator.get_panoptic`` with ``aux_outputs``
on CPU (build container only; TEST INFRASTRUCTURE), with the shims of oracle/ref_detr_image.py.  Setting ``aux_loss`` on
the built module makes ``DETR.forward`` return ``aux_outputs`` (detr.py:74-75), as DETR's default ``--aux_loss`` does."""
from __future__ import annotations

import torch

from . import ref_detr_image as rdi
from . import ref_detr_panoptic as rp
from . import ref_shims as rs

LOSSES = ["labels", "boxes", "cardinality", "masks"]


def weight_dict(dec_layers: int, masks: bool = True):
    """build()'s weight_dict (DETR/models/detr.py:344-355) for DETR's default coefficients, aux entries included"""
    wd = {"loss_ce": 1, "loss_bbox": 5, "loss_giou": 2}
    if masks:
        wd["loss_mask"], wd["loss_dice"] = 1, 1
    aux = {}
    for i in range(dec_layers - 1):
        aux.update({k + f"_{i}": v for k, v in wd.items()})
    wd.update(aux)
    return wd


def build(cfg, sd):
    m = rdi.build(cfg, sd)
    m.aux_loss = True
    return m


def _detach(o):
    if isinstance(o, dict):
        return {k: _detach(v) for k, v in o.items()}
    if isinstance(o, list):
        return [_detach(v) for v in o]
    return o.detach()


def get_panoptic(m, image: torch.Tensor, method: str):
    """``MaskGenerator(m).get_panoptic`` on one [3,H,W] image, aux_outputs included"""
    rs._ensure_path()
    from DETR.mask_generator import MaskGenerator
    with rs.cuda_is_identity():
        out = MaskGenerator(m).get_panoptic(rp.nested(image), None, method)
    return _detach(out)


def forward(m, images):
    """DETR.forward on a list of images (padded as nested_tensor_from_tensor_list pads), aux_outputs included"""
    with rs.cuda_is_identity():
        return _detach(m(images))


def criterion(num_classes: int, eos_coef: float, losses, dec_layers: int, cost=(1, 1, 1)):
    rdi._import()
    from DETR.models.detr import SetCriterion
    from DETR.models.matcher import HungarianMatcher
    matcher = HungarianMatcher(cost_class=cost[0], cost_bbox=cost[1], cost_giou=cost[2])
    return SetCriterion(num_classes, matcher, weight_dict(dec_layers, "masks" in losses), eos_coef, losses).eval()


def run(crit, outputs, targets):
    """(loss dict, [indices of layer 0 = the final output, then of each aux layer]) of the reference criterion"""
    losses = crit(outputs, targets)
    layers = [{k: v for k, v in outputs.items() if k != "aux_outputs"}] + list(outputs.get("aux_outputs", []))
    return {k: v.detach() for k, v in losses.items()}, [crit.matcher(o, targets) for o in layers]
