"""Runs the UNMODIFIED reference segmentation driver step - ``MaskGenerator.get_panoptic`` (DETR/mask_generator.py:45-155),
``PostProcess`` (DETR/models/detr.py:278-306) and ``PostProcessSegm`` (DETR/models/segmentation.py:218-242) - on CPU
(build container only; TEST INFRASTRUCTURE).  The model is oracle/ref_detr_image.py's ``build`` with its shims.

``get_panoptic`` hard-codes 100 queries (mask_generator.py:89), so the configuration here is the golden-size DETR with
DETR-R50's 100 queries.  A random-init class head keeps almost no query (softmax max > 0.5 over 6 columns), so the
golden scales ``class_embed`` by a stored factor (``scaled``)."""
from __future__ import annotations

from typing import Dict

import torch

from mmx_b200.synthetic import DetrConfig
from . import detr_backbone_oracle as bo
from . import ref_detr_image as rdi
from . import ref_shims as rs

DETR_PANOPTIC = DetrConfig(64, 2, 2, 6, 96, 100, 5)
METHODS = ("ours_no_lrp", "raw_attn", "rollout")


def init_state_dict(cfg: DetrConfig, seed: int = 0) -> Dict[str, torch.Tensor]:
    """The seeded whole-DETR state dict of oracle/detr_backbone_oracle.py (the name load_golden regenerates it by)."""
    return bo.init_state_dict(cfg, seed)


def scaled(sd: Dict[str, torch.Tensor], class_scale: float) -> Dict[str, torch.Tensor]:
    """``sd`` with class_embed's weight and bias multiplied by ``class_scale``."""
    out = dict(sd)
    out["class_embed.weight"] = sd["class_embed.weight"] * class_scale
    out["class_embed.bias"] = sd["class_embed.bias"] * class_scale
    return out


def nested(image: torch.Tensor):
    """The one-image NestedTensor the reference's data loader hands to get_panoptic (DETR/util/misc.py:306-327)."""
    *_, nested_tensor_from_tensor_list = rdi._import()
    return nested_tensor_from_tensor_list([image])


def get_panoptic(m, image: torch.Tensor, method: str):
    """``MaskGenerator(m).get_panoptic(samples, targets, method)`` on one [3,H,W] image (targets is unused there)."""
    rs._ensure_path()
    from DETR.mask_generator import MaskGenerator
    with rs.cuda_is_identity():
        out = MaskGenerator(m).get_panoptic(nested(image), None, method)
    return {k: v.detach() for k, v in out.items()}


def cams(m, image: torch.Tensor, queries, method: str) -> torch.Tensor:
    """The relevance maps [K, h*w] the reference Generator gives get_panoptic's loop for the kept ``queries`` (:90-110)."""
    rs._ensure_path()
    from DETR.modules.ExplanationGenerator import Generator
    gen = Generator(m)
    rows = []
    with rs.cuda_is_identity():
        for q in queries:
            idx = torch.tensor([int(q)])
            if method == "ours_no_lrp":
                r = gen.generate_ours(nested(image), idx, use_lrp=False)
            else:
                r = getattr(gen, "generate_" + method)(nested(image), idx)
            rows.append(r.reshape(-1).detach())
    return torch.stack(rows) if rows else torch.zeros(0)


def postprocess(outputs, orig_target_sizes, target_sizes, threshold: float = 0.5):
    """``PostProcess()(outputs, orig_target_sizes)`` then ``PostProcessSegm(threshold)(results, outputs, orig_target_sizes,
    target_sizes)``, as DETR/engine.py:188-192 runs them."""
    rs._ensure_path()
    rdi._import()
    from DETR.models.detr import PostProcess
    from DETR.models.segmentation import PostProcessSegm
    results = PostProcess()(outputs, orig_target_sizes)
    return PostProcessSegm(threshold)(results, outputs, orig_target_sizes, target_sizes)
