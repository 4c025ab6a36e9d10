"""The notebooks' visualisation step on the device, under the notebooks' names.  Each function returns device tensors
(the picture, or the printed scores) where the reference plots or writes a file; the arithmetic runs in
``csrc/visualize.cu`` (``mmx_relevance_overlay``, ``mmx_box_relevance_image``, ``mmx_clip_text_scores``).

  * ``show_image_relevance``   - CLIP_explainability.ipynb:216 (``vis`` as handed to ``axs[1].imshow``)
  * ``generate_visualization`` - Transformer_MM_explainability_ViT.ipynb:1223,1234
  * ``save_image_vis``         - LXMERT.ipynb:121, Transformer_MM_Explainability.ipynb:2571 (the 8-bit image
                                 ``cv2.imwrite`` encodes)
  * ``show_heatmap_on_text``   - CLIP_explainability.ipynb:254 (the ``text_scores`` it prints)

Batches: every function also takes a leading batch dimension and does the whole batch in one launch.
"""
from __future__ import annotations

from typing import List

import numpy as np
import torch

from ._lib import lib, check, ptr, current_stream, MmxError

VIS_SIZE = 224      # show_image_relevance's F.interpolate(size=224)


def _cuda(t, name):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise MmxError(f"{name} must be a CUDA tensor")
    return t


def _same_device(*ts):
    if len({t.device for t in ts}) != 1:
        raise MmxError("all inputs must be on the same CUDA device")


def _scale(in_size: int, out_size: int, scale_factor=None) -> float:
    """ATen's source scale of an align_corners=False resize: 1 / scale_factor when one is given, else (float)in / out."""
    if scale_factor is not None:
        return float(np.float32(1.0 / scale_factor))
    return float(np.float32(in_size) / np.float32(out_size))


def _overlay(rel: torch.Tensor, images: torch.Tensor, dim: int, size: int, scale_factor=None) -> torch.Tensor:
    """rel [B, dim*dim], images [1|B, 3, size, size] -> [B, size, size, 3] uint8."""
    _same_device(rel, images)
    B = rel.shape[0]
    if images.dim() != 4 or images.shape[1] != 3 or images.shape[0] not in (1, B):
        raise MmxError(f"image must be [1 or {B}, 3, H, W] (got {tuple(images.shape)})")
    if tuple(images.shape[2:]) != (size, size):
        raise MmxError(f"the upsampled map is {size}x{size} but the image is {tuple(images.shape[2:])}: the reference "
                       "cannot add them")
    if not rel.is_floating_point() or not images.is_floating_point():
        raise MmxError("relevance and image must be floating-point tensors")
    s = _scale(dim, size, scale_factor)
    with torch.cuda.device(rel.device):
        rel = rel.to(torch.float32).contiguous()
        images = images.to(torch.float32).contiguous()
        out = torch.empty(B, size, size, 3, dtype=torch.uint8, device=rel.device)
        check(lib().mmx_relevance_overlay(ptr(rel), B, dim, dim, s, s, ptr(images), images.shape[0], size, size, ptr(out),
                                          current_stream()))
    return out


def _square_side(P: int) -> int:
    dim = int(P ** 0.5)
    if dim < 1 or dim * dim != P:
        raise MmxError(f"the relevance map must hold a square number of patches (got {P})")
    return dim


def show_image_relevance(image_relevance: torch.Tensor, image: torch.Tensor, orig_image=None) -> torch.Tensor:
    """Drop-in for the notebook's ``show_image_relevance``: returns ``vis`` (uint8 [224, 224, 3], the array the reference
    shows next to ``orig_image``) instead of plotting it; ``orig_image`` is accepted and unused.

    ``image_relevance`` [P] or [B, P] with P a perfect square (a ``R_image`` row of ``interpret``); ``image`` [1 or B, 3,
    224, 224], the preprocessed input - with one image every map uses it, as the reference's ``image[0]`` does.  Returns
    [224, 224, 3] or [B, 224, 224, 3]."""
    _cuda(image_relevance, "image_relevance")
    _cuda(image, "image")
    if image_relevance.dim() not in (1, 2) or image_relevance.shape[-1] < 1 or image_relevance.numel() == 0:
        raise MmxError(f"image_relevance must be [P] or [B, P] (got {tuple(image_relevance.shape)})")
    single = image_relevance.dim() == 1
    rel = image_relevance.reshape(-1, image_relevance.shape[-1])
    dim = _square_side(rel.shape[1])
    out = _overlay(rel, image, dim, VIS_SIZE)
    return out[0] if single else out


def generate_visualization(model, original_image: torch.Tensor, class_index=None) -> torch.Tensor:
    """Drop-in for the ViT notebook's ``generate_visualization``; the notebook reads a global ``model``, here it is the
    first argument (a ``ViTEngine``).  ``original_image`` [3, H, W] or [B, 3, H, W]; ``class_index`` None (the top class)
    or one index per sample.  Runs ``generate_relevance``, then the overlay with ``F.interpolate(scale_factor=patch)``
    (16 for ViT-B/16, as in the notebook).  Returns uint8 [H, W, 3] or [B, H, W, 3]."""
    from .vit import ViTEngine, generate_relevance
    if not isinstance(model, ViTEngine):
        raise MmxError("model must be a mmx_b200.ViTEngine")
    _cuda(original_image, "original_image")
    if original_image.dim() not in (3, 4):
        raise MmxError(f"original_image must be [3, H, W] or [B, 3, H, W] (got {tuple(original_image.shape)})")
    single = original_image.dim() == 3
    x = original_image.unsqueeze(0) if single else original_image
    if tuple(x.shape[1:]) != (3, model.image, model.image):
        raise MmxError(f"original_image must be [B, 3, {model.image}, {model.image}] (got {tuple(x.shape)})")
    rel = generate_relevance(model, x, index=class_index).reshape(x.shape[0], -1)
    size = int(np.floor(model.grid * float(model.patch)))      # ATen's output size for a scale factor
    out = _overlay(rel, x, model.grid, size, scale_factor=model.patch)
    return out[0] if single else out


def save_image_vis(image: torch.Tensor, boxes: torch.Tensor, bbox_scores: torch.Tensor) -> torch.Tensor:
    """Drop-in for the LXMERT notebook's ``save_image_vis``: returns the uint8 image instead of writing ``new.jpg``
    (``cv2.imwrite`` of the returned array writes the same file: imwrite converts to 8 bits before it encodes).

    ``image`` [H, W, 3] or [1 or B, H, W, 3] uint8 BGR (as ``cv2.imread`` gives it); ``boxes`` [n, 4] or [B, n, 4]
    (x0, y0, x1, y1) in pixels, the reference's ``model_lrp.bboxes[0]``; ``bbox_scores`` [n] or [B, n].  The reference's
    first line rebinds ``bbox_scores`` to the global ``image_scores`` (which is what the notebook passes anyway); this
    function uses its argument.  Non-finite box coordinates raise ``ValueError``, as ``int(nan)`` does in the reference
    (the check reads one flag back from the device).  Returns [H, W, 3] or [B, H, W, 3]."""
    for t, n in ((image, "image"), (boxes, "boxes"), (bbox_scores, "bbox_scores")):
        _cuda(t, n)
    _same_device(image, boxes, bbox_scores)
    if image.dtype != torch.uint8 or image.dim() not in (3, 4) or image.shape[-1] != 3:
        raise MmxError(f"image must be uint8 [H, W, 3] or [B, H, W, 3] (got {image.dtype}, {tuple(image.shape)})")
    single = boxes.dim() == 2
    bx = boxes.unsqueeze(0) if single else boxes
    sc = bbox_scores.unsqueeze(0) if bbox_scores.dim() == 1 else bbox_scores
    img = image.unsqueeze(0) if image.dim() == 3 else image
    if bx.dim() != 3 or bx.shape[2] != 4:
        raise MmxError(f"boxes must be [n, 4] or [B, n, 4] (got {tuple(boxes.shape)})")
    B, n = bx.shape[0], bx.shape[1]
    if tuple(sc.shape) != (B, n):
        raise MmxError(f"bbox_scores must be [{n}] or [{B}, {n}] to match the boxes (got {tuple(bbox_scores.shape)})")
    if img.shape[0] not in (1, B):
        raise MmxError(f"image must hold 1 or {B} images (got {img.shape[0]})")
    if not bx.is_floating_point() or not sc.is_floating_point():
        raise MmxError("boxes and bbox_scores must be floating-point tensors")
    if not bool(torch.isfinite(bx).all()):
        raise ValueError("cannot convert a non-finite box coordinate to an integer")
    H, W = img.shape[1], img.shape[2]
    with torch.cuda.device(img.device):
        img = img.contiguous()
        bx = bx.to(torch.float32).contiguous()
        sc = sc.to(torch.float32).contiguous()
        out = torch.empty(B, H, W, 3, dtype=torch.uint8, device=img.device)
        check(lib().mmx_box_relevance_image(ptr(img), img.shape[0], H, W, ptr(bx), ptr(sc), B, n, ptr(out),
                                            current_stream()))
    return out[0] if single else out


def show_heatmap_on_text(text_encoding: torch.Tensor, R_text: torch.Tensor) -> List[torch.Tensor]:
    """The ``text_scores`` the notebook's ``show_heatmap_on_text`` prints (``R_text[eot, 1:eot] / R_text[eot,
    1:eot].sum()``, eot the first argmax of the token row), one view per prompt; the captum HTML rendering and the token
    decoding are left to the caller.  ``text_encoding`` [ctx] or [B, ctx] token ids; ``R_text`` [ctx, ctx] or [B, ctx,
    ctx].  The slice sum is taken in double and rounded once.  Costs one device-to-host copy of the B lengths."""
    _cuda(text_encoding, "text_encoding")
    _cuda(R_text, "R_text")
    _same_device(text_encoding, R_text)
    tok = text_encoding.unsqueeze(0) if text_encoding.dim() == 1 else text_encoding
    R = R_text.unsqueeze(0) if R_text.dim() == 2 else R_text
    if tok.dim() != 2 or tok.shape[1] < 1 or tok.is_floating_point():
        raise MmxError(f"text_encoding must be integer [ctx] or [B, ctx] (got {text_encoding.dtype}, "
                       f"{tuple(text_encoding.shape)})")
    B, ctx = tok.shape
    if tuple(R.shape) != (B, ctx, ctx) or not R.is_floating_point():
        raise MmxError(f"R_text must be floating-point [{ctx}, {ctx}] or [{B}, {ctx}, {ctx}] (got {tuple(R_text.shape)})")
    with torch.cuda.device(R.device):
        R = R.to(torch.float32).contiguous()
        tok = tok.to(torch.int32).contiguous()
        scores = torch.empty(B, ctx, dtype=torch.float32, device=R.device)
        lens = torch.empty(B, dtype=torch.int32, device=R.device)
        check(lib().mmx_clip_text_scores(ptr(R), ptr(tok), B, ctx, ptr(scores), ptr(lens), current_stream()))
        n = lens.tolist()
    return [scores[b, :n[b]] for b in range(B)]
