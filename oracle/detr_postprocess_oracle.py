"""Oracle restatement of DETR's two evaluation post-processors, in plain PyTorch on any device.

TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).  The reference's operations in the reference's order:
  * PostProcess.forward ......... DETR/models/detr.py:289-306
  * PostProcessSegm.forward ..... DETR/models/segmentation.py:224-242 (the bool masks stay on the input's device until
                                  the final nearest resize, which gives the same bits on CPU and CUDA)
"""
from __future__ import annotations

import torch
import torch.nn.functional as F


def postprocess(pred_logits, pred_boxes, target_sizes):
    """(scores [B,Q], labels [B,Q], boxes [B,Q,4])"""
    scores, labels = F.softmax(pred_logits, -1)[..., :-1].max(-1)
    x_c, y_c, w, h = pred_boxes.unbind(-1)
    boxes = torch.stack([(x_c - 0.5 * w), (y_c - 0.5 * h), (x_c + 0.5 * w), (y_c + 0.5 * h)], dim=-1)
    img_h, img_w = target_sizes.unbind(1)
    return scores, labels, boxes * torch.stack([img_w, img_h, img_w, img_h], dim=1)[:, None, :]


def postprocess_segm(pred_masks, sizes, orig_sizes, threshold: float = 0.5):
    """[uint8 [Q,1,oh,ow] on the CPU per image] for pred_masks [B,Q,h,w], sizes / orig_sizes [B,2] (h, w)"""
    max_h, max_w = sizes.max(0)[0].tolist()
    m = F.interpolate(pred_masks, size=(max_h, max_w), mode="bilinear", align_corners=False).sigmoid() > threshold
    return [F.interpolate(cur[:, :ih, :iw].unsqueeze(1).float(), size=(oh, ow), mode="nearest").byte().cpu()
            for cur, (ih, iw), (oh, ow) in zip(m, sizes.tolist(), orig_sizes.tolist())]
