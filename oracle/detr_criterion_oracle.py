"""Plain PyTorch + numpy restatement of DETR's HungarianMatcher and SetCriterion (DETR/models/matcher.py,
DETR/models/detr.py:103-275, DETR/models/segmentation.py:172-215), device-agnostic, in fp32 or fp64, with a pure-Python
restatement of the assignment algorithm scipy's linear_sum_assignment implements (rectangular_lsap, Crouse 2016).

TEST INFRASTRUCTURE (tests/test_detr_criterion_*.py) and the eager arm of profiles/detr_criterion_bench.py; nothing
here is imported by the product package."""
from __future__ import annotations

import math
from typing import Dict, List

import numpy as np
import torch
import torch.nn.functional as F

LOSS_KEYS = {"labels": ("loss_ce", "class_error"), "boxes": ("loss_bbox", "loss_giou"),
             "cardinality": ("cardinality_error",), "masks": ("loss_mask", "loss_dice")}


def lsa(cost) -> tuple:
    """linear_sum_assignment(cost) restated: the transpose of a tall matrix, rows in order, the reversed scan order of
    the remaining columns, the tie rule of the Dijkstra step (an unassigned column wins a tie), the dual updates and the
    output order (rows ascending).  Raises ValueError as scipy does."""
    c = np.asarray(cost, dtype=np.float64)
    nr, nc = c.shape
    if nr == 0 or nc == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    tr = nc < nr
    if tr:
        c = c.T
        nr, nc = nc, nr
    if np.isnan(c).any() or (c == -np.inf).any():
        raise ValueError("matrix contains invalid numeric entries")
    cl = c.tolist()
    u, v = [0.0] * nr, [0.0] * nc
    path, col4row, row4col = [-1] * nc, [-1] * nr, [-1] * nc
    for cur in range(nr):
        SR, SC = [False] * nr, [False] * nc
        spc = [math.inf] * nc
        remaining = [nc - it - 1 for it in range(nc)]
        nrem, minv, i, sink = nc, 0.0, cur, -1
        while sink == -1:
            index, lowest = -1, math.inf
            SR[i] = True
            ci, ui = cl[i], u[i]
            for it in range(nrem):
                j = remaining[it]
                r = minv + ci[j] - ui - v[j]
                if r < spc[j]:
                    path[j] = i
                    spc[j] = r
                if spc[j] < lowest or (spc[j] == lowest and row4col[j] == -1):
                    lowest = spc[j]
                    index = it
            minv = lowest
            if minv == math.inf:
                raise ValueError("cost matrix is infeasible")
            j = remaining[index]
            if row4col[j] == -1:
                sink = j
            else:
                i = row4col[j]
            SC[j] = True
            nrem -= 1
            remaining[index] = remaining[nrem]
        u[cur] += minv
        for r in range(nr):
            if SR[r] and r != cur:
                u[r] += minv - spc[col4row[r]]
        for j in range(nc):
            if SC[j]:
                v[j] -= minv - spc[j]
        j = sink
        while True:
            r = path[j]
            row4col[j] = r
            col4row[r], j = j, col4row[r]
            if r == cur:
                break
    if tr:
        order = np.argsort(col4row)
        return np.asarray(col4row, np.int64)[order], order.astype(np.int64)
    return np.arange(nr, dtype=np.int64), np.asarray(col4row, np.int64)


def cxcywh_to_xyxy(x):
    xc, yc, w, h = x.unbind(-1)
    return torch.stack([xc - 0.5 * w, yc - 0.5 * h, xc + 0.5 * w, yc + 0.5 * h], dim=-1)


def giou(b1, b2):
    """generalized_box_iou of xyxy boxes [N,4] x [M,4] (box_ops.py:22-68), asserting as it does"""
    assert (b1[:, 2:] >= b1[:, :2]).all()
    assert (b2[:, 2:] >= b2[:, :2]).all()
    area1 = (b1[:, 2] - b1[:, 0]) * (b1[:, 3] - b1[:, 1])
    area2 = (b2[:, 2] - b2[:, 0]) * (b2[:, 3] - b2[:, 1])
    lt = torch.max(b1[:, None, :2], b2[:, :2])
    rb = torch.min(b1[:, None, 2:], b2[:, 2:])
    wh = (rb - lt).clamp(min=0)
    inter = wh[..., 0] * wh[..., 1]
    union = area1[:, None] + area2 - inter
    iou = inter / union
    lt = torch.min(b1[:, None, :2], b2[:, :2])
    rb = torch.max(b1[:, None, 2:], b2[:, 2:])
    wh = (rb - lt).clamp(min=0)
    area = wh[..., 0] * wh[..., 1]
    return iou - (area - union) / area


def cost_blocks(outputs, targets, w_class=1.0, w_bbox=1.0, w_giou=1.0) -> List[torch.Tensor]:
    """the matcher's cost matrix split per image: [Q, T_b] per image (matcher.py:60-81)"""
    bs, nq = outputs["pred_logits"].shape[:2]
    prob = outputs["pred_logits"].flatten(0, 1).softmax(-1)
    ob = outputs["pred_boxes"].flatten(0, 1)
    ids = torch.cat([t["labels"] for t in targets])
    tb = torch.cat([t["boxes"] for t in targets])
    Cm = w_bbox * torch.cdist(ob, tb, p=1) + w_class * (-prob[:, ids]) + w_giou * (-giou(cxcywh_to_xyxy(ob), cxcywh_to_xyxy(tb)))
    Cm = Cm.view(bs, nq, -1)
    return [c[i] for i, c in enumerate(Cm.split([len(t["boxes"]) for t in targets], -1))]


def match(outputs, targets, w_class=1.0, w_bbox=1.0, w_giou=1.0, solver=None):
    """the matcher's indices per image; ``solver`` is the assignment solver (default: ``lsa``, the restatement; the
    benchmark passes scipy's compiled ``linear_sum_assignment``, which the reference calls)"""
    solver = lsa if solver is None else solver
    return [tuple(torch.as_tensor(a, dtype=torch.int64) for a in solver(c.detach().cpu().double().numpy()))
            for c in cost_blocks(outputs, targets, w_class, w_bbox, w_giou)]


def _src_idx(indices):
    return (torch.cat([torch.full_like(s, i) for i, (s, _) in enumerate(indices)]), torch.cat([s for s, _ in indices]))


def _tgt_idx(indices):
    return (torch.cat([torch.full_like(t, i) for i, (_, t) in enumerate(indices)]), torch.cat([t for _, t in indices]))


def _losses(name, outputs, targets, indices, num_boxes, empty_weight, num_classes, log=True):
    dev = outputs["pred_logits"].device
    indices = [(i.to(dev), j.to(dev)) for i, j in indices]
    if name == "labels":
        lg = outputs["pred_logits"]
        idx = _src_idx(indices)
        tco = torch.cat([t["labels"][J] for t, (_, J) in zip(targets, indices)])
        tc = torch.full(lg.shape[:2], num_classes, dtype=torch.int64, device=dev)
        tc[idx] = tco
        out = {"loss_ce": F.cross_entropy(lg.transpose(1, 2), tc, empty_weight.to(lg))}
        if log:
            if tco.numel() == 0:
                acc = torch.zeros([], device=dev, dtype=lg.dtype)
            else:
                acc = (lg[idx].topk(1, 1, True, True)[1].t() == tco.view(1, -1)).view(-1).to(lg.dtype).sum(0) * (100.0 / tco.numel())
            out["class_error"] = 100 - acc
        return out
    if name == "cardinality":
        lg = outputs["pred_logits"]
        tl = torch.as_tensor([len(t["labels"]) for t in targets], device=dev)
        card = (lg.argmax(-1) != lg.shape[-1] - 1).sum(1)
        return {"cardinality_error": F.l1_loss(card.to(lg.dtype), tl.to(lg.dtype))}
    if name == "boxes":
        idx = _src_idx(indices)
        sb = outputs["pred_boxes"][idx]
        tb = torch.cat([t["boxes"][i] for t, (_, i) in zip(targets, indices)], dim=0)
        return {"loss_bbox": F.l1_loss(sb, tb, reduction="none").sum() / num_boxes,
                "loss_giou": (1 - torch.diag(giou(cxcywh_to_xyxy(sb), cxcywh_to_xyxy(tb)))).sum() / num_boxes}
    if name == "masks":
        return mask_losses(outputs["pred_masks"], [t["masks"] for t in targets], indices, num_boxes)
    raise AssertionError(f"do you really want to compute {name} loss?")


def mask_losses(pred_masks, tgt_masks, indices, num_boxes):
    """loss_masks (detr.py:184-211): the matched planes upsampled to the padded target size, focal + dice"""
    dt = pred_masks.dtype
    sb, si = _src_idx(indices)
    tb, ti = _tgt_idx(indices)
    src = pred_masks[sb, si]
    H, W = max(m.shape[1] for m in tgt_masks), max(m.shape[2] for m in tgt_masks)
    tgt = torch.zeros(len(ti), H, W, dtype=dt, device=pred_masks.device)
    for k, (b, j) in enumerate(zip(tb.tolist(), ti.tolist())):
        m = tgt_masks[b][j]
        tgt[k, :m.shape[0], :m.shape[1]] = m.to(dt)
    x = F.interpolate(src[:, None], size=(H, W), mode="bilinear", align_corners=False)[:, 0].flatten(1)
    t = tgt.flatten(1)
    prob = x.sigmoid()
    ce = F.binary_cross_entropy_with_logits(x, t, reduction="none")
    p_t = prob * t + (1 - prob) * (1 - t)
    loss = (0.25 * t + 0.75 * (1 - t)) * (ce * ((1 - p_t) ** 2))
    num = 2 * (prob * t).sum(1)
    den = prob.sum(-1) + t.sum(-1)
    return {"loss_mask": loss.mean(1).sum() / num_boxes, "loss_dice": (1 - (num + 1) / (den + 1)).sum() / num_boxes}


def criterion(outputs, targets, num_classes, eos_coef, losses, w_class=1.0, w_bbox=1.0, w_giou=1.0, return_indices=False,
              solver=None):
    """SetCriterion.forward (detr.py:233-275): the loss dict in the reference's key order; with ``return_indices`` also
    the matcher's indices of every layer (layer 0 the final output).  ``solver``: as in ``match``."""
    ew = torch.ones(num_classes + 1)
    ew[-1] = eos_coef
    layers = [outputs] + list(outputs.get("aux_outputs", []))
    indices = [match(layers[0], targets, w_class, w_bbox, w_giou, solver)]
    nb = max(float(sum(len(t["labels"]) for t in targets)), 1.0)
    out: Dict[str, torch.Tensor] = {}
    for k in losses:
        out.update(_losses(k, outputs, targets, indices[0], nb, ew, num_classes))
    for i, aux in enumerate(layers[1:]):
        indices.append(match(aux, targets, w_class, w_bbox, w_giou, solver))
        for k in losses:
            if k == "masks":
                continue
            d = _losses(k, aux, targets, indices[-1], nb, ew, num_classes, log=False)
            out.update({f"{key}_{i}": v for key, v in d.items()})
    return (out, indices) if return_indices else out
