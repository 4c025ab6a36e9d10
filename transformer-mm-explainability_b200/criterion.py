"""DETR's evaluation losses on the device: ``HungarianMatcher`` (DETR/models/matcher.py) and ``SetCriterion``
(DETR/models/detr.py:103-275, DETR/models/segmentation.py:172-215), drop-ins for the ``criterion`` the reference's
``engine.evaluate`` calls (DETR/engine.py:174), ``aux_outputs`` included.

The matching cost of every (layer, image), scipy's linear_sum_assignment restated in double (one CTA per problem), the
box / label losses of every layer and the last layer's mask losses go through four entry points (csrc/detr_criterion.cu,
five kernels) enqueued without waiting for the host.  The one host synchronisation of a call reads the status words, so that a degenerate box
raises ``AssertionError`` and an invalid or infeasible cost matrix ``ValueError`` as the reference would, in the
reference's order."""
from __future__ import annotations

import ctypes as C
from typing import Dict

import torch

from ._lib import lib, check, ptr, current_stream, MmxError

_LOSS_KEYS = {"labels": ("loss_ce", "class_error"), "boxes": ("loss_bbox", "loss_giou"),
              "cardinality": ("cardinality_error",), "masks": ("loss_mask", "loss_dice")}
_COL = {"loss_ce": 0, "class_error": 1, "loss_bbox": 2, "loss_giou": 3, "cardinality_error": 4}
_MAX_IMAGES = 64


def _ptrs(ts):
    return (C.c_void_p * len(ts))(*[t.data_ptr() for t in ts])


class _Batch:
    """The device inputs of one call: the layers (0 = ``outputs``, then ``aux_outputs``), the concatenated targets, and
    the match of every layer.  The constructor enqueues the cost and assignment kernels; ``read`` is the host read."""

    def __init__(self, layers, targets, matcher):
        lg0 = layers[0]["pred_logits"]
        if lg0.dim() != 3:
            raise MmxError(f"pred_logits is [B, Q, C+1], got {tuple(lg0.shape)}")
        self.dev = dev = lg0.device
        self.B, self.Q, self.C1 = B, Q, C1 = lg0.shape
        if len(targets) != B:
            raise MmxError(f"{B} images of outputs and {len(targets)} targets")
        if B > _MAX_IMAGES:
            raise MmxError(f"at most {_MAX_IMAGES} images per call, got {B}")
        self.logits, self.boxes = [], []
        for o in layers:
            lg, bx = o["pred_logits"], o["pred_boxes"]
            if tuple(lg.shape) != (B, Q, C1) or tuple(bx.shape) != (B, Q, 4):
                raise MmxError(f"every layer needs pred_logits {(B, Q, C1)} and pred_boxes {(B, Q, 4)}, got "
                               f"{tuple(lg.shape)} and {tuple(bx.shape)}")
            self.logits.append(lg.detach().to(device=dev, dtype=torch.float32).contiguous())
            self.boxes.append(bx.detach().to(device=dev, dtype=torch.float32).contiguous())
        self.L = L = len(layers)
        self.sizes = [len(t["labels"]) for t in targets]
        if any(len(t["boxes"]) != n for t, n in zip(targets, self.sizes)):
            raise MmxError("every target needs as many boxes as labels")
        self.T = T = sum(self.sizes)
        self.ids = torch.cat([t["labels"].to(device=dev, dtype=torch.int64).reshape(-1) for t in targets])
        self.tboxes = torch.cat([t["boxes"].detach().to(device=dev, dtype=torch.float32).reshape(-1, 4) for t in targets])
        off = [0]
        for n in self.sizes:
            off.append(off[-1] + n)
        self.off = (C.c_int * (B + 1))(*off)
        # one int64 buffer: the indices [L, 2, T], then the status words (int32): L of the cost, L * B of the assignment
        n_status = L + L * B
        self.buf = torch.empty(2 * L * T + (n_status + 1) // 2, device=dev, dtype=torch.int64)
        self.indices = self.buf[:2 * L * T]
        self.status_words = self.buf[2 * L * T:].view(torch.int32)
        self.cost = torch.empty(L * Q * T, device=dev, dtype=torch.float32)
        l = lib()
        with torch.cuda.device(dev):
            st = current_stream()
            check(l.mmx_detr_match_cost(_ptrs(self.logits), _ptrs(self.boxes), L, B, Q, C1, ptr(self.ids),
                                        ptr(self.tboxes), self.off, float(matcher.cost_class), float(matcher.cost_bbox),
                                        float(matcher.cost_giou), ptr(self.cost), ptr(self.status_words), st))
            check(l.mmx_detr_match_lsa(ptr(self.cost), L, B, Q, self.off, ptr(self.indices),
                                       ptr(self.status_words[L:]), st))

    def read(self, with_indices: bool):
        """The one host synchronisation: the status words (and the indices when asked) in one device-to-host copy."""
        src = self.buf if with_indices else self.buf[2 * self.L * self.T:]
        host = torch.empty(src.numel(), dtype=torch.int64, pin_memory=True)
        with torch.cuda.device(self.dev):
            host.copy_(src, non_blocking=True)
            torch.cuda.current_stream().synchronize()
        st = (host[2 * self.L * self.T:] if with_indices else host).view(torch.int32)
        self.cost_status = st[:self.L].tolist()
        self.lsa_status = st[self.L:self.L + self.L * self.B].tolist()
        return host[:2 * self.L * self.T] if with_indices else None

    def raise_for_layer(self, l: int):
        """What the reference's matcher call for layer l raises, in its order: the label gather (matcher.py:66), the box
        asserts of generalized_box_iou (:73, box_ops.py:51-52), then scipy per image (:81)."""
        if self.cost_status[0] & 2:
            raise IndexError(f"a target label is outside [0, {self.C1})")
        if self.cost_status[l] & 1:
            raise AssertionError()
        for b in range(self.B):
            s = self.lsa_status[l * self.B + b]
            if s == 1:
                raise ValueError("matrix contains invalid numeric entries")
            if s == 2:
                raise ValueError("cost matrix is infeasible")

    def pairs(self, host_indices, l: int):
        """the reference's [(int64 i, int64 j)] of layer l from the host copy of the indices"""
        blk = host_indices[2 * l * self.T:2 * (l + 1) * self.T].view(2, self.T)
        out, o = [], 0
        for n in self.sizes:
            k = min(self.Q, n)
            out.append((blk[0, o:o + k].clone(), blk[1, o:o + k].clone()))
            o += n
        return out


class HungarianMatcher:
    """``HungarianMatcher`` (DETR/models/matcher.py:12-81): the same defaults and assert; ``forward`` returns the
    reference's list of (int64 CPU i, int64 CPU j) per image, from one device-to-host copy for all images."""

    def __init__(self, cost_class: float = 1, cost_bbox: float = 1, cost_giou: float = 1):
        self.cost_class = cost_class
        self.cost_bbox = cost_bbox
        self.cost_giou = cost_giou
        assert cost_class != 0 or cost_bbox != 0 or cost_giou != 0, "all costs cant be 0"

    def to(self, *args, **kwargs):
        return self

    def eval(self):
        return self

    @torch.no_grad()
    def forward(self, outputs, targets):
        batch = _Batch([outputs], targets, self)
        host = batch.read(with_indices=True)
        batch.raise_for_layer(0)
        return batch.pairs(host, 0)

    __call__ = forward


class SetCriterion:
    """``SetCriterion`` (DETR/models/detr.py:103-275): the reference's signature and attributes; ``forward`` returns
    the reference's dict of 0-d device tensors (keys in its order, the ``_i`` entries of ``aux_outputs`` included).
    ``num_boxes`` is the host count, all-reduced over the process group when one is initialised (as a device tensor,
    so no extra synchronisation), divided by the world size and clamped to >= 1 (detr.py:248-252).

    Where it differs from the reference: with "masks" and no target in the whole batch, loss_mask and loss_dice are 0
    (a sum over no masks) - the reference raises NameError there, from its ``util.misc.interpolate`` wrapper on an
    empty batch under current torchvision.  class_error's top-1 is torch.topk(1)'s on CUDA (the lowest index among
    equal maxima), which the reference's CPU topk does not promise on exactly tied logits."""

    def __init__(self, num_classes, matcher, weight_dict, eos_coef, losses):
        self.num_classes = num_classes
        self.matcher = matcher
        self.weight_dict = weight_dict
        self.eos_coef = eos_coef
        self.losses = losses
        self.empty_weight = torch.ones(self.num_classes + 1)
        self.empty_weight[-1] = self.eos_coef

    def to(self, device=None, *args, **kwargs):
        if device is not None:
            self.empty_weight = self.empty_weight.to(device)
        return self

    def eval(self):
        return self

    def _num_boxes(self, n: int, dev) -> torch.Tensor:
        nb = torch.full((1,), float(n), device=dev, dtype=torch.float32)
        import torch.distributed as dist
        world = 1
        if dist.is_available() and dist.is_initialized():
            dist.all_reduce(nb)
            world = dist.get_world_size()
        return torch.clamp(nb / world, min=1)

    @torch.no_grad()
    def forward(self, outputs, targets) -> Dict[str, torch.Tensor]:
        aux = outputs.get("aux_outputs", [])
        layers = [outputs] + list(aux)
        batch = _Batch(layers, targets, self.matcher)
        dev, L = batch.dev, batch.L
        if batch.C1 != self.num_classes + 1:
            raise MmxError(f"pred_logits has {batch.C1} columns, num_classes + 1 = {self.num_classes + 1}")
        known = [k for k in self.losses if k in _LOSS_KEYS]
        nb = self._num_boxes(batch.T, dev)
        if self.empty_weight.device != dev:                  # once, when .to(device) was not called
            self.empty_weight = self.empty_weight.to(dev)
        w = self.empty_weight.to(dtype=torch.float32).contiguous()
        box = torch.empty(L, 5, device=dev, dtype=torch.float32)
        mask = torch.empty(2, device=dev, dtype=torch.float32)
        l = lib()
        with torch.cuda.device(dev):
            st = current_stream()
            if any(k in ("labels", "boxes", "cardinality") for k in known):
                check(l.mmx_detr_set_losses(_ptrs(batch.logits), _ptrs(batch.boxes), L, batch.B, batch.Q, batch.C1,
                                            ptr(batch.ids), ptr(batch.tboxes), batch.off, ptr(batch.indices), ptr(w),
                                            ptr(nb), ptr(box), st))
            if "masks" in known and "pred_masks" in outputs:
                self._mask_losses(outputs["pred_masks"], targets, batch, nb, mask, st)
        batch.read(with_indices=False)
        # the reference's order: the last layer's matcher, its losses (get_loss's assert), then each aux layer's matcher
        batch.raise_for_layer(0)
        out: Dict[str, torch.Tensor] = {}
        for k in self.losses:
            assert k in _LOSS_KEYS, f"do you really want to compute {k} loss?"
            assert k != "masks" or "pred_masks" in outputs
            for key in _LOSS_KEYS[k]:
                out[key] = mask[0 if key == "loss_mask" else 1] if k == "masks" else box[0, _COL[key]]
        for i in range(1, L):
            batch.raise_for_layer(i)
            for k in self.losses:
                if k == "masks":
                    continue
                for key in _LOSS_KEYS[k]:
                    if key != "class_error":
                        out[f"{key}_{i - 1}"] = box[i, _COL[key]]
        return out

    __call__ = forward

    def _mask_losses(self, pred_masks, targets, batch, nb, out, st):
        pm = pred_masks
        if pm.dim() == 5 and pm.shape[2] == 1:
            pm = pm[:, :, 0]
        if pm.dim() != 4 or tuple(pm.shape[:2]) != (batch.B, batch.Q):
            raise MmxError(f"pred_masks is [B, Q, h, w] for B = {batch.B}, Q = {batch.Q}, got {tuple(pred_masks.shape)}")
        pm = pm.detach().to(device=batch.dev, dtype=torch.float32).contiguous()
        h, w = pm.shape[-2:]
        tm = [t["masks"].detach() for t in targets]
        floats = {m.dtype for m in tm} - {torch.bool, torch.uint8}
        dtype = 1 if floats else 0
        # the target masks are read in place: bool / uint8 as bytes, anything else as fp32
        tm = [m.to(device=batch.dev, dtype=torch.float32 if dtype else m.dtype).contiguous() for m in tm]
        tm = [m.view(torch.uint8) if m.dtype == torch.bool else m for m in tm]
        for m, n in zip(tm, batch.sizes):
            if m.dim() != 3 or m.shape[0] != n:
                raise MmxError(f"target masks are [T_b, H, W] with T_b = {n}, got {tuple(m.shape)}")
        hw = (C.c_int * (2 * batch.B))(*[v for m in tm for v in m.shape[1:]])
        check(lib().mmx_detr_mask_losses(ptr(pm), batch.B, batch.Q, h, w, _ptrs(tm), hw, dtype, batch.off,
                                         ptr(batch.indices), ptr(nb), ptr(out), st))
