"""DETR's image front end on libmmx (SURVEY.md §8a rows a10, a11): the ResNet body, ``input_proj`` and the mask /
sine position embedding that ``DETR.forward`` runs before the transformer (DETR/models/detr.py:63-69).

``DetrBackbone`` is built from a DETR ``state_dict`` (``backbone.0.body.*`` and ``input_proj.*``):

* every ``FrozenBatchNorm2d`` (DETR/models/backbone.py:45-55, ``scale = w rsqrt(rv + 1e-5)``, ``bias = b - rm scale``) is
  folded into the conv before it, and each weight is reordered from [Cout, Cin, kh, kw] to [Cout, kh*kw*Cin] (the
  (ky, kx, c) order of the gathered patches) and packed once for the fp16x3 tensor-core GEMM;
* the bottlenecks follow torchvision's ResNet v1.5 (stride on the 3x3 conv, downsample = 1x1 stride-s conv + BN); the
  block counts come from the keys (3/4/6/3 for ResNet-50, 3/4/23/3 for ResNet-101).  ``dilation=True`` builds the DC5
  body (DETR/models/backbone.py:88-90, ``--dilation``): layer4 as torchvision's ``_make_layer(dilate=True)``, i.e. block 0
  with stride 1 (conv2 dilation 1, padding 1, downsample stride 1) and blocks 1.. with conv2 dilation 2, padding 2, so
  the feature map has stride 16 instead of 32.  Dilation is not visible in the weights: the caller says which it is;
* activations are NHWC matrices [B*H*W, C].  Convs with fewer than 128 output channels (the stem, layer1's conv1 / conv2,
  an input_proj below 128) are padded to 128 zero rows with zero bias, so every conv meets the tensor-core GEMM's
  N >= 128 rule; their outputs keep a row stride of 128 and consumers read the real channels at that stride.

Everything runs forward only: gradients and LRP stop at the transformer input, as in the reference (no dgrad goes
below the encoder input, DETR/models/detr.py:79-92).
"""
from __future__ import annotations

import ctypes as C
import re
from typing import Dict, Optional, Tuple

import torch

from ._lib import lib, check, ptr, current_stream, MmxError
from .nn import pack_weight, ACT_NONE, ACT_RELU

MIN_ROWS = 128      # the fp16x3 / 3xTF32 GEMMs take N >= 128 (gemm_f16x3_shape_ok)
BODY = "backbone.0.body."


def has_backbone(sd: Dict[str, torch.Tensor]) -> bool:
    return any(k.startswith(BODY) for k in sd)


def fold_frozen_bn(w: torch.Tensor, bn: Dict[str, torch.Tensor], eps: float = 1e-5) -> Tuple[torch.Tensor, torch.Tensor]:
    """conv weight [Cout, ...] and FrozenBatchNorm2d buffers -> (w * scale, b - rm * scale), in fp32 like
    FrozenBatchNorm2d.forward (DETR/models/backbone.py:45-55)."""
    scale = bn["weight"].float() * (bn["running_var"].float() + eps).rsqrt()
    bias = bn["bias"].float() - bn["running_mean"].float() * scale
    return w.float() * scale.reshape(-1, *([1] * (w.dim() - 1))), bias


class _Act:
    """An NHWC activation: ``t`` [B*H*W, >= C] with row stride t.stride(0), C real channels."""
    __slots__ = ("t", "B", "H", "W", "C")

    def __init__(self, t, B, H, W, C):
        self.t, self.B, self.H, self.W, self.C = t, B, H, W, C

    def strides(self):
        ld = self.t.stride(0)
        return self.H * self.W * ld, self.W * ld, ld, 1


class Conv:
    """One conv (+ folded BN): reordered [rows, kh*kw*Cin] weight padded to >= 128 rows, its bias and packed planes."""

    def __init__(self, w: torch.Tensor, b: Optional[torch.Tensor], stride: int, pad: int, device, dilation: int = 1):
        cout, cin, kh, kw = w.shape
        self.cout, self.cin, self.kh, self.kw, self.stride, self.pad = cout, cin, kh, kw, stride, pad
        self.dilation = dilation
        self.rows = max(cout, MIN_ROWS)
        wr = torch.zeros(self.rows, kh * kw * cin, dtype=torch.float32)
        wr[:cout] = w.detach().float().permute(0, 2, 3, 1).reshape(cout, -1).cpu()
        bias = torch.zeros(self.rows, dtype=torch.float32)
        if b is not None:
            bias[:cout] = b.detach().float().cpu()
        self.w = wr.to(device).contiguous()
        self.b = bias.to(device)
        self.pw = pack_weight(self.w)

    def out_hw(self, H, W):
        d = self.dilation
        return ((H + 2 * self.pad - d * (self.kh - 1) - 1) // self.stride + 1,
                (W + 2 * self.pad - d * (self.kw - 1) - 1) // self.stride + 1)

    def __call__(self, x, strides, B, H, W, act=ACT_NONE, residual: Optional[_Act] = None) -> _Act:
        Ho, Wo = self.out_hw(H, W)
        out = torch.empty(B * Ho * Wo, self.rows, device=self.w.device, dtype=torch.float32)
        res = residual.t if residual is not None else None
        check(lib().mmx_conv2d_dilated(ptr(x), *strides, B, H, W, self.cin, ptr(self.w), self.w.stride(0), ptr(self.pw),
                                       ptr(self.b), ptr(res), 0 if res is None else res.stride(0), ptr(out), self.rows, self.rows,
                                       self.kh, self.kw, self.stride, self.pad, self.dilation, act, current_stream()))
        return _Act(out, B, Ho, Wo, self.cout)

    def on(self, a: _Act, act=ACT_NONE, residual: Optional[_Act] = None) -> _Act:
        assert a.C == self.cin, (a.C, self.cin)
        return self(a.t, a.strides(), a.B, a.H, a.W, act, residual)


class Bottleneck:
    """torchvision ResNet v1.5 bottleneck: relu(bn3(conv3(relu(bn2(conv2(relu(bn1(conv1 x)))))) + downsample(x)); conv2 is
    the 3x3 conv with padding = dilation."""

    def __init__(self, sd, p, stride, device, dilation: int = 1):
        conv = lambda n, s, pad, dil=1: Conv(*fold_frozen_bn(sd[p + f"conv{n}.weight"], _bn(sd, p + f"bn{n}.")), s, pad, device,
                                             dil)
        self.conv1, self.conv2, self.conv3 = conv(1, 1, 0), conv(2, stride, dilation, dilation), conv(3, 1, 0)
        self.down = None
        if p + "downsample.0.weight" in sd:
            self.down = Conv(*fold_frozen_bn(sd[p + "downsample.0.weight"], _bn(sd, p + "downsample.1.")), stride, 0, device)

    def __call__(self, x: _Act) -> _Act:
        identity = self.down.on(x) if self.down is not None else x
        y = self.conv2.on(self.conv1.on(x, ACT_RELU), ACT_RELU)
        return self.conv3.on(y, ACT_RELU, residual=identity)


def _bn(sd, p):
    return {n: sd[p + n] for n in ("weight", "bias", "running_mean", "running_var")}


class DetrBackbone:
    """``backbone(samples)`` -> ``input_proj(src)`` and ``pos`` of DETR.forward (DETR/models/detr.py:63-69), both
    [B*h*w, d_model] (row = b*h*w + y*w + x), plus the feature-resolution padding mask [B, h, w].  ``dilation=True``: the
    DC5 body (stride-16 layer4, module docstring)."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], device, temperature: float = 10000.0, *, dilation: bool = False):
        sd = {k: v for k, v in state_dict.items() if k.startswith((BODY, "input_proj."))}
        sd = {(k[len(BODY):] if k.startswith(BODY) else k): v.detach().to(device) for k, v in sd.items()}
        self.device = torch.device(device)
        self.temperature = temperature
        self.dilation = bool(dilation)
        self.stem = Conv(*fold_frozen_bn(sd["conv1.weight"], _bn(sd, "bn1.")), 2, 3, device)
        self.layers = []
        for li in range(1, 5):
            idx = sorted({int(m.group(1)) for k in sd for m in [re.match(rf"layer{li}\.(\d+)\.", k)] if m})
            if not idx:
                raise MmxError(f"state_dict has no {BODY}layer{li}.* keys")
            if li == 4 and self.dilation:      # _make_layer(dilate=True): stride 1; blocks after the first dilate by 2
                self.layers.append([Bottleneck(sd, f"layer4.{i}.", 1, device, 1 if i == 0 else 2) for i in idx])
                continue
            self.layers.append([Bottleneck(sd, f"layer{li}.{i}.", (1 if li == 1 else 2) if i == 0 else 1, device)
                                for i in idx])
        if "input_proj.weight" not in sd:
            raise MmxError("state_dict has backbone keys but no input_proj.weight")
        self.input_proj = Conv(sd["input_proj.weight"], sd["input_proj.bias"], 1, 0, device)
        self.d_model = self.input_proj.cout
        if self.d_model % 2:
            raise MmxError("d_model must be even (sine position embedding of d_model / 2 features per axis)")
        self.block_counts = [len(L) for L in self.layers]

    def body(self, images: torch.Tensor) -> _Act:
        """ResNet body: stem conv + BN + ReLU, 3x3/2 max-pool, layer1 .. layer4 (layer4's output, as DETR uses)."""
        B, C3, H, W = images.shape
        x = self.stem(images, (C3 * H * W, W, 1, H * W), B, H, W, ACT_RELU)
        Hp, Wp = (x.H - 1) // 2 + 1, (x.W - 1) // 2 + 1
        pooled = torch.empty(B * Hp * Wp, x.t.shape[1], device=self.device, dtype=torch.float32)
        check(lib().mmx_maxpool2d_nhwc(ptr(x.t), x.t.stride(0), ptr(pooled), pooled.stride(0), B, x.H, x.W, x.C,
                                       current_stream()))
        x = _Act(pooled, B, Hp, Wp, x.C)
        for layer in self.layers:
            for blk in layer:
                x = blk(x)
        return x

    def __call__(self, images: torch.Tensor, mask: Optional[torch.Tensor]):
        """images [B, 3, H, W] fp32 on the device, mask [B, H, W] (True / non-zero = padding) or None.  Returns
        (src [B*S, d], pos [B*S, d], mask [B, h, w] bool, (h, w))."""
        feat = self.body(images)
        src = self.input_proj.on(feat)
        B, h, w, d = feat.B, feat.H, feat.W, self.d_model
        src_t = src.t if src.t.shape[1] == d else src.t[:, :d].contiguous()
        pos = torch.empty(B * h * w, d, device=self.device, dtype=torch.float32)
        mask_out = torch.empty(B, h, w, device=self.device, dtype=torch.uint8)
        m = None if mask is None else mask.to(device=self.device, dtype=torch.uint8).contiguous()
        H, W = images.shape[-2:]
        check(lib().mmx_detr_position_sine(ptr(m), B, H, W, h, w, d // 2, C.c_float(self.temperature), ptr(pos), d,
                                           ptr(mask_out), current_stream()))
        return src_t, pos, mask_out.bool(), (h, w)


def conv_flops(bb: DetrBackbone, B: int, H: int, W: int) -> float:
    """Algorithmic FLOPs (2 * M * Cout * K with the real channel counts) of every conv of the backbone for a B x 3 x H x W
    input: the numerator of the backbone's GEMM TFLOP/s."""
    total = 0.0

    def add(c: Conv, h, w):
        nonlocal total
        ho, wo = c.out_hw(h, w)
        total += 2.0 * B * ho * wo * c.cout * c.kh * c.kw * c.cin
        return ho, wo
    h, w = add(bb.stem, H, W)
    h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    for layer in bb.layers:
        for blk in layer:
            if blk.down is not None:
                add(blk.down, h, w)
            add(blk.conv1, h, w)
            h, w = add(blk.conv2, h, w)
            add(blk.conv3, h, w)
    add(bb.input_proj, h, w)
    return total
