"""DETR's DC5 (dilated-C5) image front end: the oracle restatement and the unmodified reference module built with it.

TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).  ``--dilation`` (DETR/main.py:36) builds the ResNet with
``replace_stride_with_dilation=[False, False, True]`` (DETR/models/backbone.py:88-90): torchvision's
``_make_layer(dilate=True)`` gives layer4's block 0 stride 1 (conv2 dilation 1, padding 1; downsample 1x1 stride 1) and
blocks 1.. conv2 dilation 2, padding 2.  The feature map has stride 16; the weights (and so the state dict) are those of
the stride-32 body.  Everything else - stem, layer1..3, input_proj, mask, position embedding, heads - is
``oracle/detr_backbone_oracle.py`` unchanged.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F

from . import detr_backbone_oracle as bo


def body_forward(sd, images, stage_max: Optional[list] = None):
    """ResNet body with the dilated layer4 (layer4 output, stride 16), in the reference's operation order."""
    p = "backbone.0.body."
    x = F.relu(bo._frozen_bn(sd, p + "bn1.", F.conv2d(images, sd[p + "conv1.weight"], stride=2, padding=3)))
    if stage_max is not None:
        stage_max.append(x.abs().max().item())
    x = F.max_pool2d(x, 3, 2, 1)
    li = 1
    while f"{p}layer{li}.0.conv1.weight" in sd:
        i = 0
        while f"{p}layer{li}.{i}.conv1.weight" in sd:
            q = f"{p}layer{li}.{i}."
            if li == 4:
                s, dil = 1, (1 if i == 0 else 2)
            else:
                s, dil = (2 if (li > 1 and i == 0) else 1), 1
            y = F.relu(bo._frozen_bn(sd, q + "bn1.", F.conv2d(x, sd[q + "conv1.weight"])))
            y = F.relu(bo._frozen_bn(sd, q + "bn2.", F.conv2d(y, sd[q + "conv2.weight"], stride=s, padding=dil, dilation=dil)))
            y = bo._frozen_bn(sd, q + "bn3.", F.conv2d(y, sd[q + "conv3.weight"]))
            idn = x
            if q + "downsample.0.weight" in sd:
                idn = bo._frozen_bn(sd, q + "downsample.1.", F.conv2d(x, sd[q + "downsample.0.weight"], stride=s))
            x = F.relu(y + idn)
            i += 1
        if stage_max is not None:
            stage_max.append(x.abs().max().item())
        li += 1
    return x


def backbone(sd, images, mask=None, dtype=torch.float64, stage_max: Optional[list] = None):
    """``detr_backbone_oracle.backbone`` with the DC5 body: (src [B,d,h,w], pos [B,d,h,w] fp32, mask [B,h,w])."""
    sdd = {k: v.to(dtype) for k, v in sd.items() if k.startswith(("backbone.", "input_proj."))}
    x = body_forward(sdd, images.to(dtype), stage_max)
    src = F.conv2d(x, sdd["input_proj.weight"], sdd["input_proj.bias"])
    if mask is None:
        mask = torch.zeros(images.shape[0], *images.shape[-2:], dtype=torch.bool, device=images.device)
    m = F.interpolate(mask[None].float(), size=x.shape[-2:]).to(torch.bool)[0]
    return src, bo.position_sine(m, src.shape[1] // 2), m


PAIR_SEED, LONG_SEED = 11, 21


def pair_images(seed: int = PAIR_SEED):
    """The padded pair of ``detr_image.npz`` (3x96x160, 3x128x96; oracle/make_detr_image_golden.py ``images``)."""
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(3, 96, 160, generator=g), torch.randn(3, 128, 96, generator=g)]


def long_image(seed: int = LONG_SEED):
    """One 3x520x540 N(0, 1) image: 33 x 34 = 1122 DC5 tokens, past the 1024-key single-pass attention kernels."""
    return torch.randn(3, 520, 540, generator=torch.Generator().manual_seed(seed))


def feature_hw(H: int, W: int):
    """(h, w) of the DC5 feature map for an H x W input: stem /2, max-pool /2, layer2 /2, layer3 /2, layer4 /1."""
    for _ in range(4):
        H, W = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    return H, W


def build_reference(cfg, sd, name: str = "resnet50"):
    """The unmodified reference DETR module with the DC5 ``Backbone(name, False, False, dilation=True)``
    (build_backbone, DETR/models/backbone.py:111-119) and ``sd`` loaded strictly, as ``ref_detr_image.build``."""
    from . import ref_detr_image as rdi
    from .detr_oracle import to_checkpoint_format
    backbone, DETR, Transformer, PositionEmbeddingSine, _ = rdi._import()
    assert cfg.dec_layers == 6, "DETR.forward reads decoder output 5 (DETR/models/detr.py:72)"
    joiner = backbone.Joiner(backbone.Backbone(name, False, False, True),
                             PositionEmbeddingSine(cfg.d_model // 2, normalize=True))
    joiner.num_channels = 2048
    tr = Transformer(cfg.d_model, cfg.nhead, cfg.enc_layers, cfg.dec_layers, cfg.dim_ff, 0.0, return_intermediate_dec=True)
    m = DETR(joiner, tr, cfg.classes, cfg.queries).eval()
    missing, _ = m.load_state_dict(to_checkpoint_format(sd), strict=False)
    assert not missing, missing
    return m
