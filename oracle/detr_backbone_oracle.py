"""Oracle restatement of DETR's image front end: ResNet body, input_proj, mask and sine position embedding, box head.

TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).  Plain PyTorch over a ``state_dict`` with the reference's key names,
in the reference's operation order (conv, then the FrozenBatchNorm2d affine - no folding):
  * FrozenBatchNorm2d.forward ....... DETR/models/backbone.py:45-55
  * torchvision ResNet v1.5 ......... stem conv 7x7/2 + BN + ReLU, max-pool 3x3/2, bottlenecks with the stride on conv2
  * BackboneBase.forward ............ DETR/models/backbone.py:73-80 (nearest-resampled mask)
  * PositionEmbeddingSine ........... DETR/models/position_encoding.py:28-48 (normalize=True)
  * DETR.forward / MLP .............. DETR/models/detr.py:63-77, :309-321
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence

import torch
import torch.nn.functional as F

from mmx_b200.synthetic import DetrConfig, detr_init_state_dict

R50_BLOCKS = (3, 4, 6, 3)
DETR_IMAGE = DetrConfig(64, 2, 2, 6, 96, 7, 5)     # the golden-size transformer (DETR.forward reads decoder output 5)


def init_state_dict(cfg: DetrConfig, seed: int = 0, blocks: Sequence[int] = R50_BLOCKS) -> Dict[str, torch.Tensor]:
    """A whole DETR state dict: ResNet body (``backbone.0.body.*``), ``input_proj``, transformer, class and box heads.
    Conv weights are He-normal and the BN statistics are drawn near the identity (running_var in [0.5, 1.5], the last BN
    of each bottleneck scaled by 0.5), so activations stay O(1..100) through all blocks - far inside fp16 range."""
    sd = detr_init_state_dict(cfg, seed)
    g = torch.Generator().manual_seed(seed + 1000)

    def conv(key, cout, cin, k):
        sd[key] = torch.randn(cout, cin, k, k, generator=g) * math.sqrt(2.0 / (cin * k * k))

    def bn(p, n, gain=1.0):
        sd[p + "weight"] = gain * (1.0 + 0.1 * torch.randn(n, generator=g))
        sd[p + "bias"] = 0.1 * torch.randn(n, generator=g)
        sd[p + "running_mean"] = 0.1 * torch.randn(n, generator=g)
        sd[p + "running_var"] = 0.5 + torch.rand(n, generator=g)

    body = "backbone.0.body."
    conv(body + "conv1.weight", 64, 3, 7)
    bn(body + "bn1.", 64)
    cin = 64
    for li, nb in enumerate(blocks, start=1):
        width = 64 * 2 ** (li - 1)
        for i in range(nb):
            p = f"{body}layer{li}.{i}."
            conv(p + "conv1.weight", width, cin, 1); bn(p + "bn1.", width)
            conv(p + "conv2.weight", width, width, 3); bn(p + "bn2.", width)
            conv(p + "conv3.weight", 4 * width, width, 1); bn(p + "bn3.", 4 * width, gain=0.5)
            if i == 0:
                conv(p + "downsample.0.weight", 4 * width, cin, 1); bn(p + "downsample.1.", 4 * width)
            cin = 4 * width
    sd["input_proj.weight"] = torch.randn(cfg.d_model, cin, 1, 1, generator=g) * math.sqrt(1.0 / cin)
    sd["input_proj.bias"] = 0.05 * torch.randn(cfg.d_model, generator=g)
    for i, (o, k) in enumerate(((cfg.d_model, cfg.d_model), (cfg.d_model, cfg.d_model), (4, cfg.d_model))):
        sd[f"bbox_embed.layers.{i}.weight"] = torch.randn(o, k, generator=g) * math.sqrt(1.0 / k)
        sd[f"bbox_embed.layers.{i}.bias"] = 0.05 * torch.randn(o, generator=g)
    return sd


def nested(images: List[torch.Tensor]):
    """nested_tensor_from_tensor_list (DETR/util/misc.py:306-327): zero-padded batch and mask (True on padding)."""
    H, W = max(t.shape[1] for t in images), max(t.shape[2] for t in images)
    x = torch.zeros(len(images), images[0].shape[0], H, W, dtype=images[0].dtype, device=images[0].device)
    m = torch.ones(len(images), H, W, dtype=torch.bool, device=images[0].device)
    for i, t in enumerate(images):
        x[i, :, :t.shape[1], :t.shape[2]].copy_(t)
        m[i, :t.shape[1], :t.shape[2]] = False
    return x, m


def _frozen_bn(sd, p, x):
    w, b = sd[p + "weight"].reshape(1, -1, 1, 1), sd[p + "bias"].reshape(1, -1, 1, 1)
    rv, rm = sd[p + "running_var"].reshape(1, -1, 1, 1), sd[p + "running_mean"].reshape(1, -1, 1, 1)
    scale = w * (rv + 1e-5).rsqrt()
    return x * scale + (b - rm * scale)


def body_forward(sd, images, stage_max: Optional[list] = None):
    """ResNet body (layer4 output).  ``stage_max``: appends max|activation| after the stem and every stage."""
    p = "backbone.0.body."
    x = F.relu(_frozen_bn(sd, p + "bn1.", F.conv2d(images, sd[p + "conv1.weight"], stride=2, padding=3)))
    if stage_max is not None:
        stage_max.append(x.abs().max().item())
    x = F.max_pool2d(x, 3, 2, 1)
    li = 1
    while f"{p}layer{li}.0.conv1.weight" in sd:
        i = 0
        while f"{p}layer{li}.{i}.conv1.weight" in sd:
            q = f"{p}layer{li}.{i}."
            s = 2 if (li > 1 and i == 0) else 1
            y = F.relu(_frozen_bn(sd, q + "bn1.", F.conv2d(x, sd[q + "conv1.weight"])))
            y = F.relu(_frozen_bn(sd, q + "bn2.", F.conv2d(y, sd[q + "conv2.weight"], stride=s, padding=1)))
            y = _frozen_bn(sd, q + "bn3.", F.conv2d(y, sd[q + "conv3.weight"]))
            idn = x
            if q + "downsample.0.weight" in sd:
                idn = _frozen_bn(sd, q + "downsample.1.", F.conv2d(x, sd[q + "downsample.0.weight"], stride=s))
            x = F.relu(y + idn)
            i += 1
        if stage_max is not None:
            stage_max.append(x.abs().max().item())
        li += 1
    return x


def position_sine(mask: torch.Tensor, npf: int, temperature: float = 10000.0) -> torch.Tensor:
    """PositionEmbeddingSine(npf, temperature, normalize=True).forward on a [B,h,w] bool mask -> [B, 2 npf, h, w] fp32."""
    not_mask = ~mask
    y_embed = not_mask.cumsum(1, dtype=torch.float32)
    x_embed = not_mask.cumsum(2, dtype=torch.float32)
    eps, scale = 1e-6, 2 * math.pi
    y_embed = y_embed / (y_embed[:, -1:, :] + eps) * scale
    x_embed = x_embed / (x_embed[:, :, -1:] + eps) * scale
    dim_t = torch.arange(npf, dtype=torch.float32, device=mask.device)
    dim_t = temperature ** (2 * (dim_t // 2) / npf)
    pos_x = x_embed[:, :, :, None] / dim_t
    pos_y = y_embed[:, :, :, None] / dim_t
    pos_x = torch.stack((pos_x[:, :, :, 0::2].sin(), pos_x[:, :, :, 1::2].cos()), dim=4).flatten(3)
    pos_y = torch.stack((pos_y[:, :, :, 0::2].sin(), pos_y[:, :, :, 1::2].cos()), dim=4).flatten(3)
    return torch.cat((pos_y, pos_x), dim=3).permute(0, 3, 1, 2)


def backbone(sd, images, mask=None, dtype=torch.float64, stage_max: Optional[list] = None):
    """(src = input_proj(layer4) [B,d,h,w], pos [B,d,h,w] fp32, mask [B,h,w]) for images [B,3,H,W] and a padding mask
    [B,H,W] (None = no padding).  The convs run in ``dtype``; pos is always the fp32 reference computation."""
    sdd = {k: v.to(dtype) for k, v in sd.items() if k.startswith(("backbone.", "input_proj."))}
    x = body_forward(sdd, images.to(dtype), stage_max)
    src = F.conv2d(x, sdd["input_proj.weight"], sdd["input_proj.bias"])
    if mask is None:
        mask = torch.zeros(images.shape[0], *images.shape[-2:], dtype=torch.bool, device=images.device)
    m = F.interpolate(mask[None].float(), size=x.shape[-2:]).to(torch.bool)[0]
    return src, position_sine(m, src.shape[1] // 2), m


def boxes(sd, hs: torch.Tensor) -> torch.Tensor:
    """sigmoid(bbox_embed(hs)) (DETR/models/detr.py:73,309-321)."""
    x = hs
    for i in range(3):
        x = F.linear(x, sd[f"bbox_embed.layers.{i}.weight"].to(x.dtype), sd[f"bbox_embed.layers.{i}.bias"].to(x.dtype))
        x = F.relu(x) if i < 2 else x
    return x.sigmoid()


def decoder_output(sd, cfg: DetrConfig, src, pos, dtype=torch.float64) -> torch.Tensor:
    """hs = decoder.norm(last decoder layer) [B,Q,d], from oracle/detr_oracle.py's forward with an identity class head."""
    from .detr_oracle import detr_forward
    d = cfg.d_model
    sdd = {k: v.to(dtype) for k, v in sd.items()}
    sdd["class_embed.weight"], sdd["class_embed.bias"] = torch.eye(d, dtype=dtype), torch.zeros(d, dtype=dtype)
    return detr_forward(sdd, cfg, src.to(dtype), pos.to(dtype))[0]
