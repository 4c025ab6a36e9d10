"""Oracle restatement of the single-modality ViT relevancy path (SURVEY.md §8a row a14).

TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).

Pinning of the model forward: the ViT the notebook uses comes from another repository
(``hila-chefer/Transformer-Explainability``, ``baselines/ViT/ViT_new.py``, cloned at
Transformer_MM_explainability_ViT.ipynb:47 and imported at :1212) which is NOT vendored under /root/reference, so it
cannot be executed here.  The forward below restates the published timm ``vit_base_patch16_224`` block that file
wraps (pre-LN, eps 1e-6, packed qkv with bias, scores = (q k^T) * scale, exact-erf GELU MLP, cls-token head) and is
pinned against an independent implementation of the same architecture: torchvision's ``VisionTransformer``
(``vit_b_16``) with shared weights - logits and every block's attention probabilities, tiny and full ViT-B/16 size
(``tests/test_vit_pin.py``).
The RULE is pinned: ``avg_heads`` / ``apply_self_attention_rules`` / ``generate_relevance`` follow
Transformer_MM_explainability_ViT.ipynb:1169-1201 and are checked against the reference's own rule functions
through tests/golden/rules.npz.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict

import torch
import torch.nn.functional as F

from .rules import avg_heads


@dataclass(frozen=True)
class VitConfig:
    image: int = 224
    patch: int = 16
    dim: int = 768
    depth: int = 12
    heads: int = 12
    mlp_ratio: int = 4
    num_classes: int = 1000

    @property
    def tokens(self):
        return (self.image // self.patch) ** 2 + 1


VIT_B16 = VitConfig()
VIT_TINY = VitConfig(image=32, patch=8, dim=64, depth=2, heads=2, mlp_ratio=2, num_classes=10)


def init_state_dict(cfg: VitConfig, seed: int = 0) -> Dict[str, torch.Tensor]:
    g = torch.Generator().manual_seed(seed)

    def tn(*shape, std=0.02):
        return torch.randn(*shape, generator=g) * std

    D = cfg.dim
    sd = {"cls_token": tn(1, 1, D), "pos_embed": tn(1, cfg.tokens, D),
          "patch_embed.proj.weight": tn(D, 3, cfg.patch, cfg.patch, std=1.0 / math.sqrt(3 * cfg.patch ** 2)),
          "patch_embed.proj.bias": tn(D), "norm.weight": 1 + 0.1 * tn(D, std=1.0), "norm.bias": tn(D),
          "head.weight": tn(cfg.num_classes, D, std=0.05), "head.bias": tn(cfg.num_classes)}
    for i in range(cfg.depth):
        p = f"blocks.{i}."
        sd[p + "norm1.weight"] = 1 + 0.1 * tn(D, std=1.0); sd[p + "norm1.bias"] = tn(D)
        sd[p + "norm2.weight"] = 1 + 0.1 * tn(D, std=1.0); sd[p + "norm2.bias"] = tn(D)
        sd[p + "attn.qkv.weight"] = tn(3 * D, D, std=D ** -0.5); sd[p + "attn.qkv.bias"] = tn(3 * D)
        sd[p + "attn.proj.weight"] = tn(D, D, std=D ** -0.5); sd[p + "attn.proj.bias"] = tn(D)
        sd[p + "mlp.fc1.weight"] = tn(cfg.mlp_ratio * D, D, std=D ** -0.5); sd[p + "mlp.fc1.bias"] = tn(cfg.mlp_ratio * D)
        sd[p + "mlp.fc2.weight"] = tn(D, cfg.mlp_ratio * D, std=(cfg.mlp_ratio * D) ** -0.5); sd[p + "mlp.fc2.bias"] = tn(D)
    return sd


def vit_forward(sd, cfg: VitConfig, images, stage):
    B, D, H = images.shape[0], cfg.dim, cfg.heads
    x = F.conv2d(images, sd["patch_embed.proj.weight"], sd["patch_embed.proj.bias"], stride=cfg.patch)
    x = x.flatten(2).transpose(1, 2)
    x = torch.cat([sd["cls_token"].expand(B, -1, -1), x], dim=1) + sd["pos_embed"]
    S = x.shape[1]
    scale = (D // H) ** -0.5
    for i in range(cfg.depth):
        p = f"blocks.{i}."
        h = F.layer_norm(x, (D,), sd[p + "norm1.weight"], sd[p + "norm1.bias"], 1e-6)
        qkv = F.linear(h, sd[p + "attn.qkv.weight"], sd[p + "attn.qkv.bias"]).reshape(B, S, 3, H, D // H).permute(2, 0, 3, 1, 4)
        q, k, v = qkv[0], qkv[1], qkv[2]
        attn = ((q @ k.transpose(-1, -2)) * scale).softmax(dim=-1)        # scores scaled AFTER q k^T
        stage.append(attn)                                                # save_attn + register_hook site
        o = (attn @ v).transpose(1, 2).reshape(B, S, D)
        x = x + F.linear(o, sd[p + "attn.proj.weight"], sd[p + "attn.proj.bias"])
        h = F.layer_norm(x, (D,), sd[p + "norm2.weight"], sd[p + "norm2.bias"], 1e-6)
        h = F.gelu(F.linear(h, sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"]))
        x = x + F.linear(h, sd[p + "mlp.fc2.weight"], sd[p + "mlp.fc2.bias"])
    x = F.layer_norm(x, (D,), sd["norm.weight"], sd["norm.bias"], 1e-6)
    return F.linear(x[:, 0], sd["head.weight"], sd["head.bias"])


def generate_relevance(sd, cfg: VitConfig, images, index=None, dtype=torch.float32):
    """Transformer_MM_explainability_ViT.ipynb:1181-1201, per sample: one backward from logits[b, index_b], R = I,
    ``R += avg_heads(A_l, dA_l) @ R`` for all blocks, return R[0, 1:].  Returns ([B, S-1], logits)."""
    sd = {k: v.to(dtype) for k, v in sd.items()}
    images = images.to(dtype).requires_grad_(True)
    stage = []
    logits = vit_forward(sd, cfg, images, stage)
    B = images.shape[0]
    idx = logits.argmax(-1) if index is None else torch.as_tensor(index).reshape(B)
    y = logits[torch.arange(B), idx].sum()
    grads = torch.autograd.grad(y, stage)
    out = []
    for b in range(B):
        S = stage[0].shape[-1]
        R = torch.eye(S, dtype=dtype, device=images.device)
        for A, G in zip(stage, grads):
            cam = avg_heads(A[b].detach(), G[b])
            R = R + cam @ R
        out.append(R[0, 1:])
    return torch.stack(out), logits.detach()
