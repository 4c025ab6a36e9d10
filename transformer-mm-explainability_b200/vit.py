"""Single-modality ViT relevancy (SURVEY.md §8a row a14): ``generate_relevance(model, input, index=None)`` with the
notebook's signature (Transformer_MM_explainability_ViT.ipynb:1181-1201) over the libmmx kernels.

``ViTEngine`` takes a timm-style ``vit_base_patch16_224`` state_dict (the architecture of
``baselines/ViT/ViT_new.py`` in hila-chefer/Transformer-Explainability, which the notebook imports; that file is not
vendored in the reference tree - see oracle/vit_oracle.py for the parity status)."""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional

import torch

from ._lib import lib, check, ptr, current_stream, MmxError
from .nn import Tape, Var, Weight, AttnRecord, ACT_GELU, ATTN_SCALE_SCORES, _f32
from . import rules


class ViTEngine:
    def __init__(self, state_dict: Dict[str, torch.Tensor], heads: int = 12, device=None):
        if not torch.cuda.is_available():
            raise MmxError("mmx_b200 needs a CUDA (sm_90a) device; there is no CPU fallback")
        self.device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        sd = state_dict
        d = self.device
        w = sd["patch_embed.proj.weight"]
        self.dim, self.patch = w.shape[0], w.shape[-1]
        self.tokens = sd["pos_embed"].shape[1]
        self.grid = round((self.tokens - 1) ** 0.5)
        self.image = self.grid * self.patch
        self.heads = heads
        self.depth = len({k.split(".")[1] for k in sd if k.startswith("blocks.")})
        self.patch_w = Weight(w.reshape(self.dim, -1), sd["patch_embed.proj.bias"], d)
        self.cls = _f32(sd["cls_token"].reshape(1, self.dim), d)
        self.pos = _f32(sd["pos_embed"].reshape(self.tokens, self.dim), d)
        self.blocks = []
        for i in range(self.depth):
            p = f"blocks.{i}."
            self.blocks.append(dict(
                n1=(_f32(sd[p + "norm1.weight"], d), _f32(sd[p + "norm1.bias"], d)),
                n2=(_f32(sd[p + "norm2.weight"], d), _f32(sd[p + "norm2.bias"], d)),
                qkv=Weight(sd[p + "attn.qkv.weight"], sd[p + "attn.qkv.bias"], d),
                proj=Weight(sd[p + "attn.proj.weight"], sd[p + "attn.proj.bias"], d),
                fc1=Weight(sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"], d),
                fc2=Weight(sd[p + "mlp.fc2.weight"], sd[p + "mlp.fc2.bias"], d), attn=AttnRecord()))
        self.norm = (_f32(sd["norm.weight"], d), _f32(sd["norm.bias"], d))
        self.head = Weight(sd["head.weight"], sd["head.bias"], d)
        self.logits: Optional[torch.Tensor] = None

    def eval(self):
        return self

    def forward_backward(self, images: torch.Tensor, index=None) -> torch.Tensor:
        """Forward (staging every A_l), one-hot on logits[b, index_b], dgrad-only backward (staging every dA_l)."""
        l = lib()
        with torch.cuda.device(self.device):
            images = _f32(images, self.device)
            B, S, D, H = images.shape[0], self.tokens, self.dim, self.heads
            tape = Tape(self.device)
            G2 = self.grid * self.grid
            patches = torch.empty(B * G2, 3 * self.patch * self.patch, device=self.device)
            check(l.mmx_im2col_patches(ptr(images), ptr(patches), B, self.image, self.patch, current_stream()))
            emb = tape.linear(Var(patches), self.patch_w)                       # conv16x16/16 as a GEMM
            # tokens: [cls | patches] + pos   (glue: row gathers, no gradient needed below the first block)
            x0 = torch.empty(B * S, D, device=self.device)
            x3 = x0.view(B, S, D)
            rows_cls = torch.arange(B, device=self.device, dtype=torch.int32) * S
            pos_rep = self.pos.repeat(B, 1)
            x3[:, 1:, :] = emb.v.view(B, G2, D)                                  # torch view copy = plumbing only
            x3[:, 0, :] = self.cls
            x = tape.add_const(Var(x0), pos_rep)
            scale = float(D // H) ** -0.5
            for blk in self.blocks:
                h = tape.layernorm(x, *blk["n1"], 1e-6)
                qkv = tape.linear(h, blk["qkv"])
                q, k, v = (Var(qkv.v[:, j * D:(j + 1) * D]) for j in range(3))
                o = tape.attention(q, k, v, B, H, S, S, scale, ATTN_SCALE_SCORES, None, blk["attn"])
                self._join_qkv(tape, qkv, q, k, v)
                x = tape.add(x, tape.linear(o, blk["proj"]))
                h = tape.layernorm(x, *blk["n2"], 1e-6)
                x = tape.add(x, tape.linear(tape.linear(h, blk["fc1"], ACT_GELU), blk["fc2"]))
            xn = tape.layernorm(tape.gather_rows(x, rows_cls), *self.norm, 1e-6)
            logits = tape.linear(xn, self.head)
            self.logits = logits.v
            self.saved = dict(B=B, xn=xn)
            idx = logits.v.argmax(-1) if index is None else torch.as_tensor(index, device=self.device).reshape(B)
            one_hot = torch.zeros_like(logits.v)
            one_hot.scatter_(1, idx.long().reshape(B, 1), 1.0)                   # ipynb:1186-1190
            tape.seed(logits, one_hot, B)
            tape.backward()
        return self.logits

    @staticmethod
    def _join_qkv(tape: Tape, qkv: Var, q: Var, k: Var, v: Var):
        """q, k, v are column slices of one packed projection: stitch their gradients back (recorded BEFORE the
        attention backward in program order, so it runs AFTER it on the reversed tape)."""
        def bwd():
            if q.g is None:
                return
            D = q.cols
            g = torch.empty_like(qkv.v)
            g[:, :D], g[:, D:2 * D], g[:, 2 * D:] = q.g, k.g, v.g
            tape.accumulate(qkv, g)
        # insert before the attention op's backward entry so that it executes after it in reverse order
        tape.ops.insert(len(tape.ops) - 1, bwd)


def generate_relevance(model: ViTEngine, input: torch.Tensor, index=None) -> torch.Tensor:
    """Drop-in for the notebook's ``generate_relevance`` (Transformer_MM_explainability_ViT.ipynb:1181-1201).
    ``input`` [B,3,224,224]; returns ``R[0, 1:]`` - shape [S-1] for a single image (like the reference), else [B, S-1]."""
    if not isinstance(model, ViTEngine):
        raise MmxError("model must be a mmx_b200.ViTEngine")
    model.forward_backward(input, index)
    B, S = input.shape[0], model.tokens
    R = torch.eye(S, device=model.device).repeat(B, 1, 1)
    for blk in model.blocks:
        rec = blk["attn"]
        cam = rules.avg_heads_record(rec, B)                                         # rule 5
        R, _ = rules.self_update(R, cam)                                              # R = R + cam @ R (rule 6)
    out = R[:, 0, 1:]
    return out[0] if B == 1 else out
