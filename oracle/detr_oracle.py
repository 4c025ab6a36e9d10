"""Oracle restatement of the DETR encoder-decoder relevancy path (SURVEY.md §8a rows a10, a11).

TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).  Plain PyTorch + autograd on CPU over a ``state_dict`` with the
reference's key names.  Reference lines followed:
  * MultiheadAttention.forward ...... DETR/modules/layers.py:728-768 (separate q/k/v Linear, q*scaling, einsum scores,
                                      softmax, save_attn + register_hook; key_padding_mask / attn_mask IGNORED)
  * TransformerEncoderLayer ......... DETR/models/transformer.py:230-254 (post-norm; pos added to q and k only)
  * TransformerDecoderLayer ......... DETR/models/transformer.py:372-408
  * Transformer.forward ............. DETR/models/transformer.py:51-66; decoder norm :153-155
  * Generator.generate_ours ......... DETR/modules/ExplanationGenerator.py:142-195 (+ handlers :110-140)
The model here is the transformer + class head on given backbone features (``src`` already through input_proj), as in
the survey-time shim (SURVEY.md §8c): the ResNet-50 backbone sits below every attention layer and needs no gradient.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List

import torch
import torch.nn.functional as F

from . import rules as R_


# configs, random-init weights and synthetic inputs are shared with bench.py: they live in mmx_b200/synthetic.py
from mmx_b200.synthetic import (DetrConfig, DETR_R50, DETR_TINY, detr_init_state_dict as init_state_dict,  # noqa: E402,F401
                                detr_sine_position_embedding as sine_position_embedding, detr_synthetic_inputs as synthetic_inputs)


def _mha(sd, p, query, key, value, H, stage: List[torch.Tensor]):
    """[T,B,D] x [S,B,D] -> [T,B,D]; DETR/modules/layers.py:728-768."""
    T, B, D = query.shape
    hd = D // H
    q = F.linear(query, sd[p + "q_proj.weight"], sd[p + "q_proj.bias"]) * (float(hd) ** -0.5)
    k = F.linear(key, sd[p + "k_proj.weight"], sd[p + "k_proj.bias"])
    v = F.linear(value, sd[p + "v_proj.weight"], sd[p + "v_proj.bias"])
    q = q.contiguous().view(T, B * H, hd).transpose(0, 1)
    k = k.contiguous().view(-1, B * H, hd).transpose(0, 1)
    v = v.contiguous().view(-1, B * H, hd).transpose(0, 1)
    w = torch.einsum('bid,bjd->bij', q, k).softmax(dim=-1)
    stage.append(w)
    o = torch.einsum('bij,bjd->bid', w, v).transpose(0, 1).contiguous().view(T, B, D)
    return F.linear(o, sd[p + "out_proj.weight"], sd[p + "out_proj.bias"])


def _ln(sd, p, x):
    return F.layer_norm(x, (x.shape[-1],), sd[p + ".weight"], sd[p + ".bias"])


def detr_forward(sd, cfg: DetrConfig, src, pos):
    """src, pos: [B,d,h,w].  Returns (pred_logits [B,Q,C+1], enc self A list, dec self A list, dec cross A list),
    each A of shape [B*H, T, S] like the reference's saved attn."""
    B, d, h, w = src.shape
    x = src.flatten(2).permute(2, 0, 1)
    pe = pos.flatten(2).permute(2, 0, 1)
    qe = sd["query_embed.weight"].unsqueeze(1).repeat(1, B, 1)
    A_e, A_ds, A_dc = [], [], []
    for i in range(cfg.enc_layers):
        p = f"transformer.encoder.layers.{i}."
        qk = x + pe
        x = _ln(sd, p + "norm1", x + _mha(sd, p + "self_attn.", qk, qk, x, cfg.nhead, A_e))
        ff = F.linear(F.relu(F.linear(x, sd[p + "linear1.weight"], sd[p + "linear1.bias"])), sd[p + "linear2.weight"],
                      sd[p + "linear2.bias"])
        x = _ln(sd, p + "norm2", x + ff)
    memory = x
    t = torch.zeros_like(qe)
    for i in range(cfg.dec_layers):
        p = f"transformer.decoder.layers.{i}."
        qk = t + qe
        t = _ln(sd, p + "norm1", t + _mha(sd, p + "self_attn.", qk, qk, t, cfg.nhead, A_ds))
        t = _ln(sd, p + "norm2", t + _mha(sd, p + "multihead_attn.", t + qe, memory + pe, memory, cfg.nhead, A_dc))
        ff = F.linear(F.relu(F.linear(t, sd[p + "linear1.weight"], sd[p + "linear1.bias"])), sd[p + "linear2.weight"],
                      sd[p + "linear2.bias"])
        t = _ln(sd, p + "norm3", t + ff)
    hs = _ln(sd, "transformer.decoder.norm", t).transpose(0, 1)                     # [B,Q,d]
    return F.linear(hs, sd["class_embed.weight"], sd["class_embed.bias"]), A_e, A_ds, A_dc


def generate_ours(sd, cfg: DetrConfig, src, pos, target_index, index=None, normalize_self_attention=True,
                  apply_self_in_rule_10=True, dtype=torch.float32, return_stages=False):
    """Generator.generate_ours(use_lrp=False) per sample: ``target_index`` [B] query per image, ``index`` [B] class or
    None (argmax over the real classes, ExplanationGenerator.py:151-152).  Returns R_q_i[target] as [B, S_i]."""
    # parameters require grad like the reference's nn.Parameters: the first decoder self-attention sees only
    # query_embed (tgt = 0), and its A must still be a differentiable node to receive dA
    sd = {k: v.detach().to(dtype).requires_grad_(True) for k, v in sd.items()}
    src = src.to(dtype).requires_grad_(True)
    pos = pos.to(dtype)
    B = src.shape[0]
    H = cfg.nhead
    logits, A_e, A_ds, A_dc = detr_forward(sd, cfg, src, pos)
    tq = torch.as_tensor(target_index).reshape(B)
    cls = logits[torch.arange(B), tq, :-1].argmax(-1) if index is None else torch.as_tensor(index).reshape(B)
    y = logits[torch.arange(B), tq, cls].sum()
    grads = torch.autograd.grad(y, A_e + A_ds + A_dc)
    ne, nd = len(A_e), len(A_ds)
    G_e, G_ds, G_dc = grads[:ne], grads[ne:ne + nd], grads[ne + nd:]
    S, Q = A_e[0].shape[-1], A_ds[0].shape[-1]
    out = []
    dev = src.device
    for b in range(B):
        sl = slice(b * H, (b + 1) * H)
        R_ii, R_qq = torch.eye(S, dtype=dtype, device=dev), torch.eye(Q, dtype=dtype, device=dev)
        R_qi = torch.zeros(Q, S, dtype=dtype, device=dev)
        for A, G in zip(A_e, G_e):                                                   # :110-118
            R_ii = R_ii + R_.avg_heads(A[sl].detach(), G[sl]) @ R_ii
        for A, G, Ac, Gc in zip(A_ds, G_ds, A_dc, G_dc):
            cam = R_.avg_heads(A[sl].detach(), G[sl])                                # :120-129
            a_qq, a_qi = R_.apply_self_attention_rules(R_qq, R_qi, cam)
            R_qq, R_qi = R_qq + a_qq, R_qi + a_qi
            cam_qi = R_.avg_heads(Ac[sl].detach(), Gc[sl])                           # :131-140
            R_qi = R_qi + R_.apply_mm_attention_rules_detr(R_qq, R_ii, cam_qi, normalize_self_attention,
                                                           apply_self_in_rule_10)
        out.append(R_qi[tq[b]])
    res = torch.stack(out)
    if return_stages:
        return res, dict(logits=logits.detach(), A_e=[a.detach() for a in A_e], G_e=list(G_e),
                         A_dc=[a.detach() for a in A_dc], G_dc=list(G_dc), cls=cls)
    return res


def generate_ours_abl(sd, cfg: DetrConfig, src, pos, target_index, index=None, normalize_self_attention=False,
                      apply_self_in_rule_10=True, dtype=torch.float32):
    """GeneratorAlbationNoAgg.generate_ours_abl(use_lrp=False) per sample (DETR/modules/ExplanationGenerator.py:306-403):
    the same sweep as generate_ours with every ``+=`` replaced by ``=``.  Returns R_q_i[target] as [B, S_i]."""
    sd = {k: v.detach().to(dtype).requires_grad_(True) for k, v in sd.items()}
    src = src.to(dtype).requires_grad_(True)
    pos = pos.to(dtype)
    B, H = src.shape[0], cfg.nhead
    logits, A_e, A_ds, A_dc = detr_forward(sd, cfg, src, pos)
    tq = torch.as_tensor(target_index).reshape(B)
    cls = logits[torch.arange(B), tq, :-1].argmax(-1) if index is None else torch.as_tensor(index).reshape(B)
    grads = torch.autograd.grad(logits[torch.arange(B), tq, cls].sum(), A_e + A_ds + A_dc)
    ne, nd = len(A_e), len(A_ds)
    G_e, G_ds, G_dc = grads[:ne], grads[ne:ne + nd], grads[ne + nd:]
    S, Q = A_e[0].shape[-1], A_ds[0].shape[-1]
    out = []
    for b in range(B):
        sl = slice(b * H, (b + 1) * H)
        R_ii, R_qq, R_qi = torch.eye(S, dtype=dtype), torch.eye(Q, dtype=dtype), torch.zeros(Q, S, dtype=dtype)
        for A, G in zip(A_e, G_e):                                                   # :314-322
            R_ii = R_.avg_heads(A[sl].detach(), G[sl]) @ R_ii
        for A, G, Ac, Gc in zip(A_ds, G_ds, A_dc, G_dc):
            R_qq, R_qi = R_.apply_self_attention_rules(R_qq, R_qi, R_.avg_heads(A[sl].detach(), G[sl]))   # :324-333
            R_qi = R_.apply_mm_attention_rules_detr(R_qq, R_ii, R_.avg_heads(Ac[sl].detach(), Gc[sl]),    # :335-344
                                                    normalize_self_attention, apply_self_in_rule_10)
        out.append(R_qi[tq[b]])
    return torch.stack(out)


def generate_ours_lrp(sd, cfg: DetrConfig, src, pos, target_index, index=None, normalize_self_attention=True,
                      apply_self_in_rule_10=True, dtype=torch.float32):
    """Generator.generate_ours(use_lrp=True) per sample (DETR/modules/ExplanationGenerator.py:142-195 with the
    ``use_lrp`` branches :112-115,:122-125,:132-135): rule 5 takes the LRP relevance of A (oracle/lrp.py) instead of A."""
    from . import lrp
    B = src.shape[0]
    tq = torch.as_tensor(target_index).reshape(B)
    out = []
    for b in range(B):
        sdg = {k: v.detach().to(dtype).requires_grad_(True) for k, v in sd.items()}
        s_b = src[b:b + 1].to(dtype).requires_grad_(True)
        p_b = pos[b:b + 1].to(dtype)
        logits, A_e, A_ds, A_dc = detr_forward(sdg, cfg, s_b, p_b)
        cls = logits[0, tq[b], :-1].argmax(-1) if index is None else torch.as_tensor(index).reshape(B)[b]
        grads = torch.autograd.grad(logits[0, tq[b], cls], A_e + A_ds + A_dc)
        ne, nd = len(A_e), len(A_ds)
        G_e, G_ds, G_dc = grads[:ne], grads[ne:ne + nd], grads[ne + nd:]
        with torch.no_grad():
            sdd = {k: v.detach() for k, v in sdg.items()}
            _, enc, dec = lrp.detr_lrp_sweep(sdd, cfg, s_b.detach(), p_b, int(tq[b]), int(cls))
            S, Q = A_e[0].shape[-1], A_ds[0].shape[-1]
            R_ii, R_qq, R_qi = torch.eye(S, dtype=dtype), torch.eye(Q, dtype=dtype), torch.zeros(Q, S, dtype=dtype)
            for layer, G in zip(enc, G_e):
                R_ii = R_ii + R_.avg_heads(layer.attn.attn_cam, G) @ R_ii
            for layer, G, Gc in zip(dec, G_ds, G_dc):
                a_qq, a_qi = R_.apply_self_attention_rules(R_qq, R_qi, R_.avg_heads(layer.self_attn.attn_cam, G))
                R_qq, R_qi = R_qq + a_qq, R_qi + a_qi
                R_qi = R_qi + R_.apply_mm_attention_rules_detr(R_qq, R_ii, R_.avg_heads(layer.cross.attn_cam, Gc),
                                                               normalize_self_attention, apply_self_in_rule_10)
            out.append(R_qi[tq[b]])
    return torch.stack(out)


def generate_lrp_baseline(sd, cfg: DetrConfig, src, pos, target_index, method: str, dtype=torch.float32):
    """The two LRP-based baselines of the DETR Generator, per sample: ``transformer_att`` = rule 5 on the LAST decoder
    cross-attention (grad, LRP relevance) (DETR/modules/ExplanationGenerator.py:64-108); ``partial_lrp`` = head mean of that
    relevance, min-max normalised (:197-224).  Returns the target query's row [B, S_i]."""
    from . import lrp
    B = src.shape[0]
    tq = torch.as_tensor(target_index).reshape(B)
    out = []
    for b in range(B):
        sdg = {k: v.detach().to(dtype).requires_grad_(True) for k, v in sd.items()}
        s_b, p_b = src[b:b + 1].to(dtype).requires_grad_(True), pos[b:b + 1].to(dtype)
        logits, A_e, A_ds, A_dc = detr_forward(sdg, cfg, s_b, p_b)
        cls = logits[0, tq[b], :-1].argmax(-1)
        (G,) = torch.autograd.grad(logits[0, tq[b], cls], [A_dc[-1]])
        with torch.no_grad():
            _, enc, dec = lrp.detr_lrp_sweep({k: v.detach() for k, v in sdg.items()}, cfg, s_b.detach(), p_b, int(tq[b]), int(cls))
            cam = dec[-1].cross.attn_cam
            if method == "transformer_att":
                R = R_.avg_heads(cam, G)
            else:
                R = cam.mean(dim=0)
                R = (R - R.min()) / (R.max() - R.min())
            out.append(R[tq[b]])
    return torch.stack(out)


def to_checkpoint_format(sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """Official DETR checkpoints pack q/k/v as ``in_proj_weight`` / ``in_proj_bias``; the reference splits them in a
    load hook (DETR/modules/layers.py:711-726).  Adds the packed entries next to the split ones."""
    out = dict(sd)
    for k in list(sd):
        if k.endswith("q_proj.weight"):
            p = k[:-len("q_proj.weight")]
            out[p + "in_proj_weight"] = torch.cat([sd[p + "q_proj.weight"], sd[p + "k_proj.weight"], sd[p + "v_proj.weight"]])
            out[p + "in_proj_bias"] = torch.cat([sd[p + "q_proj.bias"], sd[p + "k_proj.bias"], sd[p + "v_proj.bias"]])
    return out
