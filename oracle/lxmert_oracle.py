"""Oracle restatement of the LXMERT bi-modal relevancy path (SURVEY.md §8a rows a12, a13).

TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).  Plain PyTorch + autograd on CPU over a ``state_dict`` with the
reference's key names (``lxmert.encoder.layer.0.attention.self.query.weight`` ...).  Reference lines followed
(lxmert/lxmert/src/lxmert_lrp.py unless noted):
  * LxmertEmbeddings.forward :285-310, LxmertVisualFeatureEncoder.forward :758-766
  * LxmertAttention.forward :385-420 (scores / sqrt(d) AFTER q k^T, additive mask, save_attn BEFORE dropout)
  * LxmertAttentionOutput :472-477, LxmertIntermediate :549-552 (exact GELU), LxmertOutput :568-573, LxmertLayer :592-599
  * LxmertXLayer.cross_att :630-655 (the i->t direction runs through a deepcopy of the SAME weights), self_att,
    output_fc, forward :701-733;  LxmertEncoder.forward :793-853;  LxmertPooler :876-884 (tanh);
    LxmertVisualAnswerHead :941-953;  extended masks :1195-1201 ((1 - mask) * -10000)
  * GeneratorOurs.generate_ours  lxmert/lxmert/src/ExplanationGenerator.py:131-211
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List

import torch
import torch.nn.functional as F

from . import rules as R_


# configs, random-init weights and synthetic inputs are shared with bench.py: they live in mmx_b200/synthetic.py
from mmx_b200.synthetic import (LxmertConfig, LXMERT_BASE, LXMERT_TINY, lxmert_init_state_dict as init_state_dict,  # noqa: E402,F401
                                lxmert_synthetic_inputs as synthetic_inputs)


def _lnorm(sd, p, x):
    return F.layer_norm(x, (x.shape[-1],), sd[p + ".weight"], sd[p + ".bias"], 1e-12)


def _lin(sd, p, x):
    return F.linear(x, sd[p + ".weight"], sd[p + ".bias"])


def _att(sd, p, hidden, context, mask, H, stage: List[torch.Tensor]):
    B, T, D = hidden.shape
    hd = D // H

    def heads(x):
        return x.view(B, -1, H, hd).permute(0, 2, 1, 3)
    q, k, v = heads(_lin(sd, p + "query", hidden)), heads(_lin(sd, p + "key", context)), heads(_lin(sd, p + "value", context))
    s = torch.matmul(q, k.transpose(-1, -2)) / math.sqrt(hd)
    if mask is not None:
        s = s + mask
    probs = s.softmax(dim=-1)
    stage.append(probs)
    return torch.matmul(probs, v).permute(0, 2, 1, 3).contiguous().view(B, T, D)


def _att_layer(sd, p, att_name, x, ctx, mask, H, stage):
    o = _att(sd, p + att_name + ".", x, ctx, mask, H, stage)
    return _lnorm(sd, p + "output.LayerNorm", _lin(sd, p + "output.dense", o) + x)


def _ffn(sd, pi, po, x):
    return _lnorm(sd, po + "LayerNorm", _lin(sd, po + "dense", F.gelu(_lin(sd, pi + "dense", x))) + x)


def lxmert_forward(sd, cfg: LxmertConfig, ids, feats, boxes, lang_mask=None, vis_mask=None):
    """Returns (answer logits [B, num_labels], dict of staged A lists: lang, vis, x_lang (t->i), x_vis (i->t),
    x_lang_self, x_vis_self), each A [B,H,T,S]."""
    B, T = ids.shape
    H = cfg.heads
    e = "lxmert.embeddings."
    pos_ids = torch.arange(T)
    emb = sd[e + "token_type_embeddings.weight"][torch.zeros_like(ids)] + sd[e + "position_embeddings.weight"][pos_ids] \
        + sd[e + "word_embeddings.weight"][ids]
    lang = _lnorm(sd, e + "LayerNorm", emb)
    lm = None if lang_mask is None else ((1.0 - lang_mask.to(lang.dtype)) * -10000.0)[:, None, None, :]
    vm = None if vis_mask is None else ((1.0 - vis_mask.to(lang.dtype)) * -10000.0)[:, None, None, :]
    v = "lxmert.encoder.visn_fc."
    vis = (_lnorm(sd, v + "visn_layer_norm", _lin(sd, v + "visn_fc", feats)) + _lnorm(sd, v + "box_layer_norm", _lin(sd, v + "box_fc", boxes))) / 2
    st = {k: [] for k in ("lang", "vis", "x_lang", "x_vis", "x_lang_self", "x_vis_self")}
    for i in range(cfg.l_layers):
        p = f"lxmert.encoder.layer.{i}."
        lang = _ffn(sd, p + "intermediate.", p + "output.", _att_layer(sd, p + "attention.", "self", lang, lang, lm, H, st["lang"]))
    for i in range(cfg.r_layers):
        p = f"lxmert.encoder.r_layers.{i}."
        vis = _ffn(sd, p + "intermediate.", p + "output.", _att_layer(sd, p + "attention.", "self", vis, vis, vm, H, st["vis"]))
    for i in range(cfg.x_layers):
        p = f"lxmert.encoder.x_layers.{i}."
        l2 = _att_layer(sd, p + "visual_attention.", "att", lang, vis, vm, H, st["x_lang"])
        v2 = _att_layer(sd, p + "visual_attention.", "att", vis, lang, lm, H, st["x_vis"])     # the deepcopy: same weights
        l3 = _att_layer(sd, p + "lang_self_att.", "self", l2, l2, lm, H, st["x_lang_self"])
        v3 = _att_layer(sd, p + "visn_self_att.", "self", v2, v2, vm, H, st["x_vis_self"])
        lang, vis = _ffn(sd, p + "lang_inter.", p + "lang_output.", l3), _ffn(sd, p + "visn_inter.", p + "visn_output.", v3)
    pooled = torch.tanh(_lin(sd, "lxmert.pooler.dense", lang[:, 0]))
    h = _lin(sd, "answer_head.logit_fc.0", pooled)
    h = F.layer_norm(F.gelu(h), (h.shape[-1],), sd["answer_head.logit_fc.2.weight"], sd["answer_head.logit_fc.2.bias"], 1e-12)
    return _lin(sd, "answer_head.logit_fc.3", h), st


def generate_ours(sd, cfg: LxmertConfig, ids, feats, boxes, index=None, normalize_self_attention=True,
                  apply_self_in_rule_10=True, dtype=torch.float32, lang_mask=None, vis_mask=None):
    """GeneratorOurs.generate_ours(use_lrp=False) per sample, with LxmertForQuestionAnswering's attention_mask /
    visual_attention_mask as ``lang_mask`` / ``vis_mask``.  Returns (R_t_t [B,T,T], R_t_i [B,T,I], logits)."""
    sd = {k: v.detach().to(dtype).requires_grad_(True) for k, v in sd.items()}
    feats, boxes = feats.to(dtype), boxes.to(dtype)
    logits, st = lxmert_forward(sd, cfg, ids, feats, boxes, lang_mask, vis_mask)
    B, T = ids.shape
    I = feats.shape[1]
    idx = logits.argmax(-1) if index is None else torch.as_tensor(index).reshape(B)
    y = logits[torch.arange(B), idx].sum()
    names = ["lang", "vis", "x_lang", "x_vis", "x_lang_self", "x_vis_self"]
    flat = [a for n in names for a in st[n]]
    grads = torch.autograd.grad(y, flat, allow_unused=True)
    G, k = {}, 0
    for n in names:
        G[n] = grads[k:k + len(st[n])]
        k += len(st[n])
    nx = cfg.x_layers
    norm, s10 = normalize_self_attention, apply_self_in_rule_10
    Rtt, Rti = [], []
    dev = feats.device
    for b in range(B):
        cam = lambda n, i: R_.avg_heads(st[n][i][b].detach(), G[n][i][b])
        R_tt, R_ii = torch.eye(T, dtype=dtype, device=dev), torch.eye(I, dtype=dtype, device=dev)
        R_ti, R_it = torch.zeros(T, I, dtype=dtype, device=dev), torch.zeros(I, T, dtype=dtype, device=dev)
        for i in range(cfg.l_layers):                                               # EG:61-71
            a, c = R_.apply_self_attention_rules(R_tt, R_ti, cam("lang", i)); R_tt, R_ti = R_tt + a, R_ti + c
        for i in range(cfg.r_layers):                                               # EG:73-83
            a, c = R_.apply_self_attention_rules(R_ii, R_it, cam("vis", i)); R_ii, R_it = R_ii + a, R_it + c
        for i in range(nx):
            last = i == nx - 1
            ti_add, tt_add = R_.apply_mm_attention_rules_lxmert(R_tt, R_ii, R_it, cam("x_lang", i), norm, s10)   # EG:107-116
            if not last:
                it_add, ii_add = R_.apply_mm_attention_rules_lxmert(R_ii, R_tt, R_ti, cam("x_vis", i), norm, s10)  # EG:118-129
            R_ti, R_tt = R_ti + ti_add, R_tt + tt_add
            if not last:
                R_it, R_ii = R_it + it_add, R_ii + ii_add
            a, c = R_.apply_self_attention_rules(R_tt, R_ti, cam("x_lang_self", i)); R_tt, R_ti = R_tt + a, R_ti + c
            if not last:
                a, c = R_.apply_self_attention_rules(R_ii, R_it, cam("x_vis_self", i)); R_ii, R_it = R_ii + a, R_it + c
        R_tt[0, 0] = 0                                                               # EG:210
        Rtt.append(R_tt); Rti.append(R_ti)
    return torch.stack(Rtt), torch.stack(Rti), logits.detach()


def generate_ours_no_agg(sd, cfg: LxmertConfig, ids, feats, boxes, index=None, normalize_self_attention=True,
                         dtype=torch.float32):
    """GeneratorOursAblationNoAggregation.generate_ours_no_agg(use_lrp=False) per sample
    (lxmert/lxmert/src/ExplanationGenerator.py:215-365): every update replaces the relevancy.  Returns
    (R_t_t [B,T,T], R_t_i [B,T,I])."""
    sd = {k: v.detach().to(dtype).requires_grad_(True) for k, v in sd.items()}
    feats, boxes = feats.to(dtype), boxes.to(dtype)
    logits, st = lxmert_forward(sd, cfg, ids, feats, boxes)
    B, T = ids.shape
    I = feats.shape[1]
    idx = logits.argmax(-1) if index is None else torch.as_tensor(index).reshape(B)
    names = ["lang", "vis", "x_lang", "x_vis", "x_lang_self", "x_vis_self"]
    flat = [a for n in names for a in st[n]]
    grads = torch.autograd.grad(logits[torch.arange(B), idx].sum(), flat, allow_unused=True)
    G, k = {}, 0
    for n in names:
        G[n] = grads[k:k + len(st[n])]
        k += len(st[n])
    nx, norm = cfg.x_layers, normalize_self_attention
    Rtt, Rti = [], []
    for b in range(B):
        cam = lambda n, i: R_.avg_heads(st[n][i][b].detach(), G[n][i][b])
        R_tt, R_ii = torch.eye(T, dtype=dtype), torch.eye(I, dtype=dtype)
        R_ti, R_it = torch.zeros(T, I, dtype=dtype), torch.zeros(I, T, dtype=dtype)
        for i in range(cfg.l_layers):
            R_tt, R_ti = R_.apply_self_attention_rules(R_tt, R_ti, cam("lang", i))
        for i in range(cfg.r_layers):
            R_ii, R_it = R_.apply_self_attention_rules(R_ii, R_it, cam("vis", i))
        for i in range(nx - 1):                                                       # EG:330-350
            ti, tt = R_.apply_mm_attention_rules_lxmert(R_tt, R_ii, R_it, cam("x_lang", i), norm)
            it, ii = R_.apply_mm_attention_rules_lxmert(R_ii, R_tt, R_ti, cam("x_vis", i), norm)
            R_ti, R_tt, R_it, R_ii = ti, tt, it, ii
            R_tt, R_ti = R_.apply_self_attention_rules(R_tt, R_ti, cam("x_lang_self", i))
            R_ii, R_it = R_.apply_self_attention_rules(R_ii, R_it, cam("x_vis_self", i))
        R_ti, R_tt = R_.apply_mm_attention_rules_lxmert(R_tt, R_ii, R_it, cam("x_lang", nx - 1), norm)   # EG:353-358
        R_tt, R_ti = R_.apply_self_attention_rules(R_tt, R_ti, cam("x_lang_self", nx - 1))
        R_tt[0, 0] = 0
        Rtt.append(R_tt); Rti.append(R_ti)
    return torch.stack(Rtt), torch.stack(Rti)


def generate_ours_lrp(sd, cfg: LxmertConfig, ids, feats, boxes, index=None, normalize_self_attention=True,
                      apply_self_in_rule_10=True, dtype=torch.float32):
    """GeneratorOurs.generate_ours(use_lrp=True) per sample: rule 5 takes the LRP relevance of A (oracle/lrp.py) in place
    of A (lxmert/lxmert/src/ExplanationGenerator.py:64-66,76-78,...).  Returns (R_t_t [B,T,T], R_t_i [B,T,I])."""
    from . import lrp
    B, T = ids.shape
    I = feats.shape[1]
    nx = cfg.x_layers
    norm, s10 = normalize_self_attention, apply_self_in_rule_10
    Rtt, Rti = [], []
    for b in range(B):
        sdg = {k: v.detach().to(dtype).requires_grad_(True) for k, v in sd.items()}
        f_b, x_b = feats[b:b + 1].to(dtype), boxes[b:b + 1].to(dtype)
        logits, st = lxmert_forward(sdg, cfg, ids[b:b + 1], f_b, x_b)
        idx = int(logits.argmax(-1)) if index is None else int(torch.as_tensor(index).reshape(B)[b])
        names = ["lang", "vis", "x_lang", "x_vis", "x_lang_self", "x_vis_self"]
        flat = [a for n in names for a in st[n]]
        grads = torch.autograd.grad(logits[0, idx], flat, allow_unused=True)
        G, k = {}, 0
        for n in names:
            G[n] = grads[k:k + len(st[n])]
            k += len(st[n])
        with torch.no_grad():
            _, layers = lrp.lxmert_lrp_sweep({k_: v.detach() for k_, v in sdg.items()}, cfg, ids[b:b + 1], f_b, x_b, idx)
            cams = {"lang": [l.att.att.attn_cam for l in layers["lang"]], "vis": [l.att.att.attn_cam for l in layers["vis"]],
                    "x_lang": [l.cross.att.attn_cam for l in layers["x"]], "x_vis": [l.cross_copy.att.attn_cam for l in layers["x"]],
                    "x_lang_self": [l.lang_self.att.attn_cam for l in layers["x"]],
                    "x_vis_self": [l.visn_self.att.attn_cam for l in layers["x"]]}
            cam = lambda n, i: R_.avg_heads(cams[n][i][0], G[n][i][0])
            R_tt, R_ii = torch.eye(T, dtype=dtype), torch.eye(I, dtype=dtype)
            R_ti, R_it = torch.zeros(T, I, dtype=dtype), torch.zeros(I, T, dtype=dtype)
            for i in range(cfg.l_layers):
                a, c = R_.apply_self_attention_rules(R_tt, R_ti, cam("lang", i)); R_tt, R_ti = R_tt + a, R_ti + c
            for i in range(cfg.r_layers):
                a, c = R_.apply_self_attention_rules(R_ii, R_it, cam("vis", i)); R_ii, R_it = R_ii + a, R_it + c
            for i in range(nx):
                last = i == nx - 1
                ti_add, tt_add = R_.apply_mm_attention_rules_lxmert(R_tt, R_ii, R_it, cam("x_lang", i), norm, s10)
                if not last:
                    it_add, ii_add = R_.apply_mm_attention_rules_lxmert(R_ii, R_tt, R_ti, cam("x_vis", i), norm, s10)
                R_ti, R_tt = R_ti + ti_add, R_tt + tt_add
                if not last:
                    R_it, R_ii = R_it + it_add, R_ii + ii_add
                a, c = R_.apply_self_attention_rules(R_tt, R_ti, cam("x_lang_self", i)); R_tt, R_ti = R_tt + a, R_ti + c
                if not last:
                    a, c = R_.apply_self_attention_rules(R_ii, R_it, cam("x_vis_self", i)); R_ii, R_it = R_ii + a, R_it + c
            R_tt[0, 0] = 0
        Rtt.append(R_tt); Rti.append(R_ti)
    return torch.stack(Rtt), torch.stack(Rti)


def generate_lrp_baseline(sd, cfg: LxmertConfig, ids, feats, boxes, method: str, index=None, dtype=torch.float32):
    """GeneratorBaselines.generate_transformer_attr (lxmert/lxmert/src/ExplanationGenerator.py:373-460: rule 5 + rule 6
    with the LRP relevance, self-attention layers only, R_t_i = the last cross layer's cam) and generate_partial_lrp
    (:462-507: head means of the last layer's relevances, min-max normalised), per sample."""
    from . import lrp
    B, T = ids.shape
    I = feats.shape[1]
    Rtt, Rti = [], []
    for b in range(B):
        sdg = {k: v.detach().to(dtype).requires_grad_(True) for k, v in sd.items()}
        f_b, x_b = feats[b:b + 1].to(dtype), boxes[b:b + 1].to(dtype)
        logits, st = lxmert_forward(sdg, cfg, ids[b:b + 1], f_b, x_b)
        idx = int(logits.argmax(-1)) if index is None else int(torch.as_tensor(index).reshape(B)[b])
        names = ["lang", "vis", "x_lang", "x_vis", "x_lang_self", "x_vis_self"]
        flat = [a for n in names for a in st[n]]
        grads = torch.autograd.grad(logits[0, idx], flat, allow_unused=True)
        G, k = {}, 0
        for n in names:
            G[n] = grads[k:k + len(st[n])]
            k += len(st[n])
        with torch.no_grad():
            _, layers = lrp.lxmert_lrp_sweep({k_: v.detach() for k_, v in sdg.items()}, cfg, ids[b:b + 1], f_b, x_b, idx)
            last = layers["x"][-1]
            if method == "partial_lrp":
                R_ti = last.cross.att.attn_cam[0].mean(dim=0)
                R_tt = last.lang_self.att.attn_cam[0].mean(dim=0)
                R_tt = (R_tt - R_tt.min()) / (R_tt.max() - R_tt.min())
                R_ti = (R_ti - R_ti.min()) / (R_ti.max() - R_ti.min())
            else:
                R_tt, R_ii = torch.eye(T, dtype=dtype), torch.eye(I, dtype=dtype)
                for i, l in enumerate(layers["lang"]):
                    R_tt = R_tt + R_.avg_heads(l.att.att.attn_cam[0], G["lang"][i][0]) @ R_tt
                for i, l in enumerate(layers["vis"]):
                    R_ii = R_ii + R_.avg_heads(l.att.att.attn_cam[0], G["vis"][i][0]) @ R_ii
                for i, l in enumerate(layers["x"][:-1]):
                    R_tt = R_tt + R_.avg_heads(l.lang_self.att.attn_cam[0], G["x_lang_self"][i][0]) @ R_tt
                    R_ii = R_ii + R_.avg_heads(l.visn_self.att.attn_cam[0], G["x_vis_self"][i][0]) @ R_ii
                R_ti = R_.avg_heads(last.cross.att.attn_cam[0], G["x_lang"][-1][0])
                R_tt = R_tt + R_.avg_heads(last.lang_self.att.attn_cam[0], G["x_lang_self"][-1][0]) @ R_tt
            R_tt[0, 0] = 0
        Rtt.append(R_tt); Rti.append(R_ti)
    return torch.stack(Rtt), torch.stack(Rti)


PERT_STEPS = [0, 0.25, 0.5, 0.75, 0.8, 0.85, 0.9, 0.95, 1]      # lxmert/lxmert/perturbation.py:42


def perturbation_image(sd, cfg, ids, feats, boxes, cam_image, is_positive_pert=False, pert_steps=PERT_STEPS):
    """ModelPert.perturbation_image (lxmert/lxmert/perturbation.py:85-133) on one item: per step keep the top
    ``int((1 - step) * I)`` boxes of ``cam_image`` (gathered in topk order, like the reference) and re-run the model.
    Returns the answer scores per step [steps, num_labels].  PARITY UNPINNED for the driver loop itself (the reference's
    ModelPert needs the Faster-RCNN extractor, the tokenizer and COCO files); the model it calls is pinned through the
    LXMERT goldens."""
    cam = cam_image.reshape(-1) * (-1 if is_positive_pert else 1)
    out = []
    with torch.no_grad():
        for step in pert_steps:
            k = int((1 - step) * cam.numel())
            _, top = cam.topk(k=k, dim=-1)
            logits, _ = lxmert_forward(sd, cfg, ids, feats[:, top, :], boxes[:, top, :])
            out.append(logits[0])
    return torch.stack(out)


def perturbation_text(sd, cfg, ids, feats, boxes, cam_text, is_positive_pert=False, pert_steps=PERT_STEPS):
    """ModelPert.perturbation_text (perturbation.py:135-194): [CLS] / [SEP] kept, top tokens kept in sentence order."""
    cam = cam_text.reshape(-1) * (-1 if is_positive_pert else 1)
    out = []
    with torch.no_grad():
        for step in pert_steps:
            pure = cam[1:-1]
            k = int((1 - step) * pure.shape[0])
            _, top = pure.topk(k=k, dim=-1)
            idx = sorted([0, cam.shape[0] - 1] + [int(t) + 1 for t in top])
            logits, _ = lxmert_forward(sd, cfg, ids[:, idx], feats, boxes)
            out.append(logits[0])
    return torch.stack(out)
