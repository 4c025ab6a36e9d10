"""Oracle restatement of the VisualBERT single-stream relevancy path (SURVEY.md §8f item 1).

TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).  Plain PyTorch + autograd on CPU over a ``state_dict`` with the
key names of ``VisualBERTForClassification`` (VisualBERT/mmf/models/visual_bert.py:263-396), i.e.
``bert.embeddings.*``, ``bert.encoder.layer.N.*``, ``classifier.0.*`` (BertPredictionHeadTransform), ``classifier.1.*``.
Reference lines followed:
  * BertVisioLinguisticEmbeddings  VisualBERT/mmf/modules/embeddings.py:305-451 (plain strategy: visual position id 0)
  * VisualBERTBase.forward  visual_bert.py:64-135 ((1 - mask) * -10000 additive mask)
  * BertSelfAttention.forward  VisualBERT/mmf/models/transformers/backends/BERT_ours.py:292-345 (scores / sqrt(d) after
    q k^T, save_attn before dropout), BertSelfOutput :397-411, BertIntermediate :422-433 (exact GELU), BertOutput
    :444-458, BertLayer :475-506, BertPredictionHeadTransform :517-531
  * VQA pooling: the second-to-last text token, visual_bert.py:380-394
  * SelfAttentionGenerator  VisualBERT/mmf/models/transformers/backends/ExplanationGenerator.py:20-214
    (generate_ours :67-107, generate_raw_attn :154-167, generate_rollout :169-185 with the NON-normalising
    compute_rollout_attention :5-18, generate_attn_gradcam :187-214)
Pinned against the unmodified reference classes run on CPU (oracle/ref_visualbert.py; tests/golden/visualbert_tiny.npz);
the embeddings module of mmf cannot be imported here (omegaconf / mmf registry), so it is restated in both.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List

import torch
import torch.nn.functional as F


@dataclass(frozen=True)
class VisualBertConfig:
    hidden: int = 768
    heads: int = 12
    intermediate: int = 3072
    layers: int = 12
    vocab: int = 30522
    max_pos: int = 512
    type_vocab: int = 2
    visual_dim: int = 2048
    num_labels: int = 3129


VISUALBERT_BASE = VisualBertConfig()
VISUALBERT_TINY = VisualBertConfig(hidden=64, heads=4, intermediate=96, layers=3, vocab=60, max_pos=24, type_vocab=2,
                                   visual_dim=20, num_labels=13)


def init_state_dict(cfg: VisualBertConfig, seed: int = 0) -> Dict[str, torch.Tensor]:
    g = torch.Generator().manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}
    Hd = cfg.hidden

    def lin(p, o, i):
        sd[p + ".weight"] = torch.randn(o, i, generator=g) * i ** -0.5
        sd[p + ".bias"] = torch.randn(o, generator=g) * 0.02

    def ln(p, d):
        sd[p + ".weight"] = 1 + 0.1 * torch.randn(d, generator=g)
        sd[p + ".bias"] = 0.05 * torch.randn(d, generator=g)

    e = "bert.embeddings."
    for name, n in (("word_embeddings", cfg.vocab), ("position_embeddings", cfg.max_pos), ("token_type_embeddings", cfg.type_vocab),
                    ("token_type_embeddings_visual", cfg.type_vocab), ("position_embeddings_visual", cfg.max_pos)):
        sd[e + name + ".weight"] = torch.randn(n, Hd, generator=g) * 0.5
    ln(e + "LayerNorm", Hd)
    lin(e + "projection", Hd, cfg.visual_dim)
    for i in range(cfg.layers):
        p = f"bert.encoder.layer.{i}."
        for n in ("query", "key", "value"):
            lin(p + "attention.self." + n, Hd, Hd)
        lin(p + "attention.output.dense", Hd, Hd); ln(p + "attention.output.LayerNorm", Hd)
        lin(p + "intermediate.dense", cfg.intermediate, Hd)
        lin(p + "output.dense", Hd, cfg.intermediate); ln(p + "output.LayerNorm", Hd)
    lin("classifier.0.dense", Hd, Hd); ln("classifier.0.LayerNorm", Hd)
    lin("classifier.1", cfg.num_labels, Hd)
    return sd


def synthetic_inputs(cfg: VisualBertConfig, B: int, T: int, V: int, seed: int = 0) -> Dict[str, torch.Tensor]:
    """The fields ``VisualBERT.forward`` hands to the model after removing the text padding (visual_bert.py:579-598)."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(3, cfg.vocab, (B, T), generator=g)
    ids[:, 0] = 1
    ids[:, -1] = 2
    return {"input_ids": ids, "token_type_ids": torch.zeros_like(ids), "input_mask": torch.ones(B, T, dtype=torch.long),
            "visual_embeddings": torch.randn(B, V, cfg.visual_dim, generator=g),
            "visual_embeddings_type": torch.ones(B, V, dtype=torch.long),
            "attention_mask": torch.ones(B, T + V, dtype=torch.long)}


def _lnorm(sd, p, x):
    return F.layer_norm(x, (x.shape[-1],), sd[p + ".weight"], sd[p + ".bias"], 1e-12)


def _lin(sd, p, x):
    return F.linear(x, sd[p + ".weight"], sd[p + ".bias"])


def visualbert_forward(sd, cfg: VisualBertConfig, inp):
    """Returns (scores [B, num_labels], list of staged A [B,H,S,S] per layer)."""
    ids, vis = inp["input_ids"], inp["visual_embeddings"]
    B, T = ids.shape
    V = vis.shape[1]
    H, hd = cfg.heads, cfg.hidden // cfg.heads
    e = "bert.embeddings."
    tt = inp.get("token_type_ids")
    tt = torch.zeros_like(ids) if tt is None else tt
    text = sd[e + "word_embeddings.weight"][ids] + sd[e + "position_embeddings.weight"][torch.arange(T)] \
        + sd[e + "token_type_embeddings.weight"][tt]
    vt = inp.get("visual_embeddings_type")
    vt = torch.zeros(B, V, dtype=torch.long) if vt is None else vt
    v_emb = _lin(sd, e + "projection", vis.to(text.dtype)) + sd[e + "position_embeddings_visual.weight"][torch.zeros(B, V, dtype=torch.long)] \
        + sd[e + "token_type_embeddings_visual.weight"][vt]
    x = _lnorm(sd, e + "LayerNorm", torch.cat((text, v_emb), dim=1))
    am = inp.get("attention_mask")
    mask = None if am is None else ((1.0 - am.to(x.dtype)) * -10000.0)[:, None, None, :]
    S = T + V
    stage: List[torch.Tensor] = []
    for i in range(cfg.layers):
        p = f"bert.encoder.layer.{i}."
        heads = lambda t: t.view(B, S, H, hd).permute(0, 2, 1, 3)
        q, k, v = (heads(_lin(sd, p + "attention.self." + n, x)) for n in ("query", "key", "value"))
        s = torch.matmul(q, k.transpose(-1, -2)) / math.sqrt(hd)
        if mask is not None:
            s = s + mask
        probs = s.softmax(dim=-1)
        stage.append(probs)
        ctx = torch.matmul(probs, v).permute(0, 2, 1, 3).contiguous().view(B, S, H * hd)
        a = _lnorm(sd, p + "attention.output.LayerNorm", _lin(sd, p + "attention.output.dense", ctx) + x)
        x = _lnorm(sd, p + "output.LayerNorm", _lin(sd, p + "output.dense", F.gelu(_lin(sd, p + "intermediate.dense", a))) + a)
    cls_index = inp["input_mask"].sum(1) - 2
    pooled = x[torch.arange(B), cls_index]
    h = _lnorm(sd, "classifier.0.LayerNorm", F.gelu(_lin(sd, "classifier.0.dense", pooled)))
    return _lin(sd, "classifier.1", h), stage


def _prep(sd, inp, dtype):
    sd = {k: v.detach().to(dtype).requires_grad_(True) for k, v in sd.items()}
    inp = dict(inp)
    inp["visual_embeddings"] = inp["visual_embeddings"].to(dtype)
    return sd, inp


def _cls_row(M, inp):
    """M [B,S,S] -> [B,S]: row cls_index with its own column zeroed (EG:95-97)."""
    B = M.shape[0]
    cls_index = inp["input_mask"].sum(1) - 2
    out = M[torch.arange(B), cls_index].clone()
    out[torch.arange(B), cls_index] = 0
    return out


def generate_ours(sd, cfg, inp, index=None, dtype=torch.float32):
    """SelfAttentionGenerator.generate_ours per sample (EG:67-107).  Returns (cls_per_token_score [B,S], scores)."""
    sd, inp = _prep(sd, inp, dtype)
    scores, st = visualbert_forward(sd, cfg, inp)
    B = scores.shape[0]
    idx = scores.argmax(-1) if index is None else torch.as_tensor(index).reshape(-1).expand(B)
    grads = torch.autograd.grad(scores[torch.arange(B), idx].sum(), st)
    S = st[0].shape[-1]
    R = torch.eye(S, dtype=dtype, device=scores.device).repeat(B, 1, 1)
    for A, G in zip(st, grads):
        cam = (G * A.detach()).clamp(min=0).mean(dim=1)
        R = R + torch.bmm(cam, R)
    return _cls_row(R, inp), scores.detach()


def generate_raw_attn(sd, cfg, inp, dtype=torch.float32):
    sd, inp = _prep(sd, inp, dtype)
    _, st = visualbert_forward(sd, cfg, inp)
    return _cls_row(st[-1].detach().mean(dim=1), inp)


def generate_rollout(sd, cfg, inp, start_layer=0, dtype=torch.float32):
    """EG:169-185 with the VisualBERT compute_rollout_attention (EG:5-18): adds I, does NOT row-normalise."""
    sd, inp = _prep(sd, inp, dtype)
    _, st = visualbert_forward(sd, cfg, inp)
    S = st[0].shape[-1]
    mats = [a.detach().mean(dim=1) + torch.eye(S, dtype=dtype) for a in st]
    joint = mats[start_layer]
    for m in mats[start_layer + 1:]:
        joint = m.bmm(joint)
    return _cls_row(joint, inp)


def generate_attn_gradcam(sd, cfg, inp, index=None, dtype=torch.float32):
    """EG:187-214: last layer, grad averaged over each head's plane, min-max normalised."""
    sd, inp = _prep(sd, inp, dtype)
    scores, st = visualbert_forward(sd, cfg, inp)
    B = scores.shape[0]
    idx = scores.argmax(-1) if index is None else torch.as_tensor(index).reshape(-1).expand(B)
    (G,) = torch.autograd.grad(scores[torch.arange(B), idx].sum(), [st[-1]])
    cam = (st[-1].detach() * G.mean(dim=[2, 3], keepdim=True)).mean(1).clamp(min=0)
    mn, mx = cam.amin(dim=(1, 2), keepdim=True), cam.amax(dim=(1, 2), keepdim=True)
    return _cls_row((cam - mn) / (mx - mn), inp)


def _lrp_per_sample(sd, cfg, inp, index, dtype):
    """(grads of the staged A, LRP layers) per sample; the relprop sweep normalises by whole-tensor sums, so one at a time."""
    from . import lrp
    B = inp["input_ids"].shape[0]
    for b in range(B):
        one = {k: v[b:b + 1] for k, v in inp.items()}
        sdg, one = _prep(sd, one, dtype)
        scores, st = visualbert_forward(sdg, cfg, one)
        idx = int(scores.argmax(-1)) if index is None else int(torch.as_tensor(index).reshape(-1).expand(B)[b])
        grads = torch.autograd.grad(scores[0, idx], st)
        with torch.no_grad():
            _, layers = lrp.visualbert_lrp_sweep({k: v.detach() for k, v in sdg.items()}, cfg, one, idx)
        yield one, grads, layers


def generate_transformer_att(sd, cfg, inp, index=None, start_layer=0, dtype=torch.float32):
    """SelfAttentionGenerator.generate_transformer_att (EG:24-66): rule 5 on (grad, LRP relevance of A) per layer, then the
    non-normalising rollout (EG:5-18) from ``start_layer``."""
    out = []
    for one, grads, layers in _lrp_per_sample(sd, cfg, inp, index, dtype):
        S = grads[0].shape[-1]
        mats = [(G[0] * L.attn_cam[0]).clamp(min=0).mean(dim=0).unsqueeze(0) + torch.eye(S, dtype=dtype) for G, L in zip(grads, layers)]
        joint = mats[start_layer]
        for m in mats[start_layer + 1:]:
            joint = m.bmm(joint)
        out.append(_cls_row(joint, one)[0])
    return torch.stack(out)


def generate_partial_lrp(sd, cfg, inp, index=None, dtype=torch.float32):
    """SelfAttentionGenerator.generate_partial_lrp (EG:109-131): head mean of the last layer's LRP relevance, min-max."""
    out = []
    for one, _, layers in _lrp_per_sample(sd, cfg, inp, index, dtype):
        cam = layers[-1].attn_cam[0].mean(dim=0).unsqueeze(0)
        cam = (cam - cam.min()) / (cam.max() - cam.min())
        out.append(_cls_row(cam, one)[0])
    return torch.stack(out)


PERT_STEPS = [0, 0.25, 0.5, 0.75, 0.8, 0.85, 0.9, 0.95, 1]      # VisualBERT/mmf/trainers/core/evaluation_loop.py:96 (text)
PERT_STEPS_IMAGE = [0, 0.5, 0.75, 0.95, 0.96, 0.97, 0.98, 0.99, 1]   # :94 (image: the 100 boxes are thinned more aggressively)


def perturbation_image(sd, cfg, inp, method_cam, is_positive_pert=False, steps=PERT_STEPS_IMAGE):
    """evaluation_loop.py:105-124 on one sample: per step keep the top ``int((1-step)*V)`` visual tokens (gathered in topk
    order) and re-run the model; returns the scores per step.  PARITY UNPINNED for the loop itself (the mmf trainer and
    dataset cannot be imported here); the model it calls is pinned through the VisualBERT goldens."""
    cam = method_cam.reshape(-1) * (-1 if is_positive_pert else 1)
    T = int(inp["input_mask"].sum())
    bbox_scores = cam[T:]
    out = []
    with torch.no_grad():
        for step in steps:
            k = int((1 - step) * bbox_scores.numel())
            _, top = bbox_scores.topk(k=k, dim=-1)
            cur = dict(inp)
            cur["visual_embeddings"] = inp["visual_embeddings"][:, top, :]
            cur["visual_embeddings_type"] = inp["visual_embeddings_type"][:, top]
            cur["attention_mask"] = torch.cat((inp["attention_mask"][:, :T], inp["attention_mask"][:, T:][:, top]), dim=1)
            out.append(visualbert_forward(sd, cfg, cur)[0][0])
    return torch.stack(out)


def perturbation_text(sd, cfg, inp, method_cam, is_positive_pert=False, steps=PERT_STEPS):
    """evaluation_loop.py:126-160: tokens 1..cls_index-1 ranked; token 0, cls_index and cls_index+1 always kept, order kept."""
    cam = method_cam.reshape(-1) * (-1 if is_positive_pert else 1)
    T = int(inp["input_mask"].sum())
    cls_index = T - 2
    text_scores = cam[1:cls_index]
    out = []
    with torch.no_grad():
        for step in steps:
            k = int((1 - step) * text_scores.numel())
            _, top = text_scores.topk(k=k, dim=-1)
            idx = sorted([0, cls_index, cls_index + 1] + [int(t) + 1 for t in top])
            cur = dict(inp)
            cur["input_ids"] = inp["input_ids"][:, idx]
            cur["token_type_ids"] = inp["token_type_ids"][:, idx]
            cur["input_mask"] = inp["input_mask"][:, :len(idx)]
            cur["attention_mask"] = torch.cat((inp["attention_mask"][:, :len(idx)], inp["attention_mask"][:, T:]), dim=1)
            out.append(visualbert_forward(sd, cfg, cur)[0][0])
    return torch.stack(out)
