"""DETR encoder-decoder relevancy (SURVEY.md §8a rows a10, a11): ``Generator(model).generate_ours(...)`` with the
reference signature (DETR/modules/ExplanationGenerator.py:142-195) over the libmmx kernels.

``DetrEngine`` holds the DETR transformer + class head (DETR/models/transformer.py, DETR/models/detr.py:46-77) built
from a reference / official-checkpoint ``state_dict``.  ``img`` takes every form ``DETR.forward`` takes
(DETR/models/detr.py:61-62, DETR/util/misc.py:306-327) when the state dict carries the ResNet backbone
(``backbone.0.body.*``, ``input_proj.*``; see ``mmx_b200.backbone``; ``dilation=True`` for the DC5 checkpoints, whose
stride-16 maps give 2500 - 4200 tokens at COCO sizes):

* a [B, 3, H, W] image tensor (no padding),
* a list of [3, H_i, W_i] images (zero-padded to the largest H and W, the padding masked),
* a ``NestedTensor`` (anything with ``.tensors`` / ``.mask``),

and always the backbone features ``(src, pos)``: ``src`` [B, d_model, h, w] (after ``input_proj``) and ``pos`` the sine
embedding [B or 1, d_model, h, w].  As in the reference the transformer ignores the mask; only ``pos`` sees it.  The
backbone runs forward only: gradients and LRP stop at the transformer input, as in the reference.  ``Generator`` and
``MaskGenerator`` also take the reference ``DETR`` ``nn.Module`` itself (its engine is built once, see ``engine_for``).
"""
from __future__ import annotations

import ctypes as C
import weakref
from typing import Dict, List, Optional

import torch

from ._lib import lib, check, ptr, current_stream, MmxError
from .nn import fp32_gemms, Tape, Var, Weight, AttnRecord, ACT_RELU, ACT_SIGMOID, _f32
from .backbone import DetrBackbone, has_backbone
from . import rules



class _Feats:
    """Transformer input of one call: x = input_proj(src) and pe = pos, both [B*S, d] (row = b*S + y*w + x)."""
    __slots__ = ("x", "pe", "B", "h", "w", "mask")

    def __init__(self, x, pe, B, h, w, mask=None):
        self.x, self.pe, self.B, self.h, self.w, self.mask = x, pe, B, h, w, mask

    def expand(self, K: int) -> "_Feats":
        """the features of one image repeated for K samples (one per query of MaskGenerator)"""
        assert self.B == 1
        return _Feats(self.x.repeat(K, 1), self.pe.repeat(K, 1), K, self.h, self.w,
                      None if self.mask is None else self.mask.expand(K, -1, -1))


def _is_features(img) -> bool:
    """(src [B,d,h,w], pos [B or 1,d,h,w] or [d,h,w]): the feature form the engine has always taken.  Image lists hold
    [3,H,W] tensors, so a 4-D first element never means an image."""
    return (isinstance(img, (tuple, list)) and len(img) == 2 and all(isinstance(t, torch.Tensor) for t in img)
            and img[0].dim() == 4 and img[1].dim() in (3, 4))


def _split_mha(sd, p, device):
    """q/k/v/out projections of one attention module; accepts split keys or the packed ``in_proj_weight`` of the
    official checkpoints (split by the reference in DETR/modules/layers.py:711-726)."""
    if p + "q_proj.weight" in sd:
        q, k, v = ((sd[p + n + ".weight"], sd[p + n + ".bias"]) for n in ("q_proj", "k_proj", "v_proj"))
    else:
        w, b = sd[p + "in_proj_weight"], sd[p + "in_proj_bias"]
        d = w.shape[1]
        q, k, v = ((w[i * d:(i + 1) * d], b[i * d:(i + 1) * d]) for i in range(3))
    return dict(q=Weight(*q, device), k=Weight(*k, device), v=Weight(*v, device),
                o=Weight(sd[p + "out_proj.weight"], sd[p + "out_proj.bias"], device), rec=AttnRecord())


class _Layer:
    pass


class DetrEngine:
    def __init__(self, state_dict: Dict[str, torch.Tensor], nhead: int = 8, device=None, dilation: bool = False):
        if not torch.cuda.is_available():
            raise MmxError("mmx_b200 needs a CUDA (sm_90a) device; there is no CPU fallback")
        self.device = d = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        sd = {(k if k.startswith(("transformer.", "class_embed", "query_embed", "backbone.", "input_proj.", "bbox_embed."))
               else "transformer." + k): v for k, v in state_dict.items()}
        self.nhead = nhead
        n_enc = len({k.split(".")[3] for k in sd if k.startswith("transformer.encoder.layers.")})
        n_dec = len({k.split(".")[3] for k in sd if k.startswith("transformer.decoder.layers.")})
        ln = lambda p: (_f32(sd[p + ".weight"], d), _f32(sd[p + ".bias"], d))
        self.encoder, self.decoder = [], []
        for i in range(n_enc):
            p = f"transformer.encoder.layers.{i}."
            L = _Layer()
            L.self_attn = _split_mha(sd, p + "self_attn.", d)
            L.l1 = Weight(sd[p + "linear1.weight"], sd[p + "linear1.bias"], d)
            L.l2 = Weight(sd[p + "linear2.weight"], sd[p + "linear2.bias"], d)
            L.n1, L.n2 = ln(p + "norm1"), ln(p + "norm2")
            self.encoder.append(L)
        for i in range(n_dec):
            p = f"transformer.decoder.layers.{i}."
            L = _Layer()
            L.self_attn = _split_mha(sd, p + "self_attn.", d)
            L.multihead_attn = _split_mha(sd, p + "multihead_attn.", d)
            L.l1 = Weight(sd[p + "linear1.weight"], sd[p + "linear1.bias"], d)
            L.l2 = Weight(sd[p + "linear2.weight"], sd[p + "linear2.bias"], d)
            L.n1, L.n2, L.n3 = ln(p + "norm1"), ln(p + "norm2"), ln(p + "norm3")
            self.decoder.append(L)
        self.dec_norm = ln("transformer.decoder.norm")
        self.query_embed = _f32(sd["query_embed.weight"], d)
        self.class_embed = Weight(sd["class_embed.weight"], sd["class_embed.bias"], d)
        self.d_model = self.query_embed.shape[1]
        self.queries = self.query_embed.shape[0]
        self.pred_logits: Optional[torch.Tensor] = None
        self.dilation = bool(dilation)
        self.backbone = DetrBackbone(sd, d, dilation=self.dilation) if has_backbone(sd) else None
        if self.backbone is not None and self.backbone.d_model != self.d_model:
            raise MmxError(f"input_proj gives {self.backbone.d_model} channels, the transformer takes {self.d_model}")
        n_box = len({k.split(".")[2] for k in sd if k.startswith("bbox_embed.layers.") and k.endswith(".weight")})
        self.bbox_embed = [Weight(sd[f"bbox_embed.layers.{i}.weight"], sd[f"bbox_embed.layers.{i}.bias"], d)
                           for i in range(n_box)]

    def eval(self):
        return self

    def zero_grad(self):
        return None

    # ------------------------------------------------------------------ inputs
    def features(self, img) -> _Feats:
        """The transformer input for any accepted form of ``img`` (module docstring)."""
        dev = self.device
        if _is_features(img):
            src, pos = img
            B, d, h, w = src.shape
            if d != self.d_model:
                raise MmxError(f"src has {d} channels, the transformer takes d_model = {self.d_model} "
                               "(images go in as a [B,3,H,W] tensor, a list of [3,H,W] tensors or a NestedTensor)")
            x = _f32(src, dev).flatten(2).permute(0, 2, 1).reshape(B * h * w, d).contiguous()
            pe = _f32(pos, dev).expand(B, d, h, w).flatten(2).permute(0, 2, 1).reshape(B * h * w, d).contiguous()
            return _Feats(x, pe, B, h, w)
        if self.backbone is None:
            raise MmxError("this DetrEngine was built without backbone weights (backbone.0.body.*, input_proj.*): pass "
                           "(src, pos) features, or build it from a full DETR state_dict to pass images")
        images, mask = self._images(img)
        with torch.cuda.device(dev):
            x, pe, m, (h, w) = self.backbone(images, mask)
        return _Feats(x, pe, images.shape[0], h, w, m)

    def _images(self, samples):
        """(images [B,3,H,W] fp32 on the device, padding mask [B,H,W] or None) as nested_tensor_from_tensor_list builds
        them (DETR/util/misc.py:306-327)."""
        dev = self.device
        if hasattr(samples, "tensors") and hasattr(samples, "mask"):
            images, mask = samples.tensors, samples.mask
        elif isinstance(samples, torch.Tensor):
            if samples.dim() != 4:
                raise MmxError(f"an image batch is [B, 3, H, W], got {tuple(samples.shape)}")
            images, mask = samples, None
        elif isinstance(samples, (list, tuple)) and samples and all(isinstance(t, torch.Tensor) for t in samples):
            if any(t.dim() != 3 for t in samples):
                raise MmxError("a list of images holds [3, H, W] tensors")
            Hm, Wm = max(t.shape[1] for t in samples), max(t.shape[2] for t in samples)
            images = torch.zeros(len(samples), samples[0].shape[0], Hm, Wm, device=dev, dtype=torch.float32)
            mask = torch.ones(len(samples), Hm, Wm, device=dev, dtype=torch.bool)
            for i, t in enumerate(samples):
                images[i, :, :t.shape[1], :t.shape[2]].copy_(t)
                mask[i, :t.shape[1], :t.shape[2]] = False
            if all(t.shape[1:] == (Hm, Wm) for t in samples):
                mask = None
        else:
            raise MmxError("img must be an image tensor [B,3,H,W], a list of [3,H,W] images, a NestedTensor or (src, pos)")
        if images.dim() != 4 or images.shape[1] != 3:
            raise MmxError(f"images must have 3 channels ([B, 3, H, W]), got {tuple(images.shape)}")
        return _f32(images, dev), mask

    # ------------------------------------------------------------------ DETR.forward
    def forward(self, samples, aux_loss: bool = False):
        """``DETR.forward`` (DETR/models/detr.py:46-77): {"pred_logits" [B,Q,C+1], "pred_boxes" [B,Q,4]} of the last decoder
        layer; pred_boxes = sigmoid(bbox_embed(hs)) (:73, MLP :309-321).  ``aux_loss=True`` adds "aux_outputs" (:74-75,
        ``_set_aux_loss`` :95-100): see ``aux_outputs``."""
        feats = self.features(samples)
        self._run(feats, None, backward=False)
        out = {"pred_logits": self.pred_logits}
        if self.bbox_embed:
            out["pred_boxes"] = self._boxes(self.saved["hs"].v)
        if aux_loss:
            out["aux_outputs"] = self.aux_outputs()
        return out

    __call__ = forward

    def aux_outputs(self) -> List[Dict[str, torch.Tensor]]:
        """The auxiliary outputs of the last forward: for decoder layers 0 .. L-2, {"pred_logits" [B,Q,C+1], "pred_boxes"
        [B,Q,4]} of class_embed / sigmoid(bbox_embed) applied to decoder.norm(layer output) (DETR/models/transformer.py:
        146-151, detr.py:70-77).  The L-1 normalised outputs form one [(L-1) B Q, d] matrix, so the class head and each
        layer of the box MLP are one GEMM for all of them; the returned tensors are views of the two results."""
        if not self.bbox_embed:
            raise MmxError("aux_outputs needs the box head (bbox_embed.*) in the state dict")
        B, S, Q = self._shape
        n, d, rows = len(self.decoder) - 1, self.d_model, B * self.queries
        if n == 0:
            return []
        hs = torch.empty(n * rows, d, device=self.device, dtype=torch.float32)
        l = lib()
        W = self.class_embed
        logits = torch.empty(n * rows, W.out_features, device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            for i, L in enumerate(self.decoder[:-1]):
                t = L.saved["out"].v
                check(l.mmx_layernorm_fwd(ptr(t), t.stride(0), None, ptr(self.dec_norm[0]), ptr(self.dec_norm[1]),
                                          ptr(hs[i * rows:]), d, None, None, rows, d, C.c_float(1e-5), current_stream()))
            check(l.mmx_linear_packed(ptr(hs), d, ptr(W.w), W.in_features, ptr(W.pw), ptr(W.b), None, 0, ptr(logits),
                                      W.out_features, None, 0, n * rows, W.out_features, W.in_features, current_stream()))
        boxes = self._mlp_boxes(hs)
        C1 = W.out_features
        return [{"pred_logits": logits[i * rows:(i + 1) * rows].view(B, Q, C1),
                 "pred_boxes": boxes[i * rows:(i + 1) * rows].view(B, Q, 4)} for i in range(n)]

    def _boxes(self, hs: torch.Tensor) -> torch.Tensor:
        B, S, Q = self._shape
        return self._mlp_boxes(hs).view(B, Q, -1)

    def _mlp_boxes(self, hs: torch.Tensor) -> torch.Tensor:
        """sigmoid(bbox_embed(hs)) for hs [rows, d]: [rows, 4]"""
        l = lib()
        x = hs
        with torch.cuda.device(self.device):
            for i, W in enumerate(self.bbox_embed):
                last = i == len(self.bbox_embed) - 1
                y = torch.empty(x.shape[0], W.out_features, device=self.device, dtype=torch.float32)
                act = ACT_SIGMOID if last else ACT_RELU
                check(l.mmx_linear_packed(ptr(x), x.stride(0), ptr(W.w), W.in_features, ptr(W.pw), ptr(W.b), None, 0, ptr(y),
                                          W.out_features, ptr(y), act, x.shape[0], W.out_features, W.in_features,
                                          current_stream()))
                x = y
        return x

    def _mha(self, tape: Tape, m, query: Var, key: Var, value: Var, B, T, S) -> Var:
        """DETR/modules/layers.py:728-768: separate projections, q scaled before q k^T, masks ignored."""
        H = self.nhead
        q, k, v = tape.linear(query, m["q"]), tape.linear(key, m["k"]), tape.linear(value, m["v"])
        o = tape.attention(q, k, v, B, H, T, S, float(self.d_model // H) ** -0.5, 0, None, m["rec"])
        m["rec"].saved.update(Xq=query, Xk=key, Xv=value)
        return tape.linear(o, m["o"])

    def forward_backward(self, *args, lrp: bool = False, **kwargs):
        """See ``_forward_backward``.  With ``lrp=True`` every GEMM of the transformer (forward, dgrad and the relprop sweep)
        runs on the fp32 FFMA backend (``nn.fp32_gemms``: the sweep amplifies tensor-core split rounding); the backbone of
        an image input runs before that on the default backend - no relevance or gradient reaches it."""
        if lrp:
            # the backbone sits below the relprop sweep: its features run on the default (tensor-core) backend first
            if args and not isinstance(args[0], _Feats):
                pos = args[1] if len(args) > 1 else kwargs.pop("pos", None)
                feats = self.features(args[0] if pos is None else (args[0], pos))
                args = (feats, None) + tuple(args[2:])
            with fp32_gemms():
                return self._forward_backward(*args, lrp=True, **kwargs)
        return self._forward_backward(*args, lrp=False, **kwargs)

    def _forward_backward(self, src, pos=None, target_index=None, index=None, backward: bool = True, lrp: bool = False):
        """Forward staging every A, one-hot on pred_logits[b, target_b, class_b], backward staging every dA
        (``backward=False``: forward only, for the raw-attention / rollout baselines); ``lrp=True`` adds the relprop
        sweep from the same one-hot (DETR/models/detr.py:79-92), staging the relevance of every A.  ``src, pos``: the
        features [B, d, h, w]; or ``src`` alone: any other accepted input (images, ``_Feats``) and ``pos=None``."""
        if isinstance(src, _Feats):
            feats = src
        else:
            feats = self.features(src if pos is None else (src, pos))
        return self._run(feats, target_index, index, backward, lrp)

    def _run(self, feats: _Feats, target_index, index=None, backward: bool = True, lrp: bool = False):
        dev = self.device
        with torch.cuda.device(dev):
            B, h, w, d = feats.B, feats.h, feats.w, self.d_model
            S, Q = h * w, self.queries
            self.spatial_dim = (h, w)
            tape = Tape(dev)
            x = Var(feats.x)
            pe = feats.pe
            qe = self.query_embed.repeat(B, 1)                                    # [B*Q, d]
            for L in self.encoder:                                                # transformer.py:230-254
                qk = tape.add_const(x, pe)
                att = self._mha(tape, L.self_attn, qk, qk, x, B, S, S)
                x1 = tape.layernorm(tape.add(x, att), *L.n1, 1e-5)
                hdn = tape.linear(x1, L.l1, ACT_RELU)
                ff = tape.linear(hdn, L.l2)
                L.saved = dict(src=x, webmd=qk, drop=att, x1=x1, h=hdn, ff=ff)
                x = tape.layernorm(tape.add(x1, ff), *L.n2, 1e-5)
            memory = x
            mem_pe = tape.add_const(memory, pe)
            t = Var(torch.zeros(B * Q, d, device=dev))
            for L in self.decoder:                                                # transformer.py:372-408
                qk = tape.add_const(t, qe)
                drop1 = self._mha(tape, L.self_attn, qk, qk, t, B, Q, Q)
                x1 = tape.layernorm(tape.add(t, drop1), *L.n1, 1e-5)
                tq = tape.add_const(x1, qe)
                drop2 = self._mha(tape, L.multihead_attn, tq, mem_pe, memory, B, Q, S)
                x2 = tape.layernorm(tape.add(x1, drop2), *L.n2, 1e-5)
                hdn = tape.linear(x2, L.l1, ACT_RELU)
                ff = tape.linear(hdn, L.l2)
                L.saved = dict(tgt=t, memory=memory, webmd=qk, drop1=drop1, x1=x1, drop2=drop2, x2=x2, h=hdn, ff=ff)
                t = tape.layernorm(tape.add(x2, ff), *L.n3, 1e-5)
                L.saved["out"] = t
            hs = tape.layernorm(t, *self.dec_norm, 1e-5)
            logits = tape.linear(hs, self.class_embed)                             # [B*Q, C+1]
            C1 = logits.cols
            self.pred_logits = logits.v.view(B, Q, C1)
            self._shape = (B, S, Q)
            self.saved = dict(B=B, memory=memory, hs=hs, logits=logits)
            if not backward:
                return {"pred_logits": self.pred_logits}
            tq_idx = torch.as_tensor(target_index, device=dev).reshape(B).long()
            rows = torch.arange(B, device=dev) * Q + tq_idx
            if index is None:                                                      # ExplanationGenerator.py:151-152
                cls = logits.v[rows, :-1].argmax(-1)
            else:
                cls = torch.as_tensor(index, device=dev).reshape(B).long()
            one_hot = torch.zeros_like(logits.v)
            one_hot.view(-1).index_fill_(0, rows * C1 + cls, 1.0)          # one_hot[rows, cls] = 1 without a host scalar (graph-capturable)
            tape.seed(logits, one_hot, B)
            tape.backward()
            if lrp:
                from .lrp import detr_sweep
                detr_sweep(self, one_hot)
        return {"pred_logits": self.pred_logits}


class Generator:
    """DETR/modules/ExplanationGenerator.py:56-195 (``generate_ours`` and its three handlers)."""

    def __init__(self, model):
        self.model = engine_for(model)
        self.model.eval()

    def _feats(self, img) -> _Feats:
        return img if isinstance(img, _Feats) else self.model.features(img)

    def handle_self_attention_image(self, blocks):                                 # :110-118
        for blk in blocks:
            cam = rules.avg_heads_record(blk.self_attn["rec"], self.B, self.use_lrp)
            self.R_i_i, _ = rules.self_update(self.R_i_i, cam)

    def handle_co_attn_self_query(self, block):                                    # :120-129
        cam = rules.avg_heads_record(block.self_attn["rec"], self.B, self.use_lrp)
        self.R_q_q, self.R_q_i = rules.self_update(self.R_q_q, cam, self.R_q_i)

    def handle_co_attn_query(self, block):                                         # :131-140
        cam_q_i = rules.avg_heads_record(block.multihead_attn["rec"], self.B, self.use_lrp)
        add, _, md = rules.mm_update_batched(self.R_q_q, self.R_i_i, None, cam_q_i,
                                             apply_normalization=self.normalize_self_attention,
                                             apply_self_in_rule_10=self.apply_self_in_rule_10, nan_to_zero=True)
        self._min_diag.append(md)
        self.R_q_i = rules.add(self.R_q_i, add)

    def generate_ours(self, img, target_index, index=None, use_lrp=True, normalize_self_attention=True,
                      apply_self_in_rule_10=True):
        self.use_lrp = bool(use_lrp)
        self.normalize_self_attention = normalize_self_attention
        self.apply_self_in_rule_10 = apply_self_in_rule_10
        m = self.model
        m.forward_backward(self._feats(img), None, target_index, index, lrp=self.use_lrp)
        B, S, Q = m._shape
        self.B = B
        dev = m.device
        self._min_diag: List[torch.Tensor] = []
        self.R_i_i = torch.eye(S, device=dev).repeat(B, 1, 1)                       # :176-180
        self.R_q_q = torch.eye(Q, device=dev).repeat(B, 1, 1)
        self.R_q_i = torch.zeros(B, Q, S, device=dev)
        self.handle_self_attention_image(m.encoder)
        for blk in m.decoder:
            self.handle_co_attn_self_query(blk)
            self.handle_co_attn_query(blk)
        self.min_diag = torch.stack(self._min_diag).min() if (normalize_self_attention and self._min_diag) else None
        if not getattr(self, "_defer_assert", False):
            self.check_min_diag()
        return self._pick(target_index)

    def check_min_diag(self):
        """handle_residual's ``assert self_attention[diag].min() >= 0`` (:50) over every cross-attention step of the last
        call (one host read; deferred to after the replay when the call runs as a CUDA graph)."""
        if getattr(self, "min_diag", None) is not None:
            assert self.min_diag.item() >= 0

    def capture(self, img, target_index, index=None, use_lrp=True, normalize_self_attention=True, apply_self_in_rule_10=True):
        """``generate_ours`` for these shapes / flags as a CUDA graph (``mmx_b200.graphs.Graphed``): returns a callable
        ``g(src, pos, target_index)`` - or ``g(images, target_index)`` when ``img`` is a [B,3,H,W] image tensor, the
        backbone then inside the graph - that replays the captured kernels on new inputs and yields the (static) result
        tensor; ``g.check()`` runs the deferred ``diag(R - I) >= 0`` assert.  ``target_index`` must be a tensor."""
        from .graphs import Graphed
        dev = self.model.device
        tq = torch.as_tensor(target_index).reshape(-1).to(dev)
        idx = None if index is None else torch.as_tensor(index).reshape(-1).to(dev)
        flags = (idx, use_lrp, normalize_self_attention, apply_self_in_rule_10)
        if _is_features(img):
            args = (img[0], img[1], tq)

            def fn(s, p, t):
                return self.generate_ours((s, p), t, *flags)
        elif isinstance(img, torch.Tensor):
            args = (img, tq)

            def fn(x, t):
                return self.generate_ours(x, t, *flags)
        else:
            raise MmxError("capture takes (src, pos) features or a [B,3,H,W] image tensor")
        self._defer_assert = True
        try:
            return Graphed(fn, args, dev, deferred_checks=[self.check_min_diag])
        finally:
            self._defer_assert = False

    def _pick(self, target_index):
        """``aggregated[:, target_index, :].unsqueeze_(0)`` (:192-194): [1,1,1,S] for a tensor index, [1,1,S] for an int;
        [B,S] for a batch."""
        B, S, Q = self.model._shape
        dev = self.model.device
        tq = torch.as_tensor(target_index, device=dev).reshape(B).long()
        picked = self.R_q_i[torch.arange(B, device=dev), tq].contiguous()
        if B == 1:
            return picked.view(1, 1, 1, S) if isinstance(target_index, torch.Tensor) else picked.view(1, 1, S)
        return picked

    # ---- baselines sharing the API (SURVEY.md §8f-2); the LRP ones need relprop and are not implemented
    def generate_raw_attn(self, img, target_index):
        """Head-mean of the last decoder layer's cross-attention (DETR/modules/ExplanationGenerator.py:224-236)."""
        m = self.model
        m.forward_backward(self._feats(img), None, target_index, backward=False)
        self.B = m._shape[0]
        self.R_q_i = rules.head_mean_record(m.decoder[-1].multihead_attn["rec"], self.B)
        return self._pick(target_index)

    def generate_rollout(self, img, target_index):
        """Attention rollout (DETR/modules/ExplanationGenerator.py:238-273): rollout of the encoder and decoder
        self-attentions, combined through the last cross-attention as R_qq^T (A_qi R_ii)."""
        m = self.model
        m.forward_backward(self._feats(img), None, target_index, backward=False)
        self.B = B = m._shape[0]
        cams_image = [rules.head_mean_record(blk.self_attn["rec"], B) for blk in m.encoder]
        cams_queries = [rules.head_mean_record(blk.self_attn["rec"], B) for blk in m.decoder]
        self.R_i_i = rules.compute_rollout_attention(cams_image)
        self.R_q_q = rules.compute_rollout_attention(cams_queries)
        cam_q_i = rules.head_mean_record(m.decoder[-1].multihead_attn["rec"], B)
        self.R_q_i, _, _ = rules.mm_update_batched(self.R_q_q, self.R_i_i, None, cam_q_i, apply_normalization=False,
                                                   apply_self_in_rule_10=True)
        return self._pick(target_index)

    def generate_attn_gradcam(self, img, target_index, index=None):
        """attn-GradCAM of the last cross-attention (DETR/modules/ExplanationGenerator.py:275-305)."""
        m = self.model
        m.forward_backward(self._feats(img), None, target_index, index)
        self.B = m._shape[0]
        self.R_q_i = rules.gradcam_record(m.decoder[-1].multihead_attn["rec"], self.B)
        return self._pick(target_index)

    def generate_partial_lrp(self, img, target_index, index=None):
        """Partial LRP (DETR/modules/ExplanationGenerator.py:197-224): head mean of the LRP relevance of the last decoder
        cross-attention, min-max normalised over the whole [Q, S] map."""
        m = self.model
        m.forward_backward(self._feats(img), None, target_index, index, lrp=True)
        self.B = B = m._shape[0]
        cam = rules.head_mean_record(m.decoder[-1].multihead_attn["rec"], B, use_cam=True).contiguous()
        self.R_q_i = rules.minmax_normalize(cam)
        return self._pick(target_index)

    def generate_transformer_att(self, img, target_index, index=None):
        """Transformer attribution (DETR/modules/ExplanationGenerator.py:64-108): rule 5 on the last decoder
        cross-attention with the LRP relevance in place of the probabilities."""
        m = self.model
        m.forward_backward(self._feats(img), None, target_index, index, lrp=True)
        self.B = B = m._shape[0]
        self.R_q_i = rules.avg_heads_record(m.decoder[-1].multihead_attn["rec"], B, use_cam=True).contiguous()
        return self._pick(target_index)


class GeneratorAlbationNoAgg(Generator):
    """DETR/modules/ExplanationGenerator.py:306-403 (sic): the ablation without aggregation - every update REPLACES the
    relevancy instead of adding to it (``R = cam R`` for the self-attention rules, ``R_q_i = rule 10`` for the
    cross-attention)."""

    def handle_self_attention_image(self, blocks):                                 # :314-322
        for blk in blocks:
            self.R_i_i = rules.bmm(rules.avg_heads_record(blk.self_attn["rec"], self.B, self.use_lrp), self.R_i_i)

    def handle_co_attn_self_query(self, block):                                    # :324-333
        cam = rules.avg_heads_record(block.self_attn["rec"], self.B, self.use_lrp)
        self.R_q_q, self.R_q_i = rules.bmm(cam, self.R_q_q), rules.bmm(cam, self.R_q_i)

    def handle_co_attn_query(self, block):                                         # :335-344
        cam_q_i = rules.avg_heads_record(block.multihead_attn["rec"], self.B, self.use_lrp)
        self.R_q_i, _, md = rules.mm_update_batched(self.R_q_q, self.R_i_i, None, cam_q_i,
                                                    apply_normalization=self.normalize_self_attention,
                                                    apply_self_in_rule_10=self.apply_self_in_rule_10, nan_to_zero=True)
        self._min_diag.append(md)

    def generate_ours_abl(self, img, target_index, index=None, use_lrp=False, normalize_self_attention=False,
                          apply_self_in_rule_10=True):                             # :346-403
        return Generator.generate_ours(self, img, target_index, index, use_lrp, normalize_self_attention, apply_self_in_rule_10)

    def generate_ours(self, *a, **k):
        raise AttributeError("GeneratorAlbationNoAgg has generate_ours_abl only (DETR/modules/ExplanationGenerator.py:346)")


class MaskGenerator:
    """The relevance -> segmentation-mask step of DETR/mask_generator.py:39-125 (``get_panoptic``): one relevance map per
    kept query through the ``method`` switch (:93-113), then min-max / Otsu (:115-121).  The reference loops over the
    kept queries with one forward + backward and one CPU cv2 call each; here the queries of an image form ONE batch and
    the masks come from one kernel launch.  ``get_panoptic`` is the whole driver step (forward, keep rule, pred_masks);
    ``PostProcess`` / ``PostProcessSegm`` below are the two post-processors the reference's ``evaluate`` runs after it.
    The visualisation and the COCO evaluator are out of scope.

    The staged A / dA of every encoder layer grow with S^2 (about 2.4 GB per query at 2500 tokens, 6.8 GB at 4200), so the
    queries run in chunks: ``max_batch`` queries per chunk when given, else as many as the free device memory holds
    (``chunk_size``).  Every query's map is the same bits whatever the chunking (the kernels are batch invariant)."""

    METHODS = ("ours_with_lrp", "ours_no_lrp", "ablation_no_self_in_10", "ablation_no_aggregation", "ours_no_lrp_no_norm",
               "transformer_att", "partial_lrp", "raw_attn", "attn_gradcam", "rollout")

    def __init__(self, model, aux_loss: bool = False):
        self.gen = Generator(model)
        self.abl = GeneratorAlbationNoAgg(self.gen.model)
        self.model = self.gen.model
        self.aux_loss = bool(aux_loss)

    def sample_bytes(self, S: int, lrp: bool) -> int:
        """Device memory one query of a chunk stages at S tokens: A and dA of every attention layer (fp32, rows padded to a
        multiple of 4), the relevancy matrices (R_i_i, rule 6's product and its operand), and half as much again under LRP
        (the relevance planes and the sweep's activations)."""
        m = self.model
        H, Q, ld = m.nhead, m.queries, -(-S // 4) * 4
        staged = 2 * H * (len(m.encoder) * S * ld + len(m.decoder) * Q * (ld + Q))
        rel = 3 * S * S + 2 * Q * S
        total = 4 * (staged + rel)
        return total * 3 // 2 if lrp else total

    def chunk_size(self, S: int, lrp: bool, budget: float = 0.7) -> int:
        """Queries per chunk: ``budget`` of the free device memory (including what PyTorch's allocator holds unused) over
        ``sample_bytes``, at least 1."""
        dev = self.model.device
        free, _ = torch.cuda.mem_get_info(dev)
        free += torch.cuda.memory_reserved(dev) - torch.cuda.memory_allocated(dev)
        return max(1, int(budget * free) // self.sample_bytes(S, lrp))

    def get_masks(self, img, queries, method: str = "ours_no_lrp", max_batch: Optional[int] = None):
        """img: one image (a [1,3,H,W] tensor, a one-image list or NestedTensor) or its features (src [1,C,h,w],
        pos [1,C,h,w]); queries: the kept query indices [K].  The backbone runs once and its features are repeated over
        the queries of each chunk (the reference re-runs the whole model per query); ``max_batch`` caps the queries per
        chunk (default: ``chunk_size``).  Returns (masks [K,h,w] in {0,255}, thresholds [K], cams [K,h*w])."""
        q = torch.as_tensor(queries).reshape(-1).long()
        K = q.numel()
        if K == 0:
            raise MmxError("no queries to segment")
        if method not in self.METHODS:
            print("please provide a valid explainability method")            # mask_generator.py:111-113
            return None
        if max_batch is not None and int(max_batch) < 1:
            raise MmxError(f"max_batch must be >= 1, got {max_batch}")
        feats = self.model.features(img)
        if feats.B != 1:
            raise MmxError(f"get_masks segments one image, got a batch of {feats.B}")
        return self._masks(feats, q, method, max_batch)

    def _masks(self, feats: _Feats, q: torch.Tensor, method: str, max_batch: Optional[int]):
        K, h, w = q.numel(), feats.h, feats.w
        lrp = method in ("ours_with_lrp", "transformer_att", "partial_lrp")
        n = int(max_batch) if max_batch is not None else self.chunk_size(h * w, lrp)
        cam = torch.cat([self._cams(feats.expand(len(qc)), qc, method) for qc in q.split(n)])
        masks, thr = rules.otsu_masks(cam)
        return masks.view(K, h, w), thr, cam

    def get_panoptic(self, samples, targets, method: str, max_batch: Optional[int] = None):
        """DETR/mask_generator.py:45-155: the segmentation driver's step 1 for one image (a [1,3,H,W] tensor, a one-image
        list or a NestedTensor; ``targets`` is ignored, as in the reference).  One forward gives pred_logits / pred_boxes
        and the keep rule ``softmax(pred_logits)[0, :, :-1].max(-1) > 0.5`` (mmx_detr_postprocess, on the device); the kept
        queries go through ``get_masks`` on the same backbone features.  Returns {"pred_logits" [1,Q,C+1], "pred_boxes"
        [1,Q,4], "pred_masks" [1,Q,h,w]} on the device, pred_masks -1 on the dropped queries and the {0, 255} Otsu mask on
        the kept ones.  Prints "no segmentation" when at most one query is kept (:65-66).  An unknown ``method`` prints
        and returns None before any work; the reference's two shape-probing forwards (:47, :80) are not needed.  With
        ``aux_loss=True`` (the reference model built with DETR's default ``aux_loss``) the dict also holds
        "aux_outputs" (``DetrEngine.aux_outputs``) between "pred_boxes" and "pred_masks", as the reference's does."""
        if method not in self.METHODS:
            print("please provide a valid explainability method")            # mask_generator.py:111-113
            return None
        m = self.model
        feats = m.features(samples)
        if feats.B != 1:
            raise MmxError(f"get_panoptic segments one image (the reference reads image 0 of --batch_size 1), got {feats.B}")
        m._run(feats, None, backward=False)
        if not m.bbox_embed:
            raise MmxError("get_panoptic needs the box head (bbox_embed.*) in the state dict")
        logits = m.pred_logits
        boxes = m._boxes(m.saved["hs"].v)
        aux = m.aux_outputs() if self.aux_loss else None
        keep = detr_postprocess(logits)["keep"][0]
        q = keep.nonzero().flatten()                                           # one host sync, as keep.nonzero() there
        K, Q, h, w = q.numel(), m.queries, feats.h, feats.w
        if K <= 1:
            print("no segmentation")
        pred_masks = torch.full((1, Q, h, w), -1.0, device=m.device, dtype=torch.float32)
        if K:
            masks, _, _ = self._masks(feats, q, method, max_batch)
            pred_masks.index_copy_(1, q, masks.view(1, K, h, w))
        if aux is not None:
            return {"pred_logits": logits, "pred_boxes": boxes, "aux_outputs": aux, "pred_masks": pred_masks}
        return {"pred_logits": logits, "pred_boxes": boxes, "pred_masks": pred_masks}

    def _cams(self, batch: _Feats, q: torch.Tensor, method: str) -> torch.Tensor:
        """the relevance maps [k, h*w] of the k queries ``q`` (one per sample of ``batch``) by ``method`` (:93-113)"""
        if method == "ours_no_lrp":
            cam = self.gen.generate_ours(batch, q, use_lrp=False)
        elif method == "ablation_no_self_in_10":
            cam = self.gen.generate_ours(batch, q, use_lrp=False, apply_self_in_rule_10=False)
        elif method == "ablation_no_aggregation":
            cam = self.abl.generate_ours_abl(batch, q, use_lrp=False, normalize_self_attention=False)
        elif method == "ours_no_lrp_no_norm":
            cam = self.gen.generate_ours(batch, q, use_lrp=False, normalize_self_attention=False)
        elif method == "raw_attn":
            cam = self.gen.generate_raw_attn(batch, q)
        elif method == "attn_gradcam":
            cam = self.gen.generate_attn_gradcam(batch, q)
        elif method == "rollout":
            cam = self.gen.generate_rollout(batch, q)
        elif method == "ours_with_lrp":                                       # mask_generator.py:93-94
            cam = self.gen.generate_ours(batch, q, use_lrp=True)
        elif method == "transformer_att":
            cam = self.gen.generate_transformer_att(batch, q)
        else:
            cam = self.gen.generate_partial_lrp(batch, q)
        return cam.reshape(q.numel(), -1)


def detr_postprocess(pred_logits: torch.Tensor, pred_boxes: Optional[torch.Tensor] = None,
                     target_sizes: Optional[torch.Tensor] = None, keep_threshold: float = 0.5) -> Dict[str, torch.Tensor]:
    """One mmx_detr_postprocess launch over pred_logits [B,Q,C+1]: {"scores" [B,Q], "labels" [B,Q] int64, "keep" [B,Q] bool
    (scores > keep_threshold)}, plus "boxes" [B,Q,4] (xyxy scaled by (w, h, w, h)) when pred_boxes and target_sizes [B,2]
    (img_h, img_w) are given.  All on pred_logits' device."""
    if pred_logits.dim() != 3:
        raise MmxError(f"pred_logits is [B, Q, C+1], got {tuple(pred_logits.shape)}")
    dev = pred_logits.device
    x = _f32(pred_logits, dev)
    B, Q, C1 = x.shape
    scores = torch.empty(B, Q, device=dev, dtype=torch.float32)
    labels = torch.empty(B, Q, device=dev, dtype=torch.int64)
    keep = torch.empty(B, Q, device=dev, dtype=torch.uint8)
    out = {"scores": scores, "labels": labels}
    bx = sz = bo = None
    if pred_boxes is not None and target_sizes is not None:
        if tuple(pred_boxes.shape) != (B, Q, 4) or tuple(target_sizes.shape) != (B, 2):
            raise MmxError(f"pred_boxes [B,Q,4] and target_sizes [B,2] for pred_logits {tuple(x.shape)}, got "
                           f"{tuple(pred_boxes.shape)} and {tuple(target_sizes.shape)}")
        bx = _f32(pred_boxes, dev)
        sz = target_sizes.to(device=dev, dtype=torch.int64).contiguous()
        bo = torch.empty(B, Q, 4, device=dev, dtype=torch.float32)
    with torch.cuda.device(dev):
        check(lib().mmx_detr_postprocess(ptr(x), C1, B, Q, C1, float(keep_threshold), ptr(scores), ptr(labels), ptr(keep),
                                         ptr(bx), ptr(sz), ptr(bo), current_stream()))
    out["keep"] = keep.bool()
    if bo is not None:
        out["boxes"] = bo
    return out


class PostProcess:
    """``PostProcess`` (DETR/models/detr.py:278-306): softmax, score / label per query (max over the classes, the
    no-object column excluded) and the boxes as xyxy in pixels of ``target_sizes`` [B,2] (img_h, img_w), in one
    kernel.  Returns the reference's list of {"scores", "labels", "boxes"} per image, on the device."""

    @torch.no_grad()
    def forward(self, outputs, target_sizes):
        out_logits, out_bbox = outputs["pred_logits"], outputs["pred_boxes"]
        assert len(out_logits) == len(target_sizes)
        assert target_sizes.shape[1] == 2
        r = detr_postprocess(out_logits, out_bbox, target_sizes)
        return [{"scores": s, "labels": l, "boxes": b} for s, l, b in zip(r["scores"], r["labels"], r["boxes"])]

    __call__ = forward


class PostProcessSegm:
    """``PostProcessSegm`` (DETR/models/segmentation.py:218-242): adds "masks" - uint8 [Q,1,oh,ow] on the CPU, 0 / 1 -
    to each result.  The bilinear resize to the batch's max size, ``sigmoid() > threshold``, the crop to each image's
    ``max_target_sizes`` row and the nearest resize to its ``orig_target_sizes`` row run as ONE kernel launch
    (mmx_detr_segm_postprocess), and only the final uint8 masks cross to the host, in one copy.  The reference instead
    materialises the fp32 bilinear masks at the padded size, copies them to the host as bool and resizes them there."""

    def __init__(self, threshold: float = 0.5):
        self.threshold = threshold

    @torch.no_grad()
    def forward(self, results, outputs, orig_target_sizes, max_target_sizes):
        assert len(orig_target_sizes) == len(max_target_sizes)
        masks = outputs["pred_masks"]
        if masks.dim() == 5 and masks.shape[2] == 1:                       # the .squeeze(2) of :227
            masks = masks[:, :, 0]
        if masks.dim() != 4 or masks.shape[2] == 1:
            raise MmxError(f"pred_masks is [B, Q, h, w] with h > 1, got {tuple(outputs['pred_masks'].shape)}")
        B, Q, h, w = masks.shape
        sizes = [tuple(int(v) for v in t) for t in max_target_sizes.tolist()]
        orig = [tuple(int(v) for v in t) for t in orig_target_sizes.tolist()]
        if len(sizes) != B or len(results) != B:
            raise MmxError(f"{B} images of pred_masks, {len(sizes)} target sizes and {len(results)} results")
        if min(min(s) for s in sizes + orig) <= 0:
            raise MmxError(f"image sizes must be positive, got {sizes} and {orig}")
        dev = masks.device
        x = _f32(masks, dev)
        n = [Q * oh * ow for oh, ow in orig]
        buf = torch.empty(sum(n), device=dev, dtype=torch.uint8)
        flat_sizes = (C.c_int * (2 * B))(*[v for s in sizes for v in s])
        flat_orig = (C.c_int * (2 * B))(*[v for s in orig for v in s])
        with torch.cuda.device(dev):
            check(lib().mmx_detr_segm_postprocess(ptr(x), B, Q, h, w, flat_sizes, flat_orig, float(self.threshold),
                                                  ptr(buf), current_stream()))
            host = torch.empty(buf.numel(), dtype=torch.uint8, pin_memory=True)
            host.copy_(buf, non_blocking=True)
            torch.cuda.current_stream().synchronize()
        for r, part, (oh, ow) in zip(results, host.split(n), orig):
            r["masks"] = part.view(Q, 1, oh, ow)
        return results

    __call__ = forward


# Engines built from reference ``DETR`` modules, keyed by the module object (dropped with it).  The engine holds a COPY of
# the weights taken at the first call, like ``mmx_b200.clip.engine_for``.
_ENGINES: "weakref.WeakKeyDictionary" = weakref.WeakKeyDictionary()


def engine_for(model, device=None) -> DetrEngine:
    """The :class:`DetrEngine` behind ``model``: the engine itself, or one built (once) from a reference ``DETR``
    ``nn.Module``'s ``state_dict()`` with ``nhead = model.transformer.nhead`` (DETR/models/detr.py:22, transformer.py:42)
    and the DC5 dilation read from ``model.backbone[0].body.layer4[-1].conv2.dilation`` (DETR/models/backbone.py:88-90)."""
    if isinstance(model, DetrEngine):
        return model
    if not (hasattr(model, "state_dict") and callable(model.state_dict)):
        raise MmxError("model must be a mmx_b200.DetrEngine or a reference DETR nn.Module (anything with state_dict())")
    eng = _ENGINES.get(model)
    if eng is None:
        try:
            nhead = int(model.transformer.nhead)
        except (AttributeError, TypeError, ValueError):
            raise MmxError("a DETR module needs model.transformer.nhead (the reference Transformer sets it)") from None
        eng = DetrEngine(model.state_dict(), nhead=nhead, device=device, dilation=_module_dilation(model))
        _ENGINES[model] = eng
    return eng


def _module_dilation(model) -> bool:
    """True for a reference DETR module with a dilated (DC5) layer4; False when it has none or no backbone."""
    try:
        d = model.backbone[0].body.layer4[-1].conv2.dilation
    except (AttributeError, IndexError, TypeError, KeyError):
        return False
    return int(d[0] if isinstance(d, (tuple, list)) else d) > 1
