"""GPU: the DETR, LXMERT, VisualBERT and ViT generators layer by layer against fp64.  The end-to-end tests
(test_detr_lxmert_gpu, test_zz_baseline_sizes_gpu, test_vit_gpu) compare R and the logits with one batch-wide number;
here every staged attention map and its gradient is held to fp64 per sample and per layer:

  * A of every attention record is recomputed in fp64 from that record's own inputs (the saved query / key rows and the
    layer's weights), so an error points at the layer that made it; masked keys and the pad columns of the staged plane
    (ld > S) must be exactly 0;
  * the logits from the engine's own last hidden state, and end to end from the inputs through the fp64 oracle;
  * dA of every layer against fp64 autograd of the whole oracle from the same inputs and masks (DETR: with the engine's
    ReLU pattern, see _engine_relu); rows that fp64 gives as exactly 0 must be exactly 0 on the device too, and a record
    no gradient reaches must stage none;
  * R per sample against the fp64 oracle's generator;
  * every sample alone and inside its (padded, differently masked) batch gives the same bits for every A, dA, the logits
    and R, on both tensor-core GEMM backends;
  * a -inf key bias gives the bits of the equivalent -10000 attention mask.

The fp64 oracles run on the device with the engine's weights; the class / answer index is the fp64 argmax, handed to the
engine and the oracle alike."""
import contextlib
import functools
import itertools
import math
import types

import pytest
import torch

from oracle import detr_oracle as do, lxmert_oracle as lo, visualbert_oracle as vbo, vit_oracle as vio

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
F64 = torch.float64

# Bounds: about twice the worst error seen over all cases below on an H100 80GB HBM3 at a 700 W power limit (in
# brackets), never looser than the op budgets (fp16x3 GEMM 2e-5, attention 5e-6, LayerNorm 2e-6).  A is the attention op
# from the record's own q and k; A_proj adds the record's q / k projection GEMMs (DETR, LXMERT); logits_h is the head GEMM
# on the engine's last hidden state.  dA, R and the end-to-end logits compound through the model and stay below 1e-4.
# DETR's dA and R take max(bound, 5 x err(fp32 oracle, fp64 oracle)) like test_zz_baseline_sizes_gpu: its fp32 arithmetic
# is itself a few 1e-5 from fp64 (DETR's worst: dA 3.8e-5 backend 1, 3.0e-5 backend 3; R 4.6e-5, the fp32 oracle's own R
# error 4.6e-5).
BOUND = dict(A=2e-6,            # [8.6e-7]
             A_proj=1.5e-5,     # [7.2e-6 backend 1, 3.1e-6 backend 3]
             logits_h=1e-5,     # [4.2e-6 backend 1, 2.0e-6 backend 3]
             logits=6e-5,       # [2.8e-5 backend 1, 1.3e-5 backend 3]
             R=3e-5)            # [1.5e-5 backend 1, 1.1e-5 backend 3]
DA_BOUND = {3: 7e-5,            # [3.4e-5]  (the tensor-core backend in use: 3 = fp16x3, 1 = 3xTF32)
            1: 1e-4}            # [7.3e-5]: capped at 1e-4
NOISE_FACTOR = 5.0


@contextlib.contextmanager
def _backend(b):
    import mmx_b200
    lib = mmx_b200.lib()
    prev = lib.mmx_get_gemm_backend()
    try:
        assert lib.mmx_set_gemm_backend(b) == b
        yield
    finally:
        lib.mmx_set_gemm_backend(prev)


def _ps(x, ref, base=None):
    """max over samples b of max|x_b - ref_b| / max|base_b| (base defaults to ref; absolute where that max is 0)"""
    B = ref.shape[0]
    x, ref = x.double().reshape(B, -1), ref.double().reshape(B, -1)
    base = ref if base is None else base.double().reshape(B, -1)
    d = torch.nan_to_num((x - ref).abs().amax(1), nan=math.inf)
    m = base.abs().amax(1)
    return float(torch.where(m > 0, d / m.clamp_min(1e-300), d).max())


def _off_diag(R):
    """R [B,n,n] with its diagonal zeroed: the part of a self relevance that is not the identity"""
    return R * (1 - torch.eye(R.shape[-1], dtype=R.dtype, device=R.device))


def _lin64(x, W):
    """x W^T + b in fp64 from a tape Var and an nn.Weight"""
    return x.v.double() @ W.w.double().t() + W.b.double()


def _softmax64(q, k, B, H, T, S, scale, bias=None):
    """q [B*T, D], k [B*S, D] -> softmax(scale q k^T + bias) [B,H,T,S] in fp64"""
    hd = q.shape[1] // H
    qh = q.double().reshape(B, T, H, hd).transpose(1, 2)
    kh = k.double().reshape(B, S, H, hd).transpose(1, 2)
    s = scale * (qh @ kh.transpose(-1, -2))
    if bias is not None:
        s = s + bias.double()[:, None, None, :]
    return torch.softmax(s, -1)


def _mask_bias(keep):
    return (1.0 - keep.to(DEV, F64)) * -10000.0


def _check_A(rec, Aref, keep=None):
    """per-sample error of the staged A against Aref [B,H,T,S]; the pad columns and the columns of removed keys exactly 0"""
    A, S = rec.A, rec.S
    assert bool((A[..., S:] == 0).all()), "pad columns of the staged A are not 0"
    A = A[..., :S]
    if keep is not None:
        dead = (keep.to(DEV) == 0)[:, None, None, :].expand_as(A)
        assert bool((A[dead] == 0).all()), "A is not 0 at a masked key"
    return _ps(A, Aref)


def _check_dA(rec, G):
    """per-sample error of the staged dA against the fp64 gradient G; rows G has as exactly 0 exactly 0"""
    dA = rec.get_attn_gradients()
    if G is None:
        assert dA is None, "a record no gradient reaches staged a dA"
        return 0.0
    assert dA is not None
    zero = (G == 0).all(-1)
    assert bool((dA[zero] == 0).all()), "dA is not 0 on a row fp64 gives as exactly 0"
    return _ps(dA, G)


def _line(tag, kind, names, errs):
    print(f"{tag} {kind}: " + " ".join(f"{n} {e:.1e}" for n, e in zip(names, errs)))


def _bad(kind, names, errs, bound):
    lim = bound if isinstance(bound, list) else [bound] * len(errs)
    return [(kind, n, e, l) for n, e, l in zip(names, errs, lim) if not e < l]


def _leaves(sd, dtype):
    """the weights as fp64 / fp32 leaves that require grad, like the reference's nn.Parameters: A of the first decoder
    self-attention of DETR sees only query_embed and must still receive a gradient"""
    return {k: v.detach().to(dtype).requires_grad_(True) for k, v in sd.items()}


def _snap(recs, logits, Rs):
    """copies of every A, dA, the logits and R of the last call (the records are overwritten by the next one)"""
    out = {}
    for r in recs:
        out[r[0] + ".A"] = r[1].A.clone()
        out[r[0] + ".dA"] = None if r[1].dA is None else r[1].dA.clone()
    out["logits"] = logits.clone()
    for i, R in enumerate(Rs):
        out[f"R{i}"] = R.clone()
    torch.cuda.synchronize()
    return out


def _same(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


# ---------------------------------------------------------------------------------------------------------------- DETR
DETR_SHAPES = {"25x34": (2, 25, 34, 5), "10x12": (3, 10, 12, 4)}


@pytest.fixture(scope="module")
def detr():
    import mmx_b200
    cfg = do.DETR_R50
    sd = do.init_state_dict(cfg, seed=9)
    packed = {k: v for k, v in do.to_checkpoint_format(sd).items() if "q_proj" not in k and "k_proj" not in k and "v_proj" not in k}
    eng = mmx_b200.DetrEngine(packed, nhead=cfg.nhead, device=DEV)
    return mmx_b200, cfg, {k: v.to(DEV) for k, v in sd.items()}, eng


def _detr_recs(eng):
    """(name, record, projections) in the oracle's order: encoder self-attentions, then decoder self / cross pairs"""
    out = [(f"e{i}", L.self_attn["rec"], L.self_attn) for i, L in enumerate(eng.encoder)]
    for i, L in enumerate(eng.decoder):
        out += [(f"d{i}s", L.self_attn["rec"], L.self_attn), (f"d{i}c", L.multihead_attn["rec"], L.multihead_attn)]
    return out


def _detr_oracle(sd, cfg, src, pos, tq, cls, dtype):
    """logits, every A and its gradient from logits[b, tq_b, cls_b] ([B,H,T,S], record order), cls (argmax over the
    real classes when None)"""
    B = src.shape[0]
    logits, A_e, A_ds, A_dc = do.detr_forward(_leaves(sd, dtype), cfg, src.to(DEV, dtype), pos.to(DEV, dtype))
    if cls is None:
        cls = logits[torch.arange(B), tq, :-1].argmax(-1).cpu()
    As = A_e + [a for pair in zip(A_ds, A_dc) for a in pair]
    G = torch.autograd.grad(logits[torch.arange(B), tq, cls].sum(), As)
    heads = lambda t: t.detach().reshape(B, cfg.nhead, t.shape[-2], t.shape[-1])
    return logits.detach(), [heads(a) for a in As], [heads(g) for g in G], cls


@contextlib.contextmanager
def _engine_relu(eng, B, S, Q):
    """The DETR oracle with the ReLU pattern of the engine's last call: every FFN ReLU keeps the units the engine kept
    (x * mask in place of relu(x)).  A pre-activation within rounding of 0 takes a sign from fp32 arithmetic that fp64
    need not share, and that unit then adds or drops a whole column of linear2 in the gradient: a discrete difference of
    up to 1e-2 in dA that says nothing about the kernels.  Yields the count of such units per FFN of the first forward."""
    masks = [(L.saved["h"].v > 0).view(B, S, -1).transpose(0, 1) for L in eng.encoder]
    masks += [(L.saved["h"].v > 0).view(B, Q, -1).transpose(0, 1) for L in eng.decoder]
    calls, flips = itertools.count(), []

    def relu(x):
        m = masks[next(calls) % len(masks)]
        if len(flips) < len(masks):
            flips.append(int(((x > 0) != m).sum()))
        return x * m
    F_ = do.F
    do.F = types.SimpleNamespace(linear=F_.linear, layer_norm=F_.layer_norm, relu=relu)
    try:
        yield flips
    finally:
        do.F = F_


def _detr_run(mmx, eng, src, pos, tq, cls):
    R = mmx.Generator(eng).generate_ours((src.to(DEV), pos.to(DEV)), tq, index=cls, use_lrp=False)
    return _snap(_detr_recs(eng), eng.pred_logits, [R])


@pytest.mark.parametrize("backend", [3, 1])
@pytest.mark.parametrize("shape", list(DETR_SHAPES))
def test_detr_stages_vs_fp64(detr, shape, backend):
    """DETR-R50 transformer, checkpoint (in_proj) keys: 25x34 features (850 keys: the 32-query attention tiles), B=2;
    10x12, B=3."""
    mmx, cfg, sd, eng = detr
    B, h, w, seed = DETR_SHAPES[shape]
    src, pos, tq = do.synthetic_inputs(cfg, B, h, w, seed=seed)
    _, _, G64_plain, cls = _detr_oracle(sd, cfg, src, pos, tq, None, F64)
    _, _, G32, _ = _detr_oracle(sd, cfg, src, pos, tq, cls, torch.float32)
    with _backend(backend):
        R = mmx.Generator(eng).generate_ours((src.to(DEV), pos.to(DEV)), tq, index=cls, use_lrp=False)
        torch.cuda.synchronize()
    with _engine_relu(eng, B, h * w, cfg.queries) as flips:
        lg64, A64, G64, _ = _detr_oracle(sd, cfg, src, pos, tq, cls, F64)
        n_flip = list(flips)
        R64 = do.generate_ours(sd, cfg, src.to(DEV), pos.to(DEV), tq, index=cls, dtype=F64)
    tag = f"DETR {shape} B={B} backend {backend}"
    recs = _detr_recs(eng)
    names = [r[0] for r in recs]
    scale = (cfg.d_model // cfg.nhead) ** -0.5
    eA, eAp, edA, ed_plain, noise = [], [], [], [], []
    for (name, rec, m), Ar, G, Gp, G_32 in zip(recs, A64, G64, G64_plain, G32):
        T, S = Ar.shape[-2:]
        eA.append(_check_A(rec, _softmax64(rec.saved["q"].v, rec.saved["k"].v, B, cfg.nhead, T, S, scale)))
        Ai = _softmax64(_lin64(rec.saved["Xq"], m["q"]), _lin64(rec.saved["Xk"], m["k"]), B, cfg.nhead, T, S, scale)
        eAp.append(_check_A(rec, Ai))
        edA.append(_check_dA(rec, G))
        ed_plain.append(_ps(rec.get_attn_gradients(), Gp))
        noise.append(_ps(G_32, Gp))
    # only the target query's row of the last cross-attention is reached by the gradient
    last = G64[-1]
    assert bool((last[torch.arange(B), :, tq] != 0).any(-1).all())
    assert int((last != 0).any(-1).sum()) == B * cfg.nhead
    W = eng.class_embed
    e_lh = _ps(eng.pred_logits, (eng.saved["hs"].v.double() @ W.w.double().t() + W.b.double()).view(B, cfg.queries, -1))
    e_lg = _ps(eng.pred_logits, lg64)
    R32 = do.generate_ours(sd, cfg, src.to(DEV), pos.to(DEV), tq, index=cls, dtype=torch.float32)
    eR, nR = _ps(R, R64), _ps(R32, do.generate_ours(sd, cfg, src.to(DEV), pos.to(DEV), tq, index=cls, dtype=F64))
    _line(tag, "A", names, eA)
    _line(tag, "A_proj", names, eAp)
    _line(tag, "dA", names, edA)
    _line(tag, "FFN units whose ReLU sign differs from fp64", [f"L{i}" for i in range(len(n_flip))], n_flip)
    _line(tag, "dA vs plain fp64", names, ed_plain)
    _line(tag, "dA fp32 oracle vs plain fp64", names, noise)
    print(f"{tag}: logits from hs {e_lh:.2e}, end to end {e_lg:.2e}; R {eR:.2e} (fp32 oracle {nR:.2e})")
    bad = (_bad("A", names, eA, BOUND["A"]) + _bad("A_proj", names, eAp, BOUND["A_proj"])
           + _bad("dA", names, edA, [max(DA_BOUND[backend], NOISE_FACTOR * n) for n in noise])
           + _bad("logits_h", ["-"], [e_lh], BOUND["logits_h"]) + _bad("logits", ["-"], [e_lg], BOUND["logits"])
           + _bad("R", ["-"], [eR], max(BOUND["R"], NOISE_FACTOR * nR)))
    assert not bad, bad


# -------------------------------------------------------------------------------------------------------------- LXMERT
LX_LENS = (20, 13, 6)                      # text lengths through attention_mask
LX_MASKED_BOXES = (1, (2, 7, 11, 19, 28, 35))     # sample 1 loses 6 boxes through visual_attention_mask
LX_KINDS = ("lang", "vis", "x_lang", "x_vis", "x_lang_self", "x_vis_self")


@pytest.fixture(scope="module")
def lxmert():
    import mmx_b200
    cfg = lo.LxmertConfig(vocab=2000, num_labels=300)
    sd = lo.init_state_dict(cfg, seed=1)
    eng = mmx_b200.LxmertEngine(sd, num_heads=cfg.heads, device=DEV)
    return mmx_b200, cfg, {k: v.to(DEV) for k, v in sd.items()}, eng


def _lx_inputs(cfg):
    """B=3, T=20, I=36: padded text (ids 0 past [SEP]) and one sample with masked boxes"""
    ids, feats, boxes = lo.synthetic_inputs(cfg, 3, 20, 36, seed=8)
    am = torch.zeros(3, 20, dtype=torch.long)
    for b, n in enumerate(LX_LENS):
        am[b, :n] = 1
        ids[b, n - 1] = 2
        ids[b, n:] = 0
    vm = torch.ones(3, 36, dtype=torch.long)
    vm[LX_MASKED_BOXES[0], list(LX_MASKED_BOXES[1])] = 0
    return ids, feats, boxes, am, vm


def _lx_recs(eng):
    """(name, record, attention weights, key side 't' / 'i') in the order of the oracle's staged lists (LX_KINDS)"""
    out = [(f"l{i}", b.att.recs[0], b.att, "t") for i, b in enumerate(eng.layer)]
    out += [(f"r{i}", b.att.recs[0], b.att, "i") for i, b in enumerate(eng.r_layers)]
    for kind, key, pick in (("ti", "i", lambda b: (b.cross.recs[0], b.cross)), ("it", "t", lambda b: (b.cross.recs[1], b.cross)),
                            ("tt", "t", lambda b: (b.lang_self.recs[0], b.lang_self)),
                            ("ii", "i", lambda b: (b.visn_self.recs[0], b.visn_self))):
        for i, b in enumerate(eng.x_layers):
            out.append((f"x{i}{kind}", *pick(b), key))
    return out


def _lx_oracle(sd, cfg, ids, feats, boxes, am, vm, idx, dtype):
    B = ids.shape[0]
    logits, st = lo.lxmert_forward(_leaves(sd, dtype), cfg, ids.to(DEV), feats.to(DEV, dtype), boxes.to(DEV, dtype),
                                   am.to(DEV), vm.to(DEV))
    if idx is None:
        idx = logits.argmax(-1).cpu()
    As = [a for n in LX_KINDS for a in st[n]]
    G = torch.autograd.grad(logits[torch.arange(B), idx].sum(), As, allow_unused=True)
    return logits.detach(), [a.detach() for a in As], list(G), idx


def _lx_generate(mmx, eng, ids, feats, boxes, idx, **masks):
    """GeneratorOurs.generate_ours(use_lrp=False) with the masks / key biases handed to the engine's forward_backward.
    Without the eq. 8-9 normalisation: a padded token is a key of no one, so its row of R_t_t stays the identity's and
    the normalisation divides 0 by 0 - in the reference too (it has no NaN guard for LXMERT) - and spreads NaN over R."""
    eng.forward_backward = functools.partial(type(eng).forward_backward, eng, **masks)
    try:
        return mmx.GeneratorOurs(eng).generate_ours((ids.to(DEV), feats.to(DEV), boxes.to(DEV)), idx, use_lrp=False,
                                                    normalize_self_attention=False)
    finally:
        del eng.forward_backward


def _lx_run(mmx, eng, ids, feats, boxes, idx, **masks):
    rtt, rti = _lx_generate(mmx, eng, ids, feats, boxes, idx, **masks)
    return _snap(_lx_recs(eng), eng.question_answering_score, [rtt, rti])


@pytest.mark.parametrize("backend", [3, 1])
def test_lxmert_stages_vs_fp64(lxmert, backend):
    """LXMERT-base (768, 12 heads, 9/5/5 layers), T=20, I=36, B=3: text lengths 20 / 13 / 6 through attention_mask, one
    sample with 6 boxes masked through visual_attention_mask."""
    mmx, cfg, sd, eng = lxmert
    ids, feats, boxes, am, vm = _lx_inputs(cfg)
    B, T, I = 3, 20, 36
    lg64, A64, G64, idx = _lx_oracle(sd, cfg, ids, feats, boxes, am, vm, None, F64)
    with _backend(backend):
        rtt, rti = _lx_generate(mmx, eng, ids, feats, boxes, idx, attention_mask=am.to(DEV), visual_attention_mask=vm.to(DEV))
        torch.cuda.synchronize()
    tag = f"LXMERT-base B={B} backend {backend}"
    recs = _lx_recs(eng)
    names = [r[0] for r in recs]
    keep = dict(t=am, i=vm)
    scale = 1.0 / math.sqrt(cfg.hidden // cfg.heads)
    eA, eAp, edA = [], [], []
    for (name, rec, att, key), Ar, G in zip(recs, A64, G64):
        Tq, S = Ar.shape[-2:]
        bias = _mask_bias(keep[key])
        eA.append(_check_A(rec, _softmax64(rec.saved["q"].v, rec.saved["k"].v, B, cfg.heads, Tq, S, scale, bias), keep[key]))
        Ai = _softmax64(_lin64(rec.saved["Xq"], att.q), _lin64(rec.saved["Xk"], att.k), B, cfg.heads, Tq, S, scale, bias)
        eAp.append(_check_A(rec, Ai, keep[key]))
        edA.append(_check_dA(rec, G))
    # the last cross layer's image->text copy feeds nothing the answer reads; its language self-attention reaches the
    # answer through token 0 only
    assert eng.x_layers[-1].cross.recs[1].get_attn_gradients() is None
    G_tt = G64[names.index(f"x{cfg.x_layers - 1}tt")]
    assert bool((G_tt[:, :, 1:] == 0).all()) and bool((G_tt[:, :, 0] != 0).any(-1).all())
    e_lh = _ps(eng.question_answering_score, _lin64(eng.saved["h"], eng.head3))
    e_lg = _ps(eng.question_answering_score, lg64)
    ott, oti, _ = lo.generate_ours(sd, cfg, ids.to(DEV), feats.to(DEV), boxes.to(DEV), index=idx, dtype=F64,
                                   normalize_self_attention=False, lang_mask=am.to(DEV), vis_mask=vm.to(DEV))
    eR = max(_ps(rtt, ott, _off_diag(ott)), _ps(rti, oti))
    _line(tag, "A", names, eA)
    _line(tag, "A_proj", names, eAp)
    _line(tag, "dA", names, edA)
    print(f"{tag}: logits from h {e_lh:.2e}, end to end {e_lg:.2e}; R {eR:.2e}")
    bad = (_bad("A", names, eA, BOUND["A"]) + _bad("A_proj", names, eAp, BOUND["A_proj"])
           + _bad("dA", names, edA, DA_BOUND[backend])
           + _bad("logits_h", ["-"], [e_lh], BOUND["logits_h"]) + _bad("logits", ["-"], [e_lg], BOUND["logits"])
           + _bad("R", ["-"], [eR], BOUND["R"]))
    assert not bad, bad


# ---------------------------------------------------------------------------------------------------------- VisualBERT
VB_LENS = (14, 9, 5)                       # text lengths: cls_index = length - 2 differs per sample
VB_MASKED_BOX = (2, 40)


@pytest.fixture(scope="module")
def visualbert():
    import mmx_b200
    cfg = vbo.VisualBertConfig(vocab=2000, num_labels=300)
    sd = vbo.init_state_dict(cfg, seed=2)
    eng = mmx_b200.VisualBertEngine(sd, num_heads=cfg.heads, device=DEV)
    return mmx_b200, cfg, {k: v.to(DEV) for k, v in sd.items()}, eng


def _vb_inputs(cfg):
    """T=14, V=100, B=3 with padded text (input_mask and attention_mask 0 past each length) and one masked box"""
    T = 14
    inp = vbo.synthetic_inputs(cfg, 3, T, 100, seed=3)
    for b, n in enumerate(VB_LENS):
        inp["input_ids"][b, n - 1] = 2
        inp["input_ids"][b, n:] = 0
        inp["input_mask"][b, n:] = 0
        inp["attention_mask"][b, n:T] = 0
    inp["attention_mask"][VB_MASKED_BOX[0], T + VB_MASKED_BOX[1]] = 0
    return inp


def _vb_oracle_inputs(inp, dtype=None):
    """on the device, except input_mask: the oracle only indexes with it"""
    out = {k: (v if k == "input_mask" else v.to(DEV)) for k, v in inp.items()}
    if dtype is not None:
        out["visual_embeddings"] = out["visual_embeddings"].to(dtype)
    return out


def _vb_recs(eng):
    return [(f"l{i}", L.rec, L) for i, L in enumerate(eng.layers)]


def _vb_run(mmx, eng, inp, idx):
    R = mmx.SelfAttentionGenerator(eng).generate_ours({k: v.to(DEV) for k, v in inp.items()}, index=idx)
    return _snap(_vb_recs(eng), eng.scores, [R])


def test_visualbert_stages_vs_fp64(visualbert):
    """VisualBERT-base (768, 12 heads, 12 layers), T=14 + V=100, B=3: text lengths 14 / 9 / 5, one masked box."""
    mmx, cfg, sd, eng = visualbert
    inp = _vb_inputs(cfg)
    B, S = 3, 114
    scores64, st = vbo.visualbert_forward(_leaves(sd, F64), cfg, _vb_oracle_inputs(inp, F64))
    idx = scores64.argmax(-1).cpu()
    G64 = torch.autograd.grad(scores64[torch.arange(B), idx].sum(), st)
    with _backend(3):
        R = mmx.SelfAttentionGenerator(eng).generate_ours({k: v.to(DEV) for k, v in inp.items()}, index=idx)
        torch.cuda.synchronize()
    cls_index = torch.tensor(VB_LENS) - 2
    assert torch.equal(eng.cls_index.cpu(), cls_index)
    tag = f"VisualBERT-base B={B} backend 3"
    recs = _vb_recs(eng)
    names = [r[0] for r in recs]
    keep = inp["attention_mask"]
    scale = 1.0 / math.sqrt(cfg.hidden // cfg.heads)
    eA, edA = [], []
    for (name, rec, L), Ar, G in zip(recs, st, G64):
        Ai = _softmax64(rec.saved["q"].v, rec.saved["k"].v, B, cfg.heads, S, S, scale, _mask_bias(keep))
        eA.append(_check_A(rec, Ai, keep))
        edA.append(_check_dA(rec, G))
    # the last layer reaches the answer through row cls_index of each sample only
    live = torch.zeros(B, S, dtype=torch.bool, device=DEV)
    live[torch.arange(B), cls_index] = True
    assert bool(((G64[-1] != 0).any(-1) == live[:, None, :]).all())
    e_lh = _ps(eng.scores, _lin64(eng.saved["h"], eng.head_out))
    e_lg = _ps(eng.scores, scores64.detach())
    ref, _ = vbo.generate_ours(sd, cfg, _vb_oracle_inputs(inp), index=idx, dtype=F64)
    eR = _ps(R, ref)
    _line(tag, "A", names, eA)
    _line(tag, "dA", names, edA)
    print(f"{tag}: logits from h {e_lh:.2e}, end to end {e_lg:.2e}; R {eR:.2e}")
    bad = (_bad("A", names, eA, BOUND["A"]) + _bad("dA", names, edA, DA_BOUND[3])
           + _bad("logits_h", ["-"], [e_lh], BOUND["logits_h"]) + _bad("logits", ["-"], [e_lg], BOUND["logits"])
           + _bad("R", ["-"], [eR], BOUND["R"]))
    assert not bad, bad


# ----------------------------------------------------------------------------------------------------------------- ViT
@pytest.fixture(scope="module")
def vit():
    import mmx_b200
    cfg = vio.VIT_B16
    sd = vio.init_state_dict(cfg, seed=3)
    eng = mmx_b200.ViTEngine(sd, heads=cfg.heads, device=DEV)
    return mmx_b200, cfg, {k: v.to(DEV) for k, v in sd.items()}, eng


def _vit_images(cfg):
    return torch.randn(2, 3, cfg.image, cfg.image, generator=torch.Generator().manual_seed(11))


def _vit_recs(eng):
    return [(f"b{i}", blk["attn"]) for i, blk in enumerate(eng.blocks)]


def _vit_run(mmx, eng, images, idx):
    R = mmx.generate_relevance(eng, images.to(DEV), idx)
    return _snap(_vit_recs(eng), eng.logits, [R])


def test_vit_stages_vs_fp64(vit):
    """ViT-B/16, B=2, 197 tokens: q / k / v are column slices of the packed qkv (row stride 3D)."""
    mmx, cfg, sd, eng = vit
    images = _vit_images(cfg)
    B, S, D = 2, cfg.tokens, cfg.dim
    st = []
    lg64 = vio.vit_forward(_leaves(sd, F64), cfg, images.to(DEV, F64), st)
    idx = lg64.argmax(-1).cpu()
    G64 = torch.autograd.grad(lg64[torch.arange(B), idx].sum(), st)
    with _backend(3):
        R = mmx.generate_relevance(eng, images.to(DEV), idx)
        torch.cuda.synchronize()
    tag = f"ViT-B/16 B={B} backend 3"
    recs = _vit_recs(eng)
    names = [r[0] for r in recs]
    eA, edA = [], []
    for (name, rec), G in zip(recs, G64):
        q, k, v = (rec.saved[n].v for n in "qkv")
        assert q.stride(0) == k.stride(0) == v.stride(0) == 3 * D
        assert k.data_ptr() - q.data_ptr() == v.data_ptr() - k.data_ptr() == 4 * D
        eA.append(_check_A(rec, _softmax64(q, k, B, cfg.heads, S, S, (D // cfg.heads) ** -0.5)))
        edA.append(_check_dA(rec, G))
    # the last block reaches the logits through the cls row only
    assert bool((G64[-1][:, :, 1:] == 0).all()) and bool((G64[-1][:, :, 0] != 0).any(-1).all())
    e_lh = _ps(eng.logits, _lin64(eng.saved["xn"], eng.head))
    e_lg = _ps(eng.logits, lg64.detach())
    ref, _ = vio.generate_relevance(sd, cfg, images.to(DEV), idx, dtype=F64)
    eR = _ps(R, ref)
    _line(tag, "A", names, eA)
    _line(tag, "dA", names, edA)
    print(f"{tag}: logits from xn {e_lh:.2e}, end to end {e_lg:.2e}; R {eR:.2e}")
    bad = (_bad("A", names, eA, BOUND["A"]) + _bad("dA", names, edA, DA_BOUND[3])
           + _bad("logits_h", ["-"], [e_lh], BOUND["logits_h"]) + _bad("logits", ["-"], [e_lg], BOUND["logits"])
           + _bad("R", ["-"], [eR], BOUND["R"]))
    assert not bad, bad


# ---------------------------------------------------------------------------------------------------- batch invariance
def _batch_case(request, engine):
    """(B, run(slice) -> snapshot) for one engine's padded batch; the engine picks the class / answer itself"""
    if engine.startswith("detr"):
        mmx, cfg, sd, eng = request.getfixturevalue("detr")
        B, h, w, seed = DETR_SHAPES[engine.split("-")[1]]
        src, pos, tq = do.synthetic_inputs(cfg, B, h, w, seed=seed)
        return B, lambda sl: _detr_run(mmx, eng, src[sl], pos[sl], tq[sl], None)
    if engine == "lxmert":
        mmx, cfg, sd, eng = request.getfixturevalue("lxmert")
        ids, feats, boxes, am, vm = _lx_inputs(cfg)
        return 3, lambda sl: _lx_run(mmx, eng, ids[sl], feats[sl], boxes[sl], None, attention_mask=am[sl].to(DEV),
                                     visual_attention_mask=vm[sl].to(DEV))
    if engine == "visualbert":
        mmx, cfg, sd, eng = request.getfixturevalue("visualbert")
        inp = _vb_inputs(cfg)
        return 3, lambda sl: _vb_run(mmx, eng, {k: v[sl] for k, v in inp.items()}, None)
    mmx, cfg, sd, eng = request.getfixturevalue("vit")
    images = _vit_images(cfg)
    return 2, lambda sl: _vit_run(mmx, eng, images[sl], None)


@pytest.mark.parametrize("backend", [3, 1])
@pytest.mark.parametrize("engine", ["detr-25x34", "detr-10x12", "lxmert", "visualbert", "vit"])
def test_batch_invariance(request, engine, backend):
    """each sample alone and inside its batch (LXMERT and VisualBERT: with a different mask per sample): every A, every dA,
    the logits and R bit for bit"""
    B, run = _batch_case(request, engine)
    with _backend(backend):
        full = run(slice(None))
        diff = []
        for b in range(B):
            one = run(slice(b, b + 1))
            for key, v in full.items():
                o = one[key]
                if v is None or o is None:
                    if not (v is None and o is None):
                        diff.append((b, key, "gradient staged in one call only"))
                    continue
                ref = v[b:b + 1]
                o = o.reshape(ref.shape)
                if not _same(o, ref):
                    diff.append((b, key, int((o != ref).sum()), float((o.double() - ref.double()).abs().max())))
    print(f"{engine} backend {backend}: {len(full)} tensors x {B} samples, {len(diff)} differ")
    assert not diff, diff[:10]


# -------------------------------------------------------------------------------------------------------- -inf = -10000
def test_neg_inf_key_bias_equals_mask_lxmert(lxmert):
    """lang_key_bias / vis_key_bias of -inf at the padded positions: the bits of attention_mask / visual_attention_mask"""
    mmx, cfg, sd, eng = lxmert
    ids, feats, boxes, am, vm = _lx_inputs(cfg)
    inf = lambda keep: torch.where(keep == 0, -math.inf, 0.0).to(DEV)
    masked = _lx_run(mmx, eng, ids, feats, boxes, None, attention_mask=am.to(DEV), visual_attention_mask=vm.to(DEV))
    biased = _lx_run(mmx, eng, ids, feats, boxes, None, lang_key_bias=inf(am), vis_key_bias=inf(vm))
    diff = [k for k, v in masked.items() if not ((v is None and biased[k] is None) or (v is not None and _same(v, biased[k])))]
    assert not diff, diff


def test_neg_inf_key_bias_equals_mask_visualbert(visualbert):
    """key_bias of -inf at the masked positions: the bits of attention_mask"""
    mmx, cfg, sd, eng = visualbert
    inp = _vb_inputs(cfg)
    masked = _vb_run(mmx, eng, inp, None)
    biased_inp = {k: v for k, v in inp.items() if k != "attention_mask"}
    biased_inp["key_bias"] = torch.where(inp["attention_mask"] == 0, -math.inf, 0.0)
    biased = _vb_run(mmx, eng, biased_inp, None)
    diff = [k for k, v in masked.items() if not ((v is None and biased[k] is None) or (v is not None and _same(v, biased[k])))]
    assert not diff, diff
