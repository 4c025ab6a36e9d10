"""GPU: the CLIP engine at ViT-B/32 stage by stage.  Every stage of every block of both towers is recomputed in fp64 from
the engine's own input to that stage (taps of the engine's arena), so an error points at the stage that made it instead of
compounding over the layers; the towers' inputs and outputs are checked the same way; the backward is checked at every
layer against fp64 autograd seeded from the engine's own x_0 and d(features); and one block per tower is replayed through
the public entry points, which must give the engine's bits - in particular fc2 with QuickGELU applied in its operand split
must equal fc1 storing QuickGELU(f) for fc2."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import clip_oracle as co

pytestmark = pytest.mark.gpu

EPS = 1e-5
QUICKGELU = 1                     # MMX_ACT_QUICKGELU

# Bounds: about twice the worst error seen over all cases below on an H100 (in brackets), never looser than the op
# budgets (fp16x3 GEMM 2e-5, attention 5e-6, LayerNorm 2e-6).  dA is the fp64-seeded backward through 12 blocks of
# dgrad GEMMs, so it takes the GEMM budget.
BOUND = dict(stats=5e-7,    # [1.9e-7]
             qkv=6e-6,      # [2.9e-6 backend 1, 1.7e-6 backend 3]
             A=2e-6,        # [6.9e-7]
             xmid=4e-6,     # [1.4e-6]
             f=6e-6,        # [3.0e-6 backend 1, 1.7e-6 backend 3]
             x_next=1e-5,   # [4.5e-6 backend 1, 2.7e-6 backend 3]
             x0=1e-5,       # [4.0e-6 backend 1, 2.1e-6 backend 3]
             feat=5e-6,     # [2.4e-6]
             featn=3e-7,    # [1.1e-7]
             dfeat=5e-7,    # [2.0e-7]
             logits=2e-6,   # [9.4e-7]
             dA=2e-5)       # [1.2e-5 backend 1, 7.5e-6 backend 3]


@pytest.fixture(scope="module")
def b32():
    import mmx_b200
    cfg = co.VIT_B32
    sd = co.init_state_dict(cfg, seed=0)
    eng = mmx_b200.ClipEngine(mmx_b200.ClipConfig(*cfg.ref_args()), sd, max_batch=64, device="cuda:0")
    sd64 = {k: v.to("cuda", torch.float64) for k, v in sd.items()}
    return mmx_b200, cfg, sd, sd64, eng


def _edge_tokens(cfg):
    """test_clip_gpu.py::test_ragged_text_edge_lengths's prompts at ViT-B/32 size: lengths 2, 77, 1 and two ordinary ones"""
    _, tokens = co.synthetic_inputs(cfg, 5, seed=3)
    ctx, eot = cfg.context_length, cfg.vocab_size - 1
    tokens[0] = 0; tokens[0, 0] = cfg.vocab_size - 2; tokens[0, 1] = eot
    g = torch.Generator().manual_seed(9)
    tokens[1] = torch.randint(1, cfg.vocab_size - 2, (ctx,), generator=g); tokens[1, 0] = cfg.vocab_size - 2
    tokens[1, ctx - 1] = eot
    tokens[2] = 0
    return tokens


def _inputs(cfg, B):
    images, tokens = co.synthetic_inputs(cfg, B, seed=0)
    return images, (tokens if B == 64 else _edge_tokens(cfg))


CASES = [(64, "B", 3), (64, "1", 3), (5, "B", 3), (5, "1", 3), (5, "B", 1)]
CASE_IDS = [f"B{B}-img{n}-backend{be}" for B, n, be in CASES]


def _run(mmx, eng, images, tokens, backend):
    lib = mmx.lib()
    prev = lib.mmx_get_gemm_backend()
    try:
        assert lib.mmx_set_gemm_backend(backend) == backend
        eng.interpret(images.cuda(), tokens.cuda(), 0, 0)
        torch.cuda.synchronize()
    finally:
        lib.mmx_set_gemm_backend(prev)


def _text_layout(tokens):
    """lens, offs, eot rows of the packed text rows and the dense row of each packed row"""
    B, T = tokens.shape
    lens = (tokens.argmax(-1) + 1).tolist()
    offs = [0]
    for n in lens[:-1]:
        offs.append(offs[-1] + n)
    idx = torch.cat([b * T + torch.arange(n) for b, n in enumerate(lens)]).cuda()
    return lens, offs, idx


def _rel(x, ref):
    x, ref = x.double(), ref.double()
    d = (x - ref).abs().max()
    return float(torch.nan_to_num(d, nan=math.inf) / ref.abs().max())


def _rel_per_sample(x, ref):
    """[B, ...]: max over b of max|x_b - ref_b| / max|ref_b|"""
    B = x.shape[0]
    x, ref = x.double().reshape(B, -1), ref.double().reshape(B, -1)
    d = torch.nan_to_num((x - ref).abs().amax(1), nan=math.inf)
    m = ref.abs().amax(1)
    return float(torch.where(m > 0, d / m.clamp_min(1e-300), d).max())


def _ln(x, g, b):
    mu = x.mean(-1, keepdim=True)
    rs = 1.0 / torch.sqrt(((x - mu) ** 2).mean(-1, keepdim=True) + EPS)
    return (x - mu) * rs * g + b, mu.squeeze(-1), rs.squeeze(-1)


def _quickgelu(f):
    return f * torch.sigmoid(1.702 * f)


def _tower_geom(cfg, tower):
    if tower == 0:
        return "visual.transformer.", cfg.vision_layers, cfg.vision_width, cfg.vision_heads, cfg.vision_tokens
    return "transformer.", cfg.transformer_layers, cfg.transformer_width, cfg.transformer_heads, cfg.context_length


def _dense(packed, idx, B, S):
    out = torch.zeros(B * S, packed.shape[1], dtype=packed.dtype, device=packed.device)
    out[idx] = packed
    return out.view(B, S, -1)


def _softmax64(q, k, H, causal, live=None):
    """q, k: [B,S,D] fp64 -> A [B,H,S,S] (rows >= live[b] zeroed)"""
    B, S, D = q.shape
    hd = D // H
    qh, kh = (t.reshape(B, S, H, hd).transpose(1, 2) for t in (q, k))
    s = (qh / math.sqrt(hd)) @ kh.transpose(-1, -2)
    if causal:
        s = s.masked_fill(torch.ones(S, S, dtype=torch.bool, device=s.device).triu(1), -math.inf)
    A = torch.softmax(s, -1)
    if live is not None:
        A = A * live[:, None, :, None]
    return A


def _check_stages(mmx, cfg, sd64, eng, tokens, images, n_img, tag):
    """every stage of every block of both towers, the towers' inputs and outputs: worst error per stage and tower"""
    B = tokens.shape[0]
    worst = {}

    def rec(tower, stage, e):
        key = (tower, stage)
        worst[key] = max(worst.get(key, 0.0), e)

    lens, offs, idx = _text_layout(tokens)
    live = (torch.arange(cfg.context_length)[None, :] < torch.tensor(lens)[:, None]).double().cuda()
    for tower in (0, 1):
        prefix, Lyr, D, H, S = _tower_geom(cfg, tower)
        text = tower == 1
        for l in range(Lyr):
            p = f"{prefix}resblocks.{l}."
            x = eng.tap("x", tower, l).cuda().double()
            st = eng.tap("stats", tower, l).cuda().double()
            qkv = eng.tap("qkv", tower, l).cuda().double()
            A = eng.tap("A", tower, l).cuda().double()
            xmid = eng.tap("xmid", tower, l).cuda().double()
            f = eng.tap("f", tower, l).cuda().double()
            xn = eng.tap("x", tower, l + 1).cuda().double()
            M = B * S if not text else sum(lens)
            assert x.shape == (M, D) and qkv.shape == (M, 3 * D) and f.shape == (M, 4 * D) and st.shape == (4, M)
            h1, mu1, rs1 = _ln(x, sd64[p + "ln_1.weight"], sd64[p + "ln_1.bias"])
            _, mu2, rs2 = _ln(xmid, sd64[p + "ln_2.weight"], sd64[p + "ln_2.bias"])
            # a mean is judged against its row's spread, a reciprocal standard deviation against itself
            rec(tower, "stats", float(max(((st[0] - mu1) * rs1).abs().max(), ((st[2] - mu2) * rs2).abs().max(),
                                          ((st[1] - rs1) / rs1).abs().max(), ((st[3] - rs2) / rs2).abs().max())))
            rec(tower, "qkv", _rel(qkv, h1 @ sd64[p + "attn.in_proj_weight"].t() + sd64[p + "attn.in_proj_bias"]))
            qd = _dense(qkv, idx, B, S) if text else qkv.view(B, S, 3 * D)
            Ar = _softmax64(qd[..., :D], qd[..., D:2 * D], H, text, live if text else None)
            rec(tower, "A", _rel_per_sample(A, Ar))
            if text:   # rows and columns past a prompt: exactly 0
                dead = (live[:, :, None] * live[:, None, :]) == 0
                assert bool((A.masked_select(dead[:, None].expand_as(A)) == 0).all()), (tag, l)
            hd = D // H
            v = qd[..., 2 * D:].reshape(B, S, H, hd).transpose(1, 2)
            o = (A @ v).transpose(1, 2).reshape(B * S, D)
            if text:
                o = o[idx]
            rec(tower, "xmid", _rel(xmid, o @ sd64[p + "attn.out_proj.weight"].t() + sd64[p + "attn.out_proj.bias"] + x))
            h2, _, _ = _ln(xmid, sd64[p + "ln_2.weight"], sd64[p + "ln_2.bias"])
            rec(tower, "f", _rel(f, h2 @ sd64[p + "mlp.c_fc.weight"].t() + sd64[p + "mlp.c_fc.bias"]))
            rec(tower, "x_next", _rel(xn, _quickgelu(f) @ sd64[p + "mlp.c_proj.weight"].t() + sd64[p + "mlp.c_proj.bias"] + xmid))

    # tower inputs: vision x_0 from the fp64 patch conv, text x_0 bit for bit against the host-packed embedding
    img = images[:n_img].cuda().double()
    pe = F.conv2d(img, sd64["visual.conv1.weight"], stride=cfg.vision_patch_size).flatten(2).transpose(1, 2)
    pe = pe[torch.arange(B) % n_img]
    tok = torch.cat([sd64["visual.class_embedding"].expand(B, 1, -1), pe], 1) + sd64["visual.positional_embedding"]
    x0r, _, _ = _ln(tok, sd64["visual.ln_pre.weight"], sd64["visual.ln_pre.bias"])
    rec(0, "x0", _rel(eng.tap("x", 0, 0).cuda(), x0r.reshape(B * cfg.vision_tokens, -1)))
    emb = sd64["token_embedding.weight"].float()
    pos = sd64["positional_embedding"].float()
    x0t = torch.cat([emb[tokens[b, :n].cuda()] + pos[:n] for b, n in enumerate(lens)])
    assert torch.equal(eng.tap("x", 1, 0).cuda().view(torch.int32), x0t.view(torch.int32)), tag
    # tower outputs: feat from the engine's x_L, featn / dfeat from the engine's feat, logits
    lse = float(sd64["logit_scale"].exp())
    feats = []
    for tower, (lnk, projk) in enumerate((("visual.ln_post.", "visual.proj"), ("ln_final.", "text_projection"))):
        _, Lyr, D, H, S = _tower_geom(cfg, tower)
        xL = eng.tap("x", tower, Lyr).cuda().double()
        rows = torch.arange(B) * S if tower == 0 else torch.tensor(offs) + torch.tensor(lens) - 1
        pooled, _, _ = _ln(xL[rows.cuda()], sd64[lnk + "weight"], sd64[lnk + "bias"])
        rec(tower, "feat", _rel(eng.tap("feat", tower).cuda(), pooled @ sd64[projk]))
        feats.append(eng.tap("feat", tower).cuda().double().requires_grad_(True))
    fn = [t / t.norm(dim=-1, keepdim=True) for t in feats]
    logits = lse * fn[0] @ fn[1].t()
    logits.diagonal().sum().backward()
    for tower in (0, 1):
        rec(tower, "featn", _rel_per_sample(eng.tap("featn", tower).cuda(), fn[tower].detach()))
        gs = eng.tap("gscale", tower).cuda()
        rec(tower, "dfeat", _rel_per_sample(eng.tap("dfeat", tower).cuda() / gs[:, None], feats[tower].grad))
    rec(0, "logits", _rel(eng.tap("logits").cuda(), logits.detach()))
    return worst


def _report(tag, worst):
    print(f"\n{tag}: worst error per (tower, stage)")
    for (tower, stage), e in sorted(worst.items()):
        print(f"  {'vision' if tower == 0 else 'text'} {stage:7s} {e:.2e}  (bound {BOUND[stage]:.0e})")


@pytest.mark.parametrize("B,n_img,backend", CASES, ids=CASE_IDS)
def test_forward_stages_vs_fp64(b32, B, n_img, backend):
    mmx, cfg, sd, sd64, eng = b32
    images, tokens = _inputs(cfg, B)
    n = B if n_img == "B" else 1
    _run(mmx, eng, images[:n], tokens, backend)
    worst = _check_stages(mmx, cfg, sd64, eng, tokens, images, n, CASE_IDS[CASES.index((B, n_img, backend))])
    _report(f"forward B {B} n_img {n} backend {backend}", worst)
    bad = {k: v for k, v in worst.items() if not v < BOUND[k[1]]}
    assert not bad, bad


def _tower64(cfg, sd64, tower, x0, lens):
    """fp64 forward of one tower from x0 ([B,S,D] dense) to its pooled feature; A_l keep their gradients"""
    prefix, Lyr, D, H, S = _tower_geom(cfg, tower)
    B, hd = x0.shape[0], D // H
    x, As = x0.detach().clone().requires_grad_(True), []
    for l in range(Lyr):
        p = f"{prefix}resblocks.{l}."
        h, _, _ = _ln(x, sd64[p + "ln_1.weight"], sd64[p + "ln_1.bias"])
        qkv = h @ sd64[p + "attn.in_proj_weight"].t() + sd64[p + "attn.in_proj_bias"]
        A = _softmax64(qkv[..., :D], qkv[..., D:2 * D], H, tower == 1)
        A.retain_grad()
        As.append(A)
        v = qkv[..., 2 * D:].reshape(B, S, H, hd).transpose(1, 2)
        o = (A @ v).transpose(1, 2).reshape(B, S, D)
        x = x + o @ sd64[p + "attn.out_proj.weight"].t() + sd64[p + "attn.out_proj.bias"]
        h, _, _ = _ln(x, sd64[p + "ln_2.weight"], sd64[p + "ln_2.bias"])
        f = h @ sd64[p + "mlp.c_fc.weight"].t() + sd64[p + "mlp.c_fc.bias"]
        x = x + _quickgelu(f) @ sd64[p + "mlp.c_proj.weight"].t() + sd64[p + "mlp.c_proj.bias"]
    if tower == 0:
        pooled, _, _ = _ln(x[:, 0], sd64["visual.ln_post.weight"], sd64["visual.ln_post.bias"])
        return pooled @ sd64["visual.proj"], As
    pooled, _, _ = _ln(x[torch.arange(B), torch.tensor(lens) - 1], sd64["ln_final.weight"], sd64["ln_final.bias"])
    return pooled @ sd64["text_projection"], As


@pytest.mark.parametrize("B,n_img,backend", CASES, ids=CASE_IDS)
def test_backward_every_layer_vs_fp64(b32, B, n_img, backend):
    """dA_l at all L layers of both towers against fp64 autograd seeded from the engine's own x_0 and dfeat / gscale,
    per sample; rows and columns past a prompt exactly 0"""
    mmx, cfg, sd, sd64, eng = b32
    images, tokens = _inputs(cfg, B)
    n = B if n_img == "B" else 1
    _run(mmx, eng, images[:n], tokens, backend)
    lens, offs, idx = _text_layout(tokens)
    live = (torch.arange(cfg.context_length)[None, :] < torch.tensor(lens)[:, None]).double().cuda()
    worst = {}
    for tower in (0, 1):
        _, Lyr, D, H, S = _tower_geom(cfg, tower)
        x0 = eng.tap("x", tower, 0).cuda().double()
        x0 = _dense(x0, idx, B, S) if tower == 1 else x0.view(B, S, D)
        feat, As = _tower64(cfg, sd64, tower, x0, lens)
        seed = eng.tap("dfeat", tower).cuda().double() / eng.tap("gscale", tower).cuda().double()[:, None]
        feat.backward(seed)
        for l in range(Lyr):
            dA = eng.tap("dA", tower, l).cuda().double()
            ref = As[l].grad
            if tower == 1:
                keep = live[:, :, None] * live[:, None, :]
                ref = ref * keep[:, None]
                assert bool((dA.masked_select((keep == 0)[:, None].expand_as(dA)) == 0).all()), l
            worst[(tower, "dA")] = max(worst.get((tower, "dA"), 0.0), _rel_per_sample(dA, ref))
    _report(f"backward B {B} n_img {n} backend {backend}", worst)
    bad = {k: v for k, v in worst.items() if not v < BOUND["dA"]}
    assert not bad, bad


@pytest.mark.parametrize("B", [64, 5])
def test_block_replay_bit_exact(b32, B):
    """One vision and one text block replayed through mmx_layernorm_fwd, mmx_linear_packed (qkv), mmx_attention_fwd or
    mmx_attention_fwd_ragged, the out-projection with its residual, LN2, fc1 storing C_act = QuickGELU(f) and fc2 on that
    C_act, all at backend 3 with mmx_pack_weight planes: qkv_l, A_l, xmid_l, f_l and x_{l+1} of the engine, whose fc2
    applies QuickGELU in its operand split instead, bit for bit."""
    mmx, cfg, sd, sd64, eng = b32
    from mmx_b200._lib import check, ptr as p, current_stream as st
    lib = mmx.lib()
    images, tokens = _inputs(cfg, B)
    _run(mmx, eng, images, tokens, 3)
    lens, offs, _ = _text_layout(tokens)
    prev = lib.mmx_get_gemm_backend()
    try:
        assert lib.mmx_set_gemm_backend(3) == 3
        for tower, l in ((0, 5), (1, 7)):
            prefix, _, D, H, S = _tower_geom(cfg, tower)
            hd = D // H
            pre = f"{prefix}resblocks.{l}."
            w = {k: sd[pre + k].cuda().contiguous() for k in ("ln_1.weight", "ln_1.bias", "ln_2.weight", "ln_2.bias",
                                                              "attn.in_proj_weight", "attn.in_proj_bias", "attn.out_proj.weight",
                                                              "attn.out_proj.bias", "mlp.c_fc.weight", "mlp.c_fc.bias",
                                                              "mlp.c_proj.weight", "mlp.c_proj.bias")}

            def pack(W):
                N, K = W.shape
                pk = torch.empty(lib.mmx_pack_weight_bytes(N, K), dtype=torch.uint8, device="cuda")
                check(lib.mmx_pack_weight(p(W), K, N, K, p(pk), st()))
                return pk

            def linear(A_, W, bias, residual, M, out, C_act=None, act=0):
                N, K = W.shape
                check(lib.mmx_linear_packed(p(A_), A_.shape[1], p(W), K, p(pack(W)), p(bias), p(residual), N, p(out), N,
                                            p(C_act), act, M, N, K, st()))

            x, stats = eng.tap("x", tower, l).cuda(), eng.tap("stats", tower, l).cuda()
            qkv_e, A_e, xmid_e = eng.tap("qkv", tower, l).cuda(), eng.tap("A", tower, l).cuda(), eng.tap("xmid", tower, l).cuda()
            f_e, xn_e = eng.tap("f", tower, l).cuda(), eng.tap("x", tower, l + 1).cuda()
            M = x.shape[0]
            h, mean, rstd = torch.empty(M, D, device="cuda"), torch.empty(M, device="cuda"), torch.empty(M, device="cuda")
            check(lib.mmx_layernorm_fwd(p(x), D, None, p(w["ln_1.weight"]), p(w["ln_1.bias"]), p(h), D, p(mean), p(rstd), M, D,
                                        C.c_float(EPS), st()))
            qkv = torch.empty(M, 3 * D, device="cuda")
            linear(h, w["attn.in_proj_weight"], w["attn.in_proj_bias"], None, M, qkv)
            ld = (S + 3) // 4 * 4
            A = torch.empty(B, H, S, ld, device="cuda")
            O = torch.empty(B * S, D, device="cuda")
            qp, kp, vp = (C.c_void_p(qkv_e.data_ptr() + 4 * i * D) for i in range(3))
            scale = C.c_float(1.0 / math.sqrt(hd))
            if tower == 0:
                check(lib.mmx_attention_fwd(qp, 3 * D, kp, 3 * D, vp, 3 * D, None, p(A), ld, p(O), D, B, H, S, S, hd, scale, 0,
                                            st()))
            else:
                qkv_b = torch.empty(B * S, 3 * D, device="cuda")     # the engine's buffers hold B*S rows; rows past M unread
                qkv_b[:M] = qkv_e
                qp, kp, vp = (C.c_void_p(qkv_b.data_ptr() + 4 * i * D) for i in range(3))
                o_d = torch.tensor(offs, dtype=torch.int32, device="cuda")
                n_d = torch.tensor(lens, dtype=torch.int32, device="cuda")
                check(lib.mmx_attention_fwd_ragged(qp, 3 * D, kp, 3 * D, vp, 3 * D, p(A), ld, p(O), D, p(o_d), p(n_d), B, H, S,
                                                   hd, scale, 1, st()))
            xmid = torch.empty(M, D, device="cuda")
            linear(O[:M], w["attn.out_proj.weight"], w["attn.out_proj.bias"], x, M, xmid)
            h2 = torch.empty(M, D, device="cuda")
            check(lib.mmx_layernorm_fwd(p(xmid_e), D, None, p(w["ln_2.weight"]), p(w["ln_2.bias"]), p(h2), D, None, None, M, D,
                                        C.c_float(EPS), st()))
            f, g = torch.empty(M, 4 * D, device="cuda"), torch.empty(M, 4 * D, device="cuda")
            linear(h2, w["mlp.c_fc.weight"], w["mlp.c_fc.bias"], None, M, f, C_act=g, act=QUICKGELU)
            xn = torch.empty(M, D, device="cuda")
            linear(g, w["mlp.c_proj.weight"], w["mlp.c_proj.bias"], xmid_e, M, xn)
            torch.cuda.synchronize()
            same = lambda a, b: torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))
            res = dict(mean1=same(mean, stats[0]), rstd1=same(rstd, stats[1]), qkv=same(qkv, qkv_e),
                       A=same(A[..., :S], A_e), xmid=same(xmid, xmid_e), f=same(f, f_e), x_next=same(xn, xn_e))
            if not res["x_next"]:
                ref = (_quickgelu(f_e.double()) @ sd64[pre + "mlp.c_proj.weight"].t() + sd64[pre + "mlp.c_proj.bias"]
                       + xmid_e.double())
                print(f"tower {tower} block {l}: fc2 differs; error vs fp64: a_act path {_rel(xn_e, ref):.2e}, "
                      f"C_act path {_rel(xn, ref):.2e}, elements differing {int((xn != xn_e).sum())}")
            assert all(res.values()), (tower, l, res)
    finally:
        lib.mmx_set_gemm_backend(prev)
