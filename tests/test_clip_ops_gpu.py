"""GPU: the CLIP engine's own kernels one op at a time through their C entry points, against fp64 - the ragged
(packed-row) self-attention of the text tower, forward and backward with the per-sample gradient scale; the packed text
embedding; the vision tokens with the fused ln_pre; the logit head with its analytic backward.  Every output starts as a
NaN sentinel (padding included), every error is measured per sample against that sample's own maximum, and batched ops are
checked for batch invariance bit for bit."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

NAN = float("nan")
T_TEXT, LD_TEXT = 77, 80          # the text tower's context length and staged plane row stride


@pytest.fixture(scope="module")
def L():
    import mmx_b200
    from mmx_b200._lib import lib, check, ptr, current_stream
    return dict(lib=lib(), check=check, ptr=ptr, st=current_stream, MmxError=mmx_b200.MmxError)


def _sentinel(*shape, fill=NAN, dtype=torch.float32):
    return torch.full(shape, fill, dtype=dtype, device="cuda")


def assert_same(a, b, what=""):
    """the same floats bit for bit, except that any NaN matches any NaN"""
    a, b = a.detach().cpu().float(), b.detach().cpu().float()
    assert a.shape == b.shape, what
    assert torch.equal(torch.isnan(a), torch.isnan(b)), f"{what}: NaN positions differ"
    m = ~torch.isnan(b)
    assert torch.equal(a[m].view(torch.int32), b[m].view(torch.int32)), f"{what}: values differ"


def per_sample_err(x, ref, sample):
    """max over samples b of max|x - ref| / max|ref| over the elements of sample b (absolute where ref_b is all zero).
    x, ref: [N, ...]; sample: [N] sample index of each leading entry"""
    x, ref = x.double().reshape(x.shape[0], -1), ref.double().reshape(ref.shape[0], -1)
    sample = sample.to(x.device)
    B = int(sample.max()) + 1
    d = torch.zeros(B, dtype=torch.float64, device=x.device).scatter_reduce(0, sample, (x - ref).abs().amax(1), "amax")
    m = torch.zeros(B, dtype=torch.float64, device=x.device).scatter_reduce(0, sample, ref.abs().amax(1), "amax")
    d = torch.where(torch.isnan(d), torch.full_like(d, math.inf), d)
    return float(torch.where(m > 0, d / m.clamp_min(1e-300), d).max())


# ---------------------------------------------------------------------------------------------------- ragged attention
def _mixed_lengths(n, seed):
    edge = [1, 2, 63, 64, 65, 76, 77]
    g = torch.Generator().manual_seed(seed)
    return [edge[i % 7] if i < 14 else int(torch.randint(1, T_TEXT + 1, (1,), generator=g)) for i in range(n)]


LEN_SETS = {
    "b1": [76],
    "b5": [1, 77, 64, 2, 65],
    "b64": _mixed_lengths(64, 5),
    "b64_all77": [77] * 64,
    "b64_all1": [1] * 64,
}


def _ragged_ref(qkv_dense, dO_dense, lens, H, causal, scale):
    """fp64 softmax attention per sample over its first lens[b] rows (dense padded [B,T,3D] operands, junk past the
    sample's rows is masked out as keys); returns A, O, dA = A.grad, dq, dk, dv with every row / column >= lens[b] zero"""
    B, T, D3 = qkv_dense.shape
    D = D3 // 3
    hd = D // H
    qkv = qkv_dense.clone().requires_grad_(True)
    q, k, v = (qkv[..., i * D:(i + 1) * D].reshape(B, T, H, hd).transpose(1, 2) for i in range(3))
    n = torch.tensor(lens, device=qkv.device)
    live = torch.arange(T, device=qkv.device)[None, :] < n[:, None]                       # [B,T]
    s = (q * scale) @ k.transpose(-1, -2)
    mask = ~live[:, None, None, :]
    if causal:
        mask = mask | torch.ones(T, T, dtype=torch.bool, device=qkv.device).triu(1)
    s = s.masked_fill(mask, -math.inf)
    A = torch.softmax(s, -1)
    A.retain_grad()
    O = (A @ v).transpose(1, 2).reshape(B, T, D)
    O.backward(dO_dense * live[..., None])
    keep = (live[:, None, :, None] & live[:, None, None, :]).double()
    return A.detach() * keep, O.detach(), A.grad * keep, qkv.grad


def _pack_index(lens, T):
    return torch.cat([b * T + torch.arange(n) for b, n in enumerate(lens)])


def _ragged_call(L, qkv, dO, lens, H, hd, causal, gscale=None):
    """forward then backward through the ragged entry points; packed rows past sum(lens) hold NaN in the inputs and
    every output starts as NaN"""
    lib, check, p, st = L["lib"], L["check"], L["ptr"], L["st"]
    B, D = len(lens), H * hd
    offs = torch.tensor([0] + list(np.cumsum(lens)[:-1]), dtype=torch.int32, device="cuda")
    lens_d = torch.tensor(lens, dtype=torch.int32, device="cuda")
    qp, kp, vp = (C.c_void_p(qkv.data_ptr() + 4 * i * D) for i in range(3))
    scale = C.c_float(1.0 / math.sqrt(hd))
    A, O = _sentinel(B, H, T_TEXT, LD_TEXT), _sentinel(B * T_TEXT, D)
    check(lib.mmx_attention_fwd_ragged(qp, 3 * D, kp, 3 * D, vp, 3 * D, p(A), LD_TEXT, p(O), D, p(offs), p(lens_d), B, H, T_TEXT,
                                       hd, scale, causal, st()))
    dA, dqkv = _sentinel(B, H, T_TEXT, LD_TEXT), _sentinel(B * T_TEXT, 3 * D)
    delta = torch.empty(B, H, T_TEXT, device="cuda")
    dq, dk, dv = (C.c_void_p(dqkv.data_ptr() + 4 * i * D) for i in range(3))
    check(lib.mmx_attention_bwd_ragged(p(dO), D, qp, 3 * D, kp, 3 * D, vp, 3 * D, p(A), p(dA), LD_TEXT, p(delta), dq, 3 * D, dk,
                                       3 * D, dv, 3 * D, p(offs), p(lens_d), B, H, T_TEXT, hd, scale, causal, p(gscale), st()))
    return A, O, dA, dqkv


def _packed_inputs(lens, D, seed):
    g = torch.Generator().manual_seed(seed)
    total = sum(lens)
    qkv = torch.full((len(lens) * T_TEXT, 3 * D), NAN)
    dO = torch.full((len(lens) * T_TEXT, D), NAN)
    qkv[:total] = torch.randn(total, 3 * D, generator=g)
    dO[:total] = torch.randn(total, D, generator=g)
    return qkv.cuda(), dO.cuda()


@pytest.mark.parametrize("hd,H", [(64, 8), (32, 4), (16, 4)])
@pytest.mark.parametrize("causal", [0, 1])
@pytest.mark.parametrize("lenset", list(LEN_SETS))
def test_attention_ragged_vs_fp64(L, hd, H, causal, lenset):
    """Ragged forward and backward against fp64 per sample (A, O, dA within 5e-6; dQ, dK, dV within 1e-5); rows and
    columns past each sample's length exactly 0 in the staged planes; packed rows past the total untouched; a sample run
    alone at offset 0 gives the bits it gets inside the batch; a power-of-two gradient scale per sample divides out."""
    lens = LEN_SETS[lenset]
    B, D, total = len(lens), H * hd, sum(lens)
    qkv, dO = _packed_inputs(lens, D, seed=hd * 7 + causal + B)
    A, O, dA, dqkv = _ragged_call(L, qkv, dO, lens, H, hd, causal)

    idx = _pack_index(lens, T_TEXT).cuda()
    row_sample = torch.repeat_interleave(torch.arange(B), torch.tensor(lens)).cuda()
    qkv_dense = torch.zeros(B * T_TEXT, 3 * D, dtype=torch.float64, device="cuda")
    dO_dense = torch.zeros(B * T_TEXT, D, dtype=torch.float64, device="cuda")
    qkv_dense[idx], dO_dense[idx] = qkv[:total].double(), dO[:total].double()
    Ar, Or, dAr, dqkv_r = _ragged_ref(qkv_dense.view(B, T_TEXT, 3 * D), dO_dense.view(B, T_TEXT, D), lens, H, causal,
                                      1.0 / math.sqrt(hd))
    Or, dqkv_r = Or.reshape(B * T_TEXT, D)[idx], dqkv_r.reshape(B * T_TEXT, 3 * D)[idx]
    bidx = torch.arange(B, device="cuda")
    errs = dict(A=per_sample_err(A[..., :T_TEXT], Ar, bidx), O=per_sample_err(O[:total], Or, row_sample),
                dA=per_sample_err(dA[..., :T_TEXT], dAr, bidx))
    for i, nm in enumerate(("dq", "dk", "dv")):
        errs[nm] = per_sample_err(dqkv[:total, i * D:(i + 1) * D], dqkv_r[:, i * D:(i + 1) * D], row_sample)
    print(f"ragged attention hd {hd} H {H} causal {causal} {lenset}:", {k: f"{v:.1e}" for k, v in errs.items()})
    # about twice the worst seen on an H100 (A / O / dA 9.2e-7, dQ / dK / dV 1.0e-6); budgets 5e-6 and 1e-5
    assert errs["A"] < 2e-6 and errs["O"] < 2e-6 and errs["dA"] < 2e-6, errs
    assert max(errs["dq"], errs["dk"], errs["dv"]) < 3e-6, errs

    # the dense staged planes: every row and column >= lens[b] (the row-stride padding included) is exactly 0
    n = torch.tensor(lens, device="cuda")
    ar = torch.arange(LD_TEXT, device="cuda")
    dead = (ar[None, :T_TEXT, None] >= n[:, None, None]) | (ar[None, None, :] >= n[:, None, None])    # [B,T,LD]
    for nm, t in (("A", A), ("dA", dA)):
        assert bool((t.masked_select(dead[:, None].expand_as(t)) == 0).all()), nm
    # packed rows past the total are neither read nor written
    assert bool(torch.isnan(O[total:]).all()) and bool(torch.isnan(dqkv[total:]).all())
    assert not bool(torch.isnan(O[:total]).any()) and not bool(torch.isnan(dqkv[:total]).any())

    # batch invariance: sample b alone, packed at offset 0, gives the same bits
    offs = [0] + list(np.cumsum(lens)[:-1])
    for b in sorted({0, B // 2, B - 1}):
        r0, nb = int(offs[b]), lens[b]
        q1 = torch.full((T_TEXT, 3 * D), NAN, device="cuda")
        d1 = torch.full((T_TEXT, D), NAN, device="cuda")
        q1[:nb], d1[:nb] = qkv[r0:r0 + nb], dO[r0:r0 + nb]
        A1, O1, dA1, dqkv1 = _ragged_call(L, q1, d1, [nb], H, hd, causal)
        assert_same(A1[0], A[b], f"A sample {b}")
        assert_same(dA1[0], dA[b], f"dA sample {b}")
        assert_same(O1[:nb], O[r0:r0 + nb], f"O sample {b}")
        assert_same(dqkv1[:nb], dqkv[r0:r0 + nb], f"dqkv sample {b}")

    # a gradient stream carrying gscale[b] = 2^12 / 2^-3: the staged dA is in true units, dQ / dK / dV carry the factor.
    # Close, not bit for bit: where a residual of the fp16 hi / lo split of dO (or of dS) is subnormal in fp16, scaling
    # the operand moves it onto a different absolute rounding grid (worst seen on an H100: 1.7e-7, a few elements in 1e3)
    gs =torch.tensor([2.0 ** 12, 2.0 ** -3] * ((B + 1) // 2), device="cuda")[:B]
    dO_s = dO.clone()
    dO_s[:total] *= gs[row_sample][:, None]
    _, _, dAs, dqkvs = _ragged_call(L, qkv, dO_s, lens, H, hd, causal, gscale=gs)
    dqkv_u = dqkvs[:total] / gs[row_sample][:, None]
    e_dA, e_d = per_sample_err(dAs, dA, bidx), per_sample_err(dqkv_u, dqkv[:total], row_sample)
    n_bits = int((dAs.view(torch.int32) != dA.view(torch.int32)).sum()), int((dqkv_u.view(torch.int32) !=
                                                                                dqkv[:total].view(torch.int32)).sum())
    print(f"  gscale vs unscaled: dA {e_dA:.1e} ({n_bits[0]} of {dA.numel()} differ), dqkv {e_d:.1e} "
          f"({n_bits[1]} of {dqkv_u.numel()} differ)")
    assert e_dA < 5e-7 and e_d < 5e-7
    assert bool(torch.isnan(dqkvs[total:]).all())


def test_attention_ragged_refusals(L):
    """ragged rows past 1024 keys, and a ragged call without offs / lens, are refused with an error"""
    lib, p, st, MmxError = L["lib"], L["ptr"], L["st"], L["MmxError"]
    T, H, hd = 1100, 1, 16
    qkv = torch.zeros(T, 3 * hd, device="cuda")
    A, O = torch.zeros(1, H, T, 1104, device="cuda"), torch.zeros(T, hd, device="cuda")
    offs = torch.zeros(1, dtype=torch.int32, device="cuda")
    lens = torch.full((1,), T, dtype=torch.int32, device="cuda")
    qp, kp, vp = (C.c_void_p(qkv.data_ptr() + 4 * i * hd) for i in range(3))
    for o, n in ((offs, lens), (None, lens), (offs, None)):
        with pytest.raises(MmxError):
            L["check"](lib.mmx_attention_fwd_ragged(qp, 3 * hd, kp, 3 * hd, vp, 3 * hd, p(A), 1104, p(O), hd, p(o), p(n), 1, H, T,
                                                    hd, C.c_float(0.25), 1, st()))
    with pytest.raises(MmxError):
        L["check"](lib.mmx_attention_bwd_ragged(p(O), hd, qp, 3 * hd, kp, 3 * hd, vp, 3 * hd, p(A), p(A), 1104, None, None, 0,
                                                None, 0, None, 0, p(offs), p(lens), 1, H, T, hd, C.c_float(0.25), 1, None, st()))
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ packed text embedding
def _first_argmax(tok):
    return np.array([int(np.argmax(r)) for r in tok.numpy()])


@pytest.mark.parametrize("B", [1, 64, 300])
def test_text_embed_packed(L, B):
    """lens / offs / eot_row / total exactly against a host first-argmax (ties: the lowest index), the packed rows bit for
    bit against tok_emb[token] + pos in fp32, rows past the total untouched"""
    lib, check, p, st = L["lib"], L["check"], L["ptr"], L["st"]
    S, D, vocab = T_TEXT, 512, 1000
    g = torch.Generator().manual_seed(B)
    tok = torch.randint(1, vocab - 1, (B, S), generator=g, dtype=torch.int32)
    eot = vocab - 1
    edge = []
    edge.append(torch.zeros(S, dtype=torch.int32))                          # all zero: length 1
    r = tok[0].clone(); r[76] = eot; edge.append(r)                        # EOT in the last slot: length 77
    r = tok[0].clone(); r[0] = eot; edge.append(r)                         # EOT in slot 0: length 1
    r = tok[0].clone(); r[40] = eot; r[5] = eot; edge.append(r)            # tie across lanes: slot 5 wins
    r = tok[0].clone(); r[35] = eot; r[3] = eot; edge.append(r)            # tie within one lane: slot 3 wins
    r = tok[0].clone(); r[31] = eot; r[32] = eot; edge.append(r)           # tie across the first lane wrap: slot 31
    edge.append(torch.full((S,), 7, dtype=torch.int32))                    # every slot tied: length 1
    if B == 1:
        tok[0, 76] = eot
    else:
        for i, r in enumerate(edge[:B]):
            tok[(i * 37) % B] = r
    emb = torch.randn(vocab, D, generator=g)
    pos = torch.randn(S, D, generator=g)
    tok_d, emb_d, pos_d = tok.cuda(), emb.cuda(), pos.cuda()
    x = _sentinel(B * S, D)
    offs, lens, eot_row = (torch.full((B,), -7, dtype=torch.int32, device="cuda") for _ in range(3))
    total = torch.full((1,), -7, dtype=torch.int32, device="cuda")
    check(lib.mmx_text_embed_packed(p(tok_d), p(emb_d), p(pos_d), p(x), p(offs), p(lens), p(eot_row), p(total), B, S, D, vocab,
                                    st()))
    n = _first_argmax(tok) + 1
    o = np.concatenate([[0], np.cumsum(n)[:-1]])
    assert lens.cpu().numpy().tolist() == n.tolist()
    assert offs.cpu().numpy().tolist() == o.tolist()
    assert eot_row.cpu().numpy().tolist() == (o + n - 1).tolist()
    assert int(total) == int(n.sum())
    if B > 1:
        for i, r in enumerate(edge[:B]):
            assert int(n[(i * 37) % B]) == [1, 77, 1, 6, 4, 32, 1][i]
    ref = torch.cat([emb[tok[b, :n[b]].long()] + pos[:n[b]] for b in range(B)])
    assert_same(x[:int(n.sum())], ref, "packed x")
    assert bool(torch.isnan(x[int(n.sum()):]).all())


# ------------------------------------------------------------------------------------------- vision tokens + ln_pre
@pytest.mark.parametrize("D", [64, 768, 1024])
@pytest.mark.parametrize("S", [50, 197, 577])
def test_vision_tokens_lnpre_vs_fp64(L, D, S):
    """LN(cat(cls, patch_emb) + pos) against fp64 within 2e-6 at row scales from 1e-2 to 1e1 (where eps matters), distinct
    images and one image broadcast to three samples (equal bits in every sample)"""
    lib, check, p, st = L["lib"], L["check"], L["ptr"], L["st"]
    B, eps = 3, 1e-5
    g = torch.Generator().manual_seed(D + S)
    row_scale = 10.0 ** (torch.rand(B * (S - 1), 1, generator=g) * 3 - 2)
    patch = torch.randn(B * (S - 1), D, generator=g) * row_scale
    cls = torch.randn(D, generator=g) * 0.05
    pos = torch.randn(S, D, generator=g) * 0.01
    gamma, beta = 1 + 0.2 * torch.randn(D, generator=g), 0.1 * torch.randn(D, generator=g)
    pd, cd, posd, gd, bd = (t.cuda() for t in (patch, cls, pos, gamma, beta))
    for n_img in (B, 1):
        x = _sentinel(B * S, D)
        check(lib.mmx_vision_tokens_lnpre(p(pd), n_img, p(cd), p(posd), p(gd), p(bd), p(x), B, S, D, C.c_float(eps), st()))
        pe = patch.double().view(-1, S - 1, D)[torch.arange(B) % n_img]
        t = torch.cat([cls.double().expand(B, 1, D), pe], 1) + pos.double()
        ref = torch.nn.functional.layer_norm(t, (D,), gamma.double(), beta.double(), eps).reshape(B * S, D)
        err = per_sample_err(x.cpu(), ref, torch.arange(B * S) // S)
        print(f"vision_tokens_lnpre D {D} S {S} n_img {n_img}: {err:.1e}")
        assert err < 5e-7           # worst seen on an H100: 2.0e-7 (LayerNorm budget 2e-6)
        if n_img == 1:
            xs = x.view(B, S, D)
            for b in range(1, B):
                assert_same(xs[b], xs[0], f"sample {b}")


# ------------------------------------------------------------------------------------------------------- logit head
def _head(L, fi, ft, lse):
    lib, check, p, st = L["lib"], L["check"], L["ptr"], L["st"]
    B, E = fi.shape
    fin, ftn, dfi, dft = (_sentinel(B, E) for _ in range(4))
    diag, gi, gt = _sentinel(B), _sentinel(B), _sentinel(B)
    check(lib.mmx_clip_head(p(fi), p(ft), C.c_float(lse), p(fin), p(ftn), p(dfi), p(dft), p(diag), p(gi), p(gt), B, E, st()))
    return fin, ftn, dfi, dft, diag, gi, gt


@pytest.mark.parametrize("E", [1, 100, 512, 768])
@pytest.mark.parametrize("B", [1, 3, 64])
@pytest.mark.parametrize("lse", [1.0, 100.0])
def test_clip_head_vs_fp64(L, E, B, lse):
    """normalised features and diag against fp64; dfeat / gscale against fp64 autograd of sum_b logits_per_image[b,b];
    gscale an exact power of two putting max|dfeat| of each sample in [16, 32); feature norms from 1e-3 to 1e3"""
    g = torch.Generator().manual_seed(E * 10 + B)
    norms = lambda: 10.0 ** (torch.rand(B, 1, generator=g) * 6 - 3)
    fi = torch.randn(B, E, generator=g)
    ft = torch.randn(B, E, generator=g)
    fi, ft = fi / fi.norm(dim=-1, keepdim=True) * norms(), ft / ft.norm(dim=-1, keepdim=True) * norms()
    fin, ftn, dfi, dft, diag, gi, gt = _head(L, fi.cuda(), ft.cuda(), lse)
    a, t = fi.double().requires_grad_(True), ft.double().requires_grad_(True)
    an, tn = a / a.norm(dim=-1, keepdim=True), t / t.norm(dim=-1, keepdim=True)
    logits = lse * an @ tn.t()
    logits.diagonal().sum().backward()
    bidx = torch.arange(B)
    # diag = scale * cos: a cosine near 0 has no relative precision, its error is judged against the scale
    errs = dict(fin=per_sample_err(fin.cpu(), an.detach(), bidx), ftn=per_sample_err(ftn.cpu(), tn.detach(), bidx),
                diag=float((diag.cpu().double() - logits.detach().diagonal()).abs().max()) / lse)
    if E > 1:
        errs.update(dfi=per_sample_err((dfi / gi[:, None]).cpu(), a.grad, bidx),
                    dft=per_sample_err((dft / gt[:, None]).cpu(), t.grad, bidx))
    else:   # a 1-d feature normalises to +-1 whatever its size: the gradient is exactly 0 (fp64 autograd leaves rounding dust)
        assert bool((dfi == 0).all() and (dft == 0).all())
        assert float((a.grad * fi.double().abs()).abs().max()) < 1e-12 * lse
    print(f"clip_head E {E} B {B} scale {lse}:", {k: f"{v:.1e}" for k, v in errs.items()})
    # about twice the worst seen on an H100 (1.4e-7 for fin / ftn, 2.6e-7 for dfi / dft)
    assert max(errs["fin"], errs["ftn"], errs["diag"]) < 4e-7 and max(errs.get("dfi", 0), errs.get("dft", 0)) < 6e-7, errs
    for gs, d in ((gi, dfi), (gt, dft)):
        gs, d = gs.cpu(), d.cpu()
        mant, _ = torch.frexp(gs)
        assert bool((mant == 0.5).all()), gs
        m = d.abs().amax(1)
        assert bool(torch.where(m > 0, (m >= 16) & (m < 32), gs == 1).all()), (m, gs)


def test_clip_head_zero_feature_row(L):
    """a zero feature gives NaN in its own sample only, with gscale 1; every other sample keeps its bits"""
    B, E = 5, 512
    g = torch.Generator().manual_seed(11)
    fi, ft = torch.randn(B, E, generator=g).cuda(), torch.randn(B, E, generator=g).cuda()
    base = _head(L, fi, ft, 100.0)
    for which in ("image", "text"):
        fz, tz = fi.clone(), ft.clone()
        (fz if which == "image" else tz)[2] = 0
        out = _head(L, fz, tz, 100.0)
        fin, ftn, dfi, dft, diag, gi, gt = out
        assert bool(torch.isnan(dfi[2]).all() and torch.isnan(dft[2]).all() and torch.isnan(diag[2]))
        assert bool(torch.isnan(fin[2] if which == "image" else ftn[2]).all())
        assert float(gi[2]) == 1.0 and float(gt[2]) == 1.0
        keep = [0, 1, 3, 4]
        for i, (x, y) in enumerate(zip(out, base)):
            assert_same(x[keep], y[keep], f"{which} output {i}")
