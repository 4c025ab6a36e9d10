"""GPU: the eleven LRP (`relprop`) primitives one op at a time through the C ABI against oracle/lrp.py - bit for bit where
the kernel does the same fp32 operations as the torch expression (split, safe_divide, clone), against fp64 for the
reductions, factors and attention relprops - and the single-pass attention kernels at the layouts the engines use
(fused QKV row strides, causal with a key bias, the gscale-carrying backward).  Pads of inputs hold NaN, outputs start as
NaN sentinels, and every batched op is checked for batch invariance."""
import ctypes as C
import math

import pytest
import torch

from oracle import lrp as olrp
from util import rel_err

pytestmark = pytest.mark.gpu

NAN, INF = float("nan"), float("inf")
TINY = 1e-40                                    # subnormal in fp32


@pytest.fixture(scope="module")
def L():
    import mmx_b200
    from mmx_b200._lib import lib, check, ptr, current_stream
    return dict(lib=lib(), check=check, ptr=ptr, st=current_stream, MmxError=mmx_b200.MmxError)


def _padded(x, ld, fill=NAN):
    buf = torch.full((*x.shape[:-1], ld), fill)
    buf[..., :x.shape[-1]] = x
    return buf.cuda()


def _sentinel(*shape, fill=NAN, dtype=torch.float32):
    return torch.full(shape, fill, dtype=dtype, device="cuda")


def assert_same(a, b):
    """the same floats bit for bit (signed zeros included), except that any NaN matches any NaN"""
    a, b = a.detach().cpu().float(), b.detach().cpu().float()
    assert a.shape == b.shape
    assert torch.equal(torch.isnan(a), torch.isnan(b)), "NaN positions differ"
    m = ~torch.isnan(b)
    assert torch.equal(a[m].view(torch.int32), b[m].view(torch.int32)), "values differ"


# the divisors where safe_divide's branches meet: 0, +-1e-9 (-1e-9 makes the denominator exactly 0), subnormal, +-inf, NaN
SPECIAL_Z = [0.0, 1e-9, -1e-9, TINY, -TINY, INF, -INF, NAN, 1.0, -2.5]


def _special(rows, cols, gen, values, scale=1.0):
    """[rows, cols] of random numbers with every special value placed at seeded positions"""
    x = torch.randn(rows, cols, generator=gen) * scale
    idx = torch.randperm(rows * cols, generator=gen)
    per = rows * cols // (2 * len(values))
    for i, v in enumerate(values):
        x.view(-1)[idx[i * per:(i + 1) * per]] = v
    return x


# ---------------------------------------------------------------------------------------------- elementwise, bitwise
def test_lrp_split_bitwise(L):
    """P = X.clamp(min=0), N = X.clamp(max=0), NaN propagating, from a padded input into a padded output"""
    rows, cols, ldx, ld = 37, 70, 75, 73
    X = _special(rows, cols, torch.Generator().manual_seed(1), [0.0, TINY, -TINY, INF, -INF, NAN, 1e-9])
    Xd = _padded(X, ldx)
    P, N = _sentinel(rows, ld), _sentinel(rows, ld)
    L["check"](L["lib"].mmx_lrp_split(L["ptr"](Xd), ldx, L["ptr"](P), L["ptr"](N), ld, rows, cols, L["st"]()))
    assert_same(P[:, :cols], X.clamp(min=0))
    assert_same(N[:, :cols], X.clamp(max=0))
    assert torch.isnan(P[:, cols:]).all() and torch.isnan(N[:, cols:]).all()


def test_lrp_safe_divide_bitwise(L):
    """S = safe_divide(R, Z) in the same fp32 operation order as layers.py:11-14, at every special divisor and with +-0,
    +-inf and NaN in R, each operand with its own row stride"""
    gen = torch.Generator().manual_seed(2)
    rows, cols = 41, 96
    R = _special(rows, cols, gen, [0.0, -0.0, INF, NAN])
    Z = _special(rows, cols, gen, SPECIAL_Z, scale=1e-3)
    Rd, Zd = _padded(R, cols + 5), _padded(Z, cols + 2)
    S = _sentinel(rows, cols + 7)
    L["check"](L["lib"].mmx_lrp_safe_divide(L["ptr"](Rd), cols + 5, L["ptr"](Zd), cols + 2, L["ptr"](S), cols + 7, rows, cols,
                                            L["st"]()))
    assert_same(S[:, :cols], olrp.safe_divide(R, Z))
    assert torch.isnan(S[:, cols:]).all()


@pytest.mark.parametrize("n", range(1, 9))
def test_lrp_clone_bitwise(L, n):
    """Clone.relprop for n = 1..8 relevance inputs, each with its own row stride: X * sum_i safe_divide(R_i, X) summed in
    input order, the same bits as oracle.lrp.clone_relprop in fp32"""
    gen = torch.Generator().manual_seed(10 + n)
    rows, cols = 29, 50
    X = _special(rows, cols, gen, SPECIAL_Z, scale=1e-2)
    Rs = [_special(rows, cols, gen, [0.0, -0.0, NAN]) for _ in range(n)]
    lds = [cols + i for i in range(n)]
    Rd = [_padded(r, ld) for r, ld in zip(Rs, lds)]
    Xd = _padded(X, cols + 3)
    out = _sentinel(rows, cols + 1)
    ptrs = (C.c_void_p * n)(*[t.data_ptr() for t in Rd])
    ldr = (C.c_int * n)(*lds)
    L["check"](L["lib"].mmx_lrp_clone(L["ptr"](Xd), cols + 3, ptrs, ldr, n, L["ptr"](out), cols + 1, rows, cols, L["st"]()))
    assert_same(out[:, :cols], olrp.clone_relprop(Rs, X))
    assert torch.isnan(out[:, cols:]).all()


# --------------------------------------------------------------------------------------------- reductions and factors
def _sums(L, Xd, ldx, rows_ps, cols, B):
    """mmx_lrp_sums -> partials [B, 64, 2] (NaN sentinel first: empty chunks must write zeros)"""
    nch = L["lib"].mmx_lrp_partials_len()
    part = _sentinel(B, nch, 2, dtype=torch.float64)
    L["check"](L["lib"].mmx_lrp_sums(L["ptr"](Xd), ldx, rows_ps, cols, B, L["ptr"](part), L["st"]()))
    return part


@pytest.mark.parametrize("B,rows_ps,cols", [(1, 3, 5), (3, 3, 5), (3, 1, 1), (1, 100, 70), (3, 40, 33)])
def test_lrp_sums_vs_fp64(L, B, rows_ps, cols):
    """{sum, sum |x|} per sample from 64 chunk partials; samples with fewer than 64 elements leave chunks empty"""
    gen = torch.Generator().manual_seed(B * 100 + rows_ps + cols)
    X = torch.randn(B, rows_ps, cols, generator=gen)
    ldx = cols + 3
    part = _sums(L, _padded(X.view(B * rows_ps, cols), ldx), ldx, rows_ps, cols, B).cpu()
    assert torch.isfinite(part).all()
    tot = part.sum(1)
    x64 = X.double()
    assert torch.allclose(tot[:, 0], x64.sum((1, 2)), rtol=1e-12, atol=1e-12)
    assert torch.allclose(tot[:, 1], x64.abs().sum((1, 2)), rtol=1e-12, atol=1e-12)
    for b in range(B):
        one = _sums(L, _padded(X[b], ldx), ldx, rows_ps, cols, 1).cpu()
        assert torch.equal(one[0], part[b])


def test_lrp_renorm_vs_fp64(L):
    """X[b] *= safe_divide(sum num[b], sum den[b]); sample 1's denominator is all zero (factor 0); pads stay NaN"""
    B, rows_ps, cols, ld = 3, 20, 30, 33
    gen = torch.Generator().manual_seed(4)
    X = torch.randn(B * rows_ps, cols, generator=gen)
    num = torch.randn(B * rows_ps, cols, generator=gen) + 0.2
    den = torch.randn(B * rows_ps, cols, generator=gen) - 0.3
    den[rows_ps:2 * rows_ps] = 0
    pn = _sums(L, num.cuda(), cols, rows_ps, cols, B)
    pd = _sums(L, den.cuda(), cols, rows_ps, cols, B)

    def run(Xs, pn_, pd_, nb):
        Xd = _padded(Xs, ld)
        L["check"](L["lib"].mmx_lrp_renorm(L["ptr"](Xd), ld, rows_ps, cols, nb, L["ptr"](pn_), L["ptr"](pd_), L["st"]()))
        return Xd.cpu()

    out = run(X, pn, pd, B)
    assert torch.isnan(out[:, cols:]).all()
    worst = 0.0
    for b in range(B):
        sl = slice(b * rows_ps, (b + 1) * rows_ps)
        fac = olrp.safe_divide(num[sl].double().sum(), den[sl].double().sum())
        worst = max(worst, rel_err(out[sl, :cols], X[sl].double() * fac))
        assert torch.equal(run(X[sl], pn[b:b + 1].contiguous(), pd[b:b + 1].contiguous(), 1)[:, :cols], out[sl, :cols])
    print(f"lrp_renorm: err {worst:.1e}")
    assert worst < 1e-6
    assert (out[rows_ps:2 * rows_ps, :cols] == 0).all()


def _add(L, R, x0, x1, rows_ps, cols, B, with_b):
    lds = dict(r=cols + 1, x0=cols + 2, x1=cols + 3, a=cols + 5, b=cols + 4)
    Rd, x0d, x1d = _padded(R, lds["r"]), _padded(x0, lds["x0"]), _padded(x1, lds["x1"])
    a = _sentinel(B * rows_ps, lds["a"])
    b = _sentinel(B * rows_ps, lds["b"]) if with_b else None
    ws = _sentinel(B, 3 * L["lib"].mmx_lrp_partials_len(), dtype=torch.float64)
    p = L["ptr"]
    L["check"](L["lib"].mmx_lrp_add(p(Rd), lds["r"], p(x0d), lds["x0"], p(x1d), lds["x1"], p(a), lds["a"], p(b), lds["b"],
                                    rows_ps, cols, B, p(ws), L["st"]()))
    assert torch.isnan(a[:, cols:]).all() and (b is None or torch.isnan(b[:, cols:]).all())
    return a[:, :cols].cpu(), (b[:, :cols].cpu() if with_b else None)


def test_lrp_add_vs_fp64(L):
    """Add.relprop per sample against oracle.lrp.add_relprop in fp64 (positive inputs, signed relevance), with b NULL and
    not; sample 1's relevance is all zero, so its sums are zero and both outputs are 0"""
    B, rows_ps, cols = 3, 17, 45
    gen = torch.Generator().manual_seed(6)
    R = torch.randn(B * rows_ps, cols, generator=gen) + 0.3
    R[rows_ps:2 * rows_ps] = 0
    x0 = torch.rand(B * rows_ps, cols, generator=gen) + 0.1
    x1 = torch.rand(B * rows_ps, cols, generator=gen) * 2 + 0.1
    a, b = _add(L, R, x0, x1, rows_ps, cols, B, True)
    a_only, _ = _add(L, R, x0, x1, rows_ps, cols, B, False)
    assert torch.equal(a_only, a)
    worst = 0.0
    for s in range(B):
        sl = slice(s * rows_ps, (s + 1) * rows_ps)
        ra, rb = olrp.add_relprop(R[sl].double(), x0[sl].double(), x1[sl].double())
        if s == 1:
            assert (a[sl] == 0).all() and (b[sl] == 0).all()
        else:
            worst = max(worst, rel_err(a[sl], ra), rel_err(b[sl], rb))
        a1, b1 = _add(L, R[sl], x0[sl], x1[sl], rows_ps, cols, 1, True)
        assert torch.equal(a1, a[sl]) and torch.equal(b1, b[sl])
    print(f"lrp_add: err {worst:.1e}")
    assert worst < 1e-6


def test_lrp_zero_value_fix_per_sample(L):
    """The all-zero-value case decided per sample on the device: sample 0's value relevance is zero after its projection
    but not before (cam_q / cam_k rescaled to share sum(cam)), sample 1's is not (left alone, bit for bit)"""
    B, rq, rk, cols = 2, 7, 11, 24
    gen = torch.Generator().manual_seed(7)
    cq = torch.randn(B * rq, cols, generator=gen) + 0.2
    ck = torch.randn(B * rk, cols, generator=gen) + 0.1
    cam = torch.randn(B * rq, cols, generator=gen) + 0.5
    v_pre = torch.randn(B * rk, cols, generator=gen)
    v_post = torch.randn(B * rk, cols, generator=gen)
    v_post[:rk] = 0

    def run(sl_q, sl_k, nb):
        s = lambda x, r: _sums(L, x[r].contiguous().cuda(), cols, x[r].shape[0] // nb, cols, nb)
        parts = [s(v_pre, sl_k), s(v_post, sl_k), s(cq, sl_q), s(ck, sl_k), s(cam, sl_q)]
        qd, kd = _padded(cq[sl_q], cols + 2), _padded(ck[sl_k], cols + 6)
        p = L["ptr"]
        L["check"](L["lib"].mmx_lrp_zero_value_fix(p(qd), cols + 2, rq, p(kd), cols + 6, rk, cols, nb, *map(p, parts), L["st"]()))
        assert torch.isnan(qd[:, cols:]).all() and torch.isnan(kd[:, cols:]).all()
        return qd[:, :cols].cpu(), kd[:, :cols].cpu()

    q, k = run(slice(None), slice(None), B)
    qs, ks, cs = cq[:rq].double().sum(), ck[:rk].double().sum(), cam[:rq].double().sum()
    k_fact = olrp.safe_divide(ks.abs(), ks.abs() + qs.abs()) * cs
    q_fact = olrp.safe_divide(qs.abs(), ks.abs() + qs.abs()) * cs
    err = max(rel_err(q[:rq], cq[:rq].double() * olrp.safe_divide(q_fact, qs)),
              rel_err(k[:rk], ck[:rk].double() * olrp.safe_divide(k_fact, ks)))
    print(f"lrp_zero_value_fix: err {err:.1e}")
    assert err < 1e-6
    assert torch.equal(q[rq:], cq[rq:]) and torch.equal(k[rk:], ck[rk:])
    for b in range(B):
        q1, k1 = run(slice(b * rq, (b + 1) * rq), slice(b * rk, (b + 1) * rk), 1)
        assert torch.equal(q1, q[b * rq:(b + 1) * rq]) and torch.equal(k1, k[b * rk:(b + 1) * rk])


# ------------------------------------------------------------------------------------------------ attention relprops
class AttnCase:
    """Positive operands; q / k / v are column views of one fused [rows, 3D] buffer (ld = 3D).  A and cam1 live in the
    [B,H,T,ldA] layout with NaN in their pad columns; R_o and O are padded with NaN as well."""

    def __init__(self, B, H, T, S, hd, seed):
        gen = torch.Generator().manual_seed(seed)
        self.B, self.H, self.T, self.S, self.hd, self.D = B, H, T, S, hd, H * hd
        D = self.D
        self.qkv = torch.rand(B * max(T, S), 3 * D, generator=gen) + 0.05
        self.q, self.k, self.v = (self.qkv[:B * n, i * D:(i + 1) * D] for i, n in ((0, T), (1, S), (2, S)))
        self.A = torch.softmax(torch.randn(B, H, T, S, generator=gen), -1)
        self.cam1 = torch.rand(B, H, T, S, generator=gen) * 0.01
        self.R_o = torch.rand(B * T, D, generator=gen)
        self.O = (self.A.double() @ self._heads(self.v, S).double()).transpose(1, 2).reshape(B * T, D).float()
        self.ldA = (S + 3) // 4 * 4 + 4
        self.qkv_d = self.qkv.cuda()
        self.A_d, self.cam1_d = _padded(self.A, self.ldA), _padded(self.cam1, self.ldA)

    def _heads(self, x, n):
        return x.reshape(self.B, n, self.H, self.hd).transpose(1, 2)

    def _cols(self, x, n):
        return x.transpose(1, 2).reshape(self.B * n, self.D)

    def view(self, i):
        """device pointer of q (0), k (1) or v (2) inside the fused buffer"""
        return C.c_void_p(self.qkv_d.data_ptr() + 4 * i * self.D)


def _attn_cases():
    out = []
    for hd in (8, 16, 32, 48, 64):
        for T, S in ((33, 65), (64, 129), (5, 7)):
            out.append((2, 3 if hd <= 32 else 2, T, S, hd))
    return out


@pytest.mark.parametrize("B,H,T,S,hd", _attn_cases())
def test_lrp_attention_relprops_vs_fp64(L, B, H, T, S, hd):
    """mmx_lrp_attn_pv / _qk / _scores against oracle.lrp.pv_relprop / scores_relprop (halved, as the attention relprop
    does) and zscale Q K^T in fp64: within 2e-5 on positive operands, no NaN from the input pads, output pads of the
    [B,H,T,ldA] planes written as zero and pads of the row outputs left alone"""
    c = AttnCase(B, H, T, S, hd, seed=T * 1000 + S * 10 + hd)
    lib, p, st = L["lib"], L["ptr"], L["st"]
    D, ld3, ldA = c.D, 3 * c.D, c.ldA
    Ro, Od = _padded(c.R_o, D + 3), _padded(c.O, D + 1)
    camA, camV = _sentinel(B, H, T, ldA), _sentinel(B * S, D + 2)
    L["check"](lib.mmx_lrp_attn_pv(p(Ro), D + 3, p(Od), D + 1, p(c.A_d), ldA, c.view(2), ld3, p(camA), p(camV), D + 2, B, H, T,
                                   S, hd, st()))
    vh = c._heads(c.v, S).double()
    rA, rV = olrp.pv_relprop(c._heads(c.R_o, T).double().reshape(B * H, T, hd), c.A.double().reshape(B * H, T, S),
                             vh.reshape(B * H, S, hd))
    errs = dict(pv_A=rel_err(camA[..., :S], rA.view(B, H, T, S) / 2),
                pv_V=rel_err(camV[:, :D], c._cols((rV / 2).view(B, H, S, hd), S)))
    assert (camA[..., S:] == 0).all() and torch.isnan(camV[:, D:]).all()

    zs = 1.0 / math.sqrt(hd)
    camQ, camK = _sentinel(B * T, D + 1), _sentinel(B * S, D + 3)
    L["check"](lib.mmx_lrp_attn_qk(p(c.cam1_d), ldA, c.view(0), ld3, c.view(1), ld3, C.c_float(zs), p(camQ), D + 1, p(camK),
                                   D + 3, B, H, T, S, hd, st()))
    qh = (c._heads(c.q, T).float() * zs).double().reshape(B * H, T, hd)
    kh = c._heads(c.k, S).double().reshape(B * H, S, hd)
    rQ, rK = olrp.scores_relprop(c.cam1.double().reshape(B * H, T, S), qh, kh)
    errs.update(qk_Q=rel_err(camQ[:, :D], c._cols((rQ / 2).view(B, H, T, hd), T)),
                qk_K=rel_err(camK[:, :D], c._cols((rK / 2).view(B, H, S, hd), S)))
    assert torch.isnan(camQ[:, D:]).all() and torch.isnan(camK[:, D:]).all()

    kb = torch.randn(B, S, generator=torch.Generator().manual_seed(hd)).cuda()
    ref_scores = (zs * (c._heads(c.q, T).double() @ c._heads(c.k, S).double().transpose(-1, -2)))
    for use_bias in (False, True):
        for use_mask in (False, True):
            scores = _sentinel(B, H, T, ldA)
            mask = _sentinel(B, H, T, ldA) if use_mask else None
            L["check"](lib.mmx_lrp_attn_scores(c.view(0), ld3, c.view(1), ld3, p(kb) if use_bias else None, C.c_float(zs),
                                               p(scores), p(mask), ldA, B, H, T, S, hd, st()))
            errs["scores"] = max(errs.get("scores", 0.0), rel_err(scores[..., :S], ref_scores))
            assert (scores[..., S:] == 0).all()
            if use_mask:
                want = kb[:, None, None, :].expand(B, H, T, S) if use_bias else torch.zeros(B, H, T, S, device="cuda")
                assert torch.equal(mask[..., :S], want) and (mask[..., S:] == 0).all()
    print("lrp attention", (B, H, T, S, hd), {k_: f"{v_:.1e}" for k_, v_ in errs.items()})
    assert max(errs.values()) < 2e-5


def test_lrp_attention_limits(L):
    """head_dim 65 and ldA < S raise MmxError on all three entry points"""
    lib, p, st = L["lib"], L["ptr"], L["st"]
    B, H, T, S = 1, 1, 4, 8
    buf = torch.zeros(64 * 65, device="cuda")
    for hd, ldA in ((65, 8), (16, 7)):
        with pytest.raises(L["MmxError"], match="head_dim"):
            L["check"](lib.mmx_lrp_attn_pv(p(buf), hd, p(buf), hd, p(buf), ldA, p(buf), hd, p(buf), p(buf), hd, B, H, T, S, hd,
                                           st()))
        with pytest.raises(L["MmxError"], match="head_dim"):
            L["check"](lib.mmx_lrp_attn_qk(p(buf), ldA, p(buf), hd, p(buf), hd, C.c_float(1.0), p(buf), hd, p(buf), hd, B, H, T,
                                           S, hd, st()))
        with pytest.raises(L["MmxError"], match="head_dim"):
            L["check"](lib.mmx_lrp_attn_scores(p(buf), hd, p(buf), hd, None, C.c_float(1.0), p(buf), None, ldA, B, H, T, S, hd,
                                               st()))


# ------------------------------------------------------------------------- single-pass attention, engine layouts
def _attn_ref(q, k, v, H, scale, causal, key_bias):
    """fp64 softmax(q scale k^T + key_bias (+ causal -inf)) v per head; A keeps its gradient"""
    B, T, Dm = q.shape
    S, hd = k.shape[1], Dm // H
    qh, kh, vh = (x.reshape(B, -1, H, hd).transpose(1, 2) for x in (q, k, v))
    s = (qh * scale) @ kh.transpose(-1, -2)
    if key_bias is not None:
        s = s + key_bias[:, None, None, :]
    if causal:
        s = s + torch.full((T, S), -INF, dtype=s.dtype).triu_(1)
    A = torch.softmax(s, -1)
    A.retain_grad()
    return A, (A @ vh).transpose(1, 2).reshape(B, T, Dm)


@pytest.mark.parametrize("B,H,S,hd,causal,bias", [(2, 12, 50, 64, 0, 0), (2, 8, 77, 64, 1, 1), (3, 4, 197, 32, 0, 1),
                                                  (1, 8, 300, 16, 1, 1), (2, 2, 17, 16, 1, 0)])
def test_attention_fused_qkv_strides(L, B, H, S, hd, causal, bias):
    """Q / K / V as column views of one fused [B*S, 3D] projection (ldq = ldk = ldv = 3D, K and V at column offsets D and
    2D), causal together with a key bias, forward and backward against fp64 with test_primitives_gpu.py's tolerances"""
    lib, check, p, st = L["lib"], L["check"], L["ptr"], L["st"]
    D = H * hd
    gen = torch.Generator().manual_seed(S * 3 + hd + causal)
    qkv = torch.randn(B * S, 3 * D, generator=gen)
    dO = torch.randn(B, S, D, generator=gen)
    kb = torch.randn(B, S, generator=gen) if bias else None
    q, k, v = (qkv[:, i * D:(i + 1) * D].reshape(B, S, D) for i in range(3))
    scale = 1.0 / math.sqrt(hd)
    ldA = (S + 3) // 4 * 4
    qkv_d, dOd = qkv.cuda(), dO.cuda()
    kbd = kb.cuda() if bias else None
    qp, kp, vp = (C.c_void_p(qkv_d.data_ptr() + 4 * i * D) for i in range(3))
    A = _sentinel(B, H, S, ldA, fill=7.0)
    O = _sentinel(B, S, D)
    check(lib.mmx_attention_fwd(qp, 3 * D, kp, 3 * D, vp, 3 * D, p(kbd), p(A), ldA, p(O), D, B, H, S, S, hd, C.c_float(scale),
                                causal, st()))
    dA = _sentinel(B, H, S, ldA, fill=7.0)
    delta = torch.empty(B, H, S, device="cuda")
    dq, dk, dv = (_sentinel(B, S, D) for _ in range(3))
    check(lib.mmx_attention_bwd_scaled(p(dOd), D, qp, 3 * D, kp, 3 * D, vp, 3 * D, p(A), p(dA), ldA, p(delta), p(dq), D, p(dk),
                                       D, p(dv), D, B, H, S, S, hd, C.c_float(scale), causal, None, st()))
    q64, k64, v64 = (t.double().requires_grad_(True) for t in (q, k, v))
    Ar, Or = _attn_ref(q64, k64, v64, H, scale, causal, kb.double() if bias else None)
    Or.backward(dO.double())
    errs = dict(A=rel_err(A[..., :S], Ar.detach()), O=rel_err(O, Or.detach()), dA=rel_err(dA[..., :S], Ar.grad),
                dq=rel_err(dq, q64.grad), dk=rel_err(dk, k64.grad), dv=rel_err(dv, v64.grad))
    print("fused-qkv attention", (B, H, S, hd, causal, bias), {k_: f"{v_:.1e}" for k_, v_ in errs.items()})
    assert errs["A"] < 5e-6 and errs["O"] < 5e-6 and errs["dA"] < 5e-6
    assert max(errs["dq"], errs["dk"], errs["dv"]) < 1e-5
    assert (A[..., S:] == 0).all() and (dA[..., S:] == 0).all()


@pytest.mark.parametrize("T,S,hd", [(50, 50, 64), (77, 77, 16), (100, 625, 32), (300, 1024, 32), (20, 36, 64)])
def test_attention_bwd_scaled_single_pass(L, T, S, hd):
    """mmx_attention_bwd_scaled on the single-pass kernels with gscale 2^12 and 2^-3 per sample: the staged dA equals the
    unscaled call's dA and dQ / dK / dV divided by gscale equal the unscaled results, to test_long_attention_gpu.py's
    bound"""
    lib, check, p, st = L["lib"], L["check"], L["ptr"], L["st"]
    B, H = 2, 256 // hd
    D = H * hd
    gen = torch.Generator().manual_seed(T + S + hd)
    q, k, v, dO = (torch.randn(B, n, D, generator=gen).cuda() for n in (T, S, S, T))
    scale = C.c_float(1.0 / math.sqrt(hd))
    ldA = (S + 3) // 4 * 4
    A, O = _sentinel(B, H, T, ldA), _sentinel(B, T, D)
    check(lib.mmx_attention_fwd(p(q), D, p(k), D, p(v), D, None, p(A), ldA, p(O), D, B, H, T, S, hd, scale, 0, st()))
    gs = torch.tensor([2.0 ** 12, 2.0 ** -3], device="cuda")

    def bwd(dO_, gscale):
        dA = _sentinel(B, H, T, ldA)
        delta = torch.empty(B, H, T, device="cuda")
        dq, dk, dv = _sentinel(B, T, D), _sentinel(B, S, D), _sentinel(B, S, D)
        check(lib.mmx_attention_bwd_scaled(p(dO_), D, p(q), D, p(k), D, p(v), D, p(A), p(dA), ldA, p(delta), p(dq), D, p(dk), D,
                                           p(dv), D, B, H, T, S, hd, scale, 0, p(gscale), st()))
        return dA, dq, dk, dv

    dA, dq, dk, dv = bwd(dO, None)
    dAs, dqs, dks, dvs = bwd(dO * gs.view(B, 1, 1), gs)
    errs = [rel_err(dAs[..., :S], dA[..., :S])] + [rel_err(xs / gs.view(B, 1, 1), x) for x, xs in ((dq, dqs), (dk, dks),
                                                                                                    (dv, dvs))]
    print("single-pass scaled vs unscaled (dA, dq, dk, dv)", (T, S, hd), [f"{e:.1e}" for e in errs])
    assert max(errs) < 1e-6
    assert (dAs[..., S:] == 0).all()
