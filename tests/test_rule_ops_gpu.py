"""GPU: the rule and evaluation-step kernels one op at a time through the C ABI - rule 5, attn-GradCAM, rules 6/7, eq. 8-9,
rules 10/11, rollout, min-max, Otsu and top-k - against fp64 restatements (or bit for bit against the fp32 torch
expression where the kernel does the same operations), at the layouts the Python wrappers never pass: padded row strides,
B > 1, both kernel paths, NaN and infinities.  Every output buffer starts as a NaN (or 7.0) sentinel, pad columns
included, so an unwritten element or a write into a pad shows."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from oracle import rules as orules
from util import rel_err

pytestmark = pytest.mark.gpu

NAN, INF = float("nan"), float("inf")
MM_NORMALIZE, MM_SELF_IN_10, MM_NAN_TO_ZERO = 1, 2, 4


@pytest.fixture(scope="module")
def L():
    import mmx_b200
    from mmx_b200._lib import lib, check, ptr, current_stream
    return dict(lib=lib(), check=check, ptr=ptr, st=current_stream, MmxError=mmx_b200.MmxError)


def _r4(n):
    return (n + 3) // 4 * 4


def _padded(x, ld, fill=NAN):
    """x [..., cols] (CPU) -> device [..., ld] with the pad columns set to `fill`"""
    buf = torch.full((*x.shape[:-1], ld), fill)
    buf[..., :x.shape[-1]] = x
    return buf.cuda()


def _sentinel(*shape, fill=NAN):
    return torch.full(shape, fill, device="cuda")


def assert_same(a, b):
    """the same floats bit for bit, except that any NaN matches any NaN (payloads differ between CPU and GPU)"""
    a, b = a.detach().cpu().float(), b.detach().cpu().float()
    assert a.shape == b.shape
    assert torch.equal(torch.isnan(a), torch.isnan(b)), "NaN positions differ"
    m = ~torch.isnan(b)
    assert torch.equal(a[m].view(torch.int32), b[m].view(torch.int32)), "values differ"


# ------------------------------------------------------------------------------------------------------------ rule 5
def _avg_heads(L, A, dA, ld_in, ld_out):
    """mmx_avg_heads of CPU [B,H,T,S] operands laid out with row strides ld_in / ld_out (NaN in every pad)"""
    B, H, T, S = A.shape
    Ad, dAd = _padded(A, ld_in), _padded(dA, ld_in)
    out = _sentinel(B, T, ld_out)
    L["check"](L["lib"].mmx_avg_heads(L["ptr"](Ad), L["ptr"](dAd), L["ptr"](out), B, H, T, S, ld_in, ld_out, L["st"]()))
    return out.cpu()


def _avg_heads64(A, dA):
    return (A.double() * dA.double()).clamp(min=0).mean(1)


@pytest.mark.parametrize("B,H,T,S", [(2, 1, 20, 36), (3, 3, 50, 52), (2, 8, 77, 77), (1, 12, 100, 100), (2, 11, 8, 40),
                                     (2, 3, 7, 13), (1, 12, 1, 3)])
def test_avg_heads_paths_vs_fp64(L, B, H, T, S):
    """The dense 128-bit kernel (ld = S, T*S % 4 == 0) and the strided scalar kernel sum the heads in the same order: the
    same data in both layouts gives the same bits, and both are within 1e-6 of fp64.  H = 3, 11 and 12 leave a remainder
    after the 8-head unroll; T*S % 4 != 0 sends the dense layout to the scalar kernel too."""
    gen = torch.Generator().manual_seed(B * 131 + H * 17 + S)
    A = torch.softmax(torch.randn(B, H, T, S, generator=gen), -1)
    dA = torch.randn(B, H, T, S, generator=gen)
    dense = _avg_heads(L, A, dA, S, S)
    strided = _avg_heads(L, A, dA, S + 5, S + 3)
    ref = _avg_heads64(A, dA)
    err = rel_err(dense, ref)
    print(f"avg_heads {(B, H, T, S)}: err {err:.1e}")
    assert err < 1e-6
    assert torch.equal(strided[..., :S], dense)
    assert torch.isnan(strided[..., S:]).all()                   # output pad columns are left alone


def test_avg_heads_nan_reaches_abar(L):
    """A NaN in A or in dA makes that Abar element NaN (clamp(min=0) propagates NaN) and touches nothing else"""
    B, H, T, S = 2, 5, 9, 16
    gen = torch.Generator().manual_seed(3)
    A = torch.rand(B, H, T, S, generator=gen)
    dA = torch.randn(B, H, T, S, generator=gen)
    A[0, 4, 2, 3] = NAN
    dA[1, 0, 8, 15] = NAN
    A[1, 2, 0, 0] = -1.0                                     # a negative product next to the NaN: clamped to 0
    ref = _avg_heads64(A, dA)
    for ld_in, ld_out in ((S, S), (S + 1, S + 2)):
        out = _avg_heads(L, A, dA, ld_in, ld_out)[..., :S]
        assert torch.isnan(out[0, 2, 3]) and torch.isnan(out[1, 8, 15])
        assert torch.isnan(out).sum() == 2
        assert rel_err(out.nan_to_num(0), ref.nan_to_num(0)) < 1e-6


# ------------------------------------------------------------------------------------------------------ attn-GradCAM
def _gradcam_case(L, B, H, T, S, ld_in, ld_out, gen):
    """Signed dA whose per-head mean nearly cancels (the plane mean is subtracted, then a small offset per head is added):
    the reduction's rounding is what the result is made of.  Returns the error of gbar (relative to |gbar|) and of the
    map (relative to max |A| |gbar|, the size of the terms it sums) against fp64."""
    A = torch.rand(B, H, T, S, device="cuda", generator=gen)
    dA = torch.randn(B, H, T, S, device="cuda", generator=gen)
    dA -= dA.mean((2, 3), keepdim=True)
    dA += torch.linspace(-2e-3, 1e-3, B * H, device="cuda").view(B, H, 1, 1)
    Ad = torch.full((B, H, T, ld_in), NAN, device="cuda"); Ad[..., :S] = A
    dAd = torch.full((B, H, T, ld_in), NAN, device="cuda"); dAd[..., :S] = dA
    del dA
    out, gbar = _sentinel(B, T, ld_out), _sentinel(B * H)
    L["check"](L["lib"].mmx_attn_gradcam(L["ptr"](Ad), L["ptr"](dAd), L["ptr"](out), L["ptr"](gbar), B, H, T, S, ld_in, ld_out,
                                         L["st"]()))
    g64 = dAd[..., :S].double().mean((2, 3))
    ref = (A.double() * g64[..., None, None]).mean(1).clamp(min=0)
    cond = (A.double() * g64.abs()[..., None, None]).mean(1)
    g_err = ((gbar.double().view(B, H) - g64).abs() / g64.abs()).max().item()
    m_err = rel_err(out[..., :S], ref, base=cond.cpu())
    assert torch.isnan(out[..., S:]).all()                   # output pad columns are left alone
    return g_err, m_err


def test_attn_gradcam_strided_batch_vs_fp64(L):
    """B*H = 6 planes, padded ld_in (NaN pads must not reach the mean), ld_out != ld_in"""
    gen = torch.Generator(device="cuda").manual_seed(11)
    g_err, m_err = _gradcam_case(L, 2, 3, 37, 50, 57, 53, gen)
    print(f"attn_gradcam B=2 H=3 37x50: gbar err {g_err:.1e}, map err {m_err:.1e}")
    assert g_err < 1e-6 and m_err < 1e-6


def test_attn_gradcam_long_plane_vs_fp64(L):
    """One DETR long-path plane, T = S = 2500: 6.25M gradient terms in one mean (about 24k per thread)"""
    gen = torch.Generator(device="cuda").manual_seed(12)
    g_err, m_err = _gradcam_case(L, 1, 2, 2500, 2500, 2504, 2500, gen)
    print(f"attn_gradcam long plane 2500x2500: gbar err {g_err:.1e}, map err {m_err:.1e}")
    assert g_err < 1e-6 and m_err < 1e-6


# ------------------------------------------------------------------------------------------------------- rules 6 + 7
def _self_update(L, Ab, R, Rq, ld_a, ld_ss, ld_sq):
    """mmx_self_update with zero-padded operands at the given row strides; returns (out_ss, out_sq, launches)"""
    B, S, _ = R.shape
    Q = Rq.shape[-1]
    Abd, Rd, Rqd = _padded(Ab, ld_a, 0.0), _padded(R, ld_ss, 0.0), _padded(Rq, ld_sq, 0.0)
    o, oq = _sentinel(B, S, ld_ss), _sentinel(B, S, ld_sq)
    lib, ptr = L["lib"], L["ptr"]
    n0 = lib.mmx_launch_count()
    L["check"](lib.mmx_self_update(ptr(Abd), ld_a, ptr(Rd), ptr(o), ld_ss, ptr(Rqd), ptr(oq), ld_sq, B, S, Q, L["st"]()))
    n = lib.mmx_launch_count() - n0
    return o.cpu(), oq.cpu(), n


@pytest.mark.parametrize("B", [1, 5])
@pytest.mark.parametrize("Q", [127, 128, 300])
@pytest.mark.parametrize("S", [127, 128, 129, 255])
def test_self_update_both_paths(L, B, S, Q):
    """Rules 6+7 around the tensor-core threshold (S, Q >= 128 with row strides % 4 == 0) and on the FFMA kernel (the
    same operands at odd row strides), against fp64; one sample alone gives the same bits as inside the batch"""
    gen = torch.Generator().manual_seed(S * 7 + Q + B)
    Ab = torch.rand(B, S, S, generator=gen) / S
    R = torch.eye(S) + torch.rand(B, S, S, generator=gen) * 0.1
    Rq = torch.rand(B, S, Q, generator=gen) * 0.1
    ref_ss = R.double() + Ab.double() @ R.double()
    ref_sq = Rq.double() + Ab.double() @ Rq.double()
    for path, lds, tol in (("ffma", (S + 1, S + 3, Q + 1), 1e-6), ("tc", (_r4(S) + 4, _r4(S) + 4, _r4(Q) + 4), 1e-5)):
        o, oq, launches = _self_update(L, Ab, R, Rq, *lds)
        e_ss, e_sq = rel_err(o[..., :S], ref_ss), rel_err(oq[..., :Q], ref_sq)
        print(f"self_update {path} B={B} S={S} Q={Q}: err ss {e_ss:.1e} sq {e_sq:.1e} ({launches} launches)")
        assert e_ss < tol and e_sq < tol
        if path == "ffma" or S < 128:
            assert launches == 2                               # one FFMA product per output
            assert torch.isnan(o[..., S:]).all() and torch.isnan(oq[..., Q:]).all()
        else:
            assert launches >= 2 + 1 + (Q >= 128)              # transpose + wgmma GEMM per tensor-core product
            assert torch.isnan(o[..., _r4(S):]).all() and torch.isnan(oq[..., _r4(Q):]).all()
        if B > 1:
            o1, oq1, _ = _self_update(L, Ab[3:4], R[3:4], Rq[3:4], *lds)
            assert torch.equal(o1[0, :, :S], o[3, :, :S]) and torch.equal(oq1[0, :, :Q], oq[3, :, :Q])


# --------------------------------------------------------------------------------------------------------- eq. 8-9
def _handle_residual64(R):
    eye = torch.eye(R.shape[-1], dtype=torch.float64)
    x = R.double() - eye
    return x / x.sum(-1, keepdim=True) + eye


def _handle_residual(L, R, ld):
    B, S, _ = R.shape
    Rd = _padded(R, ld)
    out = _sentinel(B, S, ld)
    md = _sentinel(1, fill=7.0)
    L["check"](L["lib"].mmx_handle_residual(L["ptr"](Rd), L["ptr"](out), ld, B, S, L["ptr"](md), L["st"]()))
    return out.cpu(), md.cpu()[0]


def test_handle_residual_batch_and_min_diag(L):
    """B = 3 samples of S = 100 (300 rows: more than one pass of the 256-thread min-diag loop), ld > S with NaN pads.
    *min_diag is the batch-wide fp32 min of diag(R - I): a negative entry in the last row of the last sample must be
    found, and a NaN on a diagonal must give NaN (the reference's `assert min >= 0` then fails)."""
    B, S, ld = 3, 100, 103
    gen = torch.Generator().manual_seed(21)
    R = torch.eye(S) + torch.rand(B, S, S, generator=gen) * 0.05
    out, md = _handle_residual(L, R, ld)
    err = rel_err(out[..., :S], _handle_residual64(R))
    print(f"handle_residual B=3 S=100: err {err:.1e}")
    assert err < 1e-6
    assert torch.isnan(out[..., S:]).all()
    diag = R.diagonal(dim1=-2, dim2=-1) - 1
    assert md.item() == diag.min().item()
    R[2, S - 1, S - 1] = 0.75                                    # diag(R - I) = -0.25, last row of the batch only
    _, md = _handle_residual(L, R, ld)
    assert md.item() == -0.25
    R[2, S - 1, S - 1] = R[0, 0, 0]
    R[1, 40, 40] = NAN
    _, md = _handle_residual(L, R, ld)
    assert math.isnan(md.item())


# ------------------------------------------------------------------------------------------------------ rules 10 + 11
class MmCase:
    """B = 3 samples of rules 10/11 operands, every row stride larger than its column count (NaN in the pads)"""

    def __init__(self, B, T, S, seed):
        gen = torch.Generator().manual_seed(seed)
        self.B, self.T, self.S = B, T, S
        self.R_ss = torch.eye(T) + torch.rand(B, T, T, generator=gen) * 0.05
        self.R_qq = torch.eye(S) + torch.rand(B, S, S, generator=gen) * 0.05
        self.R_qs = torch.rand(B, S, T, generator=gen) * 0.05
        self.cam = torch.rand(B, T, S, generator=gen) * 0.05
        self.ld = dict(ss=T + 3, qq=S + 5, qs=T + 2, a=S + 1, sq_add=S + 7, ss_add=T + 1)

    def run(self, L, flags, with_qs):
        B, T, S, ld = self.B, self.T, self.S, self.ld
        lib, ptr = L["lib"], L["ptr"]
        Rs, Rq, Ab = _padded(self.R_ss, ld["ss"]), _padded(self.R_qq, ld["qq"]), _padded(self.cam, ld["a"])
        Rqs = _padded(self.R_qs, ld["qs"]) if with_qs else None
        sq_add = _sentinel(B, T, ld["sq_add"])
        ss_add = _sentinel(B, T, ld["ss_add"]) if with_qs else None
        ws = _sentinel(lib.mmx_mm_update_workspace(B, T, S) // 4 + 4)
        md = _sentinel(2, fill=7.0)
        L["check"](lib.mmx_mm_update(ptr(Rs), ld["ss"], ptr(Rq), ld["qq"], ptr(Rqs), ld["qs"], ptr(Ab), ld["a"], ptr(sq_add),
                                     ld["sq_add"], ptr(ss_add), ld["ss_add"], B, T, S, flags, ptr(ws), ptr(md), L["st"]()))
        return sq_add.cpu(), (ss_add.cpu() if with_qs else None), md.cpu()

    def ref(self, b, flags):
        norm, s10 = bool(flags & MM_NORMALIZE), bool(flags & MM_SELF_IN_10)
        R_ss, R_qq, R_qs, cam = (x[b].double() for x in (self.R_ss, self.R_qq, self.R_qs, self.cam))
        sq, ss = orules.apply_mm_attention_rules_lxmert(R_ss, R_qq, R_qs, cam, norm, s10)
        if flags & MM_NAN_TO_ZERO:
            sq = orules.apply_mm_attention_rules_detr(R_ss, R_qq, cam, norm, s10)
        return sq, ss


@pytest.mark.parametrize("with_qs", [False, True])
@pytest.mark.parametrize("flags", range(8))
def test_mm_update_flags_vs_fp64(L, flags, with_qs):
    """All eight flag combinations, R_qs NULL and not, against oracle.rules per sample in fp64; both min_diag slots are
    the batch-wide minima when MMX_MM_NORMALIZE is set (also without MMX_MM_SELF_IN_10, where the product is discarded)
    and untouched otherwise; output pad columns are left alone"""
    case = MmCase(3, 20, 36, seed=31)
    sq_add, ss_add, md = case.run(L, flags, with_qs)
    T, S = case.T, case.S
    worst = 0.0
    for b in range(case.B):
        ref_sq, ref_ss = case.ref(b, flags)
        worst = max(worst, rel_err(sq_add[b, :, :S], ref_sq))
        if with_qs:
            worst = max(worst, rel_err(ss_add[b, :, :T], ref_ss))
    print(f"mm_update flags={flags} R_qs={'set' if with_qs else 'NULL'}: err {worst:.1e}")
    assert worst < 1e-5
    assert torch.isnan(sq_add[..., S:]).all()
    if with_qs:
        assert torch.isnan(ss_add[..., T:]).all()
    if flags & MM_NORMALIZE:
        assert md[0].item() == (case.R_ss.diagonal(dim1=-2, dim2=-1) - 1).min().item()
        assert md[1].item() == (case.R_qq.diagonal(dim1=-2, dim2=-1) - 1).min().item()
    else:
        assert (md == 7.0).all()


def test_mm_update_nan_to_zero_is_per_sample(L):
    """One row of sample 1's R_qq is an identity row, so eq. 8-9 gives 0/0 there and every element of that sample's
    rule-10 product is NaN.  MMX_MM_NAN_TO_ZERO zeroes exactly that sample; without it (LXMERT) that sample is all NaN
    and the other two are unchanged."""
    case = MmCase(3, 20, 36, seed=32)
    case.R_qq[1, 2] = torch.eye(case.S)[2]
    flags = MM_NORMALIZE | MM_SELF_IN_10
    detr, _, md = case.run(L, flags | MM_NAN_TO_ZERO, False)
    lx, _, _ = case.run(L, flags, False)
    S = case.S
    assert md[1].item() == 0.0
    assert (detr[1, :, :S] == 0).all() and torch.isnan(lx[1, :, :S]).all()
    for b in (0, 2):
        assert torch.isfinite(lx[b, :, :S]).all() and (lx[b, :, :S] > 0).all()
        assert torch.equal(detr[b, :, :S], lx[b, :, :S])
        assert rel_err(detr[b, :, :S], case.ref(b, flags | MM_NAN_TO_ZERO)[0]) < 1e-5
    assert torch.equal(detr[1, :, :S], case.ref(1, flags | MM_NAN_TO_ZERO)[0].float())


# ------------------------------------------------------------------------------------------------------------ rollout
@pytest.mark.parametrize("normalize", [0, 1])
@pytest.mark.parametrize("L_,start", [(1, 0), (4, 3), (4, 2), (4, 1), (4, 0)])
def test_rollout_vs_fp64(L, L_, start, normalize):
    """L = 1, start_layer = L-1 (no product), and 1, 2, 3 products (the ping-pong buffer that must end in `out` depends on
    their parity), B = 3, with and without the row normalisation"""
    B, S = 3, 45
    gen = torch.Generator().manual_seed(L_ * 10 + start)
    mats = torch.softmax(torch.randn(L_, B, S, S, generator=gen) * 2, -1)
    md = mats.cuda()
    out = _sentinel(B, S, S)
    ws = _sentinel(2, B, S, S)
    L["check"](L["lib"].mmx_rollout(L["ptr"](md), L_, B, S, start, normalize, L["ptr"](out), L["ptr"](ws), L["st"]()))
    ref = orules.compute_rollout_attention(list(mats.double()), start, normalize=bool(normalize))
    err = rel_err(out, ref)
    print(f"rollout L={L_} start={start} normalize={normalize}: err {err:.1e}")
    assert err < 1e-5


# ---------------------------------------------------------------------------------------------------------- min-max
def _minmax(L, x, inplace=False):
    B, n = x.shape
    xd = x.cuda()
    y = xd if inplace else _sentinel(B, n)
    L["check"](L["lib"].mmx_minmax_normalize(L["ptr"](xd), L["ptr"](y), B, n, L["st"]()))
    return y.cpu()


def _minmax_torch(x):
    mn, mx = x.min(-1, keepdim=True).values, x.max(-1, keepdim=True).values
    return (x - mn) / (mx - mn)


@pytest.mark.parametrize("n", [1, 255, 256, 257, 20000])
def test_minmax_normalize_bitwise(L, n):
    """The same fp32 subtraction and division as `(x - x.min()) / (x.max() - x.min())`: the same bits, per map, for 64 maps
    (n = 1 is a constant map: NaN); also in place"""
    gen = torch.Generator().manual_seed(n)
    x = torch.randn(64, n, generator=gen) * torch.logspace(-3, 3, 64).unsqueeze(1) + 0.5
    ref = _minmax_torch(x)
    assert_same(_minmax(L, x), ref)
    assert_same(_minmax(L, x, inplace=True), ref)


def test_minmax_normalize_non_finite(L):
    """A constant map gives NaN everywhere; maps with +inf, -inf or both give what torch gives; one NaN anywhere makes the
    whole map NaN, as torch's min() / max() propagate it"""
    gen = torch.Generator().manual_seed(5)
    n = 1000
    x = torch.randn(8, n, generator=gen)
    x[0] = 3.25                                   # constant
    x[1, 17] = INF
    x[2, 999] = -INF
    x[3, 0], x[3, 500] = INF, -INF
    x[4, 700] = NAN                               # one NaN
    x[5, 0] = NAN
    x[6] = NAN                                    # all NaN
    x[7, 300], x[7, 301] = INF, NAN
    y = _minmax(L, x)
    assert_same(y, _minmax_torch(x))
    assert torch.isnan(y[0]).all()
    assert torch.isnan(y[4:]).all()


# ------------------------------------------------------------------------------------------------------------- Otsu
def test_otsu_masks_degenerate_maps_bitwise(L):
    """mmx_otsu_masks against oracle.rules.otsu_masks (run on the host CPU, whose uint8 cast of NaN gives 0): an ordinary
    map, a constant map, a map with one NaN (NaN everywhere after the min-max, so threshold 0 and an all-zero mask) and an
    all-NaN map"""
    gen = torch.Generator().manual_seed(8)
    n = 1000
    cams = torch.rand(5, n, generator=gen) ** 3
    cams[1] = 0.5
    cams[2, 123] = NAN
    cams[3] = NAN
    cams[4, 999] = NAN
    cd = cams.cuda()
    masks, thr = _sentinel(5, n), torch.full((5,), -1, dtype=torch.int32, device="cuda")
    L["check"](L["lib"].mmx_otsu_masks(L["ptr"](cd), L["ptr"](masks), L["ptr"](thr), 5, n, L["st"]()))
    with np.errstate(invalid="ignore"):
        ref_m, ref_t = orules.otsu_masks(cams)
    assert (ref_m[2:] == 0).all() and (ref_t[2:] == 0).all()
    assert torch.equal(masks.cpu(), ref_m)
    assert thr.cpu().long().tolist() == ref_t.tolist()


# ------------------------------------------------------------------------------------------------------------ top-k
def _topk(L, scores, ks):
    B, n = scores.shape
    sd = scores.cuda()
    kd = torch.tensor(ks, dtype=torch.int32, device="cuda")
    keep = torch.full((B, n), -7, dtype=torch.int32, device="cuda")
    pos = torch.full((B, n), -7, dtype=torch.int32, device="cuda")
    L["check"](L["lib"].mmx_topk_select(L["ptr"](sd), L["ptr"](kd), L["ptr"](keep), L["ptr"](pos), B, n, L["st"]()))
    return keep.cpu(), pos.cpu()


def _topk_rule(row, k):
    """indices the kernel keeps: NaN first (lower index first), then by value, ties by lower index"""
    v = row.tolist()
    order = sorted(range(len(v)), key=lambda i: (0, 0.0, i) if math.isnan(v[i]) else (1, -v[i], i))
    return set(order[:max(0, min(k, len(v)))])


def _check_topk(scores, ks, keep, pos):
    for b, k in enumerate(ks):
        kept = keep[b].bool()
        n_kept = max(0, min(k, scores.shape[1]))
        assert set(torch.nonzero(kept).flatten().tolist()) == _topk_rule(scores[b], k), (b, k)
        assert kept.sum().item() == n_kept and set(keep[b].tolist()) <= {0, 1}
        assert torch.equal(pos[b][kept], torch.arange(n_kept, dtype=torch.int32))   # compacted, in index order
        assert (pos[b][~kept] == -1).all()


def test_topk_select_nan_ranks_first(L):
    """Rows of distinct scores with NaNs mixed in: the kept set is torch.topk's (NaN ranks above every number) whenever
    torch's choice is determined, exactly clamp(k, 0, n) elements are kept, and pos numbers them in index order"""
    gen = torch.Generator().manual_seed(13)
    n, n_nan = 300, 23
    ks = [0, 1, 5, n_nan - 1, n_nan, n_nan + 1, 100, n - 1, n, n + 5, -3]
    scores = torch.randn(len(ks), n, generator=gen)
    for b in range(len(ks)):
        scores[b, torch.randperm(n, generator=gen)[:n_nan]] = NAN
    keep, pos = _topk(L, scores, ks)
    _check_topk(scores, ks, keep, pos)
    for b, k in enumerate(ks):
        kk = max(0, min(k, n))
        t = torch.topk(scores[b], kk)
        assert torch.isnan(t.values).sum().item() == min(kk, n_nan)            # torch ranks NaN first too
        if kk >= n_nan:
            assert set(t.indices.tolist()) == set(torch.nonzero(keep[b]).flatten().tolist()), (b, k)


def test_topk_select_inf_and_all_nan_rows(L):
    """±inf rank between NaN and the numbers; an all-NaN row keeps its first k; a row of n = 4096 (the limit) works and
    n = 4097 raises MmxError"""
    gen = torch.Generator().manual_seed(14)
    n = 64
    rows = torch.randn(6, n, generator=gen)
    rows[0, [3, 9]] = INF
    rows[0, [4, 60]] = -INF
    rows[1, [3, 9]] = INF
    rows[1, 30] = NAN
    rows[1, [0, 63]] = -INF
    rows[2] = NAN
    rows[3] = NAN
    rows[4] = -INF
    rows[4, 50] = NAN
    rows[5, ::2] = NAN
    ks = [3, 4, 10, 0, 2, 40]
    keep, pos = _topk(L, rows, ks)
    _check_topk(rows, ks, keep, pos)
    assert keep[2, :10].all() and not keep[2, 10:].any()
    assert keep[4, 50] and keep[4, 0] and keep[4].sum() == 2
    n = 4096
    big = torch.randn(3, n, generator=gen)
    big[1, ::7] = NAN
    ks = [1, 2048, 4095]
    keep, pos = _topk(L, big, ks)
    _check_topk(big, ks, keep, pos)
    with pytest.raises(L["MmxError"], match="4096"):
        _topk(L, torch.zeros(1, 4097), [1])
