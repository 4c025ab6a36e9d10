"""GPU: the DETR backbone entry points one op at a time - mmx_conv2d / mmx_conv2d_dilated against fp64 F.conv2d, the NHWC
max-pool against F.max_pool2d, the mask / sine position embedding against the fp32 PositionEmbeddingSine restatement -
at the shapes, layouts and borders a whole ResNet never reaches (FFMA widths, Cout % 4 != 0, strided and unaligned
inputs, maps smaller than the kernel)."""
import contextlib
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

from util import rel_err

pytestmark = pytest.mark.gpu

NAN = float("nan")
ACT_NONE, ACT_GELU, ACT_RELU = 0, 2, 3
ACT_F = {ACT_NONE: lambda x: x, ACT_GELU: F.gelu, ACT_RELU: F.relu}


@pytest.fixture(scope="module")
def L():
    import mmx_b200
    from mmx_b200._lib import lib, check, ptr, current_stream
    return dict(lib=lib(), check=check, ptr=ptr, st=current_stream, MmxError=mmx_b200.MmxError)


@contextlib.contextmanager
def gemm_backend(lib, backend):
    """Runs the body under `backend` and puts back the backend and tile width it found, whatever happens."""
    prev_backend, prev_tile = lib.mmx_get_gemm_backend(), lib.mmx_set_gemm_tile_n(-1)
    try:
        if lib.mmx_set_gemm_backend(backend) != backend:
            pytest.skip("tensor-core backend not available")
        yield
    finally:
        lib.mmx_set_gemm_backend(prev_backend)
        lib.mmx_set_gemm_tile_n(prev_tile)


def _r4(n):
    return (n + 3) // 4 * 4


class ConvCase:
    """One conv: fp32 input [B, C, H, W], OIHW weight and bias on the CPU, the weight reordered to [Cout, kh*kw*C] in
    (ky, kx, c) order on the device, and its fp64 F.conv2d (before bias / residual / act)."""

    def __init__(self, B, C_, H, W, Cout, k, stride, pad, dil, seed):
        self.B, self.C, self.H, self.W, self.Cout, self.k = B, C_, H, W, Cout, k
        self.stride, self.pad, self.dil = stride, pad, dil
        gen = torch.Generator().manual_seed(seed)
        self.x = torch.randn(B, C_, H, W, generator=gen)
        self.w = torch.randn(Cout, C_, k, k, generator=gen) / math.sqrt(C_ * k * k)
        self.bias = torch.randn(Cout, generator=gen)
        self.Ho = (H + 2 * pad - dil * (k - 1) - 1) // stride + 1
        self.Wo = (W + 2 * pad - dil * (k - 1) - 1) // stride + 1
        self.M, self.K = B * self.Ho * self.Wo, k * k * C_
        self.res = torch.randn(self.M, Cout, generator=gen)
        self.wr = self.w.permute(0, 2, 3, 1).reshape(Cout, self.K).contiguous().cuda()
        self.bd = self.bias.cuda()
        self.ldres = _r4(Cout) + 8
        self.resd = torch.full((self.M, self.ldres), NAN)
        self.resd[:, :Cout] = self.res
        self.resd = self.resd.cuda()
        y = F.conv2d(self.x.double(), self.w.double(), stride=stride, padding=pad, dilation=dil)
        self.conv64 = y.permute(0, 2, 3, 1).reshape(self.M, Cout)

    def ref(self, bias, residual):
        r = self.conv64.clone()
        if bias:
            r += self.bias.double()
        if residual:
            r += self.res.double()
        return r

    def layout(self, name, x=None):
        """(device tensor kept alive, element strides sN, sY, sX, sC) of x [B, C, H, W] in one of the input layouts; pad
        columns and channels hold NaN, so a gather that reads them poisons the output."""
        x = self.x if x is None else x
        B, C_, H, W = x.shape
        if name == "nchw":
            return x.contiguous().cuda(), (C_ * H * W, W, 1, H * W)
        rows = x.permute(0, 2, 3, 1).reshape(B * H * W, C_)
        if name == "nhwc":
            return rows.contiguous().cuda(), (H * W * C_, W * C_, C_, 1)
        if name == "nhwc_ld":                    # padded row stride (the backbone's 128-row activations)
            ld = _r4(C_) + 8
            buf = torch.full((B * H * W, ld), NAN)
            buf[:, :C_] = rows
            return buf.cuda(), (H * W * ld, W * ld, ld, 1)
        if name == "nhwc_off":                   # channels 1 .. C of a wider matrix: 4 bytes off 16-byte alignment
            ld = C_ + 5
            buf = torch.full((B * H * W, ld), NAN)
            buf[:, 1:C_ + 1] = rows
            view = buf.cuda()[:, 1:]
            assert view.data_ptr() % 16 != 0
            return view, (H * W * ld, W * ld, ld, 1)
        raise ValueError(name)


LAYOUTS = ("nchw", "nhwc", "nhwc_ld", "nhwc_off")


def _conv(L, cc, xd, strides, packed, bias=False, residual=False, act=ACT_NONE, ldo=None, B=None):
    """mmx_conv2d_dilated (mmx_conv2d when the dilation is 1) into a NaN-filled [M, ldo] output; returns it."""
    lib, check, ptr, st = L["lib"], L["check"], L["ptr"], L["st"]
    B = cc.B if B is None else B
    M = B * cc.Ho * cc.Wo
    ldo = _r4(cc.Cout) + 4 if ldo is None else ldo
    out = torch.full((M, ldo), NAN, device="cuda")
    args = (ptr(xd), *strides, B, cc.H, cc.W, cc.C, ptr(cc.wr), cc.K, ptr(packed), ptr(cc.bd) if bias else None,
            ptr(cc.resd) if residual else None, cc.ldres, ptr(out), ldo, cc.Cout, cc.k, cc.k, cc.stride, cc.pad)
    if cc.dil == 1:
        check(lib.mmx_conv2d(*args, act, st()))
    else:
        check(lib.mmx_conv2d_dilated(*args, cc.dil, act, st()))
    return out


def _pack(L, Wd):
    N, K = Wd.shape
    buf = torch.empty(L["lib"].mmx_pack_weight_bytes(N, K), dtype=torch.uint8, device="cuda")
    L["check"](L["lib"].mmx_pack_weight(L["ptr"](Wd), Wd.stride(0), N, K, L["ptr"](buf), L["st"]()))
    return buf


# (name, B, C, H, W, Cout, k, stride, pad, dilation)
GEOMS = [
    ("stem7x7s2", 2, 3, 37, 53, 64, 7, 2, 3, 1),
    ("3x3s1_1x1", 2, 16, 1, 1, 130, 3, 1, 1, 1),
    ("3x3s1_2x3", 1, 32, 2, 3, 256, 3, 1, 1, 1),
    ("3x3s1_5x7", 2, 16, 5, 7, 128, 3, 1, 1, 1),
    ("3x3s1_13x9", 1, 64, 13, 9, 256, 3, 1, 1, 1),
    ("3x3s2_1x1", 2, 8, 1, 1, 3, 3, 2, 1, 1),
    ("3x3s2_2x3", 1, 16, 2, 3, 130, 3, 2, 1, 1),
    ("3x3s2_5x7", 2, 32, 5, 7, 256, 3, 2, 1, 1),
    ("3x3s2_13x9", 1, 16, 13, 9, 64, 3, 2, 1, 1),
    ("dc5_1row", 2, 32, 1, 6, 128, 3, 1, 2, 2),          # every tap off the middle row is padding
    ("dc5_2rows", 1, 16, 2, 5, 256, 3, 1, 2, 2),
    ("dc5_3rows", 2, 16, 3, 4, 130, 3, 1, 2, 2),
    ("dil2s2", 1, 8, 9, 11, 128, 3, 2, 2, 2),
    ("down1x1s2", 2, 64, 7, 5, 256, 1, 2, 0, 1),
    ("1x1_c32", 2, 32, 6, 5, 128, 1, 1, 0, 1),           # K = 32 < 64: FFMA
    ("1x1_c64", 2, 64, 6, 5, 128, 1, 1, 0, 1),
    ("1x1_c256", 1, 256, 5, 6, 256, 1, 1, 0, 1),
    ("c12_k108", 2, 12, 7, 6, 128, 3, 1, 1, 1),           # K = 108, not a multiple of 8 (backend-3 planes path)
]
# (backend, packed weight): every backend, and backend 3 without packed planes
BACKENDS = [(0, False), (1, False), (2, True), (3, True), (3, False)]


def _path(cc, strides, xd, backend, packed):
    """The code path a call takes, as a label for the error report: the 1x1 / stride-1 direct operand or the gather
    (fp32 patches, or fp16 planes under backend 3 with packed weights), then the product's kernel (the tensor cores take
    N >= 128, N % 4 == 0, K >= 64 and an aligned operand)."""
    sN, sY, sX, sC = strides
    direct = cc.k == 1 and cc.stride == 1 and cc.pad == 0 and sC == 1 and sY == cc.W * sX and sN == cc.H * sY
    tc = backend > 0 and cc.Cout >= 128 and cc.Cout % 4 == 0 and cc.K >= 64 and (
        not direct or (xd.data_ptr() % 16 == 0 and sX % 4 == 0))
    operand = "direct" if direct else ("planes" if tc and backend == 3 and packed else "patches")
    return operand + "/" + (("fp16x3" if packed else "tf32x3") if tc else "ffma")


@pytest.mark.parametrize("backend,packed", BACKENDS, ids=[f"b{b}{'p' if p else ''}" for b, p in BACKENDS])
def test_conv_vs_fp64(L, backend, packed):
    """Every geometry of GEOMS on this backend; the layout and epilogue rotate with the geometry so that each geometry
    meets every layout across the backends.  Pad columns of the output (ldo > Cout) keep their NaN sentinels."""
    tol = 5e-6 if backend == 0 else 2e-5
    worst = {}
    with gemm_backend(L["lib"], backend):
        for gi, (name, *g) in enumerate(GEOMS):
            cc = ConvCase(*g, seed=gi)
            bi = BACKENDS.index((backend, packed))
            layout = LAYOUTS[(gi + bi) % 4]
            bias, residual = bool((gi + bi) & 1), bool((gi + 2 * bi) & 2)
            act = (ACT_NONE, ACT_RELU, ACT_GELU)[(gi + 2 * bi) % 3]
            xd, strides = cc.layout(layout)
            pk = _pack(L, cc.wr) if packed else None
            out = _conv(L, cc, xd, strides, pk, bias, residual, act)
            ref = cc.ref(bias, residual)
            e = rel_err(out[:, :cc.Cout], ACT_F[act](ref), base=ref)
            what = (name, layout, bias, residual, act)
            assert e < tol, (what, e)
            assert torch.isnan(out[:, cc.Cout:]).all(), what
            p = _path(cc, strides, xd, backend, packed)
            worst[p] = max(worst.get(p, 0.0), e)
    print(f"conv backend {backend}{' packed' if packed else ''}: worst error per path " +
          ", ".join(f"{k} {v:.1e}" for k, v in sorted(worst.items())))


@pytest.mark.parametrize("backend,packed", BACKENDS, ids=[f"b{b}{'p' if p else ''}" for b, p in BACKENDS])
def test_conv_bit_identities(L, backend, packed):
    """The same values as NCHW, NHWC, NHWC with padded rows and an unaligned channel-offset NHWC view give the same bits;
    an image alone equals the same image inside a batch; tile widths 128 / 144 / 160 give the same bits."""
    with gemm_backend(L["lib"], backend):
        for gi, g in enumerate([(3, 16, 5, 7, 128, 3, 1, 1, 1), (2, 8, 9, 6, 64, 3, 2, 1, 1), (2, 16, 3, 5, 256, 3, 1, 2, 2),
                                (3, 3, 21, 18, 64, 7, 2, 3, 1)]):
            cc = ConvCase(*g, seed=100 + gi)
            pk = _pack(L, cc.wr) if packed else None
            outs = {lay: _conv(L, cc, *cc.layout(lay), pk, True, True, ACT_RELU) for lay in LAYOUTS}
            for lay in LAYOUTS[1:]:
                assert torch.equal(outs[lay][:, :cc.Cout], outs["nchw"][:, :cc.Cout]), (g, lay)
            # image 1 alone == rows of image 1 in the batch (the GEMM path never depends on M)
            x1 = cc.x[1:2]
            xd, strides = cc.layout("nhwc", x1)
            n = cc.Ho * cc.Wo
            cc_res = cc.resd
            cc.resd = cc_res[n:2 * n]
            one = _conv(L, cc, xd, strides, pk, True, True, ACT_RELU, B=1)
            cc.resd = cc_res
            assert torch.equal(one[:, :cc.Cout], outs["nhwc"][n:2 * n, :cc.Cout]), g
        if backend >= 1:
            cc = ConvCase(2, 32, 9, 11, 256, 3, 1, 1, 1, seed=7)
            pk = _pack(L, cc.wr) if packed else None
            xd, strides = cc.layout("nhwc")
            by_tile = {}
            for bn in (128, 144, 160):
                assert L["lib"].mmx_set_gemm_tile_n(bn) == bn
                by_tile[bn] = _conv(L, cc, xd, strides, pk, True, False, ACT_GELU)
            for bn in (144, 160):
                assert torch.equal(by_tile[bn][:, :cc.Cout], by_tile[128][:, :cc.Cout]), bn


def test_conv_1x1_direct_equals_gathered_planes(L):
    """Backend 3, C % 8 == 0: a 1x1 / stride-1 conv over NHWC rows reads the activation itself (the GEMM's own split pass)
    and over NCHW gathers the fp16 planes; the split is the same, so the bits are."""
    with gemm_backend(L["lib"], 3):
        for C_, Cout in ((64, 256), (256, 128), (72, 128)):
            cc = ConvCase(2, C_, 7, 9, Cout, 1, 1, 0, 1, seed=C_ + Cout)
            pk = _pack(L, cc.wr)
            direct = _conv(L, cc, *cc.layout("nhwc"), pk, True, True, ACT_RELU)
            gathered = _conv(L, cc, *cc.layout("nchw"), pk, True, True, ACT_RELU)
            assert torch.equal(direct[:, :Cout], gathered[:, :Cout]), (C_, Cout)
            assert rel_err(direct[:, :Cout], F.relu(cc.ref(True, True)), base=cc.ref(True, True)) < 2e-5


def test_conv_nan_reaches_relu(L):
    """A NaN pixel makes every output pixel whose window covers it NaN through the fused ReLU, on every backend."""
    for backend, packed in BACKENDS:
        with gemm_backend(L["lib"], backend):
            cc = ConvCase(1, 16, 6, 7, 128, 3, 1, 1, 1, seed=3)
            x = cc.x.clone()
            x[0, 5, 2, 3] = NAN
            pk = _pack(L, cc.wr) if packed else None
            out = _conv(L, cc, *cc.layout("nhwc", x), pk, True, False, ACT_RELU)[:, :cc.Cout].cpu()
            hit = torch.zeros(cc.Ho, cc.Wo, dtype=torch.bool)
            hit[1:4, 2:5] = True
            hit = hit.reshape(-1)
            assert torch.isnan(out[hit]).all(), (backend, packed)
            assert torch.isfinite(out[~hit]).all(), (backend, packed)


def _maxpool(L, x_nchw, ldi_pad=3, ldo_pad=5):
    B, C_, H, W = x_nchw.shape
    ldi, ldo = C_ + ldi_pad, C_ + ldo_pad
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    inp = torch.full((B * H * W, ldi), NAN)
    inp[:, :C_] = x_nchw.permute(0, 2, 3, 1).reshape(-1, C_)
    inp = inp.cuda()
    out = torch.full((B * Ho * Wo, ldo), 7.0, device="cuda")
    L["check"](L["lib"].mmx_maxpool2d_nhwc(L["ptr"](inp), ldi, L["ptr"](out), ldo, B, H, W, C_, L["st"]()))
    out = out.cpu()
    assert (out[:, C_:] == 7.0).all()                 # pad columns untouched
    return out[:, :C_].reshape(B, Ho, Wo, C_).permute(0, 3, 1, 2)


def _same_bits(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


@pytest.mark.parametrize("C_", [1, 3, 64, 130])
def test_maxpool_vs_torch(L, C_):
    """3x3 / 2 / pad 1 max-pool == F.max_pool2d bit for bit on every map size in {1, 2, 3, 4, 7, 8, 13}^2, with random
    values and with all-negative ones (padding that acted as 0 instead of -inf would show at the borders)."""
    sizes = (1, 2, 3, 4, 7, 8, 13)
    gen = torch.Generator().manual_seed(C_)
    for H in sizes:
        for W in sizes:
            x = torch.randn(2, C_, H, W, generator=gen)
            for xs in (x, -(x.abs() + 0.25)):
                assert _same_bits(_maxpool(L, xs), F.max_pool2d(xs, 3, 2, 1)), (H, W)


def test_maxpool_nonfinite(L):
    """NaN at the first, middle and last tap of a window propagates as in F.max_pool2d; +-inf are ordinary maxima."""
    x = -torch.rand(1, 3, 7, 7) - 1.0
    x[0, 0, 0, 0] = NAN                   # first real tap of output (0, 0)
    x[0, 0, 3, 3] = NAN                   # last tap of output (1, 1), first tap of output (2, 2)
    x[0, 1, 2, 2] = NAN                   # middle tap of output (1, 1)
    x[0, 1, 6, 6] = NAN                   # last tap of output (3, 3), whose window hangs over the bottom-right border
    x[0, 2, 1, 1] = float("inf")
    x[0, 2, 6, 6] = float("-inf")
    x[0, 2, 4, 0] = NAN
    x[0, 2, 4, 1] = float("inf")
    got, want = _maxpool(L, x), F.max_pool2d(x, 3, 2, 1)
    assert torch.isnan(want).any() and torch.isinf(want).any()
    assert _same_bits(got, want)


def _pos_ref(mask, h, w, npf, T):
    from oracle.detr_backbone_oracle import position_sine
    m = F.interpolate(mask[None].float(), size=(h, w)).bool()[0]
    pos = position_sine(m, npf, T)
    return pos.permute(0, 2, 3, 1).reshape(-1, 2 * npf), m


def _pos(L, mask, B, Hi, Wi, h, w, npf, T=10000.0, ldpos=None, want_mask=True):
    ldpos = 2 * npf if ldpos is None else ldpos
    pos = torch.full((B * h * w, ldpos), NAN, device="cuda")
    mo = torch.full((B, h, w), 7, dtype=torch.uint8, device="cuda") if want_mask else None
    md = None if mask is None else mask.to(torch.uint8).contiguous().cuda()
    L["check"](L["lib"].mmx_detr_position_sine(L["ptr"](md), B, Hi, Wi, h, w, npf, C.c_float(T), L["ptr"](pos), ldpos,
                                               L["ptr"](mo), L["st"]()))
    if ldpos > 2 * npf:
        assert torch.isnan(pos[:, 2 * npf:]).all()
    return pos[:, :2 * npf].cpu(), None if mo is None else mo.cpu()


def _padding_masks(Hi, Wi, gen):
    """B = 3: rectangular padding (a valid top-left region), an irregular random mask, a fully padded image."""
    m = torch.zeros(3, Hi, Wi, dtype=torch.bool)
    m[0, (Hi * 5) // 7:, :] = True
    m[0, :, (Wi * 2) // 3:] = True
    m[1] = torch.rand(Hi, Wi, generator=gen) < 0.3
    m[2] = True
    return m


@pytest.mark.parametrize("Hi,Wi,h,w,npf,T", [
    (97, 130, 4, 5, 128, 10000.0), (1199, 800, 38, 25, 128, 10000.0),    # non-integer resampling ratios
    (40, 9, 13, 1, 16, 20.0), (9, 40, 1, 13, 1024, 10000.0), (5, 5, 1, 1, 16, 10000.0),
    (256, 256, 128, 128, 16, 10000.0),                                    # h w = 16384, the largest map
    (111, 87, 37, 29, 64, 20.0)])                                          # h w = 1073: the last CTA is partial
def test_position_sine_vs_reference(L, Hi, Wi, h, w, npf, T):
    """pos within 1e-6 absolute of PositionEmbeddingSine(npf, T, normalize=True) of the F.interpolate-resampled mask
    (fp32 on the CPU), mask_out exact, for three different masks in one batch; a NULL mask equals an all-zero mask bit
    for bit; ldpos > 2 npf keeps the pad columns; mask_out may be NULL."""
    gen = torch.Generator().manual_seed(h * w + npf)
    mask = _padding_masks(Hi, Wi, gen)
    ref, mref = _pos_ref(mask, h, w, npf, T)
    pos, mo = _pos(L, mask, 3, Hi, Wi, h, w, npf, T, ldpos=2 * npf + 12)
    err = (pos - ref).abs().max().item()
    assert err <= 1e-6, err
    assert torch.equal(mo.bool(), mref) and mo.max().item() <= 1
    pos2, _ = _pos(L, mask, 3, Hi, Wi, h, w, npf, T, want_mask=False)
    assert torch.equal(pos2, pos)
    zero = torch.zeros(2, Hi, Wi, dtype=torch.bool)
    p0, m0 = _pos(L, zero, 2, Hi, Wi, h, w, npf, T)
    pn, mn = _pos(L, None, 2, 0, 0, h, w, npf, T)
    assert _same_bits(pn, p0) and torch.equal(mn, m0) and not m0.any()
    assert (_pos_ref(zero, h, w, npf, T)[0] - p0).abs().max().item() <= 1e-6
    print(f"position_sine {Hi}x{Wi} -> {h}x{w}, npf {npf}, T {T:g}: max abs err {err:.1e}")


def test_argument_checks(L):
    """Host-side checks raise MmxError instead of launching: a kernel larger than the padded input, ldo < Cout, and a
    position map larger than 16384 positions."""
    lib, ptr, st = L["lib"], L["ptr"], L["st"]
    xd = torch.zeros(1, 8, 2, 2, device="cuda")                 # NCHW, C = 8, 2 x 2
    strides = (32, 2, 1, 4)
    w7, w3 = torch.zeros(128, 7 * 7 * 8, device="cuda"), torch.zeros(128, 3 * 3 * 8, device="cuda")
    out = torch.empty(16, 132, device="cuda")
    with pytest.raises(L["MmxError"]):                           # 7x7 over 2 + 2 * 1 pixels
        L["check"](lib.mmx_conv2d(ptr(xd), *strides, 1, 2, 2, 8, ptr(w7), 392, None, None, None, 0, ptr(out), 132, 128,
                                  7, 7, 1, 1, 0, st()))
    with pytest.raises(L["MmxError"]):                           # dilation 2: 13-pixel taps over 2 + 2 * 3
        L["check"](lib.mmx_conv2d_dilated(ptr(xd), *strides, 1, 2, 2, 8, ptr(w7), 392, None, None, None, 0, ptr(out), 132,
                                          128, 7, 7, 1, 3, 2, 0, st()))
    with pytest.raises(L["MmxError"]):                           # ldo 64 < Cout 128
        L["check"](lib.mmx_conv2d(ptr(xd), *strides, 1, 2, 2, 8, ptr(w3), 72, None, None, None, 0, ptr(out), 64, 128,
                                  3, 3, 1, 1, 0, st()))
    pos = torch.empty(129 * 128 * 32, device="cuda")
    with pytest.raises(L["MmxError"]):
        L["check"](lib.mmx_detr_position_sine(None, 1, 0, 0, 129, 128, 16, C.c_float(10000.0), ptr(pos), 32, None, st()))
    torch.cuda.synchronize()
