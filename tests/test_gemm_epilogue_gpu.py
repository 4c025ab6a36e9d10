"""GPU: the general GEMM entry point (mmx_gemm_nt) with every epilogue, the standalone activations and the glue kernels,
called through the C ABI and compared with plain PyTorch: fp64 on the CPU for the products, torch fp32 on the device for
the elementwise activations, exact bits for the copies.  Non-finite inputs are data here: a NaN or an fp16x3 overflow
must reach the caller, through every activation."""
import contextlib
import math

import pytest
import torch
import torch.nn.functional as F

from util import rel_err

pytestmark = pytest.mark.gpu

NAN = float("nan")
INF = float("inf")


@pytest.fixture(scope="module")
def L():
    import mmx_b200
    from mmx_b200._lib import lib, check, ptr, current_stream
    return dict(lib=lib(), check=check, ptr=ptr, st=current_stream)


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


def _pack(L, Wd):
    """fp16x3 packed copy of a device [N, K] matrix (row stride Wd.stride(0))."""
    N, K = Wd.shape
    buf = torch.empty(L["lib"].mmx_pack_weight_bytes(N, K), dtype=torch.uint8, device="cuda")
    L["check"](L["lib"].mmx_pack_weight(L["ptr"](Wd), Wd.stride(0), N, K, L["ptr"](buf), L["st"]()))
    return buf


def _padded(rows, cols, ld, gen, fill=NAN, scale=1.0):
    """A [rows, cols] view (row stride ld) of a device buffer whose pad columns hold `fill` (NaN: a kernel that reads
    them poisons its result)."""
    buf = torch.full((rows, ld), fill)
    buf[:, :cols] = torch.randn(rows, cols, generator=gen) * scale
    return buf.cuda()[:, :cols]


# act(x) in the precision of x (fp64 reference / fp32 device), and ACT_MUL: the epilogue's C_act of MUL is C itself
ACT_F = {0: lambda x: x, 1: lambda x: x * torch.sigmoid(1.702 * x), 2: F.gelu, 3: F.relu, 4: torch.tanh,
         5: lambda x: x, 6: torch.sigmoid}
ACT_NAMES = {0: "none", 1: "quickgelu", 2: "gelu", 3: "relu", 4: "tanh", 5: "mul", 6: "sigmoid"}


def _act_grad(act, pre):
    """act'(pre) by autograd in the precision of pre; ACT_MUL multiplies by pre itself."""
    if act == 5:
        return pre.clone()
    p = pre.detach().clone().requires_grad_(True)
    ACT_F[act](p).sum().backward()
    return p.grad


# (name, M, N, K, row strides / A offset): the FFMA kernel (N < 128), the tensor cores with K % 32 != 0, K % 8 != 0,
# padded lda / ldb / ldc / ldpre / ldres, and an A one float off 16-byte alignment (every backend falls back to FFMA)
SHAPES = [("ffma", 37, 96, 64, {}), ("tc_k200", 300, 260, 200, {}), ("k76", 129, 384, 76, {}),
          ("padded_ld", 200, 256, 96, dict(lda=100, ldb=108, ldc=264, ldpre=260, ldres=268)),
          ("a_offset", 160, 256, 128, dict(a_off=1))]
CMODES = ("none", "separate", "same")


def _combos(backend, si):
    """A deterministic subset of (act, bias, pre, residual, C_act mode): two per act, rotated by backend and shape so that
    the whole set covers every mode of every act."""
    out = []
    for act in range(7):
        for j in range(2):
            bits = (3 * act + 5 * j + 2 * si + backend) % 8
            cmode = CMODES[(act + j + si + backend) % 3]
            pre = bool(bits & 2) or act == 5          # ACT_MUL without pre is a plain product
            out.append((act, bool(bits & 1), pre, bool(bits & 4), cmode))
    return out


@pytest.mark.parametrize("backend", [0, 1, 2, 3])
@pytest.mark.parametrize("si", range(len(SHAPES)), ids=[s[0] for s in SHAPES])
def test_gemm_nt_epilogues(L, backend, si):
    """C = ((A Bt^T + bias) (.) act'(pre)) + residual and C_act = act(C) against fp64, for every act and C_act mode; the pad
    columns of C / C_act (ldc > N) keep their NaN sentinels."""
    lib, check, ptr, st = L["lib"], L["check"], L["ptr"], L["st"]
    name, M, N, K, o = SHAPES[si]
    lda, ldb, ldc = o.get("lda", K), o.get("ldb", K), o.get("ldc", N)
    ldpre, ldres = o.get("ldpre", N), o.get("ldres", N)
    tol = 5e-6 if backend == 0 else 2e-5
    gen = torch.Generator().manual_seed(1000 * si + 17)
    if o.get("a_off"):
        flat = torch.randn(M * K + 1, generator=gen).cuda()
        Ad = flat[1:].view(M, K)
        assert Ad.data_ptr() % 16 != 0
    else:
        Ad = _padded(M, K, lda, gen)
    Bd = _padded(N, K, ldb, gen, scale=1 / math.sqrt(K))
    bias = torch.randn(N, generator=gen).cuda()
    pre = _padded(M, N, ldpre, gen)
    res = _padded(M, N, ldres, gen)
    A64, B64 = Ad.cpu().double(), Bd.cpu().double()
    prod = A64 @ B64.t()
    worst = 0.0
    with gemm_backend(lib, backend):
        pk = _pack(L, Bd) if backend >= 2 else None
        for act, use_bias, use_pre, use_res, cmode in _combos(backend, si):
            Cbuf = torch.full((M, ldc), NAN, device="cuda")
            Abuf = torch.full((M, ldc), NAN, device="cuda") if cmode == "separate" else None
            C_act = {"none": None, "separate": Abuf, "same": Cbuf}[cmode]
            check(lib.mmx_gemm_nt(ptr(Ad), Ad.stride(0), ptr(Bd), Bd.stride(0), ptr(pk), ptr(bias) if use_bias else None,
                                  ptr(pre) if use_pre else None, ldpre, ptr(res) if use_res else None, ldres, ptr(Cbuf), ldc,
                                  ptr(C_act), act, M, N, K, st()))
            ref = prod.clone()
            if use_bias:
                ref += bias.cpu().double()
            if use_pre:
                ref *= _act_grad(act, pre.cpu().double())
            if use_res:
                ref += res.cpu().double()
            what = (ACT_NAMES[act], use_bias, use_pre, use_res, cmode)
            if cmode != "same":
                e = rel_err(Cbuf[:, :N], ref)
                worst = max(worst, e)
                assert e < tol, (what, e)
            if cmode != "none":
                got = (Abuf if cmode == "separate" else Cbuf)[:, :N]
                e = rel_err(got, ACT_F[act](ref), base=ref)
                worst = max(worst, e)
                assert e < tol, (what, e)
            for buf in (Cbuf, Abuf):
                if buf is not None:
                    assert torch.isnan(buf[:, N:]).all(), what      # pad columns untouched
    print(f"gemm_nt {name} ({M}x{N}x{K}) backend {backend}: worst error {worst:.1e}")


def _nan_mask_equal(a, b):
    return torch.equal(torch.isnan(a), torch.isnan(b))


@pytest.mark.parametrize("backend", [0, 1, 2, 3])
def test_gemm_nt_nan_reaches_every_act(L, backend):
    """A NaN in row r of A makes row r of C and of C_act NaN for every act (ReLU included, as F.relu does), separate or
    C_act == C; every other row stays finite and correct.  A NaN `pre` of the ReLU dgrad passes the gradient through, as
    torch's threshold_backward does."""
    lib, check, ptr, st = L["lib"], L["check"], L["ptr"], L["st"]
    M, N, K, r = 160, 256, 128, 37
    tol = 5e-6 if backend == 0 else 2e-5
    gen = torch.Generator().manual_seed(5)
    A = torch.randn(M, K, generator=gen)
    A[r, 7] = NAN
    W = torch.randn(N, K, generator=gen) / math.sqrt(K)
    bias = torch.randn(N, generator=gen)
    Ad, Wd, bd = A.cuda(), W.cuda(), bias.cuda()
    ref = A.double() @ W.double().t() + bias.double()
    others = torch.arange(M) != r
    with gemm_backend(lib, backend):
        pk = _pack(L, Wd) if backend >= 2 else None
        for act in range(7):
            C = torch.empty(M, N, device="cuda")
            Ca = torch.empty(M, N, device="cuda")
            check(lib.mmx_gemm_nt(ptr(Ad), K, ptr(Wd), K, ptr(pk), ptr(bd), None, 0, None, 0, ptr(C), N, ptr(Ca), act, M, N, K,
                                  st()))
            Cs = torch.empty(M, N, device="cuda")
            check(lib.mmx_gemm_nt(ptr(Ad), K, ptr(Wd), K, ptr(pk), ptr(bd), None, 0, None, 0, ptr(Cs), N, ptr(Cs), act, M, N, K,
                                  st()))
            C, Ca, Cs = C.cpu(), Ca.cpu(), Cs.cpu()
            assert torch.isnan(C[r]).all(), ACT_NAMES[act]
            assert torch.isnan(Ca[r]).all(), ACT_NAMES[act]
            assert torch.isnan(Cs[r]).all(), ACT_NAMES[act]
            assert torch.isfinite(Ca[others]).all() and torch.isfinite(Cs[others]).all(), ACT_NAMES[act]
            assert rel_err(C[others], ref[others]) < tol
            assert rel_err(Ca[others], ACT_F[act](ref[others]), base=ref[others]) < tol
            assert torch.equal(Cs[others], Ca[others]), ACT_NAMES[act]
        # dgrad through ReLU: where pre is NaN the gradient passes (relu(NaN) = NaN is not <= 0), elsewhere relu'(pre)
        pre = torch.randn(M, N, generator=gen)
        pre[3, 5] = NAN
        pre[4, :] = NAN
        A2d, pred = torch.randn(M, K, generator=gen).cuda(), pre.cuda()
        C = torch.empty(M, N, device="cuda")
        check(lib.mmx_gemm_nt(ptr(A2d), K, ptr(Wd), K, ptr(pk), None, ptr(pred), N, None, 0, ptr(C), N, None, 3, M, N, K, st()))
        p = A2d.cpu().double() @ W.double().t()
        want = torch.where(torch.isnan(pre), p, p * (pre > 0).double())
        assert rel_err(C, want, base=p) < tol


@pytest.mark.parametrize("backend", [2, 3])
def test_f16x3_overflow_reaches_relu(L, backend):
    """fp16x3 with packed weights: an A entry of 7e4 (above fp16's 65504) turns its row of C into NaN; the fused ReLU must
    pass the NaN on (fmaxf(NaN, 0) would turn it into 0, a finite and wrong relevance)."""
    lib, check, ptr, st = L["lib"], L["check"], L["ptr"], L["st"]
    M, N, K, r = 256, 256, 512, 3
    gen = torch.Generator().manual_seed(11)
    A = torch.randn(M, K, generator=gen)
    A[r, 5] = 7.0e4
    # |w| in [0.5, 1.5] / sqrt(K): the hi and lo fp16 passes of the overflowing entry are +inf and -inf, which sum to NaN
    W = (torch.rand(N, K, generator=gen) + 0.5) * torch.sign(torch.randn(N, K, generator=gen)) / math.sqrt(K)
    Ad, Wd = A.cuda(), W.cuda()
    others = torch.arange(M) != r
    with gemm_backend(lib, backend):
        pk = _pack(L, Wd)
        C = torch.empty(M, N, device="cuda")
        Ca = torch.empty(M, N, device="cuda")
        check(lib.mmx_gemm_nt(ptr(Ad), K, ptr(Wd), K, ptr(pk), None, None, 0, None, 0, ptr(C), N, ptr(Ca), 3, M, N, K, st()))
        Cs = torch.empty(M, N, device="cuda")
        check(lib.mmx_gemm_nt(ptr(Ad), K, ptr(Wd), K, ptr(pk), None, None, 0, None, 0, ptr(Cs), N, ptr(Cs), 3, M, N, K, st()))
    C, Ca, Cs = C.cpu(), Ca.cpu(), Cs.cpu()
    assert torch.isnan(C[r]).any()
    assert not torch.isfinite(Ca[r]).any() and _nan_mask_equal(Ca[r], C[r])
    assert not torch.isfinite(Cs[r]).any() and _nan_mask_equal(Cs[r], C[r])
    assert torch.isfinite(C[others]).all() and torch.equal(Ca[others], F.relu(C[others]))
    assert torch.equal(Cs[others], Ca[others])
    ref = A.double() @ W.double().t()
    assert rel_err(C[others], ref[others]) < 2e-5


# inputs of the elementwise tests: a random body plus the values where activations saturate or are not finite
SPECIALS = [30.0, -30.0, 100.0, -100.0, 0.0, -0.0, INF, -INF, NAN]


def _act_inputs(rows, cols, gen):
    x = torch.randn(rows, cols, generator=gen) * 3
    flat = x.view(-1)
    idx = torch.randperm(rows * cols, generator=gen)[:4 * len(SPECIALS)]
    for i, j in enumerate(idx.tolist()):
        flat[j] = SPECIALS[i % len(SPECIALS)]
    return x


def _assert_close_nonfinite(got, ref, rtol, atol, what):
    """NaN and +-inf at exactly torch's positions, finite values within rtol / atol."""
    got, ref = got.cpu(), ref.cpu()
    assert _nan_mask_equal(got, ref), what
    assert torch.equal(torch.isposinf(got), torch.isposinf(ref)), what
    assert torch.equal(torch.isneginf(got), torch.isneginf(ref)), what
    f = torch.isfinite(ref)
    err = (got[f].double() - ref[f].double()).abs()
    assert (err <= atol + rtol * ref[f].double().abs()).all(), (what, err.max().item())


@pytest.mark.parametrize("act", range(7), ids=[ACT_NAMES[a] for a in range(7)])
def test_act_fwd_bwd(L, act):
    """mmx_act_fwd / mmx_act_bwd against torch fp32 on the device, on strided rows (rows * cols = 1665, not a multiple of
    256) that include +-30, +-100, +-0, +-inf and NaN."""
    lib, check, ptr, st = L["lib"], L["check"], L["ptr"], L["st"]
    rows, cols, ldx, ldy, lddy = 37, 45, 48, 52, 47
    gen = torch.Generator().manual_seed(100 + act)
    x = _padded(rows, cols, ldx, gen)
    x.copy_(_act_inputs(rows, cols, gen).cuda())
    dy = _padded(rows, cols, lddy, gen)
    y = torch.full((rows, ldy), NAN, device="cuda")
    check(lib.mmx_act_fwd(ptr(x), ldx, act, ptr(y), ldy, rows, cols, st()))
    _assert_close_nonfinite(y[:, :cols], ACT_F[act](x), 1e-5, 1e-6, ("fwd", ACT_NAMES[act]))
    dx = torch.full((rows, ldy), NAN, device="cuda")
    check(lib.mmx_act_bwd(ptr(dy), lddy, ptr(x), ldx, act, ptr(dx), ldy, rows, cols, st()))
    _assert_close_nonfinite(dx[:, :cols], dy * _act_grad(act, x), 1e-5, 1e-6, ("bwd", ACT_NAMES[act]))
    assert torch.isnan(y[:, cols:]).all() and torch.isnan(dx[:, cols:]).all()


def test_add(L):
    """out = a + alpha b on strided rows, within fp32 rounding of the fp64 sum; out aliasing a gives the same bits."""
    lib, check, ptr, st = L["lib"], L["check"], L["ptr"], L["st"]
    rows, cols, alpha = 67, 45, -0.75
    gen = torch.Generator().manual_seed(3)
    a, b = _padded(rows, cols, 48, gen), _padded(rows, cols, 50, gen)
    out = torch.full((rows, 52), NAN, device="cuda")
    check(lib.mmx_add(ptr(a), 48, ptr(b), 50, alpha, ptr(out), 52, rows, cols, st()))
    a64, b64 = a.cpu().double(), b.cpu().double()
    err = (out[:, :cols].cpu().double() - (a64 + alpha * b64)).abs()
    assert (err <= 2.0 ** -23 * (a64.abs() + abs(alpha) * b64.abs())).all()
    assert torch.isnan(out[:, cols:]).all()
    check(lib.mmx_add(ptr(a), 48, ptr(b), 50, alpha, ptr(a), 48, rows, cols, st()))       # in place
    assert torch.equal(a, out[:, :cols])


def test_gather_scatter_rows(L):
    """out[r] = src[row_map[r]] (repeats allowed) and dst[row_map[r]] += src[r] (distinct rows): exact fp32, rows and pad
    columns that are not addressed stay as they were."""
    lib, check, ptr, st = L["lib"], L["check"], L["ptr"], L["st"]
    gen = torch.Generator().manual_seed(4)
    n_src, cols, lds, ldo = 50, 77, 80, 84
    src = _padded(n_src, cols, lds, gen)
    rm = torch.tensor([49, 0, 7, 7, 23, 1, 48, 30, 0], dtype=torch.int32)
    out = torch.full((len(rm), ldo), NAN, device="cuda")
    rmd = rm.cuda()
    check(lib.mmx_gather_rows(ptr(src), lds, ptr(rmd), ptr(out), ldo, len(rm), cols, st()))
    assert torch.equal(out[:, :cols], src[rm.long()])
    assert torch.isnan(out[:, cols:]).all()
    rows = 13
    sm = torch.randperm(n_src, generator=gen)[:rows].to(torch.int32)
    s2 = _padded(rows, cols, 81, gen)
    dst = _padded(n_src, cols, ldo, gen)
    want = dst.clone()
    want[sm.long()] += s2
    smd = sm.cuda()
    check(lib.mmx_scatter_add_rows(ptr(s2), 81, ptr(smd), ptr(dst), ldo, rows, cols, st()))
    assert torch.equal(dst, want)
    base = dst.as_strided((n_src, ldo), (ldo, 1))
    assert torch.isnan(base[:, cols:]).all()


@pytest.mark.parametrize("n,R,p", [(2, 64, 16), (3, 96, 32), (2, 56, 14)])
def test_im2col_patches(L, n, R, p):
    """images [n, 3, R, R] -> patches [n (R/p)^2, 3 p p] in conv-weight order, bit for bit: the float4 path (p = 16, 32)
    and the scalar path (p = 14)."""
    lib, check, ptr, st = L["lib"], L["check"], L["ptr"], L["st"]
    gen = torch.Generator().manual_seed(R + p)
    img = torch.randn(n, 3, R, R, generator=gen).cuda()
    G = R // p
    out = torch.full((n * G * G, 3 * p * p), NAN, device="cuda")
    check(lib.mmx_im2col_patches(ptr(img), ptr(out), n, R, p, st()))
    want = img.unfold(2, p, p).unfold(3, p, p).permute(0, 2, 3, 1, 4, 5).reshape(n * G * G, 3 * p * p)
    assert torch.equal(out, want)


@pytest.mark.parametrize("transA", [0, 1])
@pytest.mark.parametrize("with_add", [True, False])
def test_bmm_add(L, transA, with_add):
    """C[b] = add[b] + op(A[b]) B[b] against fp64, with padded rows and batch strides larger than a sample; add = NULL."""
    lib, check, ptr, st = L["lib"], L["check"], L["ptr"], L["st"]
    batch, M, N, K = 3, 70, 45, 131
    lda, ldb, ldadd, ldc = (M + 3 if transA else K + 5), N + 2, N + 7, N + 3
    rows_a = K if transA else M
    sA, sB, sAdd, sC = (rows_a + 2) * lda, (K + 1) * ldb, (M + 3) * ldadd, (M + 1) * ldc
    gen = torch.Generator().manual_seed(10 * transA + with_add)

    def stored(rows, cols, ld, stride):
        buf = torch.full((batch * stride,), NAN)
        v = buf.as_strided((batch, rows, cols), (stride, ld, 1))
        v.copy_(torch.randn(batch, rows, cols, generator=gen))
        return buf.cuda(), v.double()

    Ad, A = stored(rows_a, (M if transA else K), lda, sA)
    Bd, Bm = stored(K, N, ldb, sB)
    addd, add = stored(M, N, ldadd, sAdd)
    Cd = torch.full((batch * sC,), NAN, device="cuda")
    check(lib.mmx_bmm_add(ptr(Ad), lda, sA, transA, ptr(Bd), ldb, sB, ptr(addd) if with_add else None, ldadd, sAdd,
                          ptr(Cd), ldc, sC, batch, M, N, K, st()))
    ref = (A.transpose(1, 2) if transA else A) @ Bm
    if with_add:
        ref = ref + add
    got = Cd.cpu().as_strided((batch, M, N), (sC, ldc, 1))
    assert rel_err(got, ref) < 5e-6
    written = torch.zeros(batch * sC, dtype=torch.bool)
    written.as_strided((batch, M, N), (sC, ldc, 1)).fill_(True)
    assert torch.isnan(Cd.cpu()[~written]).all()                   # pad columns and the gaps between samples
