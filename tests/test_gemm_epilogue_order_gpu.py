"""GPU: the tensor-core GEMM epilogue loads the whole residual / act'(pre) fragment of a tile before it stores any of it.
These pin what that order must keep: C written over its own residual (in place), pre + residual + act in one launch,
M and N that are not multiples of the tile, and every tile width giving the same bits."""
import contextlib
import math

import pytest
import torch
import torch.nn.functional as F

from util import rel_err

pytestmark = pytest.mark.gpu

NAN = float("nan")
GELU, MUL = 2, 5
TILES = (128, 144, 160)


@pytest.fixture(scope="module")
def L():
    import mmx_b200
    from mmx_b200._lib import lib, check, ptr, current_stream
    return dict(lib=lib(), check=check, ptr=ptr, st=current_stream)


@contextlib.contextmanager
def gemm_backend(lib, backend, bn=0):
    prev_backend, prev_tile = lib.mmx_get_gemm_backend(), lib.mmx_set_gemm_tile_n(-1)
    try:
        if lib.mmx_set_gemm_backend(backend) != backend:
            pytest.skip("tensor-core backend not available")
        assert lib.mmx_set_gemm_tile_n(bn) == bn
        yield
    finally:
        lib.mmx_set_gemm_backend(prev_backend)
        lib.mmx_set_gemm_tile_n(prev_tile)


def _operands(M, N, K, seed):
    gen = torch.Generator().manual_seed(seed)
    A = torch.randn(M, K, generator=gen)
    W = torch.randn(N, K, generator=gen) / math.sqrt(K)
    bias = torch.randn(N, generator=gen)
    pre = torch.randn(M, N, generator=gen)
    res = torch.randn(M, N, generator=gen)
    return A, W, bias, pre, res


def _gemm(L, A, W, pk, C, bias=None, pre=None, res=None, C_act=None, act=0):
    lib, ptr = L["lib"], L["ptr"]
    M, K = A.shape
    N = W.shape[0]
    L["check"](lib.mmx_gemm_nt(ptr(A), K, ptr(W), K, ptr(pk), ptr(bias), ptr(pre), N, ptr(res), N, ptr(C), N, ptr(C_act),
                               act, M, N, K, L["st"]()))


def _pack(L, W):
    N, K = W.shape
    buf = torch.empty(L["lib"].mmx_pack_weight_bytes(N, K), dtype=torch.uint8, device="cuda")
    L["check"](L["lib"].mmx_pack_weight(L["ptr"](W), K, N, K, L["ptr"](buf), L["st"]()))
    return buf


# M and N off every tile multiple (BM = 128; BN = 128 / 144 / 160), K off the slab width
SHAPE = (300, 420, 200)


@pytest.mark.parametrize("backend", [1, 2, 3])
def test_in_place_residual(L, backend):
    """C = A W^T + bias + residual written over the residual itself equals the out-of-place result bit for bit, at every
    tile width, and all tile widths agree."""
    M, N, K = SHAPE
    A, W, bias, _, res = _operands(M, N, K, 21 + backend)
    Ad, Wd, bd, rd = A.cuda(), W.cuda(), bias.cuda(), res.cuda()
    ref = A.double() @ W.double().t() + bias.double() + res.double()
    first = None
    for bn in TILES:
        with gemm_backend(L["lib"], backend, bn):
            pk = _pack(L, Wd) if backend >= 2 else None
            C = torch.full((M, N), NAN, device="cuda")
            _gemm(L, Ad, Wd, pk, C, bias=bd, res=rd)
            Ci = rd.clone()
            _gemm(L, Ad, Wd, pk, Ci, bias=bd, res=Ci)
        assert rel_err(C, ref) < 2e-5, bn
        assert torch.equal(Ci, C), bn
        first = C if first is None else first
        assert torch.equal(C, first), bn


@pytest.mark.parametrize("backend", [1, 2, 3])
@pytest.mark.parametrize("act", [GELU, MUL], ids=["gelu", "mul"])
def test_pre_residual_act(L, backend, act):
    """C = (A W^T + bias) act'(pre) + residual and C_act = act(C) in one launch (the LRP form) against fp64; in place over
    the residual with the same bits, and the same bits at every tile width."""
    M, N, K = SHAPE
    A, W, bias, pre, res = _operands(M, N, K, 40 + 3 * backend + act)
    Ad, Wd, bd, pd, rd = A.cuda(), W.cuda(), bias.cuda(), pre.cuda(), res.cuda()
    if act == MUL:
        grad = pre.double()
        fwd = lambda x: x
    else:
        p = pre.double().requires_grad_(True)
        F.gelu(p).sum().backward()
        grad, fwd = p.grad, F.gelu
    ref = (A.double() @ W.double().t() + bias.double()) * grad + res.double()
    first = None
    for bn in TILES:
        with gemm_backend(L["lib"], backend, bn):
            pk = _pack(L, Wd) if backend >= 2 else None
            C = torch.full((M, N), NAN, device="cuda")
            Ca = torch.full((M, N), NAN, device="cuda")
            _gemm(L, Ad, Wd, pk, C, bias=bd, pre=pd, res=rd, C_act=Ca, act=act)
            Ci = rd.clone()
            Cai = torch.full((M, N), NAN, device="cuda")
            _gemm(L, Ad, Wd, pk, Ci, bias=bd, pre=pd, res=Ci, C_act=Cai, act=act)
        assert rel_err(C, ref) < 2e-5, bn
        assert rel_err(Ca, fwd(ref), base=ref) < 2e-5, bn
        assert torch.equal(Ci, C) and torch.equal(Cai, Ca), bn
        first = (C, Ca) if first is None else first
        assert torch.equal(C, first[0]) and torch.equal(Ca, first[1]), bn
