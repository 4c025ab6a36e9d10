"""GPU: the two-pass attention kernels for rows longer than the single-pass kernels take (S > 1024; DETR's DC5 maps and
padded COCO batches), through the unchanged C ABI, against fp64 autograd - with the tolerances of test_primitives_gpu.py."""
import ctypes as C
import math

import pytest
import torch

from util import rel_err

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L():
    import mmx_b200
    from mmx_b200._lib import lib, check, ptr, current_stream, MmxError
    return dict(lib=lib(), check=check, ptr=ptr, st=current_stream, err=MmxError)


def _ref(q, k, v, H, scale):
    """fp64 softmax(q scale k^T) v per head, on the device; A keeps its gradient."""
    B, T, Dm = q.shape
    S, hd = k.shape[1], Dm // H
    qh, kh, vh = (x.view(B, -1, H, hd).transpose(1, 2) for x in (q, k, v))
    A = torch.softmax((qh * scale) @ kh.transpose(-1, -2), -1)
    A.retain_grad()
    return A, (A @ vh).transpose(1, 2).reshape(B, T, Dm)


def _inputs(B, H, T, S, hd, seed):
    gen = torch.Generator().manual_seed(seed)
    Dm = H * hd
    return [torch.randn(B, n, Dm, generator=gen).cuda() for n in (T, S, S, T)]    # q, k, v, dO


def _run(L, q, k, v, dO, H, hd, ldA, full=True, gscale=None):
    """(A, O, dA, dq, dk, dv) from mmx_attention_fwd / _bwd (/ _bwd_scaled); pad columns start at 7 to catch unwritten ones."""
    lib, check, ptr, st = L["lib"], L["check"], L["ptr"], L["st"]
    B, T, Dm = q.shape
    S = k.shape[1]
    scale = C.c_float(1.0 / math.sqrt(hd))
    A = torch.full((B, H, T, ldA), 7.0, device="cuda")
    O = torch.empty(B, T, Dm, device="cuda")
    check(lib.mmx_attention_fwd(ptr(q), Dm, ptr(k), Dm, ptr(v), Dm, None, ptr(A), ldA, ptr(O), Dm, B, H, T, S, hd, scale, 0,
                                st()))
    dA = torch.full((B, H, T, ldA), 7.0, device="cuda")
    delta = torch.empty(B, H, T, device="cuda")
    dq, dk, dv = (torch.empty_like(t) for t in (q, k, v)) if full else (None, None, None)
    args = [ptr(dO), Dm, ptr(q), Dm, ptr(k), Dm, ptr(v), Dm, ptr(A), ptr(dA), ldA, ptr(delta) if full else None,
            ptr(dq), Dm, ptr(dk), Dm, ptr(dv), Dm, B, H, T, S, hd, scale, 0]
    if gscale is None:
        check(lib.mmx_attention_bwd(*args, st()))
    else:
        check(lib.mmx_attention_bwd_scaled(*args, ptr(gscale), st()))
    torch.cuda.synchronize()
    return A, O, dA, dq, dk, dv


def _ld(S):
    """a row stride with pad columns inside the last 64-key tile and beyond it"""
    return (S + 3) // 4 * 4 + 68


@pytest.mark.parametrize("T,S,hd", [(1024, 1024, 32), (1025, 1025, 32), (2500, 2500, 32), (100, 3350, 32), (1100, 1100, 64),
                                    (100, 4200, 64)])
def test_long_attention_vs_fp64(L, T, S, hd):
    """S = 1024 runs the single-pass kernel, every longer row the two-pass one; both meet the same fp64 tolerance."""
    H = 256 // hd
    q, k, v, dO = _inputs(1, H, T, S, hd, seed=T * 7 + S)
    ldA = _ld(S)
    A, O, dA, dq, dk, dv = _run(L, q, k, v, dO, H, hd, ldA)
    q64, k64, v64 = (t.double().requires_grad_(True) for t in (q, k, v))
    Ar, Or = _ref(q64, k64, v64, H, 1.0 / math.sqrt(hd))
    Or.backward(dO.double())
    errs = dict(A=rel_err(A[..., :S], Ar.detach()), O=rel_err(O, Or.detach()), dA=rel_err(dA[..., :S], Ar.grad),
                dq=rel_err(dq, q64.grad), dk=rel_err(dk, k64.grad), dv=rel_err(dv, v64.grad))
    print("long attention errors", (T, S, hd), {k_: f"{v_:.1e}" for k_, v_ in errs.items()})
    assert errs["A"] < 5e-6 and errs["O"] < 5e-6 and errs["dA"] < 5e-6
    assert max(errs["dq"], errs["dk"], errs["dv"]) < 1e-5
    assert (A[..., S:] == 0).all() and (dA[..., S:] == 0).all()     # pad columns zero-filled
    # stop after dA (the last relevant block): the same dA bits
    _, _, dA2, *_ = _run(L, q, k, v, dO, H, hd, ldA, full=False)
    assert torch.equal(dA2, dA)


def test_long_attention_bwd_scaled_stages_the_unscaled_dA(L):
    """dO carrying a power-of-two factor per sample: dA is staged in true units (the unscaled call's dA up to the fp16
    split of the scaled operand), dQ / dK / dV stay scaled"""
    B, H, T, S, hd = 2, 8, 300, 1500, 32
    q, k, v, dO = _inputs(B, H, T, S, hd, seed=5)
    gs = torch.tensor([2.0 ** 12, 2.0 ** -3], device="cuda")
    A, O, dA, dq, dk, dv = _run(L, q, k, v, dO, H, hd, _ld(S))
    _, _, dAs, dqs, dks, dvs = _run(L, q, k, v, dO * gs.view(B, 1, 1), H, hd, _ld(S), gscale=gs)
    errs = [rel_err(dAs, dA)] + [rel_err(xs / gs.view(B, 1, 1), x) for x, xs in ((dq, dqs), (dk, dks), (dv, dvs))]
    print("scaled vs unscaled (dA, dq, dk, dv):", [f"{e:.1e}" for e in errs])
    assert max(errs) < 1e-6
    assert (dAs[..., S:] == 0).all()


def test_long_attention_is_batch_invariant(L):
    """a sample alone and the same sample inside a batch of 3: the same bits for A, O, dA, dQ, dK, dV"""
    H, T, S, hd = 8, 200, 1300, 32
    q, k, v, dO = _inputs(3, H, T, S, hd, seed=9)
    ldA = _ld(S)
    full = _run(L, q, k, v, dO, H, hd, ldA)
    one = _run(L, *(t[1:2].contiguous() for t in (q, k, v, dO)), H, hd, ldA)
    for name, a, b in zip(("A", "O", "dA", "dq", "dk", "dv"), full, one):
        assert torch.equal(a[1:2], b), name


def test_long_attention_limits(L):
    """S above 16384 and ragged batches past 1024 keys raise MmxError (no silent fall-back)"""
    lib, check, ptr, st = L["lib"], L["check"], L["ptr"], L["st"]
    H, hd, T, S = 1, 32, 1, 16385
    q, k = torch.zeros(1, T, 32, device="cuda"), torch.zeros(1, S, 32, device="cuda")
    A, O = torch.empty(1, 1, T, S + 3, device="cuda"), torch.empty(1, T, 32, device="cuda")
    with pytest.raises(L["err"], match="16384"):
        check(lib.mmx_attention_fwd(ptr(q), 32, ptr(k), 32, ptr(k), 32, None, ptr(A), S + 3, ptr(O), 32, 1, H, T, S, hd,
                                    C.c_float(1.0), 0, st()))
    # the CLIP text tower is ragged (packed rows up to each sample's EOT); a 1100-token context is past the ragged kernels
    import mmx_b200
    from oracle import clip_oracle as co
    cfg = co.ClipConfig(64, 64, 1, 128, 16, 1100, 512, 64, 2, 1)
    sd = co.init_state_dict(cfg, seed=1)
    images, tokens = co.synthetic_inputs(cfg, 1, seed=2)
    eng = mmx_b200.ClipEngine(mmx_b200.ClipConfig(*cfg.ref_args()), sd, max_batch=1, device="cuda:0")
    with pytest.raises(L["err"], match="ragged"):
        mmx_b200.interpret(images.cuda(), tokens.cuda(), eng, "cuda:0", -1, -1)
        torch.cuda.synchronize()
