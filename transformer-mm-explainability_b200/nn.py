"""Host-side tape for the DETR / LXMERT / ViT relevancy generators.

The reference obtains A (attention probabilities) and dA (their gradients) with PyTorch forward / backward hooks
and ``loss.backward()`` (DETR/modules/layers.py:758-759, lxmert/lxmert/src/lxmert_lrp.py:407-408).  Here the forward
is a sequence of libmmx kernel launches recorded on a tape, and the backward replays the tape in reverse with the
matching dgrad kernels (no weight gradients are ever needed: only dA).  PyTorch owns buffers and the stream only.

All activations are row-major matrices ``[B*S, D]`` (row = b*S + s).
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Callable, List, Optional

import torch

from ._lib import lib, check, ptr, current_stream, MmxError

ACT_NONE, ACT_QUICKGELU, ACT_GELU, ACT_RELU, ACT_TANH = 0, 1, 2, 3, 4
ACT_SIGMOID = 6
ATTN_CAUSAL, ATTN_SCALE_SCORES = 1, 2


def _f32(t: torch.Tensor, device) -> torch.Tensor:
    return t.detach().to(device=device, dtype=torch.float32).contiguous()


class Var:
    """A device matrix (2-D torch view, unit column stride) with an optional accumulated gradient."""
    __slots__ = ("v", "g")

    def __init__(self, v: torch.Tensor):
        assert v.dim() == 2 and v.stride(1) == 1 and v.is_cuda and v.dtype == torch.float32
        self.v = v
        self.g: Optional[torch.Tensor] = None

    @property
    def rows(self):
        return self.v.shape[0]

    @property
    def cols(self):
        return self.v.shape[1]


def pack_weight(w: torch.Tensor) -> Optional[torch.Tensor]:
    """fp16 hi / lo planes of a static [N, K] GEMM operand for the fp16x3 tensor-core backend (``mmx_pack_weight``);
    None when the matrix is below the tensor-core kernel's minimum tile (N < 128 or K < 64: the fp32 path runs)."""
    N, K = w.shape
    if N < 128 or K < 64:
        return None
    l = lib()
    buf = torch.empty(l.mmx_pack_weight_bytes(N, K), dtype=torch.uint8, device=w.device)
    with torch.cuda.device(w.device):
        check(l.mmx_pack_weight(ptr(w), w.stride(0), N, K, ptr(buf), current_stream()))
    return buf


class Weight:
    """Linear weight [out, in] plus its transpose (the K-major operand of the dgrad GEMM), their packed fp16x3 copies
    and the optional bias."""

    def __init__(self, w: torch.Tensor, b: Optional[torch.Tensor], device):
        self.w = _f32(w, device)
        self.wt = self.w.t().contiguous()
        self.b = _f32(b, device) if b is not None else None
        self.out_features, self.in_features = self.w.shape
        self.pw, self.pwt = pack_weight(self.w), pack_weight(self.wt)


class fp32_gemms:
    """Context manager: every linear inside runs on the fp32 FFMA GEMM backend (``mmx_set_gemm_backend(0)``), restored on
    exit.  Used by the LRP paths: relprop divides by activations, attention scores and whole-tensor sums that nearly cancel,
    so the ~1e-6 (of max|C|) rounding of the tensor-core fp16x3 / 3xTF32 products - harmless for the gradient path - is
    amplified to the 1e-1 level there, against ~1e-7-grade fp32 products for which the sweep's own fp32 noise dominates
    (the reference's fp32 sweep is itself 1e-2 .. 1e-1 away from its fp64 evaluation at DETR-R50 / LXMERT-base size with
    random-init weights; tests/test_lrp_gpu.py measures both on the same box)."""

    def __enter__(self):
        l = lib()
        self.prev = l.mmx_get_gemm_backend()
        l.mmx_set_gemm_backend(0)
        return self

    def __exit__(self, *exc):
        lib().mmx_set_gemm_backend(self.prev)
        return False


class Tape:
    # Power-of-two factor the seed gradient is multiplied by (and every staged dA divided by, exactly): keeps the
    # operands of the fp16x3 dgrad GEMMs well inside fp16's exponent range (csrc/gemm_wgmma.cu).
    GRAD_SCALE = 256.0

    def __init__(self, device):
        self.device = torch.device(device)
        self.ops: List[Callable[[], None]] = []
        self.lib = lib()
        self.gscale: Optional[torch.Tensor] = None

    def seed(self, var: "Var", one_hot: torch.Tensor, B: int):
        """var.g = GRAD_SCALE * one_hot; the attention backwards stage dA / GRAD_SCALE (the true gradient)."""
        var.g = one_hot * self.GRAD_SCALE
        self.gscale = torch.full((B,), self.GRAD_SCALE, device=self.device, dtype=torch.float32)

    # ------------------------------------------------------------------ helpers
    def new(self, rows, cols) -> torch.Tensor:
        return torch.empty(rows, cols, device=self.device, dtype=torch.float32)

    def accumulate(self, var: Var, buf: torch.Tensor):
        """var.g += buf (buf is consumed: it becomes the gradient buffer when there was none)."""
        if var.g is None:
            var.g = buf
        else:
            check(self.lib.mmx_add(ptr(var.g), var.g.stride(0), ptr(buf), buf.stride(0), C.c_float(1.0), ptr(var.g),
                                   var.g.stride(0), var.rows, var.cols, current_stream()))

    def backward(self):
        for fn in reversed(self.ops):
            fn()

    # ------------------------------------------------------------------ ops
    def linear(self, x: Var, W: Weight, act: int = ACT_NONE) -> Var:
        """y = act(x W^T + b)   (F.linear + activation)."""
        M, K, N = x.rows, x.cols, W.out_features
        assert K == W.in_features, (K, W.in_features)
        pre = self.new(M, N)
        out = self.new(M, N) if act else None
        check(self.lib.mmx_linear_packed(ptr(x.v), x.v.stride(0), ptr(W.w), K, ptr(W.pw), ptr(W.b), None, 0, ptr(pre), N,
                                         ptr(out), act, M, N, K, current_stream()))
        y = Var(out if act else pre)

        def bwd():
            if y.g is None:
                return
            dy = y.g
            if act:
                dpre = self.new(M, N)
                check(self.lib.mmx_act_bwd(ptr(dy), dy.stride(0), ptr(pre), N, act, ptr(dpre), N, M, N, current_stream()))
                dy = dpre
            dx = self.new(M, K)
            check(self.lib.mmx_linear_dgrad_packed(ptr(dy), dy.stride(0), ptr(W.wt), N, ptr(W.pwt), None, 0, 0, ptr(dx), K,
                                                   M, N, K, current_stream()))
            self.accumulate(x, dx)
        self.ops.append(bwd)
        return y

    def layernorm(self, x: Var, gamma: torch.Tensor, beta: torch.Tensor, eps: float) -> Var:
        M, D = x.rows, x.cols
        out = self.new(M, D)
        mean = torch.empty(M, device=self.device)
        rstd = torch.empty(M, device=self.device)
        check(self.lib.mmx_layernorm_fwd(ptr(x.v), x.v.stride(0), None, ptr(gamma), ptr(beta), ptr(out), D, ptr(mean), ptr(rstd),
                                         M, D, C.c_float(eps), current_stream()))
        y = Var(out)

        def bwd():
            if y.g is None:
                return
            dx = self.new(M, D)
            check(self.lib.mmx_layernorm_bwd(ptr(y.g), y.g.stride(0), ptr(x.v), x.v.stride(0), None, ptr(gamma), ptr(mean),
                                             ptr(rstd), None, 0, ptr(dx), D, M, D, current_stream()))
            self.accumulate(x, dx)
        self.ops.append(bwd)
        return y

    def add(self, a: Var, b: Var) -> Var:
        out = self.new(a.rows, a.cols)
        check(self.lib.mmx_add(ptr(a.v), a.v.stride(0), ptr(b.v), b.v.stride(0), C.c_float(1.0), ptr(out), a.cols, a.rows,
                               a.cols, current_stream()))
        y = Var(out)

        def bwd():
            if y.g is None:
                return
            for t in (a, b):
                if t.g is None:
                    t.g = y.g.clone() if t is a else y.g      # second consumer may own the buffer
                else:
                    self.accumulate(t, y.g)
        self.ops.append(bwd)
        return y

    def add_const(self, a: Var, const: torch.Tensor) -> Var:
        """a + const (const carries no gradient: positional / query embeddings)."""
        out = self.new(a.rows, a.cols)
        check(self.lib.mmx_add(ptr(a.v), a.v.stride(0), ptr(const), const.stride(0), C.c_float(1.0), ptr(out), a.cols, a.rows,
                               a.cols, current_stream()))
        y = Var(out)

        def bwd():
            if y.g is not None:
                self.accumulate(a, y.g)
        self.ops.append(bwd)
        return y

    def gather_rows(self, x: Var, row_map: torch.Tensor) -> Var:
        """out[r] = x[row_map[r]] (e.g. the pooled [CLS] token x[:, 0])."""
        R = row_map.numel()
        out = self.new(R, x.cols)
        check(self.lib.mmx_gather_rows(ptr(x.v), x.v.stride(0), ptr(row_map), ptr(out), x.cols, R, x.cols, current_stream()))
        y = Var(out)

        def bwd():
            if y.g is None:
                return
            if x.g is None:
                x.g = torch.zeros(x.rows, x.cols, device=self.device, dtype=torch.float32)
            check(self.lib.mmx_scatter_add_rows(ptr(y.g), y.g.stride(0), ptr(row_map), ptr(x.g), x.g.stride(0), R, x.cols,
                                                current_stream()))
        self.ops.append(bwd)
        return y

    def attention(self, q: Var, k: Var, v: Var, B: int, H: int, T: int, S: int, scale: float, flags: int = 0,
                  key_bias: Optional[torch.Tensor] = None, record: Optional["AttnRecord"] = None) -> Var:
        """softmax(scale * q k^T + bias) v per head, staging A; the backward stages dA into `record`."""
        Dm = q.cols
        hd = Dm // H
        ldA = (S + 3) // 4 * 4
        A = torch.empty(B, H, T, ldA, device=self.device, dtype=torch.float32)
        out = self.new(B * T, Dm)
        check(self.lib.mmx_attention_fwd(ptr(q.v), q.v.stride(0), ptr(k.v), k.v.stride(0), ptr(v.v), v.v.stride(0), ptr(key_bias),
                                         ptr(A), ldA, ptr(out), Dm, B, H, T, S, hd, C.c_float(scale), flags, current_stream()))
        y = Var(out)
        if record is not None:
            record.A, record.S, record.dA, record.cam = A, S, None, None
            # what the relprop sweep of this attention reads (mmx_b200/lrp.py); references only, nothing is copied
            record.saved = dict(q=q, k=k, v=v, o=y, B=B, H=H, T=T, S=S, hd=hd)

        def bwd():
            if y.g is None:
                return
            dA = torch.empty_like(A)
            delta = torch.empty(B, H, T, device=self.device, dtype=torch.float32)
            dq, dk, dv = self.new(B * T, Dm), self.new(B * S, Dm), self.new(B * S, Dm)
            check(self.lib.mmx_attention_bwd_scaled(ptr(y.g), y.g.stride(0), ptr(q.v), q.v.stride(0), ptr(k.v), k.v.stride(0),
                                                    ptr(v.v), v.v.stride(0), ptr(A), ptr(dA), ldA, ptr(delta), ptr(dq), Dm,
                                                    ptr(dk), Dm, ptr(dv), Dm, B, H, T, S, hd, C.c_float(scale), flags,
                                                    ptr(self.gscale), current_stream()))
            if record is not None:
                record.dA = dA
            self.accumulate(q, dq)
            self.accumulate(k, dk)
            self.accumulate(v, dv)
        self.ops.append(bwd)
        return y


class AttnRecord:
    """What the reference attention modules expose through get_attn() / get_attn_gradients()
    (DETR/modules/layers.py:693-709): A and dA of the last forward / backward, [B, H, T, S]."""

    def __init__(self):
        self.A: Optional[torch.Tensor] = None
        self.dA: Optional[torch.Tensor] = None
        self.cam: Optional[torch.Tensor] = None      # LRP relevance of A (``get_attn_cam()``), staged by mmx_b200.lrp
        self.saved: dict = {}
        self.S = 0

    def get_attn(self) -> torch.Tensor:
        return self.A[..., :self.S]

    def get_attn_gradients(self) -> Optional[torch.Tensor]:
        return None if self.dA is None else self.dA[..., :self.S]

    def get_attn_cam(self) -> Optional[torch.Tensor]:
        return None if self.cam is None else self.cam[..., :self.S]

    def padded(self, use_cam: bool = False):
        """(A, dA, ld) with the zero-padded row stride the rule-5 kernel can read directly; ``use_cam``: the LRP relevance
        of A in place of A (the ``use_lrp`` branches of the generators, DETR/modules/ExplanationGenerator.py:112-115)."""
        if use_cam:
            if self.cam is None:
                raise MmxError("no LRP relevance recorded for this attention (run the relprop sweep first)")
            return self.cam, self.dA, self.A.shape[-1]
        return self.A, self.dA, self.A.shape[-1]
