"""Micro-benchmark of the linear GEMM through the C ABI (both backends) on the CLIP ViT-B/32 batch-64 shapes.
usage (GPU box): python profiles/gemm_bench.py
  --epilogue bias|residual|gelu|dgelu   the CLIP shapes that run each epilogue, through mmx_gemm_nt: bias + residual
                                        (out-proj, fc2), bias + C_act = QuickGELU(C) (fc1), C * QuickGELU'(pre) (the fc2
                                        dgrad); default: bias on every shape, through mmx_linear_packed
  --tree DIR                            time the library of another checkout (same C ABI), e.g. the parent commit's"""
import ctypes as C
import json
import os
import sys

import torch

TREE = sys.argv[sys.argv.index("--tree") + 1] if "--tree" in sys.argv else os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.abspath(TREE))
import mmx_b200  # noqa: E402
from mmx_b200._lib import lib, check, ptr, current_stream  # noqa: E402

SHAPES = [(3200, 2304, 768), (3200, 768, 768), (3200, 3072, 768), (3200, 768, 3072),
          (4928, 1536, 512), (4928, 512, 512), (4928, 2048, 512), (4928, 512, 2048), (3136, 768, 3072), (3200, 768, 2304)]
# vision (3200 rows) and text (4928 rows) blocks: out-proj and fc2 add the residual, fc1 stores QuickGELU(C) beside C,
# the fc2 dgrad (dX [M, 4D] = dY [M, D] W_fc2) multiplies by QuickGELU'(f)
EPILOGUE_SHAPES = {"residual": [(3200, 768, 768), (3200, 768, 3072), (4928, 512, 512), (4928, 512, 2048)],
                   "gelu": [(3200, 3072, 768), (4928, 2048, 512)],
                   "dgelu": [(3200, 3072, 768), (4928, 2048, 512)]}
QUICKGELU = 1


def main():
    l = lib()
    out = []
    global SHAPES
    epi = sys.argv[sys.argv.index("--epilogue") + 1] if "--epilogue" in sys.argv else None
    if epi in EPILOGUE_SHAPES:
        SHAPES = EPILOGUE_SHAPES[epi]
    elif epi not in (None, "bias"):
        sys.exit(f"unknown --epilogue {epi}")
    backends = (1, 2) if "--tiles" in sys.argv else (0, 1, 2)
    if "--only" in sys.argv:            # e.g. --only 3200,2304,768  (tensor-core backend only; for ncu captures)
        SHAPES = [tuple(int(v) for v in sys.argv[sys.argv.index("--only") + 1].split(","))]
        backends = (2,)
    if "--backend" in sys.argv:
        backends = (int(sys.argv[sys.argv.index("--backend") + 1]),)
    for backend in backends:
        if l.mmx_set_gemm_backend(backend) != backend:
            continue
        widths = (128, 144, 160, 0) if (backend >= 1 and "--tiles" in sys.argv) else (0,)    # 0 = automatic tile width
        for (M, N, K), bn in [(sh, w) for sh in SHAPES for w in widths]:
            l.mmx_set_gemm_tile_n(bn)
            g = torch.Generator(device="cuda").manual_seed(1)
            A = torch.randn(M, K, device="cuda", generator=g)
            W = torch.randn(N, K, device="cuda", generator=g) / K ** 0.5
            bias = torch.randn(N, device="cuda", generator=g)
            Cm = torch.empty(M, N, device="cuda")
            res = torch.randn(M, N, device="cuda", generator=g) if epi == "residual" else None
            pre = torch.randn(M, N, device="cuda", generator=g) if epi == "dgelu" else None
            Ca = torch.empty(M, N, device="cuda") if epi == "gelu" else None
            pk = None
            if backend >= 2:      # fp16x3: the weight's hi / lo planes are built once (static weights)
                pk = torch.empty(l.mmx_pack_weight_bytes(N, K), dtype=torch.uint8, device="cuda")
                check(l.mmx_pack_weight(ptr(W), K, N, K, ptr(pk), current_stream()))
            if epi is None:
                def call():
                    check(l.mmx_linear_packed(ptr(A), K, ptr(W), K, ptr(pk), ptr(bias), None, 0, ptr(Cm), N, None, 0, M, N, K,
                                              current_stream()))
            else:
                def call():
                    check(l.mmx_gemm_nt(ptr(A), K, ptr(W), K, ptr(pk), None if epi == "dgelu" else ptr(bias), ptr(pre), N, ptr(res),
                                        N, ptr(Cm), N, ptr(Ca), QUICKGELU if epi in ("gelu", "dgelu") else 0, M, N, K, current_stream()))
            for _ in range(3):
                call()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            reps = 20
            if "--graph" in sys.argv:       # replay 20 launches from a CUDA graph: no host time (ctypes, tensor-map encodes) in the figure
                gr = torch.cuda.CUDAGraph()
                with torch.cuda.graph(gr):
                    for _ in range(reps):
                        call()
                gr.replay()
                torch.cuda.synchronize()
                e0.record()
                gr.replay()
                e1.record()
            else:
                e0.record()
                for _ in range(reps):
                    call()
                e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / reps
            ref = A[:256].double() @ W.double().t()
            if epi == "dgelu":
                s = torch.sigmoid(1.702 * pre[:256].double())
                ref = ref * (s + 1.702 * pre[:256].double() * s * (1 - s))
            else:
                ref = ref + bias.double()
            if epi == "residual":
                ref = ref + res[:256].double()
            err = ((Cm[:256].double() - ref).abs().max() / ref.abs().max()).item()
            out.append(dict(backend=backend, epilogue=epi or "bias", tile_n=bn, M=M, N=N, K=K, us=ms * 1e3, tflops=2.0 * M * N * K / (ms * 1e-3) / 1e12, rel_err=err))
            print(out[-1], flush=True)
    l.mmx_set_gemm_backend(2)
    l.mmx_set_gemm_tile_n(0)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
