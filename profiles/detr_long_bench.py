"""DETR past 1024 tokens on one GPU: the DC5 (dilated layer4) ResNet-50 backbone, generate_ours and MaskGenerator on DC5
maps, and the two-pass long-row attention kernels alone.  Prints one JSON line.

    python profiles/detr_long_bench.py [--reps 5]

Weights: the seeded DETR-R50 state dict of oracle/detr_backbone_oracle.py (ResNet-50 + d_model 256, 8 heads, 6 + 6 layers,
100 queries), built with dilation=True; inputs N(0, 1) images.  Times are CUDA-event medians after warm-up.

* backbone: ms per image (gathers, max-pool and position embedding included) and the GEMM TFLOP/s of the convs
  (algorithmic 2 M N K over the summed GEMM launch time, mmx_profile_gemm window).
* attention: mmx_attention_fwd / mmx_attention_bwd (dQ, dK, dV) at T = S, H = 8, hd = 32.  FLOPs are the algorithmic fp32
  products (forward QK^T and PV; backward dO V^T, dS K, A^T dO, dS^T Q), each run as three fp16 tensor-core products.
  Bytes are the staged fp32 planes: the forward writes A once; the backward writes dA and reads A three times and dA
  twice (two passes of the query kernel, the key kernel).  "bound" names the larger of the two times at the H100 SXM
  data-sheet peaks (989 dense fp16 tensor TFLOP/s, 3.35 TB/s HBM3).
* rules: the encoder's rule 5 + rule 6 (R_ii += avg_heads(A, dA) R_ii, 6 layers; O(S^3)) as a share of one
  generate_ours call.
"""
import argparse
import ctypes as C
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import mmx_b200  # noqa: E402
from mmx_b200.backbone import conv_flops  # noqa: E402
from mmx_b200._lib import ptr, current_stream, check  # noqa: E402
from oracle import detr_backbone_oracle as bo, detr_oracle as do  # noqa: E402
from detr_image_bench import timed, gpu_info  # noqa: E402

PEAK_F16_TFLOPS, PEAK_HBM_TBS = 989.0, 3.35


def attention_alone(l, S, reps, H=8, hd=32):
    g = torch.Generator().manual_seed(S)
    D = H * hd
    q, k, v, dO = (torch.randn(S, D, generator=g).cuda() for _ in range(4))
    ldA = (S + 3) // 4 * 4
    A, dA = (torch.empty(H, S, ldA, device="cuda") for _ in range(2))
    O, dq, dk, dv = (torch.empty(S, D, device="cuda") for _ in range(4))
    delta = torch.empty(H, S, device="cuda")
    sc = C.c_float(hd ** -0.5)
    fwd = lambda: check(l.mmx_attention_fwd(ptr(q), D, ptr(k), D, ptr(v), D, None, ptr(A), ldA, ptr(O), D, 1, H, S, S, hd, sc,
                                            0, current_stream()))
    bwd = lambda: check(l.mmx_attention_bwd(ptr(dO), D, ptr(q), D, ptr(k), D, ptr(v), D, ptr(A), ptr(dA), ldA, ptr(delta),
                                            ptr(dq), D, ptr(dk), D, ptr(dv), D, 1, H, S, S, hd, sc, 0, current_stream()))
    out = {}
    for name, fn, nprod, nplanes in (("fwd", fwd, 2, 1), ("bwd", bwd, 4, 6)):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        ms = timed(fn, reps)
        flops = 2.0 * H * S * S * hd * nprod
        nbytes = 4.0 * H * S * ldA * nplanes
        t_c, t_m = 3 * flops / (PEAK_F16_TFLOPS * 1e12), nbytes / (PEAK_HBM_TBS * 1e12)
        out[name] = dict(ms=round(ms, 3), tflops=round(flops / (ms * 1e-3) / 1e12, 1), tb_per_s=round(nbytes / (ms * 1e-3) / 1e12, 2),
                         bound="memory" if t_m > t_c else "compute",
                         share_of_bound=round(max(t_c, t_m) / (ms * 1e-3), 2))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    l = mmx_b200.lib()
    cfg = do.DETR_R50
    sd = bo.init_state_dict(cfg, seed=5)
    eng = mmx_b200.DetrEngine(sd, nhead=cfg.nhead, device="cuda:0", dilation=True)
    name, power = gpu_info()
    res = dict(gpu=name, power_limit=power, gemm_backend=l.mmx_get_gemm_backend(), backbone={}, attention={})
    g = torch.Generator().manual_seed(0)
    for H, W in ((800, 800), (800, 1066)):
        B = 4
        x = torch.randn(B, 3, H, W, generator=g).cuda()
        for _ in range(2):
            eng.features(x)
        torch.cuda.synchronize()
        ms = timed(lambda: eng.features(x), args.reps)
        l.mmx_profile_gemm(1)
        f = eng.features(x)
        l.mmx_profile_gemm(0)
        gms, gfl, n = C.c_double(), C.c_double(), C.c_int()
        l.mmx_profile_gemm_report(C.byref(gms), C.byref(gfl), C.byref(n))
        flops = conv_flops(eng.backbone, B, H, W)
        res["backbone"][f"dc5_{H}x{W}_b{B}"] = dict(
            tokens=f.h * f.w, backbone_ms_per_image=round(ms / B, 3), backbone_gflop_per_image=round(flops / B / 1e9, 1),
            backbone_gemm_tflops=round(flops / (gms.value * 1e-3) / 1e12, 1), gemm_launches=n.value)
        del x, f
        torch.cuda.empty_cache()
    # generate_ours from images: 4 images x 1 query, 800 x 800 DC5 (2500 tokens)
    gen = mmx_b200.Generator(eng)
    x = torch.randn(4, 3, 800, 800, generator=g).cuda()
    tq = torch.randint(0, cfg.queries, (4,), generator=g)
    for _ in range(2):
        gen.generate_ours(x, tq, use_lrp=False)
    torch.cuda.synchronize()
    ms = timed(lambda: gen.generate_ours(x, tq, use_lrp=False), args.reps)
    # the encoder's rule 5 + rule 6 alone, on the A / dA the last call staged
    m = gen.model

    def enc_rules():
        gen.R_i_i = torch.eye(m._shape[1], device=m.device).repeat(gen.B, 1, 1)
        gen.handle_self_attention_image(m.encoder)
    enc_rules()
    torch.cuda.synchronize()
    rms = timed(enc_rules, args.reps)
    res["generate_ours_dc5_800x800_b4"] = dict(tokens=m._shape[1], ms=round(ms, 2), maps_per_s=round(4 / (ms * 1e-3), 2),
                                               encoder_rules_5_6_ms=round(rms, 2), encoder_rules_share=round(rms / ms, 3))
    # MaskGenerator: one image, 10 queries (backbone once; chunked by free memory)
    mg = mmx_b200.MaskGenerator(eng)
    one = x[:1].contiguous()
    q = torch.arange(10)
    del x
    torch.cuda.empty_cache()
    mg.get_masks(one, q)
    torch.cuda.synchronize()
    res["mask_generator_dc5_800x800_1img_10q"] = dict(ms=round(timed(lambda: mg.get_masks(one, q), max(2, args.reps // 2)), 1),
                                                      chunk=mg.chunk_size(2500, False))
    torch.cuda.empty_cache()
    for S in (2500, 3350):
        res["attention"][f"S{S}_T{S}_H8_hd32"] = attention_alone(l, S, args.reps)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
