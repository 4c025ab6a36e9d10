"""DETR from images on one GPU: ResNet-50 backbone time and GEMM throughput, generate_ours maps/s and MaskGenerator time,
beside the same backbone in eager fp32 PyTorch on the same GPU.  Prints one JSON line.

    python profiles/detr_image_bench.py [--reps 5]

Weights: the seeded DETR-R50 state dict of oracle/detr_backbone_oracle.py (ResNet-50 + d_model 256, 8 heads, 6 + 6 layers,
100 queries), inputs N(0, 1) images.  Times are CUDA-event medians after warm-up.  backbone_gemm_tflops is the algorithmic
FLOPs of the 53 convs + input_proj (2 M N K from the conv shapes) over the summed GEMM launch time of one backbone call
(mmx_profile_gemm window); backbone_ms includes the gathers, the max-pool and the position embedding."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import mmx_b200  # noqa: E402
from mmx_b200.backbone import conv_flops  # noqa: E402
from oracle import detr_backbone_oracle as bo, detr_oracle as do  # noqa: E402


def timed(fn, reps):
    times = []
    for _ in range(reps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        times.append(s.elapsed_time(e))
    return sorted(times)[len(times) // 2]


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = (x.strip() for x in out.split(","))
        return name, power
    except Exception:                     # noqa: BLE001 - the numbers stand without it
        return torch.cuda.get_device_name(0), "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    l = mmx_b200.lib()
    cfg = do.DETR_R50
    sd = bo.init_state_dict(cfg, seed=5)
    eng = mmx_b200.DetrEngine(sd, nhead=cfg.nhead, device="cuda:0")
    sd_cuda = {k: v.cuda() for k, v in sd.items()}
    name, power = gpu_info()
    res = dict(gpu=name, power_limit=power, gemm_backend=l.mmx_get_gemm_backend(),
               eager="torch fp32 on the same GPU, torch.backends.cudnn.enabled=False, "
                     "torch.backends.cuda.matmul.allow_tf32=False, torch.backends.cudnn.allow_tf32=False",
               backbone={})
    g = torch.Generator().manual_seed(0)
    for H, W in ((800, 800), (800, 1066)):
        for B in (1, 16):
            x = torch.randn(B, 3, H, W, generator=g).cuda()
            for _ in range(2):
                eng.features(x)
            torch.cuda.synchronize()
            ms = timed(lambda: eng.features(x), args.reps)
            l.mmx_profile_gemm(1)
            eng.features(x)
            l.mmx_profile_gemm(0)
            import ctypes as C
            gms, gfl, n = C.c_double(), C.c_double(), C.c_int()
            l.mmx_profile_gemm_report(C.byref(gms), C.byref(gfl), C.byref(n))
            flops = conv_flops(eng.backbone, B, H, W)
            # eager fp32 PyTorch, no cuDNN / TF32
            cudnn, tf32m, tf32c = (torch.backends.cudnn.enabled, torch.backends.cuda.matmul.allow_tf32,
                                   torch.backends.cudnn.allow_tf32)
            torch.backends.cudnn.enabled = False
            torch.backends.cuda.matmul.allow_tf32 = False
            torch.backends.cudnn.allow_tf32 = False
            try:
                with torch.no_grad():
                    bo.backbone(sd_cuda, x, dtype=torch.float32)
                    torch.cuda.synchronize()
                    ems = timed(lambda: bo.backbone(sd_cuda, x, dtype=torch.float32), max(2, args.reps // 2))
            finally:
                torch.backends.cudnn.enabled, torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = \
                    cudnn, tf32m, tf32c
            res["backbone"][f"{H}x{W}_b{B}"] = dict(
                backbone_ms_per_image=round(ms / B, 3), backbone_gflop_per_image=round(flops / B / 1e9, 1),
                backbone_gemm_tflops=round(flops / (gms.value * 1e-3) / 1e12, 1), gemm_launches=n.value,
                gemm_share_of_backbone=round(gms.value / ms, 3),
                eager_fp32_ms_per_image=round(ems / B, 3), speedup_vs_eager=round(ems / ms, 2))
            del x
            torch.cuda.empty_cache()
    # generate_ours from images: 16 images x 1 query, 800 x 800
    gen = mmx_b200.Generator(eng)
    x = torch.randn(16, 3, 800, 800, generator=g).cuda()
    tq = torch.randint(0, cfg.queries, (16,), generator=g)
    for _ in range(2):
        gen.generate_ours(x, tq, use_lrp=False)
    torch.cuda.synchronize()
    ms = timed(lambda: gen.generate_ours(x, tq, use_lrp=False), args.reps)
    res["generate_ours_images_800x800_b16"] = dict(ms=round(ms, 2), maps_per_s=round(16 / (ms * 1e-3), 1))
    # MaskGenerator: one image, 10 queries (backbone once)
    mg = mmx_b200.MaskGenerator(eng)
    one = x[:1].contiguous()
    q = torch.arange(10)
    for _ in range(2):
        mg.get_masks(one, q)
    torch.cuda.synchronize()
    res["mask_generator_800x800_1img_10q_ms"] = round(timed(lambda: mg.get_masks(one, q), args.reps), 2)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
