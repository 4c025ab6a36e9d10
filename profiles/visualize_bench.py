"""Visualisation step: the device calls (csrc/visualize.cu through mmx_b200.visualize) plus their one device-to-host copy,
against the notebooks' form on the same machine - a per-map Python loop of torch CUDA interpolate, .cpu(), numpy and cv2
(the oracle's numpy LUT step when cv2 is absent).

Workloads: the 64 CLIP ViT-B/32 image maps of one interpret batch (one repeated image, and 64 images); ViT-B/16 overlays at
B = 16; LXMERT, one 640 x 480 image, 36 boxes, 8 questions.  Each form is warmed up, then the two alternate; times are
host clocks around synchronised work (the whole call, copy included), and the kernel alone is timed with CUDA events over
repeated launches.  bytes: what the call must move at least (inputs read once, output written once); hbm_share: those bytes
at 3.35 TB/s over the kernel time.  Writes one JSON object to stdout and to --out.

    python profiles/visualize_bench.py --out /tmp/visualize_bench_h100.json
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import mmx_b200  # noqa: E402
from mmx_b200.visualize import _scale  # noqa: E402

try:
    import cv2
except ImportError:
    cv2 = None

HBM = 3.35e12
# without cv2, the notebook form looks the heat map up in cv2's JET table as the golden fixture holds it
_JET = None if cv2 is not None else np.load(os.path.join(ROOT, "tests", "golden", "visualize.npz"))["jet"]


def _jet(q):
    return cv2.applyColorMap(q, cv2.COLORMAP_JET) if cv2 is not None else _JET[q]


def _swap(vis):
    return cv2.cvtColor(vis, cv2.COLOR_RGB2BGR) if cv2 is not None else np.ascontiguousarray(vis[..., ::-1])


def notebook_overlay(rel, images, dim, size=None, scale_factor=None):
    """The notebooks' per-map loop (show_image_relevance / generate_visualization)."""
    outs = []
    for b in range(rel.shape[0]):
        r = F.interpolate(rel[b].reshape(1, 1, dim, dim), size=size, scale_factor=scale_factor, mode="bilinear")
        r = r.reshape(r.shape[-2], r.shape[-1]).cpu().numpy()
        r = (r - r.min()) / (r.max() - r.min())
        img = images[b if images.shape[0] > 1 else 0].permute(1, 2, 0).cpu().numpy()
        img = (img - img.min()) / (img.max() - img.min())
        heat = np.float32(_jet(np.uint8(255 * r))) / 255
        cam = heat + np.float32(img)
        cam = cam / np.max(cam)
        outs.append(_swap(np.uint8(255 * cam)))
    return outs


def notebook_boxes(img, boxes, scores):
    """save_image_vis's loop per question, up to the 8-bit image imwrite encodes (OpenCV's rounding, restated)."""
    outs = []
    for b in range(boxes.shape[0]):
        mask = torch.zeros(img.shape[0], img.shape[1])
        for i in range(boxes.shape[1]):
            x, y, w, h = boxes[b, i]
            cur = mask[int(y):int(h), int(x):int(w)]
            mask[int(y):int(h), int(x):int(w)] = torch.max(torch.ones_like(cur) * scores[b, i].item(), cur)
        mask = (mask - mask.min()) / (mask.max() - mask.min())
        out = img * mask.unsqueeze(-1).expand(img.shape).numpy()
        outs.append(np.clip(np.rint(np.nan_to_num(out)), 0, 255).astype(np.uint8))
    return outs


def host_ms(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3


def kernel_ms(fn, reps=50):
    fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def compare(name, device_call, device_kernel, notebook, nbytes, warmup, reps):
    for _ in range(warmup):
        device_call()
        notebook()
    dev, nb = [], []
    for _ in range(reps):                                         # alternate the two forms
        dev.append(host_ms(device_call))
        nb.append(host_ms(notebook))
    k = kernel_ms(device_kernel)
    return dict(workload=name, device_call_ms=float(np.median(dev)), device_call_ms_min=float(np.min(dev)),
                notebook_ms=float(np.median(nb)), notebook_ms_min=float(np.min(nb)),
                speedup=float(np.median(nb) / np.median(dev)), kernel_ms=k, bytes=int(nbytes),
                hbm_share=nbytes / HBM / (k * 1e-3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = "cuda:0"
    gen = torch.Generator().manual_seed(0)
    res = []

    for n_img in (1, 64):
        rel = torch.rand(64, 49, generator=gen).to(dev)
        img = torch.randn(n_img, 3, 224, 224, generator=gen).to(dev)
        nbytes = rel.numel() * 4 + img.numel() * 4 + 64 * 224 * 224 * 3
        res.append(compare(f"clip_b32_64maps_{n_img}img", lambda: mmx_b200.show_image_relevance(rel, img).cpu(),
                           lambda: mmx_b200.show_image_relevance(rel, img),
                           lambda: notebook_overlay(rel, img, 7, size=224), nbytes, a.warmup, a.reps))
    one, img1 = rel[:1], img[:1]                                  # the notebook's B = 1: launch latency dominates
    res.append(compare("clip_b32_1map", lambda: mmx_b200.show_image_relevance(one, img1).cpu(),
                       lambda: mmx_b200.show_image_relevance(one, img1),
                       lambda: notebook_overlay(one, img1, 7, size=224), 49 * 4 + 3 * 224 * 224 * 7, a.warmup, a.reps))

    rel = torch.rand(16, 196, generator=gen).to(dev)
    img = torch.randn(16, 3, 224, 224, generator=gen).to(dev)
    s = _scale(0, 1, scale_factor=16)

    def vit_device():
        l, out = mmx_b200.lib(), torch.empty(16, 224, 224, 3, dtype=torch.uint8, device=dev)
        from mmx_b200._lib import check, ptr, current_stream
        check(l.mmx_relevance_overlay(ptr(rel), 16, 14, 14, s, s, ptr(img), 16, 224, 224, ptr(out), current_stream()))
        return out

    res.append(compare("vit_b16_16maps", lambda: vit_device().cpu(), vit_device,
                       lambda: notebook_overlay(rel, img, 14, scale_factor=16),
                       rel.numel() * 4 + img.numel() * 4 + 16 * 224 * 224 * 3, a.warmup, a.reps))

    H, W, n, B = 480, 640, 36, 8
    bimg = torch.randint(0, 256, (H, W, 3), dtype=torch.uint8, generator=gen)
    x0, y0 = torch.rand(B, n, generator=gen) * (W - 40), torch.rand(B, n, generator=gen) * (H - 40)
    boxes = torch.stack([x0, y0, x0 + torch.rand(B, n, generator=gen) * 300, y0 + torch.rand(B, n, generator=gen) * 200], -1)
    scores = torch.rand(B, n, generator=gen)
    bimg_d, boxes_d, scores_d = bimg.to(dev), boxes.to(dev), scores.to(dev)
    bimg_np = bimg.numpy()
    res.append(compare("lxmert_640x480_36boxes_8q",
                       lambda: mmx_b200.save_image_vis(bimg_d, boxes_d, scores_d).cpu(),
                       lambda: mmx_b200.save_image_vis(bimg_d, boxes_d, scores_d),
                       lambda: notebook_boxes(bimg_np, boxes, scores),
                       H * W * 3 + boxes.numel() * 4 + scores.numel() * 4 + B * H * W * 3, a.warmup, a.reps))

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    line = dict(bench="visualize", gpu=torch.cuda.get_device_name(0), nvidia_smi=q[0] if q else None,
                cv2=cv2.__version__ if cv2 is not None else None, torch=torch.__version__, results=res)
    text = json.dumps(line)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
