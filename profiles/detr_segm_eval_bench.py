"""DETR segmentation evaluation step on one GPU: PostProcess + PostProcessSegm at COCO shapes against the reference's eager
PyTorch form, and MaskGenerator.get_panoptic + both post-processors per image at DETR-R50 dimensions.  Writes one JSON file.

    python profiles/detr_segm_eval_bench.py [--reps 20] [--out profiles/detr_segm_eval_bench_h100.json]

* postprocess: B = 1 (pred_masks [1,100,25,34], size 800x1066, original 480x640) and a padded B = 2 batch (sizes 800x1066
  and 704x1066, originals 480x640 and 427x640).  pred_masks hold get_panoptic's values (-1 rows, {0, 255} kept rows).
  "ours" is mmx_b200.PostProcess + PostProcessSegm (one kernel each, one uint8 copy to the host); "eager" is the reference's
  PostProcess / PostProcessSegm arithmetic in PyTorch on the same GPU: bilinear to the padded size in fp32, sigmoid > 0.5,
  the bool masks copied to the host, the crop and the float nearest resize on the CPU (DETR/models/segmentation.py:224-242).
  Both end when the masks are on the host; host-clock medians.  host_bytes: the bytes each form copies to the host.
* panoptic: get_panoptic("ours_no_lrp") + PostProcess + PostProcessSegm for one 800x1066 N(0, 1) image, DETR-R50 dimensions
  (seeded ResNet-50 + d_model 256, 8 heads, 6 + 6 layers, 100 queries), with class_embed scaled so that some queries are kept.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import mmx_b200  # noqa: E402
from oracle import detr_backbone_oracle as bo, detr_oracle as do  # noqa: E402
from oracle.ref_detr_panoptic import scaled  # noqa: E402
from detr_image_bench import gpu_info  # noqa: E402


def host_timed(fn, reps):
    times = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
    return sorted(times)[len(times) // 2]


def eager(outputs, orig, sizes, threshold=0.5):
    """PostProcess + PostProcessSegm as the reference computes them (detr.py:289-306, segmentation.py:224-242)."""
    prob = F.softmax(outputs["pred_logits"], -1)
    scores, labels = prob[..., :-1].max(-1)
    x_c, y_c, w, h = outputs["pred_boxes"].unbind(-1)
    boxes = torch.stack([(x_c - 0.5 * w), (y_c - 0.5 * h), (x_c + 0.5 * w), (y_c + 0.5 * h)], dim=-1)
    img_h, img_w = orig.unbind(1)
    boxes = boxes * torch.stack([img_w, img_h, img_w, img_h], dim=1)[:, None, :]
    results = [{"scores": s, "labels": l, "boxes": b} for s, l, b in zip(scores, labels, boxes)]
    max_h, max_w = sizes.max(0)[0].tolist()
    m = F.interpolate(outputs["pred_masks"], size=(max_h, max_w), mode="bilinear", align_corners=False)
    m = (m.sigmoid() > threshold).cpu()
    for i, (cur, t, tt) in enumerate(zip(m, sizes, orig)):
        r = cur[:, :t[0], :t[1]].unsqueeze(1)
        results[i]["masks"] = F.interpolate(r.float(), size=tuple(tt.tolist()), mode="nearest").byte()
    return results


def postprocess_case(B, sizes, origs, reps):
    g = torch.Generator().manual_seed(B)
    Q, h, w = 100, 25, 34
    pm = torch.where(torch.rand(B, Q, h, w, generator=g) < 0.4, 255.0, 0.0)
    pm[:, torch.rand(Q, generator=g) < 0.9] = -1.0
    outputs = {"pred_logits": torch.randn(B, Q, 92, generator=g).cuda(), "pred_boxes": torch.rand(B, Q, 4, generator=g).cuda(),
               "pred_masks": pm.cuda()}
    size, orig = torch.tensor(sizes).cuda(), torch.tensor(origs).cuda()
    post, segm = mmx_b200.PostProcess(), mmx_b200.PostProcessSegm()
    ours = lambda: segm(post(outputs, orig), outputs, orig, size)
    ref = lambda: eager(outputs, orig, size)
    a, b = ours(), ref()
    same = all(torch.equal(x["masks"], y["masks"]) and torch.equal(x["labels"], y["labels"]) for x, y in zip(a, b))
    t_ours, t_ref = [], []
    for _ in range(3):                         # alternate the two forms
        t_ours.append(host_timed(ours, reps))
        t_ref.append(host_timed(ref, reps))
    mo, mr = float(np.median(t_ours)), float(np.median(t_ref))
    return dict(B=B, pred_masks=[B, Q, h, w], sizes=sizes, orig_sizes=origs, ours_ms=round(mo, 3), eager_ms=round(mr, 3),
                speedup=round(mr / mo, 2), masks_identical=same,
                host_bytes_ours=sum(Q * oh * ow for oh, ow in origs),
                host_bytes_eager=B * Q * max(s[0] for s in sizes) * max(s[1] for s in sizes))


def panoptic_case(reps):
    cfg = do.DETR_R50
    sd = bo.init_state_dict(cfg, seed=5)
    x = torch.randn(1, 3, 800, 1066, generator=torch.Generator().manual_seed(1)).cuda()
    lg = mmx_b200.DetrEngine(sd, nhead=cfg.nhead, device="cuda:0")(x)["pred_logits"][0].double()
    kept = lambda s: int(((s * lg).softmax(-1)[:, :-1].max(-1).values > 0.5).sum())
    scale = min((abs(kept(s) - 5), float(s)) for s in np.arange(1.0, 400.0, 0.05) if kept(s) >= 1)[1]   # ~5 kept
    eng = mmx_b200.DetrEngine(scaled(sd, scale), nhead=cfg.nhead, device="cuda:0")
    mg, post, segm = mmx_b200.MaskGenerator(eng), mmx_b200.PostProcess(), mmx_b200.PostProcessSegm()
    orig, size = torch.tensor([[480, 640]]).cuda(), torch.tensor([[800, 1066]]).cuda()
    state = {}

    def step():
        out = mg.get_panoptic(x, None, "ours_no_lrp")
        state["kept"] = int((out["pred_masks"][0] != -1).flatten(1).any(1).sum())
        segm(post(out, orig), out, orig, size)

    step()
    ms = host_timed(step, reps)
    return dict(image=[800, 1066], class_scale=scale, kept=state["kept"], ms_per_image=round(ms, 2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=os.path.join(os.path.dirname(os.path.abspath(__file__)), "detr_segm_eval_bench_h100.json"))
    args = ap.parse_args()
    name, power = gpu_info()
    res = {"gpu": name, "power_limit": power,
           "postprocess": [postprocess_case(1, [[800, 1066]], [[480, 640]], args.reps),
                           postprocess_case(2, [[800, 1066], [704, 1066]], [[480, 640], [427, 640]], args.reps)],
           "panoptic": panoptic_case(max(3, args.reps // 4))}
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        f.write(json.dumps(res) + "\n")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
