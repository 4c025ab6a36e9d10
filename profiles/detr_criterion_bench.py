"""DETR's evaluation criterion per batch on the H100: mmx_b200.SetCriterion (cost, assignment, box / label and mask
losses on the device, one host synchronisation) against the eager restatement (oracle/detr_criterion_oracle.py: torch
on the same GPU, the assignment on the host), at COCO shapes: Q = 100, 92 logit columns, 6 decoder layers (aux_outputs
on), 25x34 mask planes, targets padded to 800x1066; T in {7, 20, 60} targets per image, B = 1 and a padded B = 2
(800x1066 and 704x1066).  The eager arm solves each assignment with scipy's compiled linear_sum_assignment, as the
reference's matcher does.  One sample is a window of --calls calls timed on the host clock and closed by a synchronise
(a single device call is about 1 ms, too short to time alone); the two forms alternate sample by sample, and the median
per call is recorded with the 10th and 90th percentiles of the samples.  Also records the largest relative loss
difference and the host synchronisations per call (torch's CUDA sync debug mode counts them).

    python profiles/detr_criterion_bench.py [--reps 15] [--calls 20] [--out profiles/detr_criterion_bench_h100.json]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
from scipy.optimize import linear_sum_assignment  # noqa: E402

import mmx_b200  # noqa: E402
from oracle import detr_criterion_oracle as co  # noqa: E402

LOSSES = ["labels", "boxes", "cardinality", "masks"]
Q, C1, LAYERS, h, w = 100, 92, 6, 25, 34
SIZES = ((800, 1066), (704, 1066))


def case(B, T, seed=0):
    g = torch.Generator().manual_seed(seed)
    layers = []
    for _ in range(LAYERS):
        lg = 3.0 * torch.randn(B, Q, C1, generator=g)
        bx = torch.cat([0.2 + 0.6 * torch.rand(B, Q, 2, generator=g), 0.05 + 0.4 * torch.rand(B, Q, 2, generator=g)], -1)
        layers.append({"pred_logits": lg.cuda(), "pred_boxes": bx.cuda()})
    out = dict(layers[-1])
    out["aux_outputs"] = layers[:-1]
    out["pred_masks"] = (4.0 * torch.randn(B, Q, h, w, generator=g)).cuda()
    tg = []
    for b in range(B):
        tg.append({"labels": torch.randint(0, C1 - 1, (T,), generator=g).cuda(),
                   "boxes": torch.cat([0.2 + 0.6 * torch.rand(T, 2, generator=g),
                                       0.05 + 0.4 * torch.rand(T, 2, generator=g)], -1).cuda(),
                   "masks": (torch.rand(T, *SIZES[b], generator=g) < 0.3).cuda()})
    return out, tg


def syncs(fn):
    """host synchronisations torch sees in one call (sync debug mode warns on each)"""
    torch.cuda.set_sync_debug_mode("warn")
    try:
        with warnings.catch_warnings(record=True) as rec:
            warnings.simplefilter("always")
            fn()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    return sum("synchroniz" in str(r.message) for r in rec)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15, help="samples per form and case")
    ap.add_argument("--calls", type=int, default=20, help="calls per timed sample")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "detr_criterion_bench_h100.json"))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    crit = mmx_b200.SetCriterion(C1 - 1, mmx_b200.HungarianMatcher(), {}, 0.1, LOSSES).to("cuda")
    rows = []
    for B in (1, 2):
        for T in (7, 20, 60):
            out, tg = case(B, T, seed=B * 100 + T)
            dev_fn = lambda: crit(out, tg)
            ref_fn = lambda: co.criterion(out, tg, C1 - 1, 0.1, LOSSES, solver=linear_sum_assignment)
            for _ in range(3):
                dev_fn(); ref_fn()
            torch.cuda.synchronize()
            td, tr = [], []
            for _ in range(a.reps):
                for fn, acc in ((dev_fn, td), (ref_fn, tr)):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    for _ in range(a.calls):
                        fn()
                    torch.cuda.synchronize()
                    acc.append((time.perf_counter() - t0) / a.calls)
            got, ref = dev_fn(), ref_fn()
            err = max(abs(float(got[k]) - float(ref[k])) / max(abs(float(ref[k])), 1e-30) for k in ref)
            q = lambda xs: [1e3 * x for x in statistics.quantiles(xs, n=10)[::8]]     # p10, p90
            row = {"B": B, "T_per_image": T, "mmx_ms": 1e3 * statistics.median(td), "mmx_ms_p10_p90": q(td),
                   "eager_ms": 1e3 * statistics.median(tr), "eager_ms_p10_p90": q(tr),
                   "max_rel_loss_diff": err, "keys_equal": list(got) == list(ref),
                   "host_syncs_mmx": syncs(dev_fn), "host_syncs_eager": syncs(ref_fn)}
            row["speedup"] = row["eager_ms"] / row["mmx_ms"]
            print(json.dumps(row), flush=True)
            rows.append(row)
    res = {"gpu": smi, "torch": torch.__version__, "reps": a.reps, "calls_per_sample": a.calls,
           "eager_solver": "scipy.optimize.linear_sum_assignment", "shape": {"Q": Q, "C1": C1, "layers": LAYERS,
           "mask_plane": [h, w], "target_sizes": SIZES}, "rows": rows}
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
