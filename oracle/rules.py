"""Oracle restatement of the relevancy *rules* (Chefer et al., rules 5, 6, 7, 10, 11, eq. 8-9, rollout).

TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).  Plain PyTorch on CPU, fp32 by default (callers may
pass fp64 tensors for headroom).  Every function cites the reference lines it follows; the reference tree is
``hila-chefer/Transformer-MM-Explainability`` and paths are relative to it.
"""
from __future__ import annotations

import torch


def avg_heads(cam: torch.Tensor, grad: torch.Tensor) -> torch.Tensor:
    """Rule 5, single sample.  DETR/modules/ExplanationGenerator.py:19-24 (same text in
    lxmert/lxmert/src/ExplanationGenerator.py:18-23): flatten heads, ``(grad*cam).clamp(min=0).mean(0)``."""
    cam = cam.reshape(-1, cam.shape[-2], cam.shape[-1])
    grad = grad.reshape(-1, grad.shape[-2], grad.shape[-1])
    return (grad * cam).clamp(min=0).mean(dim=0)


def avg_heads_batched(cam: torch.Tensor, grad: torch.Tensor, batch: int) -> torch.Tensor:
    """Rule 5, batched, head index ``b*H+h``.  CLIP_explainability.ipynb:176-181 (cell 6):
    ``cam.reshape(batch, -1, S, S).clamp(min=0).mean(dim=1)`` applied to ``grad*cam``."""
    t, s = cam.shape[-2], cam.shape[-1]
    prod = (grad.reshape(-1, t, s) * cam.reshape(-1, t, s)).reshape(batch, -1, t, s)
    return prod.clamp(min=0).mean(dim=1)


def apply_self_attention_rules(R_ss, R_sq, cam_ss):
    """Rules 6+7.  DETR/modules/ExplanationGenerator.py:27-30: both additions from the pre-update state."""
    R_sq_addition = torch.matmul(cam_ss, R_sq)
    R_ss_addition = torch.matmul(cam_ss, R_ss)
    return R_ss_addition, R_sq_addition


def handle_residual(orig_self_attention: torch.Tensor) -> torch.Tensor:
    """Eq. 8-9.  DETR/modules/ExplanationGenerator.py:46-53: ``(R-I)/rowsum(R-I) + I`` with the
    ``diag(R-I) >= 0`` assertion (AssertionError on violation, like the reference)."""
    n = orig_self_attention.shape[-1]
    eye = torch.eye(n, dtype=orig_self_attention.dtype, device=orig_self_attention.device)
    sa = orig_self_attention.clone() - eye
    assert sa.diagonal().min() >= 0
    sa = sa / sa.sum(dim=-1, keepdim=True)
    return sa + eye


def apply_mm_attention_rules_detr(R_ss, R_qq, cam_sq, apply_normalization=True, apply_self_in_rule_10=True):
    """Rule 10 as DETR uses it.  DETR/modules/ExplanationGenerator.py:33-43; NaN -> 0 at :42."""
    R_ss_n, R_qq_n = R_ss, R_qq
    if apply_normalization:
        R_ss_n = handle_residual(R_ss)
        R_qq_n = handle_residual(R_qq)
    add = torch.matmul(R_ss_n.t(), torch.matmul(cam_sq, R_qq_n))
    if not apply_self_in_rule_10:
        add = cam_sq.clone()
    add[torch.isnan(add)] = 0
    return add


def apply_mm_attention_rules_lxmert(R_ss, R_qq, R_qs, cam_sq, apply_normalization=True,
                                    apply_self_in_rule_10=True):
    """Rules 10+11 as LXMERT uses them.  lxmert/lxmert/src/ExplanationGenerator.py:32-42 (no NaN guard)."""
    R_ss_n, R_qq_n = R_ss, R_qq
    if apply_normalization:
        R_ss_n = handle_residual(R_ss)
        R_qq_n = handle_residual(R_qq)
    R_sq_addition = torch.matmul(R_ss_n.t(), torch.matmul(cam_sq, R_qq_n))
    if not apply_self_in_rule_10:
        R_sq_addition = cam_sq
    R_ss_addition = torch.matmul(cam_sq, R_qs)
    return R_sq_addition, R_ss_addition


def compute_rollout_attention(all_layer_matrices, start_layer=0, normalize=True):
    """Attention rollout.  DETR/modules/ExplanationGenerator.py:5-16 (``normalize=True``); the VisualBERT copy
    (VisualBERT/mmf/models/transformers/backends/ExplanationGenerator.py:5-17) is batched and skips the
    row-normalisation (``normalize=False``)."""
    n = all_layer_matrices[0].shape[-1]
    eye = torch.eye(n, dtype=all_layer_matrices[0].dtype)
    mats = [m + eye for m in all_layer_matrices]
    if normalize:
        mats = [m / m.sum(dim=-1, keepdim=True) for m in mats]
    joint = mats[start_layer]
    for i in range(start_layer + 1, len(mats)):
        joint = mats[i].matmul(joint)
    return joint


def otsu_threshold_u8(img) -> int:
    """Otsu's threshold of a uint8 image as OpenCV computes it for ``cv2.threshold(..., THRESH_BINARY + THRESH_OTSU)``
    (DETR/mask_generator.py:119).  OpenCV is a third-party dependency (reference pin: opencv_python == 3.4.2.17,
    requirements.txt:6; 4.13.0 in this image), absent from the reference tree, so its published algorithm
    (imgproc/thresh.cpp ``getThreshVal_Otsu_8u``) is restated: 256-bin histogram, one pass over the bins in double
    precision maximising the between-class variance q1*q2*(mu1-mu2)^2, first maximum wins, bins with a class weight
    below FLT_EPSILON skipped.  Pinned against cv2 itself in tests/golden/otsu.npz (oracle/make_golden.py)."""
    import numpy as np
    img = np.asarray(img, dtype=np.uint8).reshape(-1)
    h = np.bincount(img, minlength=256).astype(np.float64)
    scale = 1.0 / img.size
    mu = 0.0
    for i in range(256):
        mu += i * h[i]
    mu *= scale
    mu1 = q1 = max_sigma = 0.0
    max_val = 0
    eps = float(np.finfo(np.float32).eps)
    for i in range(256):
        p_i = h[i] * scale
        mu1 *= q1
        q1 += p_i
        q2 = 1.0 - q1
        if min(q1, q2) < eps or max(q1, q2) > 1.0 - eps:
            continue
        mu1 = (mu1 + i * p_i) / q1
        mu2 = (mu - q1 * mu1) / q2
        sigma = q1 * q2 * (mu1 - mu2) * (mu1 - mu2)
        if sigma > max_sigma:
            max_sigma, max_val = sigma, i
    return max_val


def otsu_masks(cams: torch.Tensor):
    """The mask step of ``MaskGenerator.get_panoptic`` (DETR/mask_generator.py:115-121) for a batch of maps [B, n]:
    ``(cam - min) / (max - min) * 255`` -> uint8 (truncation) -> Otsu -> ``255 where pixel > threshold else 0``.
    Returns (masks [B,n] float32, thresholds [B] int64)."""
    import numpy as np
    masks, ths = [], []
    for cam in cams.float():
        q = ((cam - cam.min()) / (cam.max() - cam.min()) * 255).numpy().astype(np.uint8)
        t = otsu_threshold_u8(q)
        masks.append(torch.from_numpy(np.where(q > t, 255, 0).astype(np.float32)))
        ths.append(t)
    return torch.stack(masks), torch.tensor(ths)
