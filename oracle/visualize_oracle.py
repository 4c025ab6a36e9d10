"""numpy restatement of the notebooks' visualisation step (TEST INFRASTRUCTURE ONLY), pinned bit for bit to the
reference's own outputs in ``tests/golden/visualize.npz`` (``oracle/make_visualize_golden.py``) and used by the GPU tests
at shapes the golden does not hold.

  * ``overlay``      - show_image_relevance / generate_visualization after F.interpolate (CLIP_explainability.ipynb:216,
                       Transformer_MM_explainability_ViT.ipynb:1223): the upsampled map is an input, as the device kernel
                       is compared against torch's own interpolate
  * ``box_image``    - save_image_vis (LXMERT.ipynb:121) up to the 8-bit image cv2.imwrite encodes
  * ``text_scores``  - show_heatmap_on_text's text_scores (CLIP_explainability.ipynb:254), slice sum in float64

Every step is one numpy fp32 operation, as in the reference; casts to uint8 are written out (truncation, NaN -> 0, which is
what numpy's cast gives on x86) instead of relying on the platform's cast.
"""
from __future__ import annotations

import numpy as np

F32 = np.float32


def _trunc_u8(x: np.ndarray) -> np.ndarray:
    """np.uint8(x) for x in [0, 255] or NaN: truncation, NaN -> 0."""
    return np.where(np.isnan(x), F32(0), x).astype(np.uint8)


def _minmax(x: np.ndarray) -> np.ndarray:
    return (x - x.min()) / (x.max() - x.min())


def overlay(up: np.ndarray, image: np.ndarray, jet: np.ndarray) -> np.ndarray:
    """up [H, W] fp32 (the F.interpolate output), image [3, H, W] fp32, jet [256, 3] uint8 (cv2 COLORMAP_JET, BGR) ->
    the notebook's vis after cvtColor, [H, W, 3] uint8."""
    with np.errstate(invalid="ignore", divide="ignore"):
        m = _minmax(up.astype(F32))
        img = _minmax(np.ascontiguousarray(image.astype(F32).transpose(1, 2, 0)))
        heat = jet[_trunc_u8(F32(255) * m)].astype(F32) / F32(255)
        cam = heat + img                                  # BGR channel c + RGB channel c, as the reference adds them
        cam = cam / np.max(cam)
        vis = _trunc_u8(F32(255) * cam)
    return np.ascontiguousarray(vis[..., ::-1])           # cv2.cvtColor(RGB2BGR)


def cv_to_u8(x: np.ndarray) -> np.ndarray:
    """OpenCV's float -> 8U conversion (what imwrite applies to a float image): round half to even to int32, saturate.
    The x86 conversion gives INT_MIN for NaN, infinities and values beyond int32, so those give 0."""
    r = np.rint(np.where(np.abs(x) < F32(2 ** 31), x, F32(0)).astype(np.float64))
    return np.clip(r, 0, 255).astype(np.uint8)


def box_mask(H: int, W: int, boxes: np.ndarray, scores: np.ndarray) -> np.ndarray:
    """The reference's mask: each box's Python slice [int(y0):int(y1), int(x0):int(x1)] takes the elementwise max with its
    score (np.maximum propagates NaN, as torch.max does)."""
    mask = np.zeros((H, W), F32)
    for (x0, y0, x1, y1), s in zip(boxes.astype(F32), scores.astype(F32)):
        ys, xs = slice(int(y0), int(y1)), slice(int(x0), int(x1))
        mask[ys, xs] = np.maximum(np.full_like(mask[ys, xs], s), mask[ys, xs])
    return mask


def box_image(img: np.ndarray, boxes: np.ndarray, scores: np.ndarray) -> np.ndarray:
    """img [H, W, 3] uint8, boxes [n, 4] (x0, y0, x1, y1), scores [n] -> the 8-bit image imwrite encodes, [H, W, 3]."""
    H, W = img.shape[:2]
    with np.errstate(invalid="ignore", divide="ignore"):
        m = _minmax(box_mask(H, W, boxes, scores))
        prod = img * m[:, :, None]                       # uint8 x fp32 -> fp32
    assert prod.dtype == F32
    return cv_to_u8(prod)


def eot_index(tokens: np.ndarray) -> int:
    return int(np.argmax(tokens))


def text_scores(R_text: np.ndarray, tokens: np.ndarray) -> np.ndarray:
    """R_text [ctx, ctx], tokens [ctx] -> R_text[eot, 1:eot] / s, s the slice's float64 sum rounded once to fp32."""
    eot = eot_index(tokens)
    row = R_text[eot, 1:eot].astype(F32)
    s = F32(row.astype(np.float64).sum())
    with np.errstate(invalid="ignore", divide="ignore"):
        return row / s


def block_image_u8(H: int, W: int, seed: int, block: int = 16) -> np.ndarray:
    """A seeded uint8 [H, W, 3] picture of block x block tiles of random colour: a picture (and an overlay on it) that
    compresses well in the fixture."""
    g = np.random.default_rng(seed).integers(0, 256, size=(-(-H // block), -(-W // block), 3), dtype=np.uint8)
    return np.ascontiguousarray(np.repeat(np.repeat(g, block, 0), block, 1)[:H, :W])


CLIP_MEAN = np.array([0.48145466, 0.4578275, 0.40821073], F32)
CLIP_STD = np.array([0.26862954, 0.26130258, 0.27577711], F32)


def preprocess(u8: np.ndarray) -> np.ndarray:
    """uint8 [H, W, 3] RGB -> fp32 [3, H, W], CLIP's ToTensor + Normalize (one fp32 operation per step)."""
    x = u8.astype(F32) / F32(255)
    return np.ascontiguousarray(((x - CLIP_MEAN) / CLIP_STD).transpose(2, 0, 1))
