"""Golden fixture of the notebooks' visualisation step, ``tests/golden/visualize.npz``, from the UNMODIFIED notebook code.

TEST INFRASTRUCTURE ONLY.  Run in the build container (needs the reference tree and cv2)::

    python -m oracle.make_visualize_golden

The four functions are exec'd straight from the notebooks' JSON, as ``ref_shims.reference_interpret`` does for
``interpret``: ``show_image_relevance`` and ``show_heatmap_on_text`` (CLIP_explainability.ipynb), ``show_cam_on_image`` +
``generate_visualization`` (Transformer_MM_explainability_ViT.ipynb) and ``save_image_vis`` (LXMERT.ipynb).  matplotlib,
captum's ``visualization`` and the tokenizer are stubbed; ``.cuda()`` is an identity.  Captured: ``vis`` where it reaches
``axs[1].imshow`` (or is returned), the array handed to ``cv2.imwrite`` converted to 8 bits by OpenCV itself (a lossless
PNG round trip through ``imencode`` / ``imdecode``: imwrite's own conversion), the printed ``text_scores``, and the
upsampled map ``F.interpolate`` returned.
"""
from __future__ import annotations

import json
import os
import types

import cv2
import numpy as np
import torch

from . import ref_shims as rs
from . import visualize_oracle as vo

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "visualize.npz")


def _cell(nb_name, head):
    with open(os.path.join(rs.REFERENCE_ROOT, nb_name)) as f:
        nb = json.load(f)
    for cell in nb["cells"]:
        s = "".join(cell["source"])
        if cell["cell_type"] == "code" and head in s:
            return s
    raise AssertionError(f"{head} not found in {nb_name}")


def _defs(src, *names):
    """The source of the named top-level functions of a cell (the rest of the cell loads models)."""
    out = []
    lines = src.split("\n")
    for n in names:
        i = next(k for k, l in enumerate(lines) if l.startswith(f"def {n}("))
        j = next((k for k in range(i + 1, len(lines)) if lines[k].strip() and not lines[k][0].isspace()), len(lines))
        out.append("\n".join(lines[i:j]))
    return "\n\n".join(out)


class _Axes:
    def __init__(self, sink):
        self.sink = sink

    def imshow(self, x, *a, **k):
        self.sink.append(np.array(x))

    def axis(self, *a, **k):
        pass


def _plt(sink):
    axs = [_Axes([]), _Axes(sink)]
    return types.SimpleNamespace(subplots=lambda *a, **k: (None, axs))


def _imwrite_u8(img):
    """What cv2.imwrite encodes for a float image: OpenCV's own 8U conversion, read back through a lossless PNG."""
    ok, buf = cv2.imencode(".png", np.ascontiguousarray(img))
    assert ok
    return cv2.imdecode(buf, cv2.IMREAD_UNCHANGED)


def _with_interpolate_spy(fn):
    captured = {}
    orig = torch.nn.functional.interpolate

    def spy(x, *a, **k):
        y = orig(x, *a, **k)
        captured["up"] = y.detach().clone().reshape(y.shape[-2], y.shape[-1]).numpy()
        return y

    torch.nn.functional.interpolate = spy
    try:
        with rs.cuda_is_identity():
            res = fn()
    finally:
        torch.nn.functional.interpolate = orig
    return res, captured["up"]


def clip_cases(out):
    src = _cell("CLIP_explainability.ipynb", "def show_image_relevance(")
    rng = np.random.default_rng(11)
    img = vo.preprocess(vo.block_image_u8(224, 224, seed=1))
    const_img = np.full_like(img, 0.25)
    nan_map = rng.random(49).astype(np.float32)
    nan_map[17] = np.nan
    cases = {"clip.rand0": (rng.random(49).astype(np.float32), img),
             "clip.grid14": (rng.random(196).astype(np.float32), img),
             "clip.const_map": (np.full(49, 0.5, np.float32), img),
             "clip.nan_map": (nan_map, img),
             "clip.const_image": (rng.random(49).astype(np.float32), const_img)}
    out["clip.image_u8"] = vo.block_image_u8(224, 224, seed=1)
    for tag, (rel, im) in cases.items():
        sink = []
        ns = {"torch": torch, "np": np, "cv2": cv2, "plt": _plt(sink)}
        exec(compile(src, "CLIP_explainability.ipynb:show_image_relevance", "exec"), ns)
        _, up = _with_interpolate_spy(lambda: ns["show_image_relevance"](torch.from_numpy(rel), torch.from_numpy(im)[None], None))
        out[f"{tag}.rel"] = rel
        out[f"{tag}.vis"] = sink[0]
        if tag == "clip.rand0":
            # one captured map (a [224, 224] fp32 array does not compress); the tests recompute the others with torch's
            # CPU interpolate, which they check against this one
            out[f"{tag}.up"] = up
        if im is const_img:
            out[f"{tag}.image"] = im


def vit_cases(out):
    src = _defs(_cell("Transformer_MM_explainability_ViT.ipynb", "def generate_visualization("),
                "show_cam_on_image", "generate_visualization")
    img = vo.preprocess(vo.block_image_u8(224, 224, seed=1))      # the CLIP cases' image, clip.image_u8
    rng = np.random.default_rng(12)
    for k in range(1):
        rel = rng.random(196).astype(np.float32)
        ns = {"torch": torch, "np": np, "cv2": cv2, "model": None,
              "generate_relevance": lambda model, x, index=None, r=rel: torch.from_numpy(r)[None]}
        exec(compile(src, "Transformer_MM_explainability_ViT.ipynb:generate_visualization", "exec"), ns)
        vis, _ = _with_interpolate_spy(lambda: ns["generate_visualization"](torch.from_numpy(img)))
        out[f"vit.rand{k}.rel"] = rel
        out[f"vit.rand{k}.vis"] = vis


def lxmert_cases(out):
    src = _cell("LXMERT.ipynb", "def save_image_vis(")
    H, W, n = 120, 160, 36
    rng = np.random.default_rng(13)
    img = vo.block_image_u8(H, W, seed=3)                 # read as BGR, as cv2.imread gives it
    out["lxmert.image"] = img

    def boxes_rand():
        x0, y0 = rng.uniform(0, W - 10, n), rng.uniform(0, H - 10, n)
        return np.stack([x0, y0, x0 + rng.uniform(5, 80, n), y0 + rng.uniform(5, 60, n)], 1).astype(np.float32)

    edge = boxes_rand()
    edge[0] = [-30.7, -20.2, -3.9, -1.5]          # negative: both bounds wrap once
    edge[1] = [50.0, 40.0, 20.0, 10.0]            # reversed: empty
    edge[2] = [100.0, 90.0, 400.0, 300.0]         # past the image: clamped
    edge[3] = [-500.0, -400.0, 30.0, 20.0]        # far negative start: clamps to 0
    edge[4] = [-0.9, -0.5, 12.7, 9.99]            # int() truncates toward zero
    edge[5] = [155.0, 115.0, 2000.0, 1000.0]
    s_rand = rng.random(n).astype(np.float32)
    s_nan = rng.random(n).astype(np.float32)
    s_nan[7] = np.nan
    s_nan_empty = rng.random(n).astype(np.float32)
    s_nan_empty[1] = np.nan                       # its box (edge[1]) is empty: no effect
    cases = {"lxmert.rand": (boxes_rand(), s_rand), "lxmert.edge": (edge, rng.random(n).astype(np.float32)),
             "lxmert.nan_score": (edge, s_nan), "lxmert.nan_empty_box": (edge, s_nan_empty),
             "lxmert.neg_scores": (boxes_rand(), -rng.random(n).astype(np.float32))}
    for tag, (boxes, scores) in cases.items():
        sink = []
        cv = types.SimpleNamespace(imread=lambda path: img.copy(), imwrite=lambda path, x: sink.append(_imwrite_u8(x)))
        ns = {"torch": torch, "np": np, "cv2": cv, "image_scores": torch.from_numpy(scores),
              "model_lrp": types.SimpleNamespace(bboxes=torch.from_numpy(boxes)[None])}
        exec(compile(src, "LXMERT.ipynb:save_image_vis", "exec"), ns)
        ns["save_image_vis"]("unused.jpg", torch.from_numpy(scores))
        out[f"{tag}.boxes"], out[f"{tag}.scores"], out[f"{tag}.out"] = boxes, scores, sink[0]


def text_cases(out):
    src = _defs(_cell("CLIP_explainability.ipynb", "def show_heatmap_on_text("), "show_heatmap_on_text")
    rng = np.random.default_rng(14)
    ctx = 77
    for k, eot in enumerate((8, 1, 40, 76, 2)):
        tokens = rng.integers(1, 49405, ctx).astype(np.int64)
        tokens[0], tokens[eot], tokens[eot + 1:] = 49406, 49407, 0
        R = np.zeros((ctx, ctx), np.float32)          # the function reads only the EOT row
        R[eot] = rng.random(ctx).astype(np.float32)
        printed = []
        ns = {"torch": torch, "print": lambda x, *a, **kw: printed.append(x.detach().clone().numpy()),
              "_tokenizer": types.SimpleNamespace(encode=lambda t: [], decode=lambda t: ""),
              "visualization": types.SimpleNamespace(VisualizationDataRecord=lambda *a: None,
                                                     visualize_text=lambda *a: None)}
        exec(compile(src, "CLIP_explainability.ipynb:show_heatmap_on_text", "exec"), ns)
        ns["show_heatmap_on_text"]("unused", torch.from_numpy(tokens), torch.from_numpy(R))
        out[f"text{k}.tokens"], out[f"text{k}.R"], out[f"text{k}.scores"] = tokens, R, printed[0]


def main():
    out = {}
    out["jet"] = cv2.applyColorMap(np.arange(256, dtype=np.uint8).reshape(256, 1), cv2.COLORMAP_JET).reshape(256, 3)
    conv = np.array([0.5, 1.5, 2.5, 3.5, 127.5, 128.5, 253.5, 254.5, 255.49, 255.5, 256.0, 300.0, 1e9, -0.4, -0.5, -0.6,
                     -3.0, -1e9, np.inf, -np.inf, np.nan, 0.49999997, 1.4999999], np.float32)
    conv = np.pad(conv, (0, (-len(conv)) % 3)).reshape(1, -1, 3)
    out["cv8u.in"], out["cv8u.out"] = conv, _imwrite_u8(conv)
    clip_cases(out)
    vit_cases(out)
    lxmert_cases(out)
    text_cases(out)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
