"""CPU: the numpy visualisation oracle (oracle/visualize_oracle.py) equals the unmodified notebook code's outputs in
tests/golden/visualize.npz bit for bit: show_image_relevance / generate_visualization's vis, save_image_vis's 8-bit image,
show_heatmap_on_text's text_scores, cv2's JET table and cv2's float -> 8U conversion."""
import os

import numpy as np
import pytest
import torch

from oracle import visualize_oracle as vo


@pytest.fixture(scope="module")
def g(golden_dir):
    return np.load(os.path.join(golden_dir, "visualize.npz"))


def _cpu_up(rel, size=None, scale_factor=None):
    d = int(rel.size ** 0.5)
    x = torch.from_numpy(rel).reshape(1, 1, d, d)
    y = torch.nn.functional.interpolate(x, size=size, scale_factor=scale_factor, mode="bilinear")
    return y.reshape(y.shape[-2], y.shape[-1]).numpy()


def _clip_image(g, tag):
    key = f"{tag}.image"
    return g[key] if key in g.files else vo.preprocess(g["clip.image_u8"])


@pytest.mark.parametrize("tag", ["clip.rand0", "clip.grid14", "clip.const_map", "clip.nan_map", "clip.const_image"])
def test_clip_overlay_matches_notebook(g, tag):
    up = _cpu_up(g[f"{tag}.rel"], size=224)
    if f"{tag}.up" in g.files:
        np.testing.assert_array_equal(up, g[f"{tag}.up"])
    got = vo.overlay(up, _clip_image(g, tag), g["jet"])
    np.testing.assert_array_equal(got, g[f"{tag}.vis"])


def test_degenerate_inputs_are_what_the_notebook_draws(g):
    # a constant map or a NaN in it normalises to NaN, which the uint8 cast turns into 0: JET[0] everywhere
    assert (g["clip.const_map.vis"] == g["clip.nan_map.vis"]).all()
    # a constant image normalises to NaN everywhere: cam / max is NaN, every byte 0
    assert not g["clip.const_image.vis"].any()


def test_vit_overlay_matches_notebook(g):
    up = _cpu_up(g["vit.rand0.rel"], scale_factor=16)
    got = vo.overlay(up, vo.preprocess(g["clip.image_u8"]), g["jet"])
    np.testing.assert_array_equal(got, g["vit.rand0.vis"])


@pytest.mark.parametrize("tag", ["lxmert.rand", "lxmert.edge", "lxmert.nan_score", "lxmert.nan_empty_box",
                                 "lxmert.neg_scores"])
def test_box_image_matches_notebook(g, tag):
    got = vo.box_image(g["lxmert.image"], g[f"{tag}.boxes"], g[f"{tag}.scores"])
    np.testing.assert_array_equal(got, g[f"{tag}.out"])


def test_nan_score_cases(g):
    assert not g["lxmert.nan_score.out"].any()                        # a covering NaN box: mask NaN, image 0
    np.testing.assert_array_equal(g["lxmert.nan_empty_box.out"],       # a NaN on an empty box changes nothing
                                  vo.box_image(g["lxmert.image"], g["lxmert.edge.boxes"],
                                               np.nan_to_num(g["lxmert.nan_empty_box.scores"], nan=-1.0)))


@pytest.mark.parametrize("k", range(5))
def test_text_scores_match_notebook(g, k):
    got = vo.text_scores(g[f"text{k}.R"], g[f"text{k}.tokens"])
    want = g[f"text{k}.scores"]
    assert got.shape == want.shape
    # the reference's R.sum() is fp32 in torch's order; the library (and the oracle) sum in float64 and round once, which
    # is at least as close to the exact sum.  The two sums differ by at most 1 ulp, so the quotients by at most 2
    np.testing.assert_array_max_ulp(got, want, maxulp=2)
    row = g[f"text{k}.R"][vo.eot_index(g[f"text{k}.tokens"]), 1:len(got) + 1]
    np.testing.assert_allclose(got, row / row.astype(np.float64).sum(), rtol=2e-7, atol=0)


def test_jet_and_cv8u_conversion(g):
    jet = g["jet"]
    assert jet.shape == (256, 3) and jet.dtype == np.uint8
    assert tuple(jet[0]) == (128, 0, 0) and tuple(jet[255]) == (0, 0, 128)
    np.testing.assert_array_equal(vo.cv_to_u8(g["cv8u.in"]), g["cv8u.out"])
