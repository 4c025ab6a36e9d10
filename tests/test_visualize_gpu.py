"""GPU: the visualisation kernels (csrc/visualize.cu) against the notebook goldens (tests/golden/visualize.npz) and the
numpy oracle (oracle/visualize_oracle.py), bit for bit: the CLIP / ViT heat-map overlay, LXMERT's box-relevance image,
CLIP's text scores; batching, n_img = 1, CUDA-graph replay and the façade's errors."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import visualize_oracle as vo

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def g(golden_dir):
    return np.load(os.path.join(golden_dir, "visualize.npz"))


@pytest.fixture(scope="module")
def mmx(built_lib):
    import mmx_b200
    return mmx_b200


def _lib():
    import mmx_b200
    from mmx_b200._lib import check, ptr, current_stream
    return mmx_b200.lib(), check, ptr, current_stream


def _overlay_abi(rel, images, h, w, H, W, scale_h, scale_w):
    l, check, ptr, cs = _lib()
    rel, images = rel.to(DEV).float().contiguous(), images.to(DEV).float().contiguous()
    out = torch.empty(rel.shape[0], H, W, 3, dtype=torch.uint8, device=DEV)
    check(l.mmx_relevance_overlay(ptr(rel), rel.shape[0], h, w, scale_h, scale_w, ptr(images), images.shape[0], H, W,
                                  ptr(out), cs()))
    return out


def _box_abi(img, boxes, scores):
    l, check, ptr, cs = _lib()
    img, boxes, scores = img.to(DEV).contiguous(), boxes.to(DEV).float().contiguous(), scores.to(DEV).float().contiguous()
    B, n = boxes.shape[:2]
    H, W = img.shape[1:3]
    out = torch.empty(B, H, W, 3, dtype=torch.uint8, device=DEV)
    check(l.mmx_box_relevance_image(ptr(img), img.shape[0], H, W, ptr(boxes), ptr(scores), B, n, ptr(out), cs()))
    return out


def _text_abi(R, tokens):
    l, check, ptr, cs = _lib()
    R, tokens = R.to(DEV).float().contiguous(), tokens.to(DEV).int().contiguous()
    B, ctx = tokens.shape
    scores = torch.full((B, ctx), float("nan"), device=DEV)
    lens = torch.full((B,), -1, dtype=torch.int32, device=DEV)
    check(l.mmx_clip_text_scores(ptr(R), ptr(tokens), B, ctx, ptr(scores), ptr(lens), cs()))
    return scores, lens


def _scale(i, o):
    return float(np.float32(i) / np.float32(o))


# -- overlay -------------------------------------------------------------------------------------------------------------

def test_equal_size_copy_reproduces_golden(mmx, g):
    """The golden's own upsampled map fed through equal sizes (ATen's copy case) gives the notebook's vis."""
    tag = "clip.rand0"
    up = torch.from_numpy(g[f"{tag}.up"]).reshape(1, -1)
    img = torch.from_numpy(vo.preprocess(g["clip.image_u8"]))[None]
    out = _overlay_abi(up, img, 224, 224, 224, 224, 1.0, 1.0)
    np.testing.assert_array_equal(out[0].cpu().numpy(), g[f"{tag}.vis"])


@pytest.mark.parametrize("tag", ["clip.const_map", "clip.nan_map", "clip.const_image"])
def test_degenerate_golden_cases_through_facade(mmx, g, tag):
    """A constant map, a NaN in the map and a constant image: vis does not depend on the upsample's last bits."""
    key = f"{tag}.image"
    img = torch.from_numpy(g[key] if key in g.files else vo.preprocess(g["clip.image_u8"]))[None].to(DEV)
    out = mmx.show_image_relevance(torch.from_numpy(g[f"{tag}.rel"]).to(DEV), img)
    assert out.shape == (224, 224, 3) and out.dtype == torch.uint8
    np.testing.assert_array_equal(out.cpu().numpy(), g[f"{tag}.vis"])


@pytest.mark.parametrize("d,size", [(7, 224), (14, 224), (24, 336)])
def test_overlay_matches_oracle_on_torch_interpolate(mmx, g, d, size):
    gen = torch.Generator().manual_seed(d)
    B = 3
    rel = torch.rand(B, d * d, generator=gen)
    rel[1] = rel[1] * 1e-4 - 3.0                                  # a narrow, offset range
    images = torch.randn(B, 3, size, size, generator=gen)
    out = _overlay_abi(rel, images, d, d, size, size, _scale(d, size), _scale(d, size)).cpu().numpy()
    up = F.interpolate(rel.to(DEV).reshape(B, 1, d, d), size=size, mode="bilinear").cpu().numpy()
    for b in range(B):
        np.testing.assert_array_equal(out[b], vo.overlay(up[b, 0], images[b].numpy(), g["jet"]), err_msg=f"map {b}")


def test_overlay_scale_factor_form(mmx, g):
    """The ViT form: F.interpolate(scale_factor=16), source scale 1/16."""
    gen = torch.Generator().manual_seed(5)
    rel = torch.rand(2, 196, generator=gen)
    images = torch.randn(2, 3, 224, 224, generator=gen)
    out = _overlay_abi(rel, images, 14, 14, 224, 224, 1.0 / 16, 1.0 / 16).cpu().numpy()
    up = F.interpolate(rel.to(DEV).reshape(2, 1, 14, 14), scale_factor=16, mode="bilinear").cpu().numpy()
    for b in range(2):
        np.testing.assert_array_equal(out[b], vo.overlay(up[b, 0], images[b].numpy(), g["jet"]))


def test_jet_table_equals_golden(mmx, g):
    """A map that visits every level 0..255 and an image that is 0 except one channel of one pixel (1, where the heat map's
    channel is 0): max(cam) = 1 and each output byte is f(JET[q][c]) = uint8(255 * (JET/255)).  f is injective, so equal
    outputs mean equal tables."""
    jet = g["jet"]
    f = vo._trunc_u8(np.float32(255) * (np.arange(256, dtype=np.float32) / np.float32(255)))
    assert len(np.unique(f)) == 256
    n = 224 * 224
    k = np.arange(n) % 256
    m = np.where(k < 255, k + 0.5, 255.0).astype(np.float32)
    m[0] = 0.0
    img = np.zeros((3, 224, 224), np.float32)
    assert tuple(jet[255]) == (0, 0, 128)
    img[0].reshape(-1)[255] = 1.0                                  # pixel 255 has q = 255, JET[255] channel 0 = 0
    out = _overlay_abi(torch.from_numpy(m)[None], torch.from_numpy(img)[None], 224, 224, 224, 224, 1.0, 1.0)
    out = out[0].cpu().numpy().reshape(-1, 3)
    want = vo.overlay(m.reshape(224, 224), img, jet).reshape(-1, 3)
    np.testing.assert_array_equal(out, want)
    # and directly: each level's bytes (channels back in BGR order) are f of the golden's entry
    q = vo._trunc_u8(np.float32(255) * (m / np.float32(255)))
    sel = np.arange(n) != 255
    for lvl in range(256):
        rows = out[sel & (q == lvl)][:, ::-1]
        assert len(rows) and (rows == f[jet[lvl]]).all(), lvl


def test_batching_and_shared_image(mmx, g):
    """A map alone, inside a batch of 64, and with n_img = 1 against 64 copies of the image: identical bytes."""
    gen = torch.Generator().manual_seed(8)
    rel = torch.rand(64, 49, generator=gen)
    img = torch.randn(1, 3, 224, 224, generator=gen)
    s = _scale(7, 224)
    shared = _overlay_abi(rel, img, 7, 7, 224, 224, s, s)
    copies = _overlay_abi(rel, img.expand(64, -1, -1, -1), 7, 7, 224, 224, s, s)
    assert torch.equal(shared, copies)
    for b in (0, 31, 63):
        alone = _overlay_abi(rel[b:b + 1], img, 7, 7, 224, 224, s, s)
        assert torch.equal(alone[0], shared[b])


def test_graph_replay_equals_eager(mmx, g):
    l, check, ptr, cs = _lib()
    gen = torch.Generator().manual_seed(9)
    rel = torch.rand(16, 49, generator=gen).to(DEV)
    img = torch.randn(16, 3, 224, 224, generator=gen).to(DEV)
    bimg = torch.randint(0, 256, (1, 96, 128, 3), dtype=torch.uint8, generator=gen).to(DEV)
    boxes = (torch.rand(4, 36, 4, generator=gen) * 140 - 10).to(DEV)
    scores = torch.rand(4, 36, generator=gen).to(DEV)
    R = torch.rand(4, 77, 77, generator=gen).to(DEV)
    tok = torch.arange(77, dtype=torch.int32).flip(0).roll(9).repeat(4, 1).to(DEV)
    s = _scale(7, 224)
    outs = [torch.empty(16, 224, 224, 3, dtype=torch.uint8, device=DEV), torch.empty(4, 96, 128, 3, dtype=torch.uint8,
                                                                                     device=DEV),
            torch.empty(4, 77, device=DEV), torch.empty(4, dtype=torch.int32, device=DEV)]

    def run():
        st = cs()
        check(l.mmx_relevance_overlay(ptr(rel), 16, 7, 7, s, s, ptr(img), 16, 224, 224, ptr(outs[0]), st))
        check(l.mmx_box_relevance_image(ptr(bimg), 1, 96, 128, ptr(boxes), ptr(scores), 4, 36, ptr(outs[1]), st))
        check(l.mmx_clip_text_scores(ptr(R), ptr(tok), 4, 77, ptr(outs[2]), ptr(outs[3]), st))

    run()
    torch.cuda.synchronize()
    eager = [o.clone() for o in outs]
    for o in outs:
        o.zero_()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=side):
            run()
    torch.cuda.current_stream().wait_stream(side)
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(eager, outs):
        assert torch.equal(a, b)


# -- box relevance image -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("tag", ["lxmert.rand", "lxmert.edge", "lxmert.nan_score", "lxmert.nan_empty_box",
                                 "lxmert.neg_scores"])
def test_box_image_matches_golden(mmx, g, tag):
    img = torch.from_numpy(g["lxmert.image"]).to(DEV)
    out = mmx.save_image_vis(img, torch.from_numpy(g[f"{tag}.boxes"]).to(DEV),
                             torch.from_numpy(g[f"{tag}.scores"]).to(DEV))
    assert out.shape == img.shape and out.dtype == torch.uint8
    np.testing.assert_array_equal(out.cpu().numpy(), g[f"{tag}.out"])


@pytest.mark.parametrize("shared", [True, False])
def test_box_image_matches_oracle(mmx, shared):
    """LXMERT's size (640 x 480, 36 boxes), several questions, random and edge-case boxes."""
    gen = torch.Generator().manual_seed(21 + shared)
    B, n, H, W = 4, 36, 480, 640
    imgs = torch.randint(0, 256, (1 if shared else B, H, W, 3), dtype=torch.uint8, generator=gen)
    x0, y0 = torch.rand(B, n, generator=gen) * 800 - 100, torch.rand(B, n, generator=gen) * 600 - 100
    boxes = torch.stack([x0, y0, x0 + torch.rand(B, n, generator=gen) * 400 - 50,
                         y0 + torch.rand(B, n, generator=gen) * 300 - 50], -1)
    scores = torch.randn(B, n, generator=gen)
    scores[2, 5] = float("nan")
    out = _box_abi(imgs, boxes, scores).cpu().numpy()
    for b in range(B):
        want = vo.box_image(imgs[0 if shared else b].numpy(), boxes[b].numpy(), scores[b].numpy())
        np.testing.assert_array_equal(out[b], want, err_msg=f"question {b}")


def test_box_image_rejects_non_finite_boxes(mmx):
    img = torch.zeros(8, 8, 3, dtype=torch.uint8, device=DEV)
    boxes = torch.tensor([[0.0, 0.0, float("nan"), 4.0]], device=DEV)
    with pytest.raises(ValueError):
        mmx.save_image_vis(img, boxes, torch.ones(1, device=DEV))


# -- text scores ---------------------------------------------------------------------------------------------------------

def test_text_scores(mmx, g):
    toks = torch.stack([torch.from_numpy(g[f"text{k}.tokens"]) for k in range(5)])
    R = torch.stack([torch.from_numpy(g[f"text{k}.R"]) for k in range(5)])
    scores, lens = _text_abi(R, toks)
    scores, lens = scores.cpu().numpy(), lens.cpu().numpy()
    Rd = R.to(DEV)
    for k in range(5):
        want = vo.text_scores(g[f"text{k}.R"], g[f"text{k}.tokens"])
        assert lens[k] == len(want) == len(g[f"text{k}.scores"])
        got = scores[k, :lens[k]]
        np.testing.assert_array_max_ulp(got, want, maxulp=1)                     # the fp64-summed host value
        eot = int(toks[k].argmax())
        ref = Rd[k, eot, 1:eot] / Rd[k, eot, 1:eot].sum()                          # torch's own expression
        np.testing.assert_allclose(got, ref.cpu().numpy(), rtol=1e-5, atol=0)
        assert (scores[k, lens[k]:] == 0).all()
    assert lens[1] == 0                                                          # eot = 1: the empty slice
    views = mmx.show_heatmap_on_text(toks.to(DEV), Rd)
    assert [len(v) for v in views] == list(lens)
    single = mmx.show_heatmap_on_text(toks[0].to(DEV), Rd[0])
    assert len(single) == 1 and torch.equal(single[0], views[0])


# -- end to end ----------------------------------------------------------------------------------------------------------

def test_interpret_then_show_image_relevance_b32(mmx, g):
    from oracle import clip_oracle as co
    cfg = co.VIT_B32
    sd = co.init_state_dict(cfg, seed=0)
    eng = mmx.ClipEngine(mmx.ClipConfig(*cfg.ref_args()), sd, max_batch=64, device=DEV)
    images, tokens = co.synthetic_inputs(cfg, 64, seed=3)
    images = images.to(DEV)
    _, R_image = mmx.interpret(images, tokens.to(DEV), eng, DEV)
    out = mmx.show_image_relevance(R_image, images)
    assert out.shape == (64, 224, 224, 3)
    up = F.interpolate(R_image.reshape(64, 1, 7, 7), size=224, mode="bilinear").cpu().numpy()
    out, imgs = out.cpu().numpy(), images.cpu().numpy()
    for b in range(0, 64, 7):
        np.testing.assert_array_equal(out[b], vo.overlay(up[b, 0], imgs[b], g["jet"]), err_msg=f"map {b}")
    one = mmx.show_image_relevance(R_image[5], images[5:6])
    np.testing.assert_array_equal(one.cpu().numpy(), out[5])


@pytest.mark.parametrize("which,B", [("VIT_TINY", 3), ("VIT_B16", 1)])
def test_generate_visualization(mmx, g, which, B):
    from oracle import vit_oracle as vio
    cfg = getattr(vio, which)
    sd = vio.init_state_dict(cfg, seed=3)
    eng = mmx.ViTEngine(sd, heads=cfg.heads, device=DEV)
    images = torch.randn(B, 3, cfg.image, cfg.image, generator=torch.Generator().manual_seed(4)).to(DEV)
    x = images[0] if B == 1 else images
    out = mmx.generate_visualization(eng, x)
    assert out.shape == ((cfg.image, cfg.image, 3) if B == 1 else (B, cfg.image, cfg.image, 3))
    rel = mmx.generate_relevance(eng, images).reshape(B, 1, eng.grid, eng.grid)
    up = F.interpolate(rel, scale_factor=eng.patch, mode="bilinear").cpu().numpy()
    out = out.reshape(B, cfg.image, cfg.image, 3).cpu().numpy()
    for b in range(B):
        np.testing.assert_array_equal(out[b], vo.overlay(up[b, 0], images[b].cpu().numpy(), g["jet"]))


def test_facade_errors(mmx):
    img = torch.randn(1, 3, 224, 224, device=DEV)
    with pytest.raises(mmx.MmxError):
        mmx.show_image_relevance(torch.rand(48, device=DEV), img)              # not a square
    with pytest.raises(mmx.MmxError):
        mmx.show_image_relevance(torch.rand(49, device=DEV), torch.randn(1, 3, 112, 112, device=DEV))   # size mismatch
    with pytest.raises(mmx.MmxError):
        mmx.show_image_relevance(torch.rand(4, 49, device=DEV), torch.randn(2, 3, 224, 224, device=DEV))  # 2 images, 4 maps
    with pytest.raises(mmx.MmxError):
        mmx.show_image_relevance(torch.rand(2, 3, 49, device=DEV), img)        # bad rank
    with pytest.raises(mmx.MmxError):
        mmx.show_image_relevance(torch.rand(49), img)                           # host tensor
    with pytest.raises(mmx.MmxError):
        mmx.save_image_vis(torch.zeros(8, 8, 3, dtype=torch.uint8, device=DEV), torch.zeros(2, 4, device=DEV),
                           torch.zeros(3, device=DEV))
    with pytest.raises(mmx.MmxError):
        mmx.show_heatmap_on_text(torch.zeros(2, 77, dtype=torch.int64, device=DEV), torch.zeros(2, 76, 76, device=DEV))
