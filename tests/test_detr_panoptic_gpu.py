"""GPU: the DETR segmentation evaluation step on the device - MaskGenerator.get_panoptic, PostProcess and PostProcessSegm
(mmx_b200/detr.py, csrc/detr_postprocess.cu) - against the unmodified reference (tests/golden/detr_panoptic.npz) and
against the plain-PyTorch restatement of the post-processors run with torch's CUDA kernels (oracle/detr_postprocess_oracle.py)."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import detr_postprocess_oracle as po, rules as R
from oracle.ref_detr_panoptic import DETR_PANOPTIC as CFG, METHODS, scaled
from util import rel_err, TOL, load_golden

pytestmark = pytest.mark.gpu


class _Nested:
    def __init__(self, tensors, mask):
        self.tensors, self.mask = tensors, mask


def _golden(golden_dir):
    g = load_golden(golden_dir, "detr_panoptic.npz")
    sd = {k[3:]: torch.from_numpy(v) for k, v in g.items() if k.startswith("sd.")}
    gen = torch.Generator().manual_seed(int(g["images.seed"]))
    imgs = [torch.randn(3, *g[f"{b}.size"].tolist(), generator=gen) for b in (0, 1)]
    return g, sd, imgs


@pytest.fixture(scope="module")
def panoptic(golden_dir):
    import mmx_b200
    g, sd, imgs = _golden(golden_dir)
    sds = scaled(sd, float(g["weights.class_scale"]))
    eng = mmx_b200.DetrEngine(sds, nhead=CFG.nhead, device="cuda:0")
    return g, sd, sds, imgs, eng


def _forms(img):
    x = img[None].cuda()
    return x, _Nested(x, torch.zeros(1, *x.shape[-2:], dtype=torch.bool, device="cuda"))


@pytest.mark.parametrize("method", METHODS)
def test_get_panoptic_vs_reference(panoptic, method, capsys):
    """keep identical; pred_logits / pred_boxes / the kept cams to TOL; pred_masks -1 off the kept rows and the oracle's
    Otsu of OUR cams on them; PostProcess to TOL (labels identical); PostProcessSegm identical wherever pred_masks are."""
    import mmx_b200
    g, sd, sds, imgs, eng = panoptic
    mg = mmx_b200.MaskGenerator(eng)
    for b, img in enumerate(imgs):
        x, nt = _forms(img)
        out = mg.get_panoptic(x, None, method)
        assert set(out) == {"pred_logits", "pred_boxes", "pred_masks"}
        out_nt = mg.get_panoptic(nt, [{}], method)
        assert all(torch.equal(out[k], out_nt[k]) for k in out)
        pm, pl, pb = out["pred_masks"], out["pred_logits"], out["pred_boxes"]
        assert pm.dtype == torch.float32 and pm.is_cuda and tuple(pm.shape) == tuple(g[f"{b}.{method}.pred_masks"].shape)
        keep = mmx_b200.detr_postprocess(pl)["keep"][0].cpu()
        gk = torch.from_numpy(g[f"{b}.keep"])
        assert torch.equal(keep, gk)
        assert rel_err(pl, g[f"{b}.pred_logits"]) < TOL and rel_err(pb, g[f"{b}.pred_boxes"]) < TOL
        q = gk.nonzero().flatten()
        masks, _, cams = mg.get_masks(x, q, method)
        # the relevancy path on the reference's own features: TOL (from the image, DETR's maps also move with the 2e-5
        # rounding of the features; tests/test_detr_image_gpu.py bounds that part)
        feats = (torch.from_numpy(g[f"{b}.src"]).cuda(), torch.from_numpy(g[f"{b}.pos"]).cuda())
        e_cam = rel_err(mg.get_masks(feats, q, method)[2], g[f"{b}.{method}.cams"])
        print(f"image {b} {method}: {q.numel()} kept, cams on the reference's features {e_cam:.2e}, from the image "
              f"{rel_err(cams, g[f'{b}.{method}.cams']):.2e}")
        assert e_cam < TOL
        om, _ = R.otsu_masks(cams.cpu())
        assert torch.equal(pm[0, q].reshape(q.numel(), -1).cpu(), om)
        assert (pm[0, ~gk.cuda()] == -1).all()
        assert torch.equal(pm[0, q], masks)
        # the post-processors
        orig, size = torch.from_numpy(g[f"{b}.orig_size"])[None].cuda(), torch.from_numpy(g[f"{b}.size"])[None].cuda()
        res = mmx_b200.PostProcess()(out, orig)
        assert len(res) == 1 and set(res[0]) == {"scores", "labels", "boxes"}
        assert torch.equal(res[0]["labels"].cpu(), torch.from_numpy(g[f"{b}.labels"]))
        assert rel_err(res[0]["scores"], g[f"{b}.scores"]) < TOL and rel_err(res[0]["boxes"], g[f"{b}.boxes"]) < TOL
        res = mmx_b200.PostProcessSegm()(res, out, orig, size)
        got = res[0]["masks"]
        assert got.dtype == torch.uint8 and not got.is_cuda
        same = (pm.cpu() == torch.from_numpy(g[f"{b}.{method}.pred_masks"]))[0].flatten(1).all(1)
        print(f"image {b} {method}: pred_masks equal to the reference's on {int(same.sum())} / {same.numel()} queries")
        assert np.array_equal(got.numpy()[same.numpy()], g[f"{b}.{method}.masks"][same.numpy()])
    capsys.readouterr()


def test_get_panoptic_zero_one_kept_lrp_and_errors(panoptic, capsys):
    import mmx_b200
    g, sd, sds, imgs, eng = panoptic
    x = imgs[1][None].cuda()
    # zero kept: a zero class head gives uniform probabilities 1/6; get_masks is skipped
    mg0 = mmx_b200.MaskGenerator(mmx_b200.DetrEngine(scaled(sd, 0.0), nhead=CFG.nhead, device="cuda:0"))
    out = mg0.get_panoptic(x, None, "ours_no_lrp")
    assert "no segmentation" in capsys.readouterr().out
    assert (out["pred_masks"] == -1).all()
    # one kept: the scale in the middle of the range where exactly one query passes 0.5 (found from the unscaled logits)
    lg = mmx_b200.DetrEngine(sd, nhead=CFG.nhead, device="cuda:0")(x)["pred_logits"][0].double()
    scales = [s for s in np.arange(0.5, 40.0, 0.01)
              if int(((s * lg).softmax(-1)[:, :-1].max(-1).values > 0.5).sum()) == 1]
    assert scales
    s1 = float(scales[len(scales) // 2])
    mg1 = mmx_b200.MaskGenerator(mmx_b200.DetrEngine(scaled(sd, s1), nhead=CFG.nhead, device="cuda:0"))
    out = mg1.get_panoptic(x, None, "raw_attn")
    assert "no segmentation" in capsys.readouterr().out
    kept = (out["pred_masks"][0] != -1).flatten(1).any(1)
    assert int(kept.sum()) == 1
    # two or more kept: no message
    mg = mmx_b200.MaskGenerator(eng)
    mg.get_panoptic(x, None, "raw_attn")
    assert "no segmentation" not in capsys.readouterr().out
    # an LRP method: the shape, and the kept rows are get_masks' masks
    out = mg.get_panoptic(x, None, "ours_with_lrp")
    q = mmx_b200.detr_postprocess(out["pred_logits"])["keep"][0].nonzero().flatten()
    assert tuple(out["pred_masks"].shape) == (1, CFG.queries, *eng.spatial_dim)
    assert torch.equal(out["pred_masks"][0, q], mg.get_masks(x, q, "ours_with_lrp")[0])
    # an unknown method prints and returns None; a batch of two is refused
    assert mg.get_panoptic(x, None, "no_such_method") is None
    assert "valid explainability method" in capsys.readouterr().out
    with pytest.raises(mmx_b200.MmxError):
        mg.get_panoptic(torch.cat([x, x]), None, "raw_attn")


def _segm(pm, sizes, orig, thr):
    """mmx_detr_segm_postprocess called directly: [uint8 [Q,1,oh,ow] per image] on the CPU"""
    from mmx_b200._lib import lib, check, ptr, current_stream
    B, Q, h, w = pm.shape
    n = [Q * oh * ow for oh, ow in orig]
    out = torch.full((sum(n),), 7, dtype=torch.uint8, device="cuda")
    fs = (C.c_int * (2 * B))(*[v for s in sizes for v in s])
    fo = (C.c_int * (2 * B))(*[v for s in orig for v in s])
    check(lib().mmx_detr_segm_postprocess(ptr(pm), B, Q, h, w, fs, fo, thr, ptr(out), current_stream()))
    return [p.view(Q, 1, oh, ow).cpu() for p, (oh, ow) in zip(out.split(n), orig)]


def _planes(kind, B, Q, h, w, gen):
    if kind == "pm":                         # get_panoptic's -1 / {0, 255} rows
        x = torch.where(torch.rand(B, Q, h, w, generator=gen) < 0.4, 255.0, 0.0)
        x[:, torch.rand(Q, generator=gen) < 0.7] = -1.0
        return x
    x = torch.randn(B, Q, h, w, generator=gen)
    if kind in ("zeros", "nonfinite"):
        x[torch.rand(x.shape, generator=gen) < 0.2] = 0.0
    if kind == "nonfinite":
        for v in (float("nan"), float("inf"), -float("inf")):
            x[torch.rand(x.shape, generator=gen) < 0.02] = v
    return x


SEGM_CASES = {
    "r50_coco": (100, 25, 34, [(800, 1066)], [(480, 640)]),
    "dc5": (100, 50, 67, [(800, 1066)], [(480, 640)]),
    "odd_ratio": (9, 5, 7, [(15, 22)], [(31, 17)]),
    "orig_eq_size": (9, 8, 10, [(40, 50)], [(40, 50)]),
    "orig_2x_size": (9, 8, 10, [(40, 50)], [(80, 100)]),
    "same_size_bilinear": (9, 12, 16, [(12, 16)], [(20, 30)]),
    "downsample": (9, 30, 40, [(12, 17)], [(9, 13)]),
    "batch_crop": (100, 25, 34, [(800, 1066), (640, 1000)], [(480, 640), (427, 640)]),
}


@pytest.mark.parametrize("case", list(SEGM_CASES))
def test_segm_kernel_vs_torch_cuda(case):
    """bit for bit against the restatement on torch's CUDA kernels, for {-1, 0, 255} planes, N(0,1), exact zeros, NaN / inf,
    at thresholds 0.5 and 0.85"""
    Q, h, w, sizes, orig = SEGM_CASES[case]
    gen = torch.Generator().manual_seed(len(case))
    for kind in ("pm", "randn", "zeros", "nonfinite"):
        pm = _planes(kind, len(sizes), Q, h, w, gen).cuda()
        for thr in (0.5, 0.85):
            got = _segm(pm, sizes, orig, thr)
            ref = po.postprocess_segm(pm, torch.tensor(sizes).cuda(), torch.tensor(orig).cuda(), thr)
            for i, (a, r) in enumerate(zip(got, ref)):
                assert a.shape == r.shape and a.dtype == r.dtype
                assert torch.equal(a, r), (case, kind, thr, i, int((a != r).sum()))


def test_segm_kernel_vs_cpu_golden(golden_dir):
    g = load_golden(golden_dir, "detr_panoptic.npz")
    got = _segm(torch.from_numpy(g["syn.pred_masks"]).cuda(), g["syn.size"].tolist(), g["syn.orig_size"].tolist(), 0.5)
    for i in (0, 1):
        assert np.array_equal(got[i].numpy(), g[f"syn.masks.{i}"])


def _ulps(a, b):
    ai, bi = a.view(torch.int32).long(), b.view(torch.int32).long()
    return (ai - bi).abs()


@pytest.mark.parametrize("B,C1", [(1, 92), (3, 92), (1, 251), (3, 251), (2, 6)])
def test_postprocess_kernel_vs_torch(B, C1):
    """mmx_detr_postprocess against the restatement on torch's CUDA kernels: boxes bit-identical, scores within 2 ulp, labels
    identical (a tied row takes the lower index; a NaN row gives NaN and label 0, as torch), keep == scores > 0.5."""
    from mmx_b200._lib import lib, check, ptr, current_stream
    Q = 100
    gen = torch.Generator().manual_seed(B * 1000 + C1)
    logits = (4.0 * torch.randn(B, Q, C1, generator=gen)).cuda()
    logits[0, 1, :] = 0.0
    logits[0, 1, 1] = logits[0, 1, 3] = 5.0                       # tie between classes 1 and 3
    logits[0, 2, 5] = float("nan")
    logits[0, 3, 1] = float("inf")
    logits[0, 4, :] = -float("inf")
    logits[0, 4, 2] = 1.0
    boxes = torch.rand(B, Q, 4, generator=gen).cuda()
    sizes = torch.randint(100, 1400, (B, 2), generator=gen).cuda()
    scores = torch.empty(B, Q, device="cuda")
    labels = torch.empty(B, Q, dtype=torch.int64, device="cuda")
    keep = torch.empty(B, Q, dtype=torch.uint8, device="cuda")
    bo_ = torch.empty(B, Q, 4, device="cuda")
    check(lib().mmx_detr_postprocess(ptr(logits), C1, B, Q, C1, 0.5, ptr(scores), ptr(labels), ptr(keep), ptr(boxes), ptr(sizes),
                                     ptr(bo_), current_stream()))
    rs, rl, rb = po.postprocess(logits, boxes, sizes)
    assert torch.equal(bo_, rb)
    assert torch.equal(labels, rl)
    nan = torch.isnan(rs)
    assert torch.equal(torch.isnan(scores), nan) and nan[0, 2] and nan[0, 3]
    assert int(_ulps(scores[~nan], rs[~nan]).max()) <= 2
    assert int(labels[0, 1]) == 1 and int(labels[0, 2]) == 0
    assert torch.equal(keep.bool(), scores > 0.5)
    # the Python form, and the NULL outputs
    import mmx_b200
    r = mmx_b200.detr_postprocess(logits, boxes, sizes)
    assert torch.equal(r["scores"].nan_to_num(-1.0), scores.nan_to_num(-1.0)) and torch.equal(r["labels"], labels) and torch.equal(r["boxes"], bo_)
    check(lib().mmx_detr_postprocess(ptr(logits), C1, B, Q, C1, 0.5, None, None, ptr(keep), None, None, None, current_stream()))
    assert torch.equal(keep.bool(), scores > 0.5)


def test_host_checks():
    import mmx_b200
    from mmx_b200._lib import lib, ptr, current_stream
    x = torch.zeros(1, 4, 2, device="cuda")
    with pytest.raises(mmx_b200.MmxError):
        mmx_b200.detr_postprocess(x[..., :1])                       # C + 1 = 1
    post = mmx_b200.PostProcessSegm()
    size, orig = torch.tensor([[10, 12]]), torch.tensor([[20, 24]])
    with pytest.raises(mmx_b200.MmxError):                          # h == 1: the reference's squeeze(2) would drop it
        post([{}], {"pred_masks": torch.zeros(1, 4, 1, 6, device="cuda")}, orig, size)
    with pytest.raises(mmx_b200.MmxError):
        post([{}], {"pred_masks": torch.zeros(1, 4, 3, 6, device="cuda")}, orig, torch.tensor([[0, 12]]))
    with pytest.raises(mmx_b200.MmxError):
        post([{}], {"pred_masks": torch.zeros(1, 4, 3, 6, device="cuda")}, torch.tensor([[20, -1]]), size)
    # a [B, Q, 1, h, w] input is squeezed as the reference does
    r = post([{}], {"pred_masks": torch.zeros(1, 4, 1, 3, 6, device="cuda")}, orig, size)
    assert tuple(r[0]["masks"].shape) == (4, 1, 20, 24) and not r[0]["masks"].any()
    assert lib().mmx_detr_segm_postprocess(None, 1, 4, 3, 6, None, None, 0.5, None, current_stream()) != 0
