"""GPU: DETR with the DC5 (dilated layer4, stride-16) backbone - dilated convs, the long-row attention path its maps
need (1122 tokens and up), MaskGenerator chunking - against the fp64 oracle (oracle/detr_dc5_oracle.py) and the
unmodified reference built with ``dilation=True`` (tests/golden/detr_dc5.npz); and plain DETR-R50 on a padded COCO-size
batch past 1024 tokens."""
import pytest
import torch

from oracle import detr_backbone_oracle as bo, detr_dc5_oracle as dc5, detr_oracle as do
from util import rel_err, TOL

pytestmark = pytest.mark.gpu
CFG = bo.DETR_IMAGE


def _bchw(t, B, h, w):
    return t.view(B, h, w, -1).permute(0, 3, 1, 2)


def _golden(golden_dir):
    from util import load_golden
    g = load_golden(golden_dir, "detr_dc5.npz")
    return g, {k[3:]: torch.from_numpy(v) for k, v in g.items() if k.startswith("sd.")}


@pytest.fixture(scope="module")
def case(golden_dir):
    import mmx_b200
    g, sd = _golden(golden_dir)
    eng = mmx_b200.DetrEngine(sd, nhead=CFG.nhead, device="cuda:0", dilation=True)
    return dict(g=g, sd=sd, eng=eng, imgs=dc5.pair_images(int(g["images.seed"])), big=dc5.long_image(int(g["long.seed"])))


def test_features_mask_pos_vs_oracle(case):
    eng, sd = case["eng"], case["sd"]
    x, m = bo.nested(case["imgs"])
    src, pos, mf = dc5.backbone(sd, x, m)
    f = eng.features([t.cuda() for t in case["imgs"]])
    assert (f.h, f.w) == tuple(src.shape[-2:]) == (8, 10)
    assert torch.equal(f.mask.cpu(), mf) and mf.any()
    e_pos = (_bchw(f.pe, f.B, f.h, f.w).cpu() - pos).abs().max().item()
    e_src = rel_err(_bchw(f.x, f.B, f.h, f.w), src)
    print(f"DC5 features vs fp64 oracle {e_src:.2e}, pos max abs err {e_pos:.2e}")
    assert e_pos <= 1e-6 and e_src < TOL
    # the stride-32 engine on the same weights still gives the stride-32 map
    import mmx_b200
    f32 = mmx_b200.DetrEngine(sd, nhead=CFG.nhead, device="cuda:0").features(x.cuda())
    assert (f32.h, f32.w) == (4, 5)


def test_golden_unmodified_reference(case):
    """the padded pair (mask, pos, src, logits, boxes), per-image maps and baselines, and the 1122-token image's maps"""
    import mmx_b200
    g, sd, eng = case["g"], case["sd"], case["eng"]
    cimgs = [t.cuda() for t in case["imgs"]]
    f = eng.features(cimgs)
    assert torch.equal(f.mask.cpu(), torch.from_numpy(g["mask"]))
    e_pos = (_bchw(f.pe, f.B, f.h, f.w).cpu() - torch.from_numpy(g["pos"])).abs().max().item()
    out = eng(cimgs)
    e = dict(src=rel_err(_bchw(f.x, f.B, f.h, f.w), g["src"]), logits=rel_err(out["pred_logits"], g["pred_logits"]),
             boxes=rel_err(out["pred_boxes"], g["pred_boxes"]))
    print(f"DC5 vs reference: pos {e_pos:.2e} abs, " + ", ".join(f"{k} {v:.2e}" for k, v in e.items()))
    assert e_pos <= 1e-6 and max(e.values()) < TOL
    gen = mmx_b200.Generator(eng)
    cases = [(f"R.{b}", f"base.{b}", img, int(g["tq"][b])) for b, img in enumerate(case["imgs"])]
    cases.append(("long.R", None, case["big"], int(g["long.tq"])))
    for rkey, bkey, img, t in cases:
        one = img[None].cuda()
        tq = torch.tensor([t])
        fb = eng.features(one)
        own = (_bchw(fb.x, 1, fb.h, fb.w).cpu().double(), _bchw(fb.pe, 1, fb.h, fb.w).cpu())
        ref_feats = dc5.backbone(sd, img[None], dtype=torch.float32)[:2]      # the reference's features to 1e-5
        for norm, s10 in ((1, 1), (0, 1), (1, 0)):
            kw = dict(normalize_self_attention=bool(norm), apply_self_in_rule_10=bool(s10))
            got = gen.generate_ours(one, tq, use_lrp=False, **kw)
            assert tuple(got.shape) == (1, 1, 1, fb.h * fb.w)
            r64_own = _oracle_on_device(sd, CFG, *own, tq, torch.float64, **kw)
            sens = rel_err(r64_own, _oracle_on_device(sd, CFG, ref_feats[0].double(), ref_feats[1], tq, torch.float64, **kw))
            e_own, e_img = rel_err(got, r64_own), rel_err(got, g[f"{rkey}.n{norm}s{s10}"])
            print(f"{rkey} ({fb.h * fb.w} tokens) n{norm}s{s10}: vs fp64 on own features {e_own:.2e}, vs reference "
                  f"{e_img:.2e} (sensitivity {sens:.2e})")
            assert e_own < TOL and e_img < max(TOL, 2.0 * sens)
        if bkey:
            for method in ("raw_attn", "rollout", "attn_gradcam"):
                e_b = rel_err(getattr(gen, "generate_" + method)(one, tq), g[f"{bkey}.{method}"])
                print(f"{bkey} {method}: {e_b:.2e}")
                assert e_b < TOL


def test_reference_module_form(case):
    """a module with the reference key set whose layer4 conv2 reports dilation (2, 2) gets a DC5 engine"""
    import mmx_b200
    from mmx_b200.detr import engine_for
    g, sd = case["g"], case["sd"]
    mod = torch.nn.Module()
    for k in g["ref.state_dict_keys"].tolist():
        *path, leaf = k.split(".")
        node = mod
        for p in path:
            if not hasattr(node, p):
                node.add_module(p, torch.nn.Sequential() if p in ("backbone", "layer4") else torch.nn.Module())
            node = getattr(node, p)
        node.register_buffer(leaf, sd[k].clone())
    mod.transformer.nhead = CFG.nhead
    mod.backbone[0].body.layer4[-1].conv2.dilation = (2, 2)
    gen = mmx_b200.Generator(mod)
    assert engine_for(mod).dilation and engine_for(mod) is gen.model
    img = case["big"][None].cuda()
    cam = gen.generate_ours(img, torch.tensor([2]), use_lrp=False)
    assert cam.numel() == 33 * 34
    assert torch.equal(cam, mmx_b200.Generator(case["eng"]).generate_ours(img, torch.tensor([2]), use_lrp=False))


def test_lrp_long_image_vs_fp64_oracle(case):
    """use_lrp=True at 1122 tokens: the criterion of test_lrp_gpu.py (max(1e-4, 5 x the fp32 oracle's own error))"""
    import mmx_b200
    eng, sd = case["eng"], case["sd"]
    img = case["big"][None].cuda()
    tq = torch.tensor([2])
    out = mmx_b200.Generator(eng).generate_ours(img, tq)
    f = eng.features(img)
    src, pos = _bchw(f.x, 1, f.h, f.w).cpu(), _bchw(f.pe, 1, f.h, f.w).cpu()
    r64 = do.generate_ours_lrp(sd, CFG, src, pos, tq, dtype=torch.float64)
    noise = rel_err(do.generate_ours_lrp(sd, CFG, src, pos, tq, dtype=torch.float32), r64)
    gen = torch.Generator().manual_seed(0)
    for _ in range(2):                                    # test_detr_r50_lrp_vs_oracle's floor: one-ulp input moves, fp64
        s_ulp = src * (1 + 2.0 ** -23 * torch.randn(src.shape, generator=gen))
        noise = max(noise, rel_err(do.generate_ours_lrp(sd, CFG, s_ulp, pos, tq, dtype=torch.float64), r64))
    e = rel_err(out.reshape(1, -1), r64)
    print(f"DC5 1122 tokens lrp vs fp64 oracle {e:.2e} (noise floor {noise:.2e})")
    assert e < max(TOL, 5.0 * noise)


def test_bitwise_identities(case):
    """CUDA-graph replay == eager, and MaskGenerator in chunks == one batch, at 1122 tokens"""
    import mmx_b200
    eng = case["eng"]
    img = case["big"][None].cuda()
    gen = mmx_b200.Generator(eng)
    tq = torch.tensor([3])
    eager = gen.generate_ours(img, tq, use_lrp=False).clone()
    gr = gen.capture(img, tq, use_lrp=False)
    rep = gr(img, tq.cuda())
    gr.check()
    assert torch.equal(rep, eager)
    mg = mmx_b200.MaskGenerator(eng)
    q = torch.tensor([0, 2, 3, 5, 6])
    assert mg.chunk_size(1122, False) >= len(q)           # the default is one batch here
    ref = mg.get_masks(img, q)
    for n in (1, 2, 3):
        got = mg.get_masks(img, q, max_batch=n)
        for a, b in zip(got, ref):
            assert torch.equal(a, b), n
    assert torch.equal(ref[2][2:3], eager.reshape(1, -1))
    with pytest.raises(mmx_b200.MmxError):
        mg.get_masks(img, q, max_batch=0)


def _oracle_on_device(sd, cfg, src, pos, tq, dtype, **kw):
    """the fp64 / fp32 oracle maps, run on the device (rule 6 is O(S^3): 2500 - 3350 tokens are minutes on a CPU)"""
    sdc = {k: v.cuda() for k, v in sd.items()}
    with torch.device("cuda"):
        return do.generate_ours(sdc, cfg, src.cuda(), pos.cuda(), tq.cuda(), dtype=dtype, **kw).cpu()


def _full_size(eng, sd, cfg, images, tq, backbone):
    """test_full_size_r50's criterion, with the fp64 oracle on the device: features and logits to 1e-4 of the fp64 oracle;
    maps on the engine's own features within max(1e-4, 5 x the fp32 oracle's own error), and end to end within that plus
    twice what the 2e-5 rounding of the features moves the exact map by (fp64, as test_golden_unmodified_reference).
    images: a [B,3,H,W] tensor or a list of [3,H,W] images (padded)."""
    import mmx_b200
    f = eng.features(images)
    x, m = (images, None) if isinstance(images, torch.Tensor) else bo.nested(images)
    with torch.no_grad():
        src, pos, _ = backbone({k: v.cuda() for k, v in sd.items()}, x, m)
    e_src = rel_err(_bchw(f.x, f.B, f.h, f.w), src)
    src, pos = src.cpu(), pos.cpu()
    out = eng(images)
    with torch.device("cuda"), torch.no_grad():
        logits = do.detr_forward({k: v.double().cuda() for k, v in sd.items()}, cfg, src.cuda(), pos.double().cuda())[0].cpu()
    e_log = rel_err(out["pred_logits"], logits)
    cam = mmx_b200.Generator(eng).generate_ours(images, tq, use_lrp=False)
    own = (_bchw(f.x, f.B, f.h, f.w).cpu(), _bchw(f.pe, f.B, f.h, f.w).cpu())
    r64_own = _oracle_on_device(sd, cfg, own[0].double(), own[1], tq, torch.float64)
    noise = rel_err(_oracle_on_device(sd, cfg, *own, tq, torch.float32), r64_own)
    r64 = _oracle_on_device(sd, cfg, src, pos, tq, torch.float64)
    cam = cam.reshape(r64.shape)
    e_own, e64, sens = rel_err(cam, r64_own), rel_err(cam, r64), rel_err(r64_own, r64)
    print(f"{f.h}x{f.w} = {f.h * f.w} tokens, B={f.B}: features {e_src:.2e}, logits {e_log:.2e}, maps vs fp64 on own "
          f"features {e_own:.2e} (fp32 oracle noise {noise:.2e}), end to end {e64:.2e} (sensitivity {sens:.2e})")
    assert e_src < TOL and e_log < TOL
    assert e_own < max(TOL, 5.0 * noise)
    assert e64 < max(TOL, 5.0 * noise) + 2.0 * sens


@pytest.mark.parametrize("H,W", [(800, 800), (800, 1066)])
def test_full_size_dc5_r50(H, W):
    """ResNet-50 DC5 + the DETR-R50 transformer at the reference's input sizes: 2500 and 3350 tokens."""
    import mmx_b200
    cfg = do.DETR_R50
    sd = bo.init_state_dict(cfg, seed=5)
    x = torch.randn(1, 3, H, W, generator=torch.Generator().manual_seed(H + W)).cuda()
    eng = mmx_b200.DetrEngine(sd, nhead=cfg.nhead, device="cuda:0", dilation=True)
    _full_size(eng, sd, cfg, x, torch.tensor([3]), dc5.backbone)


def test_full_size_r50_padded_mixed_orientation():
    """plain ResNet-50 on 800x1199 + 1199x800 padded to one batch: 38x38 = 1444 tokens"""
    import mmx_b200
    cfg = do.DETR_R50
    sd = bo.init_state_dict(cfg, seed=6)
    gen = torch.Generator().manual_seed(1)
    imgs = [torch.randn(3, 800, 1199, generator=gen).cuda(), torch.randn(3, 1199, 800, generator=gen).cuda()]
    eng = mmx_b200.DetrEngine(sd, nhead=cfg.nhead, device="cuda:0")
    _full_size(eng, sd, cfg, imgs, torch.tensor([3, 17]), bo.backbone)
