"""GPU: DETR from images - the ResNet backbone, input_proj, mask / sine position embedding and box head on libmmx
(mmx_b200/backbone.py, csrc/conv.cu) against the plain-PyTorch oracle (oracle/detr_backbone_oracle.py), in fp64 for the
convs and fp32 for the position embedding, as the reference computes it."""
import pytest
import torch

from oracle import detr_backbone_oracle as bo, detr_oracle as do
from util import rel_err, TOL

pytestmark = pytest.mark.gpu
CFG = bo.DETR_IMAGE


def _images(seed=0):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(3, 96, 160, generator=g), torch.randn(3, 128, 96, generator=g)]


@pytest.fixture(scope="module")
def case():
    import mmx_b200
    sd = bo.init_state_dict(CFG, seed=3)
    imgs = _images()
    x, m = bo.nested(imgs)
    src, pos, mf = bo.backbone(sd, x, m)
    eng = mmx_b200.DetrEngine(sd, nhead=CFG.nhead, device="cuda:0")
    return dict(sd=sd, imgs=imgs, x=x, m=m, src=src, pos=pos, mask=mf, eng=eng)


def _bchw(t, B, h, w):
    return t.view(B, h, w, -1).permute(0, 3, 1, 2)


def test_features_mask_pos_vs_oracle(case):
    import mmx_b200
    eng = case["eng"]
    f = eng.features([t.cuda() for t in case["imgs"]])
    B, h, w = f.B, f.h, f.w
    assert (B, h, w) == tuple(case["src"].shape[:1]) + tuple(case["src"].shape[2:])
    assert torch.equal(f.mask.cpu(), case["mask"]) and case["mask"].any()
    e_pos = (_bchw(f.pe, B, h, w).cpu() - case["pos"]).abs().max().item()
    e_src = rel_err(_bchw(f.x, B, h, w), case["src"])
    print(f"features vs fp64 oracle {e_src:.2e}, pos max abs err {e_pos:.2e}")
    assert e_pos <= 1e-6
    assert e_src < TOL
    # the NestedTensor form gives the same bits as the list form
    nt = type("NestedTensor", (), {})()
    nt.tensors, nt.mask = case["x"].cuda(), case["m"].cuda()
    g = eng.features(nt)
    assert torch.equal(g.x, f.x) and torch.equal(g.pe, f.pe)
    assert isinstance(eng, mmx_b200.DetrEngine)


def test_forward_logits_boxes_and_maps_vs_oracle(case):
    import mmx_b200
    eng, sd = case["eng"], case["sd"]
    imgs = [t.cuda() for t in case["imgs"]]
    out = eng(imgs)
    assert tuple(out["pred_logits"].shape) == (2, CFG.queries, CFG.classes + 1)
    assert tuple(out["pred_boxes"].shape) == (2, CFG.queries, 4)
    sd64 = {k: v.double() for k, v in sd.items()}
    logits = do.detr_forward(sd64, CFG, case["src"], case["pos"].double())[0]
    hs = bo.decoder_output(sd, CFG, case["src"], case["pos"])
    e_log, e_box = rel_err(out["pred_logits"], logits), rel_err(out["pred_boxes"], bo.boxes(sd64, hs))
    tq = torch.tensor([1, 4])
    gen = mmx_b200.Generator(eng)
    print(f"logits {e_log:.2e}, boxes {e_box:.2e} vs fp64 oracle")
    assert e_log < TOL and e_box < TOL
    # maps.  (1) Given the features the engine computed, the relevancy path is held to 1e-4 of the fp64 oracle on those
    # features.  (2) End to end, DETR's relevancy amplifies a change of its input: at this random-init size the 2e-5
    # (of max|src|) fp16x3 rounding of the features moves the exact map by up to ~1e-4 by itself.  The end-to-end error is
    # held to max(1e-4, 2 x that sensitivity), the sensitivity measured in fp64 on the same features.
    f = eng.features(imgs)
    own = (_bchw(f.x, f.B, f.h, f.w).cpu().double(), _bchw(f.pe, f.B, f.h, f.w).cpu())
    for kw in (dict(), dict(normalize_self_attention=False), dict(apply_self_in_rule_10=False)):
        got = gen.generate_ours(imgs, tq, use_lrp=False, **kw)
        r64 = do.generate_ours(sd, CFG, case["src"], case["pos"], tq, dtype=torch.float64, **kw)
        r64_own = do.generate_ours(sd, CFG, *own, tq, dtype=torch.float64, **kw)
        e_own, e64, sens = rel_err(got, r64_own), rel_err(got, r64), rel_err(r64_own, r64)
        print(f"maps {kw}: vs fp64 oracle on the engine's features {e_own:.2e}; end to end {e64:.2e} "
              f"(sensitivity to the feature rounding {sens:.2e})")
        assert e_own < TOL
        assert e64 < max(TOL, 2.0 * sens)
    # baselines take images too
    for fn in (gen.generate_raw_attn, gen.generate_rollout, gen.generate_attn_gradcam):
        assert tuple(fn(imgs, tq).shape) == (2, eng._shape[1])
    # single image: the reference's return shapes
    one = imgs[0][None]
    S = eng.features(one).h * eng.features(one).w
    assert tuple(gen.generate_ours(one, torch.tensor([2]), use_lrp=False).shape) == (1, 1, 1, S)
    assert tuple(gen.generate_ours(one, 2, use_lrp=False).shape) == (1, 1, S)
    assert tuple(mmx_b200.GeneratorAlbationNoAgg(eng).generate_ours_abl(one, 2).shape) == (1, 1, S)


def test_every_backend_and_tile_width(case):
    import mmx_b200
    l = mmx_b200.lib()
    eng = case["eng"]
    x = case["x"].cuda()
    prev = l.mmx_get_gemm_backend()
    try:
        for be in (0, 1, 2, 3):
            assert l.mmx_set_gemm_backend(be) == be
            f = eng.features(x)
            e = rel_err(_bchw(f.x, f.B, f.h, f.w), bo.backbone(case["sd"], case["x"])[0])
            print(f"backend {be}: features vs fp64 oracle {e:.2e}")
            assert e < TOL
        l.mmx_set_gemm_backend(prev)
        outs = []
        for bn in (128, 160):
            l.mmx_set_gemm_tile_n(bn)
            outs.append(eng.features(x).x.clone())
        assert torch.equal(outs[0], outs[1])
    finally:
        l.mmx_set_gemm_tile_n(0)
        l.mmx_set_gemm_backend(prev)


def test_bitwise_identities(case):
    import mmx_b200
    eng = case["eng"]
    g = torch.Generator().manual_seed(7)
    batch = torch.randn(3, 3, 96, 128, generator=g).cuda()
    gen = mmx_b200.Generator(eng)
    tq = torch.tensor([0, 3, 5])
    # an image alone == the same image inside a batch of same-size images
    full = gen.generate_ours(batch, tq, use_lrp=False).clone()
    alone = gen.generate_ours(batch[1:2], tq[1:2], use_lrp=False)
    assert torch.equal(alone.reshape(-1), full[1])
    # images == the engine's own backbone outputs passed as (src, pos)
    f = eng.features(batch)
    src, pos = _bchw(f.x, f.B, f.h, f.w), _bchw(f.pe, f.B, f.h, f.w)
    assert torch.equal(gen.generate_ours((src, pos), tq, use_lrp=False), full)
    # a CUDA-graph replay (backbone inside the graph) == the eager call
    gr = gen.capture(batch, tq, use_lrp=False)
    rep = gr(batch, tq.cuda())
    gr.check()
    assert torch.equal(rep, full)
    # MaskGenerator: backbone once, features expanded over the queries == the (src, pos) path
    mg = mmx_b200.MaskGenerator(eng)
    q = torch.tensor([0, 2, 6])
    m1, t1, c1 = mg.get_masks(batch[:1], q)
    m2, t2, c2 = mg.get_masks((src[:1], pos[:1]), q)
    assert torch.equal(c1, c2) and torch.equal(m1, m2) and torch.equal(t1, t2)
    assert tuple(m1.shape) == (3, f.h, f.w)


def _golden(golden_dir):
    from util import load_golden
    g = load_golden(golden_dir, "detr_image.npz")
    sd = {k[3:]: torch.from_numpy(v) for k, v in g.items() if k.startswith("sd.")}
    return g, sd, [torch.from_numpy(g["images.0"]), torch.from_numpy(g["images.1"])]


def test_golden_unmodified_reference(golden_dir):
    """Against the unmodified reference DETR run from the same images (oracle/make_detr_image_golden.py): mask exact, pos
    to 1e-6, input_proj(src), pred_logits, pred_boxes to 1e-4; per-image maps (three flag sets) and baselines."""
    import mmx_b200
    g, sd, imgs = _golden(golden_dir)
    eng = mmx_b200.DetrEngine(sd, nhead=CFG.nhead, device="cuda:0")
    cimgs = [t.cuda() for t in imgs]
    f = eng.features(cimgs)
    B, h, w = f.B, f.h, f.w
    assert torch.equal(f.mask.cpu(), torch.from_numpy(g["mask"]))
    e_pos = (_bchw(f.pe, B, h, w).cpu() - torch.from_numpy(g["pos"])).abs().max().item()
    out = eng(cimgs)
    e = dict(src=rel_err(_bchw(f.x, B, h, w), g["src"]), logits=rel_err(out["pred_logits"], g["pred_logits"]),
             boxes=rel_err(out["pred_boxes"], g["pred_boxes"]))
    print(f"vs reference: pos {e_pos:.2e} abs, " + ", ".join(f"{k} {v:.2e}" for k, v in e.items()))
    assert e_pos <= 1e-6 and max(e.values()) < TOL
    gen = mmx_b200.Generator(eng)
    for b, img in enumerate(cimgs):
        tq = torch.tensor([int(g["tq"][b])])
        one = img[None]
        fb = eng.features(one)
        own = (_bchw(fb.x, 1, fb.h, fb.w).cpu().double(), _bchw(fb.pe, 1, fb.h, fb.w).cpu())
        ref_feats = (torch.from_numpy(g[f"single.{b}.src"]), torch.from_numpy(g[f"single.{b}.pos"]))
        for norm, s10 in ((1, 1), (0, 1), (1, 0)):
            kw = dict(normalize_self_attention=bool(norm), apply_self_in_rule_10=bool(s10))
            ref = g[f"R.{b}.n{norm}s{s10}"]
            got = gen.generate_ours(one, tq, use_lrp=False, **kw)
            assert tuple(got.shape) == (1, 1, 1, fb.h * fb.w)
            # the relevancy path on the reference's own features: 1e-4
            e_feat = rel_err(gen.generate_ours((ref_feats[0].cuda(), ref_feats[1].cuda()), tq, use_lrp=False, **kw), ref)
            # end to end: plus what the 2e-5 rounding of the features moves the exact map by (fp64, same features)
            sens = rel_err(do.generate_ours(sd, CFG, *own, tq, dtype=torch.float64, **kw),
                           do.generate_ours(sd, CFG, ref_feats[0].double(), ref_feats[1], tq, dtype=torch.float64, **kw))
            e_img = rel_err(got, ref)
            print(f"image {b} n{norm}s{s10}: on reference features {e_feat:.2e}, from the image {e_img:.2e} "
                  f"(sensitivity {sens:.2e})")
            assert e_feat < TOL and e_img < max(TOL, 2.0 * sens)
        for method in ("raw_attn", "rollout", "attn_gradcam"):
            e_b = rel_err(getattr(gen, "generate_" + method)(one, tq), g[f"base.{b}.{method}"])
            print(f"image {b} {method}: {e_b:.2e}")
            assert e_b < TOL


def test_reference_module_form(golden_dir):
    """Generator / MaskGenerator / engine_for take an nn.Module whose state_dict() has the reference DETR's exact key set
    (stored with the golden) and `transformer.nhead`; the engine is built once per module."""
    import mmx_b200
    from mmx_b200.detr import engine_for
    g, sd, imgs = _golden(golden_dir)
    keys = g["ref.state_dict_keys"].tolist()
    mod = torch.nn.Module()
    for k in keys:
        *path, leaf = k.split(".")
        node = mod
        for p in path:
            if not hasattr(node, p):
                node.add_module(p, torch.nn.Module())
            node = getattr(node, p)
        node.register_buffer(leaf, sd[k].clone())
    mod.transformer.nhead = CFG.nhead
    assert sorted(mod.state_dict()) == sorted(keys)
    gen = mmx_b200.Generator(mod)
    assert mmx_b200.MaskGenerator(mod).model is gen.model and engine_for(mod) is gen.model
    img = imgs[0][None].cuda()
    out = engine_for(mod)(img)
    assert tuple(out["pred_logits"].shape) == (1, CFG.queries, CFG.classes + 1) and tuple(out["pred_boxes"].shape) == (1, CFG.queries, 4)
    cam = gen.generate_ours(img, torch.tensor([1]), use_lrp=False)
    eng = mmx_b200.DetrEngine(sd, nhead=CFG.nhead, device="cuda:0")
    assert torch.equal(cam, mmx_b200.Generator(eng).generate_ours(img, torch.tensor([1]), use_lrp=False))


def test_lrp_from_images_and_feature_forms(case):
    """use_lrp=True from images equals use_lrp=True on the engine's own features (the backbone runs on the default
    backend, outside the FFMA scope of the sweep); a 3-D pos [d,h,w] is broadcast as before."""
    import mmx_b200
    eng = case["eng"]
    img = case["imgs"][0][None].cuda()
    gen = mmx_b200.Generator(eng)
    a = gen.generate_ours(img, torch.tensor([2]))
    f = eng.features(img)
    src, pos = _bchw(f.x, 1, f.h, f.w), _bchw(f.pe, 1, f.h, f.w)
    assert torch.equal(a, gen.generate_ours((src, pos), torch.tensor([2])))
    eng.forward_backward(img, None, torch.tensor([2]), lrp=True)
    assert torch.equal(gen.generate_ours((src, pos[0]), torch.tensor([2]), use_lrp=False),
                       gen.generate_ours((src, pos), torch.tensor([2]), use_lrp=False))


def test_errors(case):
    import mmx_b200
    feats_only = mmx_b200.DetrEngine(do.init_state_dict(CFG, 3), nhead=CFG.nhead, device="cuda:0")
    img = torch.randn(1, 3, 64, 64, device="cuda")
    with pytest.raises(mmx_b200.MmxError):
        mmx_b200.Generator(feats_only).generate_ours(img, 0, use_lrp=False)
    with pytest.raises(mmx_b200.MmxError):
        case["eng"].features(torch.randn(1, 4, 64, 64, device="cuda"))
    # a features-only engine still runs (src, pos) exactly as before
    src, pos, tq = do.synthetic_inputs(CFG, 1, 3, 4, seed=1)
    a = mmx_b200.Generator(feats_only).generate_ours((src.cuda(), pos.cuda()), tq, use_lrp=False)
    b = mmx_b200.Generator(case["eng"]).generate_ours((src.cuda(), pos.cuda()), tq, use_lrp=False)
    assert torch.equal(a, b)


@pytest.mark.parametrize("H,W", [(800, 800), (800, 1066)])
def test_full_size_r50(H, W):
    """ResNet-50 + the DETR-R50 transformer (d 256, 8 heads, 6 + 6 layers, 100 queries) at the reference's input sizes,
    batch 2.  Maps: the criterion of test_zz_baseline_sizes_gpu.py (DETR's own fp32 noise at this size)."""
    import mmx_b200
    cfg = do.DETR_R50
    sd = bo.init_state_dict(cfg, seed=5)
    g = torch.Generator().manual_seed(H + W)
    x = torch.randn(2, 3, H, W, generator=g)
    tq = torch.tensor([3, 17])
    eng = mmx_b200.DetrEngine(sd, nhead=cfg.nhead, device="cuda:0")
    f = eng.features(x.cuda())
    with torch.no_grad():
        src, pos, _ = bo.backbone({k: v.cuda() for k, v in sd.items()}, x.cuda())
    src, pos = src.cpu(), pos.cpu()
    e_src = rel_err(_bchw(f.x, f.B, f.h, f.w), src)
    out = eng(x.cuda())
    logits = do.detr_forward({k: v.double() for k, v in sd.items()}, cfg, src, pos.double())[0]
    e_log = rel_err(out["pred_logits"], logits)
    cam = mmx_b200.Generator(eng).generate_ours(x.cuda(), tq, use_lrp=False)
    r64 = do.generate_ours(sd, cfg, src, pos, tq, dtype=torch.float64)
    r32 = do.generate_ours(sd, cfg, src.float(), pos, tq)
    e64, noise = rel_err(cam, r64), rel_err(r32, r64)
    print(f"R50 {H}x{W} B=2: features {e_src:.2e}, logits {e_log:.2e}, maps vs fp64 {e64:.2e} (fp32 oracle noise {noise:.2e})")
    assert e_src < TOL
    assert e_log < TOL
    assert e64 < max(TOL, 5.0 * noise)
