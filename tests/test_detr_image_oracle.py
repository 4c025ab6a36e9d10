"""CPU: the oracle restatement of DETR's image front end (oracle/detr_backbone_oracle.py) - bounded activations for the
seeded ResNet-50, BN folding against conv-then-affine, the mask / position embedding against the all-valid formula, the
padded-batch construction."""
import math

import torch
import torch.nn.functional as F

from oracle import detr_backbone_oracle as bo
from oracle import detr_oracle as do


def _images(seed=0):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(3, 96, 160, generator=g), torch.randn(3, 128, 96, generator=g)]


def test_seeded_r50_activations_stay_in_fp16_range():
    sd = bo.init_state_dict(bo.DETR_IMAGE, seed=3)
    x, m = bo.nested(_images())
    stage_max = []
    src, pos, mf = bo.backbone(sd, x, m, stage_max=stage_max)
    print("max |activation| per stage (stem, layer1..4):", ["%.1f" % v for v in stage_max])
    assert len(stage_max) == 5
    assert all(1e-2 < v < 1e3 for v in stage_max), stage_max
    assert src.shape == (2, 64, 4, 5) and pos.shape == (2, 64, 4, 5) and mf.shape == (2, 4, 5)
    assert torch.isfinite(src).all() and src.abs().max() < 1e3


def test_padding_mask_reaches_feature_resolution():
    x, m = bo.nested(_images())
    assert x.shape == (2, 3, 128, 160)
    assert not m[0, :96, :].any() and m[0, 96:, :].all() and m[1, :, 96:].all() and not m[1, :, :96].any()
    mf = F.interpolate(m[None].float(), size=(4, 5)).to(torch.bool)[0]
    assert mf.any() and not mf.all()            # some positions are padding at feature resolution, some are not


def test_position_sine_matches_all_valid_formula():
    mask = torch.zeros(2, 5, 7, dtype=torch.bool)
    assert torch.equal(bo.position_sine(mask, 32), do.sine_position_embedding(2, 5, 7, 64))


def test_bn_folding_matches_conv_then_affine():
    g = torch.Generator().manual_seed(1)
    w = torch.randn(16, 8, 3, 3, generator=g, dtype=torch.float64)
    bn = dict(weight=1 + 0.1 * torch.randn(16, generator=g, dtype=torch.float64),
              bias=0.1 * torch.randn(16, generator=g, dtype=torch.float64),
              running_mean=0.1 * torch.randn(16, generator=g, dtype=torch.float64),
              running_var=0.5 + torch.rand(16, generator=g, dtype=torch.float64))
    from mmx_b200.backbone import fold_frozen_bn
    x = torch.randn(2, 8, 9, 9, generator=g, dtype=torch.float64)
    ref = bo._frozen_bn({k: v for k, v in bn.items()}, "", F.conv2d(x, w, padding=1))
    wf, bf = fold_frozen_bn(w, bn)
    got = F.conv2d(x, wf.double(), bf.double(), padding=1)
    assert (got - ref).abs().max() / ref.abs().max() < 1e-6     # fp32 fold: rounding of the folded weights only


def test_reordered_weight_is_the_patch_order():
    """[Cout, Cin, kh, kw] -> [Cout, kh*kw*Cin] in (ky, kx, c) order: a GEMM of the NHWC patches reproduces conv2d."""
    g = torch.Generator().manual_seed(2)
    x = torch.randn(1, 5, 6, 7, generator=g, dtype=torch.float64)
    w = torch.randn(4, 5, 3, 3, generator=g, dtype=torch.float64)
    ref = F.conv2d(x, w, stride=2, padding=1)
    xp = F.pad(x, (1, 1, 1, 1)).permute(0, 2, 3, 1)                   # NHWC, padded
    Ho, Wo = ref.shape[-2:]
    rows = [torch.cat([xp[0, 2 * oy + ky, 2 * ox + kx] for ky in range(3) for kx in range(3)])
            for oy in range(Ho) for ox in range(Wo)]
    got = torch.stack(rows) @ w.permute(0, 2, 3, 1).reshape(4, -1).t()
    assert torch.allclose(got.t().reshape(1, 4, Ho, Wo), ref)


def test_state_dict_keys_match_a_detr_checkpoint_layout():
    sd = bo.init_state_dict(bo.DETR_IMAGE, seed=0)
    body = [k for k in sd if k.startswith("backbone.0.body.")]
    assert len([k for k in body if k.endswith("conv1.weight") and "layer" in k]) == sum(bo.R50_BLOCKS)
    convs = [k for k in body if k.endswith(".weight") and sd[k].dim() == 4]
    assert len(convs) == 53                                             # ResNet-50: 53 convs
    for k in ("input_proj.weight", "input_proj.bias", "bbox_embed.layers.2.weight", "query_embed.weight"):
        assert k in sd
    assert math.isclose(sd["input_proj.weight"].shape[1], 2048)


# ---- pinned to the unmodified reference DETR run from images (tests/golden/detr_image.npz, oracle/make_detr_image_golden.py)
def _golden(golden_dir):
    from util import load_golden
    g = load_golden(golden_dir, "detr_image.npz")
    sd = {k[3:]: torch.from_numpy(v) for k, v in g.items() if k.startswith("sd.")}
    return g, sd, [torch.from_numpy(g["images.0"]), torch.from_numpy(g["images.1"])]


def test_oracle_front_end_vs_reference_golden(golden_dir):
    from util import rel_err
    g, sd, imgs = _golden(golden_dir)
    x, m = bo.nested(imgs)
    src, pos, mf = bo.backbone(sd, x, m, dtype=torch.float32)
    assert torch.equal(mf, torch.from_numpy(g["mask"])) and mf.any() and not mf.all()
    assert (pos - torch.from_numpy(g["pos"])).abs().max().item() <= 1e-6
    assert rel_err(src, g["src"]) < 1e-5


def test_oracle_logits_boxes_maps_vs_reference_golden(golden_dir):
    from util import rel_err
    g, sd, imgs = _golden(golden_dir)
    cfg = bo.DETR_IMAGE
    x, m = bo.nested(imgs)
    src, pos, _ = bo.backbone(sd, x, m, dtype=torch.float32)
    logits = do.detr_forward(sd, cfg, src, pos)[0]
    boxes = bo.boxes(sd, bo.decoder_output(sd, cfg, src, pos, dtype=torch.float32))
    assert rel_err(logits, g["pred_logits"]) < 1e-5 and rel_err(boxes, g["pred_boxes"]) < 1e-5
    for b, img in enumerate(imgs):
        s1, p1, _ = bo.backbone(sd, img[None], dtype=torch.float32)
        assert rel_err(s1, g[f"single.{b}.src"]) < 1e-5 and (p1 - torch.from_numpy(g[f"single.{b}.pos"])).abs().max() <= 1e-6
        for norm, s10 in ((1, 1), (0, 1), (1, 0)):
            r = do.generate_ours(sd, cfg, s1, p1, torch.tensor([int(g["tq"][b])]), normalize_self_attention=bool(norm),
                                 apply_self_in_rule_10=bool(s10))
            assert rel_err(r, g[f"R.{b}.n{norm}s{s10}"][None]) < 1e-4, (b, norm, s10)


def test_oracle_state_dict_has_the_reference_key_set(golden_dir):
    g, sd, _ = _golden(golden_dir)
    assert set(sd) == set(g["ref.state_dict_keys"].tolist())
