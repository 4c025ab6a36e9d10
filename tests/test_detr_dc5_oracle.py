"""CPU: the oracle restatement of DETR's DC5 front end (oracle/detr_dc5_oracle.py) against the unmodified reference DETR
built with ``dilation=True`` (tests/golden/detr_dc5.npz, oracle/make_detr_dc5_golden.py), the stride-16 feature size, and
the DC5 state dict's key set."""
import torch

from oracle import detr_backbone_oracle as bo
from oracle import detr_dc5_oracle as dc5
from oracle import detr_oracle as do


def _golden(golden_dir, name="detr_dc5.npz"):
    from util import load_golden
    g = load_golden(golden_dir, name)
    sd = {k[3:]: torch.from_numpy(v) for k, v in g.items() if k.startswith("sd.")}
    return g, sd


def test_dc5_front_end_and_heads_vs_reference_golden(golden_dir):
    from util import rel_err
    g, sd = _golden(golden_dir)
    cfg = bo.DETR_IMAGE
    x, m = bo.nested(dc5.pair_images(int(g["images.seed"])))
    src, pos, mf = dc5.backbone(sd, x, m, dtype=torch.float32)
    assert torch.equal(mf, torch.from_numpy(g["mask"])) and mf.any() and not mf.all()
    assert (pos - torch.from_numpy(g["pos"])).abs().max().item() <= 1e-6
    assert rel_err(src, g["src"]) < 1e-5
    logits = do.detr_forward(sd, cfg, src, pos)[0]
    boxes = bo.boxes(sd, bo.decoder_output(sd, cfg, src, pos, dtype=torch.float32))
    assert rel_err(logits, g["pred_logits"]) < 1e-5 and rel_err(boxes, g["pred_boxes"]) < 1e-5


def test_dc5_maps_vs_reference_golden(golden_dir):
    from util import rel_err
    g, sd = _golden(golden_dir)
    cfg = bo.DETR_IMAGE
    for b, img in enumerate(dc5.pair_images(int(g["images.seed"]))):
        s1, p1, _ = dc5.backbone(sd, img[None], dtype=torch.float32)
        for norm, s10 in ((1, 1), (0, 1), (1, 0)):
            r = do.generate_ours(sd, cfg, s1, p1, torch.tensor([int(g["tq"][b])]), normalize_self_attention=bool(norm),
                                 apply_self_in_rule_10=bool(s10))
            assert rel_err(r, g[f"R.{b}.n{norm}s{s10}"][None]) < 1e-4, (b, norm, s10)


def test_dc5_long_image_maps_vs_reference_golden(golden_dir):
    """3x520x540: 33x34 = 1122 tokens, the size where the engine switches to the two-pass attention kernels."""
    from util import rel_err
    g, sd = _golden(golden_dir)
    cfg = bo.DETR_IMAGE
    s1, p1, _ = dc5.backbone(sd, dc5.long_image(int(g["long.seed"]))[None], dtype=torch.float32)
    assert s1.shape[-2:] == (33, 34)
    r = do.generate_ours(sd, cfg, s1, p1, torch.tensor([int(g["long.tq"])]))
    assert rel_err(r, g["long.R.n1s1"][None]) < 1e-4


def test_dc5_feature_map_has_stride_16():
    sd = bo.init_state_dict(bo.DETR_IMAGE, seed=0)
    x = torch.randn(1, 3, 100, 132, generator=torch.Generator().manual_seed(0))
    src, pos, m = dc5.backbone(sd, x, dtype=torch.float32)
    src32, _, _ = bo.backbone(sd, x, dtype=torch.float32)
    assert src.shape[-2:] == dc5.feature_hw(100, 132) == (7, 9)
    assert src32.shape[-2:] == (4, 5)                    # the stride-32 body on the same weights
    assert pos.shape == (1, 64, 7, 9) and m.shape == (1, 7, 9)
    for H, W in ((800, 800), (800, 1066), (800, 1333)):  # 2500, 3350 and 4200 tokens at COCO evaluation sizes
        h, w = dc5.feature_hw(H, W)
        assert h * w == {(800, 800): 2500, (800, 1066): 3350, (800, 1333): 4200}[(H, W)]


def test_dc5_state_dict_keys_equal_the_stride_32_ones(golden_dir):
    g, sd = _golden(golden_dir)
    g32, _ = _golden(golden_dir, "detr_image.npz")
    keys = set(g["ref.state_dict_keys"].tolist())
    assert keys == set(g32["ref.state_dict_keys"].tolist())
    assert keys == set(sd)
