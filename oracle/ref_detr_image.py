"""Runs the UNMODIFIED reference ``DETR`` - ResNet ``Backbone`` + ``Joiner`` + ``PositionEmbeddingSine`` + ``Transformer``
+ heads (DETR/models/detr.py:22-77) - on CPU from images (build container only; TEST INFRASTRUCTURE).

Shims (SURVEY.md §8c): the torchvision version guard at DETR/util/misc.py:21 (as oracle/ref_detr.py), ``.cuda()`` identity
(DETR.forward hard-codes ``torch.tensor([5]).cuda()``, :72), and ``DETR.models.backbone.is_main_process -> False`` so that
torchvision builds the ResNet without downloading ImageNet weights (backbone.py:88-90); the weights come from the state
dict.  DETR.forward reads decoder output 5, so the transformer needs 6 decoder layers."""
from __future__ import annotations

import torch

from . import ref_shims as rs


def _import():
    rs._ensure_path()
    import torchvision
    tv = torchvision.__version__
    torchvision.__version__ = "0.9.9"
    try:
        import DETR.models.backbone as backbone
        from DETR.models.detr import DETR
        from DETR.models.transformer import Transformer
        from DETR.models.position_encoding import PositionEmbeddingSine
        from DETR.util.misc import nested_tensor_from_tensor_list
    finally:
        torchvision.__version__ = tv
    backbone.is_main_process = lambda: False
    return backbone, DETR, Transformer, PositionEmbeddingSine, nested_tensor_from_tensor_list


def build(cfg, sd, name: str = "resnet50"):
    """The reference DETR module with ``sd`` loaded (strict: every reference parameter / buffer must come from ``sd``)."""
    backbone, DETR, Transformer, PositionEmbeddingSine, _ = _import()
    from .detr_oracle import to_checkpoint_format
    assert cfg.dec_layers == 6, "DETR.forward reads decoder output 5 (DETR/models/detr.py:72)"
    joiner = backbone.Joiner(backbone.Backbone(name, False, False, False),
                             PositionEmbeddingSine(cfg.d_model // 2, normalize=True))        # build_backbone, backbone.py:111-119
    joiner.num_channels = 2048
    tr = Transformer(cfg.d_model, cfg.nhead, cfg.enc_layers, cfg.dec_layers, cfg.dim_ff, 0.0, return_intermediate_dec=True)
    m = DETR(joiner, tr, cfg.classes, cfg.queries).eval()
    missing, _ = m.load_state_dict(to_checkpoint_format(sd), strict=False)
    assert not missing, missing
    return m


def front_end(m, images):
    """mask, pos and input_proj(src) of DETR.forward (detr.py:63-69) for a list of [3,H_i,W_i] images."""
    *_, nested = _import()
    samples = nested(images)
    features, pos = m.backbone(samples)
    src, mask = features[-1].decompose()
    return mask, pos[-1].detach(), m.input_proj(src).detach()


def forward(m, images):
    with rs.cuda_is_identity():       # not under no_grad: the reference's attention registers gradient hooks
        return {k: v.detach() for k, v in m(images).items()}


def generator_maps(m, image, tq, method="ours", **kw):
    """The reference Generator's ``generate_<method>`` (DETR/modules/ExplanationGenerator.py) on ONE image [3,H,W]."""
    from DETR.modules.ExplanationGenerator import Generator
    gen = Generator(m)
    fn = gen.generate_ours if method == "ours" else getattr(gen, "generate_" + method)
    with rs.cuda_is_identity():
        if method == "ours":
            r = fn(image[None], torch.tensor([int(tq)]), use_lrp=False, **kw)
        else:
            r = fn(image[None], torch.tensor([int(tq)]))
    return r.reshape(-1).detach()
