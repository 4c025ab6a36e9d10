"""Small end-to-end exercise of every kernel family for `compute-sanitizer --tool memcheck` (run on the GPU box):
   compute-sanitizer --tool memcheck --error-exitcode 3 python profiles/sanitize_run.py"""
import os, sys
import numpy as np
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import mmx_b200
from mmx_b200._lib import lib, check, ptr, current_stream
from oracle import clip_oracle as co, detr_oracle as do, lxmert_oracle as lo, vit_oracle as vo

l = lib()
# CLIP (fp32 FFMA GEMMs at this size), both start modes, ragged text
cfg = co.SMALL
sd = co.init_state_dict(cfg, seed=3)
images, tokens = co.synthetic_inputs(cfg, 4, seed=5)
eng = mmx_b200.ClipEngine(mmx_b200.ClipConfig(*cfg.ref_args()), sd, max_batch=3, device="cuda:0")   # micro-batched 3+1
for sl in (-1, 0):
    mmx_b200.interpret(images.cuda(), tokens.cuda(), eng, "cuda:0", sl, sl)
# wgmma GEMM with ragged edges in M, N, K + every epilogue input
M, N, K = 300, 260, 200
A = torch.randn(M, K, device="cuda"); W = torch.randn(N, K, device="cuda"); b = torch.randn(N, device="cuda")
res = torch.randn(M, N, device="cuda"); C = torch.empty(M, N, device="cuda"); Ca = torch.empty(M, N, device="cuda")
for backend in (1, 2):
    if l.mmx_set_gemm_backend(backend) == backend:
        check(l.mmx_linear(ptr(A), K, ptr(W), K, ptr(b), ptr(res), N, ptr(C), N, ptr(Ca), 2, M, N, K, current_stream()))
# fp16x3 kernels on packed weight planes: in-kernel split (2) and pre-split (3), epilogue with every input
pk = torch.empty(l.mmx_pack_weight_bytes(N, K), dtype=torch.uint8, device="cuda")
check(l.mmx_pack_weight(ptr(W), K, N, K, ptr(pk), current_stream()))
for backend in (2, 3):
    if l.mmx_set_gemm_backend(backend) == backend:
        check(l.mmx_linear_packed(ptr(A), K, ptr(W), K, ptr(pk), ptr(b), ptr(res), N, ptr(C), N, ptr(Ca), 2, M, N, K, current_stream()))
        check(l.mmx_linear_packed(ptr(A), K, ptr(W), K, ptr(pk), ptr(b), None, 0, ptr(C), N, None, 0, M, N, K, current_stream()))
l.mmx_set_gemm_backend(1)
# tensor-core rule update (S >= 128: one batched launch, tiles spill into the next sample's rows) and the FFMA one
for S in (197, 50):
    R = torch.eye(S, device="cuda").repeat(2, 1, 1); Ab = torch.rand(2, S, S, device="cuda") * 0.01
    mmx_b200.self_update(R, Ab)
# DETR / LXMERT / ViT generators on tiny configs
dcfg = do.DETR_TINY
src, pos, tq = do.synthetic_inputs(dcfg, 2, 3, 4, seed=1)
g = mmx_b200.Generator(mmx_b200.DetrEngine(do.init_state_dict(dcfg, 5), nhead=dcfg.nhead, device="cuda:0"))
g.generate_ours((src.cuda(), pos.cuda()), tq, use_lrp=False); g.generate_rollout((src.cuda(), pos.cuda()), tq)
g.generate_attn_gradcam((src.cuda(), pos.cuda()), tq)
lcfg = lo.LXMERT_TINY
ids, feats, boxes = lo.synthetic_inputs(lcfg, 2, 6, 5, seed=2)
le = mmx_b200.LxmertEngine(lo.init_state_dict(lcfg, 3), num_heads=lcfg.heads, device="cuda:0")
mmx_b200.GeneratorOurs(le).generate_ours((ids.cuda(), feats.cuda(), boxes.cuda()), use_lrp=False)
mmx_b200.GeneratorBaselines(le).generate_rollout((ids.cuda(), feats.cuda(), boxes.cuda()))
vcfg = vo.VIT_TINY
ve = mmx_b200.ViTEngine(vo.init_state_dict(vcfg, 3), heads=vcfg.heads, device="cuda:0")
mmx_b200.generate_relevance(ve, torch.randn(2, 3, vcfg.image, vcfg.image).cuda())
# tile-width instantiations of the wgmma GEMM
for bn in (128, 144, 160, 0):
    l.mmx_set_gemm_tile_n(bn)
    check(l.mmx_linear(ptr(A), K, ptr(W), K, ptr(b), ptr(res), N, ptr(C), N, ptr(Ca), 2, M, N, K, current_stream()))
# VisualBERT generator + perturbation drivers, Otsu masks, min-max, top-k
from oracle import visualbert_oracle as vbo
vbcfg = vbo.VISUALBERT_TINY
vinp = {k: v.cuda() for k, v in vbo.synthetic_inputs(vbcfg, 1, 8, 7, seed=2).items()}
vbe = mmx_b200.VisualBertEngine(vbo.init_state_dict(vbcfg, 3), num_heads=vbcfg.heads, device="cuda:0")
vgen = mmx_b200.SelfAttentionGenerator(vbe)
cam = vgen.generate_ours(vinp); vgen.generate_rollout(vinp); vgen.generate_attn_gradcam(vinp)
vp = mmx_b200.VisualBertPerturbation(vbe)
vp.perturbation_image(vinp, cam); vp.perturbation_text(vinp, cam, True)
item = (ids[:1].cuda(), feats[:1].cuda(), boxes[:1].cuda())
rtt, rti = mmx_b200.GeneratorOurs(le).generate_ours(item, use_lrp=False)
lp = mmx_b200.LxmertPerturbation(le)
lp.perturbation_image(item, rti[0], rtt[0]); lp.perturbation_text(item, rti[0], rtt[0], True)
mmx_b200.GeneratorOursAblationNoAggregation(le).generate_ours_no_agg(item, normalize_self_attention=False)
mmx_b200.MaskGenerator(g.model).get_masks((src[:1].cuda(), pos[:1].cuda()), torch.tensor([0, 1]), "ours_no_lrp")
mmx_b200.otsu_masks(torch.rand(3, 850, device="cuda")); mmx_b200.minmax_normalize(torch.rand(2, 77, device="cuda"))
# long-sequence attention (32-row tile instantiation)
q = torch.randn(1, 850, 64, device="cuda"); Aa = torch.empty(1, 2, 850, 852, device="cuda"); Oo = torch.empty(1, 850, 64, device="cuda")
import ctypes as C
check(l.mmx_attention_fwd(ptr(q), 64, ptr(q), 64, ptr(q), 64, None, ptr(Aa), 852, ptr(Oo), 64, 1, 2, 850, 850, 32, C.c_float(0.17), 0,
                          current_stream()))
# ---- round 2: LRP sweeps (lrp.cu), the rule-6 chain kernel, the plane-based attention (pre-pass + ring, and the backward at a
# long sequence), CUDA-graph capture of a generator call
g.generate_ours((src.cuda(), pos.cuda()), tq)                                 # use_lrp=True (reference default)
g.generate_transformer_att((src.cuda(), pos.cuda()), tq); g.generate_partial_lrp((src.cuda(), pos.cuda()), tq)
mmx_b200.GeneratorOurs(le).generate_ours((ids.cuda(), feats.cuda(), boxes.cuda()))
mmx_b200.GeneratorBaselines(le).generate_transformer_attr((ids.cuda(), feats.cuda(), boxes.cuda()))
vgen.generate_transformer_att(vinp); vgen.generate_partial_lrp(vinp)
for S_, L_ in ((77, 3), (50, 2), (128, 1), (5, 2)):
    ld_ = (S_ + 3) // 4 * 4
    Ab_ = torch.rand(L_, 2, S_, ld_, device="cuda") * 0.01; Ro_ = torch.empty(2, S_, ld_, device="cuda")
    check(l.mmx_self_chain(ptr(Ab_), 2 * S_ * ld_, ld_, ptr(Ro_), ld_, 2, S_, L_, current_stream()))
for S_, hd_ in ((197, 64), (300, 32), (850, 16)):                                # pre-pass planes, 2-4 stage K / V ring, 64- and 32-row tiles
    H_ = 2; D_ = H_ * hd_; ld_ = (S_ + 3) // 4 * 4
    qkv_ = torch.randn(S_, 3 * D_, device="cuda"); do_ = torch.randn(S_, D_, device="cuda")
    A_ = torch.empty(1, H_, S_, ld_, device="cuda"); dA_ = torch.empty_like(A_); O_ = torch.empty(S_, D_, device="cuda")
    dl_ = torch.empty(H_ * S_, device="cuda"); dqkv_ = torch.empty_like(qkv_)
    check(l.mmx_attention_fwd(ptr(qkv_), 3 * D_, ptr(qkv_[:, D_:]), 3 * D_, ptr(qkv_[:, 2 * D_:]), 3 * D_, None, ptr(A_), ld_, ptr(O_), D_,
                              1, H_, S_, S_, hd_, C.c_float(hd_ ** -0.5), 0, current_stream()))
    check(l.mmx_attention_bwd(ptr(do_), D_, ptr(qkv_), 3 * D_, ptr(qkv_[:, D_:]), 3 * D_, ptr(qkv_[:, 2 * D_:]), 3 * D_, ptr(A_), ptr(dA_),
                              ld_, ptr(dl_), ptr(dqkv_), 3 * D_, ptr(dqkv_[:, D_:]), 3 * D_, ptr(dqkv_[:, 2 * D_:]), 3 * D_, 1, H_, S_, S_, hd_,
                              C.c_float(hd_ ** -0.5), 0, current_stream()))
gr = g.capture((src.cuda(), pos.cuda()), tq, use_lrp=False)
gr(src.cuda(), pos.cuda(), tq.cuda()); gr.check()
# ---- DETR from images (conv.cu): im2col into fp16 planes (backend 3) and into fp32 (backend 1), NCHW stem, strided 1x1,
# max-pool, mask / position embedding with padding, sigmoid box head
from oracle import detr_backbone_oracle as dbo
ieng = mmx_b200.DetrEngine(dbo.init_state_dict(dbo.DETR_IMAGE, 3), nhead=dbo.DETR_IMAGE.nhead, device="cuda:0")
ims = [torch.randn(3, 70, 90, device="cuda"), torch.randn(3, 64, 100, device="cuda")]
for backend in (3, 1):
    l.mmx_set_gemm_backend(backend)
    ieng(ims)
mmx_b200.Generator(ieng).generate_ours(ims, torch.tensor([0, 1]), use_lrp=False)
# ---- rows past 1024 keys: the two-pass attention kernels at S = 1100 (forward, backward with dQ / dK / dV, stop after
# dA, pad columns beyond the last key tile) and dilated convs (the DC5 backbone, fp16 planes and fp32 gathers)
for hd_ in (16, 32, 64):
    H_, S_ = 2, 1100
    D_ = H_ * hd_; ld_ = S_ + 68
    qkv_ = torch.randn(S_, 3 * D_, device="cuda"); do_ = torch.randn(S_, D_, device="cuda")
    A_ = torch.empty(1, H_, S_, ld_, device="cuda"); dA_ = torch.empty_like(A_); O_ = torch.empty(S_, D_, device="cuda")
    dl_ = torch.empty(H_ * S_, device="cuda"); dqkv_ = torch.empty_like(qkv_)
    check(l.mmx_attention_fwd(ptr(qkv_), 3 * D_, ptr(qkv_[:, D_:]), 3 * D_, ptr(qkv_[:, 2 * D_:]), 3 * D_, None, ptr(A_), ld_, ptr(O_), D_,
                              1, H_, S_, S_, hd_, C.c_float(hd_ ** -0.5), 0, current_stream()))
    for full in (True, False):
        check(l.mmx_attention_bwd(ptr(do_), D_, ptr(qkv_), 3 * D_, ptr(qkv_[:, D_:]), 3 * D_, ptr(qkv_[:, 2 * D_:]), 3 * D_, ptr(A_),
                                  ptr(dA_), ld_, ptr(dl_) if full else None, ptr(dqkv_) if full else None, 3 * D_,
                                  ptr(dqkv_[:, D_:]) if full else None, 3 * D_, ptr(dqkv_[:, 2 * D_:]) if full else None, 3 * D_,
                                  1, H_, S_, S_, hd_, C.c_float(hd_ ** -0.5), 0, current_stream()))
deng = mmx_b200.DetrEngine(dbo.init_state_dict(dbo.DETR_IMAGE, 3), nhead=dbo.DETR_IMAGE.nhead, device="cuda:0", dilation=True)
for backend in (3, 1):
    l.mmx_set_gemm_backend(backend)
    deng(ims)
# ---- DETR evaluation post-processing (detr_postprocess.cu): PostProcess with boxes, the keep-only launch, and the fused
# PostProcessSegm on a padded two-image batch (16-byte and byte stores, crop) and on a same-size plane (the copy case)
l.mmx_set_gemm_backend(3)
pout = deng(ims)
pout["pred_masks"] = torch.randn(2, dbo.DETR_IMAGE.queries, 5, 7, device="cuda")
res = mmx_b200.PostProcess()(pout, torch.tensor([[70, 90], [64, 100]], device="cuda"))
mmx_b200.detr_postprocess(pout["pred_logits"])
mmx_b200.PostProcessSegm()(res, pout, torch.tensor([[61, 93], [33, 47]]), torch.tensor([[70, 90], [64, 100]]))
mmx_b200.PostProcessSegm(0.85)(res[:1], {"pred_masks": pout["pred_masks"][:1]}, torch.tensor([[9, 21]]), torch.tensor([[5, 7]]))
torch.cuda.synchronize()
print("sanitize_run: all kernels executed")
