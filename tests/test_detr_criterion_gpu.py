"""GPU: DETR's evaluation losses on the device - HungarianMatcher, SetCriterion and the decoder's auxiliary outputs
(mmx_b200/criterion.py, csrc/detr_criterion.cu) - against the unmodified reference (tests/golden/detr_criterion.npz),
scipy's answers stored there, and the plain-PyTorch restatement (oracle/detr_criterion_oracle.py) run on CUDA or in fp64."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import detr_criterion_oracle as co
from oracle.ref_detr_panoptic import DETR_PANOPTIC as CFG, scaled
from test_detr_criterion_oracle import outputs as golden_outputs, targets as golden_targets, RUNS
from util import TOL, load_golden, rel_err

pytestmark = pytest.mark.gpu
LOSSES = ["labels", "boxes", "cardinality", "masks"]


@pytest.fixture(scope="module")
def golden(golden_dir):
    return load_golden(golden_dir, "detr_criterion.npz")


def _cuda(o):
    if isinstance(o, dict):
        return {k: _cuda(v) for k, v in o.items()}
    if isinstance(o, list):
        return [_cuda(v) for v in o]
    return o.cuda()


def _ptrs(ts):
    return (C.c_void_p * len(ts))(*[t.data_ptr() for t in ts])


def _offsets(sizes):
    off = [0]
    for n in sizes:
        off.append(off[-1] + n)
    return (C.c_int * len(off))(*off)


def _lsa(cost_blocks, L, B, Q, sizes):
    """mmx_detr_match_lsa on [L][B] blocks [Q, T_b]: (indices [L, 2, T] on the CPU, status [L, B])"""
    from mmx_b200._lib import lib, check, ptr, current_stream
    T = sum(sizes)
    flat = torch.cat([torch.as_tensor(c, dtype=torch.float32).reshape(-1) for blocks in cost_blocks for c in blocks]).cuda()
    idx = torch.full((L * 2 * T,), 7, dtype=torch.int64, device="cuda")
    st = torch.full((L * B,), 9, dtype=torch.int32, device="cuda")
    check(lib().mmx_detr_match_lsa(ptr(flat), L, B, Q, _offsets(sizes), ptr(idx), ptr(st), current_stream()))
    return idx.view(L, 2, T).cpu(), st.view(L, B).cpu()


def _random_outputs(L, B, Q, C1, gen, nan_logit=False, bad_box=False):
    layers = []
    for l in range(L):
        lg = 3.0 * torch.randn(B, Q, C1, generator=gen)
        bx = torch.cat([0.2 + 0.6 * torch.rand(B, Q, 2, generator=gen), 0.05 + 0.4 * torch.rand(B, Q, 2, generator=gen)], -1)
        layers.append({"pred_logits": lg, "pred_boxes": bx})
    if nan_logit:
        layers[0]["pred_logits"][0, 3, 2] = float("nan")
    if bad_box:
        layers[-1]["pred_boxes"][B - 1, 5, 2] = -0.1
    out = dict(layers[0])
    out["aux_outputs"] = layers[1:]
    return out


def _random_targets(sizes, C, gen, hw=None):
    out = []
    for b, n in enumerate(sizes):
        t = {"labels": torch.randint(0, C, (n,), generator=gen),
             "boxes": torch.cat([0.2 + 0.6 * torch.rand(n, 2, generator=gen), 0.05 + 0.4 * torch.rand(n, 2, generator=gen)], -1)}
        if hw is not None:
            t["masks"] = torch.rand(n, *hw[b], generator=gen) < 0.3
        out.append(t)
    return out


def test_cost_vs_restatement_and_status():
    from mmx_b200._lib import lib, check, ptr, current_stream
    gen = torch.Generator().manual_seed(1)
    L, Q, C1, sizes = 3, 100, 92, [7, 0, 20]
    B = len(sizes)
    out = _cuda(_random_outputs(L, B, Q, C1, gen))
    tg = _cuda(_random_targets(sizes, C1 - 1, gen))
    layers = [out] + out["aux_outputs"]
    T = sum(sizes)
    cost = torch.full((L * Q * T,), float("nan"), device="cuda")
    st = torch.full((L,), 5, dtype=torch.int32, device="cuda")
    ids, tb = torch.cat([t["labels"] for t in tg]), torch.cat([t["boxes"] for t in tg])
    w = (2.0, 5.0, 2.0)
    check(lib().mmx_detr_match_cost(_ptrs([o["pred_logits"] for o in layers]), _ptrs([o["pred_boxes"] for o in layers]), L, B,
                                    Q, C1, ptr(ids), ptr(tb), _offsets(sizes), *w, ptr(cost), ptr(st), current_stream()))
    assert st.tolist() == [0] * L
    o = 0
    for l, lay in enumerate(layers):
        ref = co.cost_blocks(lay, tg, *w)
        for b, n in enumerate(sizes):
            got = cost[o:o + Q * n].view(Q, n)
            o += Q * n
            assert (got - ref[b]).abs().max().item() <= 1e-6 * ref[b].abs().max().item() if n else True
    # a degenerate predicted box raises AssertionError, a NaN logit ValueError (through the public classes)
    import mmx_b200
    crit = mmx_b200.SetCriterion(C1 - 1, mmx_b200.HungarianMatcher(1, 5, 2), {}, 0.1, ["labels", "boxes"])
    with pytest.raises(AssertionError):
        crit(_cuda(_random_outputs(L, B, Q, C1, gen, bad_box=True)), tg)
    nanb = _cuda(_random_outputs(L, B, Q, C1, gen))
    nanb["aux_outputs"][1]["pred_boxes"][0, 0, 0] = float("nan")
    with pytest.raises(AssertionError):
        crit(nanb, tg)
    with pytest.raises(ValueError, match="invalid numeric entries"):
        mmx_b200.HungarianMatcher()(_cuda(_random_outputs(1, B, Q, C1, gen, nan_logit=True)), tg)
    bad = [dict(tg[0]), tg[1], tg[2]]
    bad[0]["boxes"] = bad[0]["boxes"].clone()
    bad[0]["boxes"][1, 3] = -1.0
    with pytest.raises(AssertionError):
        mmx_b200.HungarianMatcher()(_cuda(_random_outputs(1, B, Q, C1, gen)), bad)


def test_lsa_golden_cases(golden):
    names = sorted({k[4:-5] for k in golden.files if k.startswith("lsa.") and k.endswith(".cost")})
    for n in names:
        c = golden[f"lsa.{n}.cost"]
        Q, T = c.shape
        if max(Q, T) > 1024:
            continue
        idx, st = _lsa([[c]], 1, 1, Q, [T])
        if f"lsa.{n}.error" in golden.files:
            want = {"matrix contains invalid numeric entries": 1, "cost matrix is infeasible": 2}[str(golden[f"lsa.{n}.error"])]
            assert int(st[0, 0]) == want, n
            continue
        assert int(st[0, 0]) == 0, n
        k = min(Q, T)
        assert np.array_equal(idx[0, 0, :k].numpy(), golden[f"lsa.{n}.i"]), n
        assert np.array_equal(idx[0, 1, :k].numpy(), golden[f"lsa.{n}.j"]), n
        assert (idx[0, :, k:] == -1).all()


def test_lsa_random_sizes_batched_and_repeatable():
    """random and tied 100 x T problems, several layers x images in one launch: each equals the problem alone, scipy's
    answer (the Python restatement, itself equal to scipy), and two runs give the same bits; T > Q and the 1024 limit"""
    from mmx_b200 import MmxError
    rng = np.random.default_rng(5)
    Q, sizes, L = 100, [0, 1, 7, 20, 63, 100, 120], 3
    blocks = [[(rng.integers(0, 3, (Q, n)) if l == 1 else rng.standard_normal((Q, n))).astype(np.float32) for n in sizes]
              for l in range(L)]
    idx, st = _lsa(blocks, L, len(sizes), Q, sizes)
    idx2, _ = _lsa(blocks, L, len(sizes), Q, sizes)
    assert torch.equal(idx, idx2) and (st == 0).all()
    o = 0
    for b, n in enumerate(sizes):
        for l in range(L):
            i, j = co.lsa(blocks[l][b].astype(np.float64))
            k = min(Q, n)
            assert np.array_equal(idx[l, 0, o:o + k].numpy(), i) and np.array_equal(idx[l, 1, o:o + k].numpy(), j), (l, n)
            alone, _ = _lsa([[blocks[l][b]]], 1, 1, Q, [n])
            assert torch.equal(alone[0, :, :n], idx[l, :, o:o + n])
        o += n
    from mmx_b200._lib import lib, ptr, current_stream
    big = torch.zeros(1025 * 3, device="cuda")
    out = torch.empty(2 * 3, dtype=torch.int64, device="cuda")
    s = torch.empty(1, dtype=torch.int32, device="cuda")
    assert lib().mmx_detr_match_lsa(ptr(big), 1, 1, 1025, _offsets([3]), ptr(out), ptr(s), current_stream()) != 0


def _check_losses(got, ref_keys, ref, rtol):
    """same keys in the same order; class_error and cardinality_error exact, the rest within rtol"""
    assert list(got) == list(ref_keys)
    for k in ref_keys:
        v, r = float(got[k]), float(ref[k])
        assert got[k].dim() == 0 and got[k].is_cuda
        if k.startswith(("class_error", "cardinality_error")):
            assert v == r, (k, v, r)
        else:
            assert abs(v - r) <= rtol * max(abs(r), 1e-30), (k, v, r)


@pytest.mark.parametrize("run", list(RUNS))
def test_criterion_on_reference_outputs(golden, run):
    import mmx_b200
    g = golden
    out = _cuda(golden_outputs(g, run))
    tg = _cuda(golden_targets(g, RUNS[run]))
    crit = mmx_b200.SetCriterion(int(g["num_classes"]), mmx_b200.HungarianMatcher(), {}, float(g["eos_coef"]), LOSSES).to("cuda")
    assert crit.eval() is crit and crit.empty_weight[-1].item() == pytest.approx(float(g["eos_coef"]))
    got = crit(out, tg)
    keys = g[f"{run}.keys"].tolist()
    _check_losses(got, keys, {k: g[f"{run}.loss.{k}"] for k in keys}, 1e-5)
    for l, lay in enumerate([out] + out["aux_outputs"]):
        for b, (i, j) in enumerate(crit.matcher(lay, tg)):
            assert i.dtype == torch.int64 and not i.is_cuda
            assert np.array_equal(i.numpy(), g[f"{run}.idx.{l}.{b}.i"]) and np.array_equal(j.numpy(), g[f"{run}.idx.{l}.{b}.j"])


def test_mask_losses_coco_size():
    """25x34 planes, padded targets 800x1066 (images 800x1066 and 704x1066), 20 matched masks, logits with +-large
    values and get_panoptic's -1 / 0 / 255 rows, bool, uint8 and float targets: <= 1e-5 relative to fp64"""
    from mmx_b200._lib import lib, check, ptr, current_stream
    gen = torch.Generator().manual_seed(7)
    Q, h, w, hw, sizes = 100, 25, 34, [(800, 1066), (704, 1066)], [12, 8]
    pm = 4.0 * torch.randn(2, Q, h, w, generator=gen)
    pm[0, :30] = torch.where(torch.rand(30, h, w, generator=gen) < 0.4, 255.0, 0.0)
    pm[0, 30:40] = -1.0
    pm[1, :10] = 80.0 * torch.randn(10, h, w, generator=gen)
    tg = _random_targets(sizes, 5, gen, hw)
    rng = np.random.default_rng(0)
    indices = [(torch.as_tensor(np.sort(rng.choice(Q, n, replace=False))), torch.as_tensor(rng.permutation(n))) for n in sizes]
    T = sum(sizes)
    idx = torch.cat([torch.cat([i for i, _ in indices]), torch.cat([j for _, j in indices])]).cuda()
    ref = co.mask_losses(pm.double(), [t["masks"].double() for t in tg], indices, 20.0)
    nb = torch.full((1,), 20.0, device="cuda")
    pmc = pm.cuda()
    for dt in (torch.bool, torch.uint8, torch.float32):
        ms = [t["masks"].to(dt).cuda() for t in tg]
        ms_b = [m.view(torch.uint8) if dt == torch.bool else m for m in ms]
        out = torch.full((2,), float("nan"), device="cuda")
        fhw = (C.c_int * 4)(*[v for m in ms for v in m.shape[1:]])
        check(lib().mmx_detr_mask_losses(ptr(pmc), 2, Q, h, w, _ptrs(ms_b), fhw, 1 if dt == torch.float32 else 0,
                                         _offsets(sizes), ptr(idx), ptr(nb), ptr(out), current_stream()))
        for k, v in zip(("loss_mask", "loss_dice"), out.tolist()):
            r = float(ref[k])
            print(f"{dt} {k}: {v:.9g} vs {r:.9g} ({abs(v - r) / abs(r):.2e})")
            assert abs(v - r) <= 1e-5 * abs(r), (dt, k)
    assert T == 20


def test_set_losses_direct_and_edges(golden):
    """mmx_detr_set_losses called directly equals the public form; a batch with an image without targets, a losses
    subset, the all-empty target list and an unknown loss name"""
    import mmx_b200
    from mmx_b200._lib import lib, check, ptr, current_stream
    gen = torch.Generator().manual_seed(3)
    L, Q, C1, sizes = 2, 100, 92, [6, 0, 11]
    B = len(sizes)
    out = _cuda(_random_outputs(L, B, Q, C1, gen))
    tg = _cuda(_random_targets(sizes, C1 - 1, gen))
    ref = co.criterion(out, tg, C1 - 1, 0.1, ["labels", "boxes", "cardinality"])
    crit = mmx_b200.SetCriterion(C1 - 1, mmx_b200.HungarianMatcher(), {}, 0.1, ["labels", "boxes", "cardinality"])
    got = crit(out, tg)
    _check_losses(got, list(ref), ref, 1e-5)
    # directly, with the matcher's indices
    layers = [out] + out["aux_outputs"]
    T = sum(sizes)
    blk = []
    for o in layers:
        pairs = crit.matcher(o, tg)
        ii = torch.full((T,), -1, dtype=torch.int64)
        jj = torch.full((T,), -1, dtype=torch.int64)
        off = 0
        for (i, j), n in zip(pairs, sizes):
            ii[off:off + len(i)], jj[off:off + len(j)] = i, j
            off += n
        blk.append(torch.cat([ii, jj]))
    idx = torch.cat(blk).cuda()
    res = torch.full((L, 5), float("nan"), device="cuda")
    ew = torch.ones(C1, device="cuda")
    ew[-1] = 0.1
    nb = torch.full((1,), float(T), device="cuda")
    ids, tb = torch.cat([t["labels"] for t in tg]), torch.cat([t["boxes"] for t in tg])
    check(lib().mmx_detr_set_losses(_ptrs([o["pred_logits"] for o in layers]), _ptrs([o["pred_boxes"] for o in layers]), L, B,
                                    Q, C1, ptr(ids), ptr(tb), _offsets(sizes), ptr(idx), ptr(ew), ptr(nb), ptr(res),
                                    current_stream()))
    assert torch.equal(res[0, [0, 1, 2, 3, 4]], torch.stack([got[k] for k in ("loss_ce", "class_error", "loss_bbox",
                                                                               "loss_giou", "cardinality_error")]))
    # a losses subset keeps the reference's key set and order
    sub = mmx_b200.SetCriterion(C1 - 1, mmx_b200.HungarianMatcher(), {}, 0.1, ["cardinality", "boxes"])(out, tg)
    assert list(sub) == ["cardinality_error", "loss_bbox", "loss_giou", "cardinality_error_0", "loss_bbox_0", "loss_giou_0"]
    # every image without targets: the reference's values (golden), no error without masks
    g = golden
    empty = [{k: v[:0] for k, v in golden_targets(g, (0,))[0].items()}]
    got = mmx_b200.SetCriterion(int(g["num_classes"]), mmx_b200.HungarianMatcher(), {}, float(g["eos_coef"]),
                                ["labels", "boxes", "cardinality"])(_cuda(golden_outputs(g, "0")), _cuda(empty))
    keys = [k[11:] for k in g.files if k.startswith("empty.loss.")]
    _check_losses(got, [k for k in got], {k: g[f"empty.loss.{k}"] for k in keys}, 1e-5)
    with pytest.raises(AssertionError, match="do you really want"):
        mmx_b200.SetCriterion(C1 - 1, mmx_b200.HungarianMatcher(), {}, 0.1, ["labels", "nope"])(out, tg)
    with pytest.raises(AssertionError):
        mmx_b200.HungarianMatcher(0, 0, 0)


def test_end_to_end_aux_outputs(golden, golden_dir):
    """MaskGenerator(aux_loss=True).get_panoptic on the golden images: aux_outputs within TOL of the reference's, and
    SetCriterion on those outputs gives the reference's indices and losses to 1e-4; aux_loss=False is bitwise unchanged"""
    import mmx_b200
    g = golden
    sd = {k[3:]: torch.from_numpy(v) for k, v in g.items() if k.startswith("sd.")}
    eng = mmx_b200.DetrEngine(scaled(sd, float(g["weights.class_scale"])), nhead=CFG.nhead, device="cuda:0")
    gen = torch.Generator().manual_seed(int(g["images.seed"]))
    p = load_golden(golden_dir, "detr_panoptic.npz")
    imgs = [torch.randn(3, *p[f"{b}.size"].tolist(), generator=gen) for b in (0, 1)]
    mg, mga = mmx_b200.MaskGenerator(eng), mmx_b200.MaskGenerator(eng, aux_loss=True)
    crit = mmx_b200.SetCriterion(int(g["num_classes"]), mmx_b200.HungarianMatcher(), {}, float(g["eos_coef"]), LOSSES)
    for b, img in enumerate(imgs):
        x = img[None].cuda()
        plain = mg.get_panoptic(x, None, "raw_attn")
        o = mga.get_panoptic(x, None, "raw_attn")
        assert list(o) == ["pred_logits", "pred_boxes", "aux_outputs", "pred_masks"]
        assert all(torch.equal(o[k], plain[k]) for k in plain)
        again = mg.get_panoptic(x, None, "raw_attn")
        assert list(again) == ["pred_logits", "pred_boxes", "pred_masks"] and all(torch.equal(again[k], plain[k]) for k in plain)
        assert len(o["aux_outputs"]) == CFG.dec_layers - 1
        for i, a in enumerate(o["aux_outputs"]):
            assert rel_err(a["pred_logits"], g[f"{b}.aux.{i}.pred_logits"]) < TOL
            assert rel_err(a["pred_boxes"], g[f"{b}.aux.{i}.pred_boxes"]) < TOL
        fw = eng.forward(x, aux_loss=True)
        assert torch.equal(fw["aux_outputs"][2]["pred_logits"], o["aux_outputs"][2]["pred_logits"])
        assert list(eng.forward(x)) == ["pred_logits", "pred_boxes"]
        tg = _cuda(golden_targets(g, (b,)))
        got = crit(o, tg)
        keys = g[f"{b}.keys"].tolist()
        _check_losses(got, keys, {k: g[f"{b}.loss.{k}"] for k in keys}, 1e-4)
        for l, lay in enumerate([o] + o["aux_outputs"]):
            (i, j), = crit.matcher(lay, tg)
            assert np.array_equal(i.numpy(), g[f"{b}.idx.{l}.0.i"]) and np.array_equal(j.numpy(), g[f"{b}.idx.{l}.0.j"])


def test_mask_losses_with_images_without_targets():
    """masks with an image that has no targets (first and last in the batch, and the tallest / widest one, so the padded
    size still counts it) against the restatement on CUDA; every image without targets: the mask losses are 0 where the
    reference's own interpolate wrapper raises NameError on the empty batch, the other losses are the reference's"""
    import mmx_b200
    gen = torch.Generator().manual_seed(11)
    Q, C1, h, w = 100, 92, 25, 34
    sizes, hw = [0, 9, 4, 0], [(300, 420), (256, 320), (224, 288), (200, 448)]
    out = _cuda(_random_outputs(2, len(sizes), Q, C1, gen))
    out["pred_masks"] = (4.0 * torch.randn(len(sizes), Q, h, w, generator=gen)).cuda()
    tg = _cuda(_random_targets(sizes, C1 - 1, gen, hw))
    crit = mmx_b200.SetCriterion(C1 - 1, mmx_b200.HungarianMatcher(), {}, 0.1, LOSSES)
    got = crit(out, tg)
    ref = co.criterion(out, tg, C1 - 1, 0.1, LOSSES)
    _check_losses(got, list(ref), ref, 1e-5)
    empty = [{k: v[:0] for k, v in t.items()} for t in tg]
    got = crit(out, empty)
    ref = co.criterion(out, empty, C1 - 1, 0.1, ["labels", "boxes", "cardinality"])
    assert float(got["loss_mask"]) == 0.0 and float(got["loss_dice"]) == 0.0
    _check_losses({k: v for k, v in got.items() if k not in ("loss_mask", "loss_dice")}, list(ref), ref, 1e-5)


def test_class_error_tie_rule_is_cuda_topk():
    """class_error's top-1 on rows with tied (and NaN) maxima follows torch.topk(1) on CUDA - the device the reference's
    evaluate runs the criterion on - : the lowest index among equal maxima, NaN above every number"""
    from mmx_b200._lib import lib, check, ptr, current_stream
    gen = torch.Generator().manual_seed(13)
    B, Q, C1, sizes = 2, 100, 92, [30, 25]
    out = _cuda(_random_outputs(1, B, Q, C1, gen))
    lg = torch.randint(0, 3, (B, Q, C1), generator=gen).float()          # every row has tied maxima
    lg[:, 50:, 0] = lg[:, 50:, 20] = 3.0                                 # ... and here classes 0 and 20 tie above the rest
    lg[0, :10, 5] = float("nan")
    lg[1, :10, 7] = lg[1, :10, 60] = float("nan")
    out["pred_logits"] = lg.cuda()
    tg = _random_targets(sizes, C1 - 1, gen)
    for t in tg:                                                         # targets on the tied classes
        t["labels"] = torch.randint(0, 2, (len(t["labels"]),), generator=gen) * 20
    tg = _cuda(tg)
    tied = out["pred_logits"][1, 20:24]
    top = tied.topk(1, 1, True, True)[1].flatten()
    assert torch.equal(top, torch.stack([torch.nonzero(r == r.max())[0, 0] for r in tied]))
    T = sum(sizes)
    pairs = [(torch.arange(n) * 3, torch.randperm(n, generator=gen)) for n in sizes]   # rows 0 .. 87, NaN rows included
    idx = torch.cat([torch.cat([i for i, _ in pairs]), torch.cat([j for _, j in pairs])]).cuda()
    res = torch.full((1, 5), float("nan"), device="cuda")
    ew = torch.ones(C1, device="cuda")
    ew[-1] = 0.1
    nb = torch.full((1,), float(T), device="cuda")
    ids, tb = torch.cat([t["labels"] for t in tg]), torch.cat([t["boxes"] for t in tg])
    check(lib().mmx_detr_set_losses(_ptrs([out["pred_logits"]]), _ptrs([out["pred_boxes"]]), 1, B, Q, C1, ptr(ids), ptr(tb),
                                    _offsets(sizes), ptr(idx), ptr(ew), ptr(nb), ptr(res), current_stream()))
    ref = co._losses("labels", out, tg, pairs, float(T), ew.cpu(), C1 - 1)
    assert float(res[0, 1]) == float(ref["class_error"]) and float(ref["class_error"]) < 100.0
    card = co._losses("cardinality", out, tg, pairs, float(T), ew.cpu(), C1 - 1)
    assert float(res[0, 4]) == float(card["cardinality_error"])
