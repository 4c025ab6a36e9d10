"""CPU: the plain-PyTorch restatement of DETR's HungarianMatcher / SetCriterion (oracle/detr_criterion_oracle.py) against
the unmodified reference (tests/golden/detr_criterion.npz), and its restatement of scipy's linear_sum_assignment against
scipy itself."""
import json

import numpy as np
import pytest
import torch
from scipy.optimize import linear_sum_assignment

from oracle import detr_criterion_oracle as co
from util import load_golden

RUNS = {"0": (0,), "1": (1,), "batch": (0, 1)}


def outputs(g, prefix, dtype=torch.float32):
    t = lambda k: torch.from_numpy(g[f"{prefix}.{k}"]).to(dtype)
    n = len({k.split(".")[2] for k in g.files if k.startswith(prefix + ".aux.")})
    return {"pred_logits": t("pred_logits"), "pred_boxes": t("pred_boxes"),
            "aux_outputs": [{"pred_logits": t(f"aux.{i}.pred_logits"), "pred_boxes": t(f"aux.{i}.pred_boxes")}
                            for i in range(n)],
            "pred_masks": t("pred_masks")}


def targets(g, images, dtype=torch.float32):
    return [{"labels": torch.from_numpy(g[f"{b}.labels"]), "boxes": torch.from_numpy(g[f"{b}.boxes"]).to(dtype),
             "masks": torch.from_numpy(g[f"{b}.masks"])} for b in images]


@pytest.fixture(scope="module")
def golden(golden_dir):
    return load_golden(golden_dir, "detr_criterion.npz")


@pytest.mark.parametrize("run", list(RUNS))
def test_restatement_reproduces_reference(golden, run):
    g = golden
    prefix = run if run != "batch" else "batch"
    losses, idx = co.criterion(outputs(g, prefix), targets(g, RUNS[run]), int(g["num_classes"]), float(g["eos_coef"]),
                               ["labels", "boxes", "cardinality", "masks"], return_indices=True)
    assert list(losses) == g[f"{run}.keys"].tolist()
    for k, v in losses.items():
        ref = float(g[f"{run}.loss.{k}"])
        assert abs(float(v) - ref) <= 1e-6 * max(abs(ref), 1e-30), (k, float(v), ref)
    for l, ind in enumerate(idx):
        for b, (i, j) in enumerate(ind):
            assert np.array_equal(i.numpy(), g[f"{run}.idx.{l}.{b}.i"]) and np.array_equal(j.numpy(), g[f"{run}.idx.{l}.{b}.j"])
    wd = json.loads(str(g["weight_dict"]))
    assert {k for k in losses if k[-1].isdigit() and not k.startswith("cardinality")} <= set(wd)


def test_empty_targets(golden):
    g = golden
    empty = [{k: v[:0] for k, v in targets(g, (0,))[0].items()}]
    losses = co.criterion(outputs(g, "0"), empty, int(g["num_classes"]), float(g["eos_coef"]),
                          ["labels", "boxes", "cardinality"])
    for k, v in losses.items():
        assert abs(float(v) - float(g[f"empty.loss.{k}"])) <= 1e-6 * max(abs(float(g[f"empty.loss.{k}"])), 1e-30), k
    assert str(g["empty.error"]) == "NameError"     # the reference's interpolate wrapper on an empty mask batch


def test_lsa_golden_cases(golden):
    names = sorted({k[4:-5] for k in golden.files if k.startswith("lsa.") and k.endswith(".cost")})
    assert len(names) > 30
    for n in names:
        c = golden[f"lsa.{n}.cost"]
        if f"lsa.{n}.error" in golden.files:
            with pytest.raises(ValueError, match=str(golden[f"lsa.{n}.error"])):
                co.lsa(c)
        else:
            i, j = co.lsa(c)
            assert np.array_equal(i, golden[f"lsa.{n}.i"]) and np.array_equal(j, golden[f"lsa.{n}.j"]), n


def test_lsa_matches_scipy_on_seeded_matrices():
    """4000 seeded matrices: small-integer ties, duplicated rows / columns, +inf entries, wide and tall"""
    rng = np.random.default_rng(1)
    for trial in range(4000):
        r, c = (int(x) for x in rng.integers(1, 10, 2))
        kind = trial % 4
        if kind == 0:
            m = rng.integers(0, 3, (r, c)).astype(float)
        elif kind == 1:
            m = rng.standard_normal((r, c))
        elif kind == 2:
            m = rng.integers(0, 2, (r, c)).astype(float)
            m[-1] = m[0]
            m[:, -1] = m[:, 0]
        else:
            m = rng.integers(0, 4, (r, c)).astype(float)
            m[rng.random((r, c)) < 0.2] = np.inf
        try:
            ref = linear_sum_assignment(m)
        except ValueError as e:
            with pytest.raises(ValueError, match=str(e)):
                co.lsa(m)
            continue
        got = co.lsa(m)
        assert np.array_equal(got[0], ref[0]) and np.array_equal(got[1], ref[1]), (trial, m)
