"""oracle/proposals.py against golden vectors produced by the reference's own GenerateProposalsOp (CPU, unmodified;
tests/golden/make_golden_proposals.py), and oracle_nms_cython against the reference's live Cython NMS."""
import os

import numpy as np
import pytest

from detectron.pytorch_b200 import synthetic as S
from oracle import cpu as O
from oracle import proposals as P
from tests import proposal_cases as PC

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "proposals.npz"))
CASES = sorted({k.split("/")[0] for k in GOLD.files if k.endswith("/params")})


def case(name):
    g = {k.split("/", 1)[1]: GOLD[k] for k in GOLD.files if k.startswith(name + "/")}
    if "scores" not in g:                                        # inputs regenerated from the case seed, pinned by their digest
        g["scores"], g["deltas"] = PC.golden_inputs(name)[:2]
        assert PC.sha256(g["scores"], g["deltas"]) == str(g["input_sha256"])
    stride, pre, post, thresh, min_size = g["params"]
    return g, float(stride), int(pre), int(post), float(thresh), float(min_size)


@pytest.mark.parametrize("name", CASES)
def test_oracle_reproduces_the_reference_op_bit_for_bit(name):
    g, stride, pre, post, thresh, min_size = case(name)
    rois, probs = P.generate_proposals(g["scores"], g["deltas"], g["im_info"], g["anchors"], stride, pre, post, thresh,
                                       min_size, nms="cython")
    assert rois.shape == g["rois"].shape
    assert np.array_equal(rois, g["rois"])
    assert np.array_equal(probs, g["probs"])


@pytest.mark.parametrize("name", CASES)
def test_cuda_nms_semantics_give_the_same_proposals_on_these_inputs(name):
    """IoU > t (CUDA kernel) vs IoU >= t (Cython): identical unless some pair sits exactly on the threshold."""
    g, stride, pre, post, thresh, min_size = case(name)
    rois, probs = P.generate_proposals(g["scores"], g["deltas"], g["im_info"], g["anchors"], stride, pre, post, thresh,
                                       min_size, nms="cuda")
    assert np.array_equal(rois, g["rois"]) and np.array_equal(probs, g["probs"])


def test_new_golden_cases_reach_the_edges_they_are_for():
    """nonfinite: NaN scores exist but none is selected, NaN- and inf-delta candidates are among the pre-NMS top k, and the
    reference dropped every NaN box; clip_edges: dw / dh at all three float32 neighbours of the clip reach the decode."""
    g, stride, pre, post, thresh, min_size = case("nonfinite")
    for i in range(2):
        s = g["scores"][i].transpose(1, 2, 0).reshape(-1)
        d = g["deltas"][i].reshape(-1, 4, s.size // 3).transpose(2, 0, 1).reshape(-1, 4)
        top = PC.stable_topk(g["scores"][i], pre)
        assert np.isnan(s).any() and not np.isnan(s[top]).any()
        for c in range(4):
            assert np.isnan(d[top, c]).any()
        assert np.isinf(d[top]).any()
    assert not np.isnan(g["rois"]).any() and not np.isnan(g["probs"]).any()
    g, stride, pre, post, thresh, min_size = case("clip_edges")
    d = g["deltas"][0].reshape(-1, 4, g["scores"][0][0].size).transpose(2, 0, 1).reshape(-1, 4)
    top = PC.stable_topk(g["scores"][0], pre)
    for v in PC.CLIP_NEIGHBOURS:
        assert (d[top, 2] == v).any() and (d[top, 3] == v).any()


@pytest.mark.parametrize("n", [1, 65, 1000, 3000])
def test_nms_cython_restatement_matches_the_live_cython_routine(n):
    b = S.make_nms_boxes(n, seed=n)
    assert np.array_equal(np.asarray(O.nms_cython(b, 0.7)).reshape(-1), GOLD["cython_nms/%d/keep" % n])


def test_proposal_properties():
    g, stride, pre, post, thresh, min_size = case("min_size")
    rois, probs = P.generate_proposals(g["scores"], g["deltas"], g["im_info"], g["anchors"], stride, pre, post, thresh, min_size)
    im_h, im_w, scale = g["im_info"][0]
    assert np.all(rois[:, 1] >= 0) and np.all(rois[:, 3] <= im_w - 1) and np.all(rois[:, 2] >= 0) and np.all(rois[:, 4] <= im_h - 1)
    assert np.all(rois[:, 3] - rois[:, 1] + 1 >= min_size * scale) and np.all(rois[:, 4] - rois[:, 2] + 1 >= min_size * scale)
    assert np.all(np.diff(probs.reshape(-1)) <= 0) and len(rois) <= post
