"""The RPN proposal layer on the device (b200_topk_batched -> b200_proposal_decode -> b200_nms_batched, then collect /
distribute) against oracle/proposals.py and oracle/fpn.py, on the inputs an RPN produces: float32 sigmoid scores whose k-th
value is tied, saturated maps, NaN / inf scores and deltas, at the shapes of an FPN pyramid and of C4, at the top-k's limits
and past them.  Inputs come from tests/proposal_cases.py.

The pre-NMS top-k is exactly np.argsort(-scores_hwa, kind="stable")[:k] (NaN last, -0.0 == +0.0); the layer is compared with
the bar the golden tests use: probabilities and batch column exact, coordinates within 1e-4, at least 99.9 % bit-equal."""
import os

import numpy as np
import pytest
import torch

from tests import proposal_cases as PC

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "proposals.npz")


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def make_op(shape_name, pre, post, thresh=0.7, min_size=0, return_tensors=False):
    from detectron.pytorch_b200.modeling.generate_proposals import GenerateProposalsOp
    anchors, stride = PC.anchors_and_stride(shape_name)
    mode = dict(RPN_PRE_NMS_TOP_N=pre, RPN_POST_NMS_TOP_N=post, RPN_NMS_THRESH=thresh, RPN_MIN_SIZE=min_size)
    return GenerateProposalsOp(anchors, 1.0 / stride, train=mode, test=mode, return_tensors=return_tensors), anchors, stride


def oracle(scores, deltas, im_info, anchors, stride, pre, post, thresh=0.7, min_size=0):
    from oracle import proposals as OP
    return OP.generate_proposals(scores, deltas, im_info, anchors, float(stride), pre, post, thresh, min_size)


def assert_matches(rois, probs, ref_rois, ref_probs):
    rois, probs = np.asarray(rois), np.asarray(probs)
    assert rois.shape == ref_rois.shape and probs.shape == ref_probs.shape
    assert np.array_equal(probs, ref_probs, equal_nan=True)        # same candidates survive, in the same order
    assert np.array_equal(rois[:, 0], ref_rois[:, 0])
    np.testing.assert_allclose(rois, ref_rois, rtol=0, atol=1e-4)
    if rois.size:
        assert np.mean(rois == ref_rois) > 0.999


def im_info_for(N):
    return np.stack([PC.IM_INFO[i % 2] for i in range(N)])


def pyramid(score_kind, delta_kinds, k, seed, N=2):
    """{level name: ((N, A, H, W) scores, (N, 4A, H, W) deltas)}; the (level, image) maps take the delta kinds in turn."""
    out = {}
    for j, (name, lvl) in enumerate(PC.FPN_LEVELS):
        maps = [PC.batch(score_kind, delta_kinds[(j * N + i) % len(delta_kinds)], name, k, seed + 31 * lvl + 7 * i, N=1)
                for i in range(N)]
        out[name] = (np.concatenate([m[0] for m in maps]), np.concatenate([m[1] for m in maps]))
    return out


def run_pyramid(inputs, pre, post, min_size=0, N=2):
    """The pyramid through generate_proposals_batched and through per-level op calls (must be identical); returns the batched
    result per level and the oracle's."""
    from detectron.pytorch_b200.modeling.generate_proposals import generate_proposals_batched
    info = im_info_for(N)
    ops, cls, box, refs = [], [], [], []
    for name, _ in PC.FPN_LEVELS:
        op, anchors, stride = make_op(name, pre, post, min_size=min_size)
        s, d = inputs[name]
        ops.append(op); cls.append(dev(s)); box.append(dev(d))
        refs.append(oracle(s, d, info, anchors, stride, pre, post, min_size=min_size))
    fused = generate_proposals_batched(ops, cls, box, torch.from_numpy(info))
    for (rois, probs), op, c, b in zip(fused, ops, cls, box):
        r1, p1 = op(c, b, torch.from_numpy(info))
        assert np.array_equal(rois, r1) and np.array_equal(probs, p1, equal_nan=True)
    return fused, refs


# ------------------------------------------------------------------------------------------------ top-k alone
def _topk_problems():
    """64 (map, k) problems mixing every shape and score kind, k in {0, 1, 2000, n, 8192, 8193, 12000, 16384} where k <= n,
    plus a cut through the -0.0 / +0.0 run of a nonfinite map."""
    ks = (0, 1, 2000, "n", 8192, 8193, 12000, 16384)
    probs = []
    names = list(PC.SHAPES)
    for j in range(63):
        name, kind = names[j % len(names)], PC.SCORE_KINDS[(j // len(names) + j) % len(PC.SCORE_KINDS)]
        A, H, W = PC.SHAPES[name]
        n = A * H * W
        allowed = [n if k == "n" else k for k in ks if (k == "n" and n <= 16384) or (k != "n" and k <= n)]
        k = allowed[(j // len(names)) % len(allowed)]
        probs.append((PC.scores(kind, (A, H, W), max(k, 1), seed=j), k))
    x = PC.scores("nonfinite", PC.SHAPES["p4"], 2000, seed=99)
    probs.append((x, int((x > 0).sum()) + int((x == 0).sum()) // 2))
    return probs


def test_topk_batched_is_the_stable_argsort():
    """One b200_topk_batched call over 64 problems: indices exactly np.argsort(-x_hwa, kind="stable")[:k] -- tied scores
    straddling the cut taken in (h, w, a) order, NaN after every number, -0.0 tied with +0.0 -- and scores equal to x_hwa[order]
    (NaN where the score is NaN); a second call is bit-identical."""
    from detectron.pytorch_b200 import ops
    probs = _topk_problems()
    assert len(probs) == 64
    ks = [k for _, k in probs]
    assert {0, 1, 2000, 8192, 8193, 12000, 16384} <= set(ks)
    maps = [dev(x) for x, _ in probs]
    order, top = ops.topk_batched_raw(maps, ks)
    order2, top2 = ops.topk_batched_raw(maps, ks)
    assert torch.equal(order, order2) and torch.equal(top.view(torch.int32), top2.view(torch.int32))
    order, top = order.cpu().numpy(), top.cpu().numpy()
    off = 0
    for p, (x, k) in enumerate(probs):
        x_hwa = x.transpose(1, 2, 0).reshape(-1)
        ref = PC.stable_topk(x, k)
        assert np.array_equal(order[off:off + k], ref), "problem %d: %s k=%d" % (p, x.shape, k)
        assert np.array_equal(top[off:off + k], x_hwa[ref], equal_nan=True), "problem %d" % p
        off += k


def test_torch_sort_fallback_is_the_stable_argsort():
    """The fallback for k > 16384 candidates follows the same rule as the device top-k (torch.sort alone puts NaN first)."""
    from detectron.pytorch_b200.modeling.generate_proposals import _stable_descending_order
    for kind in ("nonfinite", "saturated", "sigmoid", "quantised"):
        x = PC.scores(kind, PC.SHAPES["p3"], 16385, seed=5)
        flat = dev(x).permute(1, 2, 0).reshape(-1)
        assert np.array_equal(_stable_descending_order(flat).cpu().numpy(), PC.stable_topk(x, x.size)), kind


# ------------------------------------------------------------------------------------------------ whole layer vs oracle
@pytest.mark.parametrize("mode,score_kind", [("fpn_train", "sigmoid"), ("fpn_train", "saturated"), ("fpn_test", "sigmoid"),
                                             ("fpn_test", "saturated"), ("min_size", "sigmoid")])
def test_fpn_pyramid_vs_oracle(mode, score_kind):
    """The five levels of an 800 x 1333 pyramid, two images of different size in one padded map; the ten (level, image) maps
    take every delta kind."""
    pre, post, _, min_size = PC.MODES[mode]
    shift = len(mode) + len(score_kind)
    kinds = PC.DELTA_KINDS[shift % 8:] + PC.DELTA_KINDS[:shift % 8]
    fused, refs = run_pyramid(pyramid(score_kind, kinds, pre, seed=shift), pre, post, min_size)
    for (rois, probs), (rr, pp) in zip(fused, refs):
        assert_matches(rois, probs, rr, pp)


def test_c4_train_saturated_vs_oracle():
    pre, post, _, _ = PC.MODES["c4_train"]
    op, anchors, stride = make_op("c4", pre, post)
    s, d = PC.batch("saturated", "normal", "c4", pre, seed=4)
    rois, probs = op(dev(s), dev(d), torch.from_numpy(PC.IM_INFO))
    assert_matches(rois, probs, *oracle(s, d, PC.IM_INFO, anchors, stride, pre, post))


# ------------------------------------------------------------------------------------------------ limits and fallbacks
@pytest.mark.parametrize("pre", [16384, 16385])
def test_pre_nms_top_n_at_the_device_top_k_limit_and_past_it(pre):
    """16384: the device top-k at its largest k; 16385: the torch.sort fallback.  Both on a C4 map with more exact 1.0 scores
    than k, and both past the 13000-candidate limit of the batched NMS."""
    op, anchors, stride = make_op("c4", pre, 2000)
    s, d = PC.batch("saturated", "normal", "c4", pre, seed=8, N=1)
    rois, probs = op(dev(s), dev(d), torch.from_numpy(PC.IM_INFO[:1]))
    assert_matches(rois, probs, *oracle(s, d, PC.IM_INFO[:1], anchors, stride, pre, 2000))


def test_all_candidates_on_p3_single_problem_nms():
    """pre_nms_topN <= 0: all 50 400 P3 candidates, sorted by the fallback and suppressed by one single-problem NMS."""
    op, anchors, stride = make_op("p3", -1, 1000)
    s, d = PC.batch("sigmoid", "normal", "p3", 2000, seed=6, N=1)
    rois, probs = op(dev(s), dev(d), torch.from_numpy(PC.IM_INFO[:1]))
    assert_matches(rois, probs, *oracle(s, d, PC.IM_INFO[:1], anchors, stride, -1, 1000))


def test_65_problems_chunk_the_top_k_and_the_nms():
    """13 images x 5 levels = 65 (level, image) problems: two batched top-k calls and two batched NMS calls."""
    pre, post, _, _ = PC.MODES["fpn_test"]
    fused, refs = run_pyramid(pyramid("sigmoid", ("normal",), pre, seed=13, N=13), pre, post, N=13)
    for (rois, probs), (rr, pp) in zip(fused, refs):
        assert_matches(rois, probs, rr, pp)


# ------------------------------------------------------------------------------------------------ non-finite inputs
def test_nonfinite_scores_and_deltas_vs_oracle():
    """NaN scores are never selected while finite ones remain (P2..P5: pre_nms_topN below the finite count; P6 takes all its
    819 candidates, NaN ones last as in the oracle); a candidate whose deltas hold a NaN is dropped; +-inf deltas give the
    oracle's boxes."""
    pre, post, _, _ = PC.MODES["fpn_train"]
    inputs = pyramid("nonfinite", ("nan_dx", "nan_dy", "nan_dw", "nan_dh", "inf"), pre, seed=17)
    fused, refs = run_pyramid(inputs, pre, post)
    for (name, _), (rois, probs), (rr, pp) in zip(PC.FPN_LEVELS, fused, refs):
        assert not np.isnan(rois).any()
        finite = min(int((~np.isnan(s)).sum()) for s in inputs[name][0])
        if pre < finite:
            assert not np.isnan(probs).any()
        assert_matches(rois, probs, rr, pp)


@pytest.mark.parametrize("name", sorted(PC.GOLDEN))
def test_new_golden_cases_through_the_device_layer(name):
    """The reference op's own output on NaN / inf inputs, at the clip's float32 neighbours and on an FPN P2 level."""
    g = np.load(GOLDEN)
    s, d, im_info, anchors, stride, pre, post, thresh, min_size, training = PC.golden_inputs(name)
    assert PC.sha256(s, d) == str(g[name + "/input_sha256"])
    op, _, _ = make_op(PC.GOLDEN[name][2], pre, post, thresh, min_size)
    op.train(training)
    rois, probs = op(dev(s), dev(d), torch.from_numpy(im_info))
    assert_matches(rois, probs, g[name + "/rois"], g[name + "/probs"])


# ------------------------------------------------------------------------------------------------ collect and distribute
def test_collect_and_distribute_with_scores_tied_across_levels():
    """Saturated maps: thousands of proposals score exactly 1.0 on every level, so the collect's cut falls inside a tie that
    spans levels.  Device collect / distribute on the device proposals equal oracle/fpn.py on the same proposals exactly, and
    those proposals match oracle/proposals.py."""
    from detectron.pytorch_b200.modeling.collect_and_distribute_fpn_rpn_proposals import collect, distribute
    from detectron.pytorch_b200.modeling.generate_proposals import generate_proposals_batched
    from oracle import fpn as OF
    pre, post, _, _ = PC.MODES["fpn_train"]
    inputs = pyramid("saturated", ("normal",), pre, seed=23)
    ops, cls, box, refs = [], [], [], []
    for name, _ in PC.FPN_LEVELS:
        op, anchors, stride = make_op(name, pre, post, return_tensors=True)
        s, d = inputs[name]
        ops.append(op); cls.append(dev(s)); box.append(dev(d))
        refs.append(oracle(s, d, PC.IM_INFO, anchors, stride, pre, post))
    out = generate_proposals_batched(ops, cls, box, torch.from_numpy(PC.IM_INFO))
    for (r, p), (rr, pp) in zip(out, refs):
        assert_matches(r.cpu().numpy(), p.cpu().numpy(), rr, pp)
    lvl_rois, lvl_probs = [r for r, _ in out], [p for _, p in out]
    assert sum(int((p == 1).sum()) for p in lvl_probs) > post                  # the cut falls inside the tie
    rois = collect(lvl_rois, lvl_probs, post)
    blobs = distribute(rois, 2, 5)
    r_ref = OF.collect([r.cpu().numpy() for r in lvl_rois], [p.cpu().numpy() for p in lvl_probs], post)
    b_ref = OF.distribute(r_ref, 2, 5)
    assert np.array_equal(rois.cpu().numpy(), r_ref)
    assert np.array_equal(blobs["rois_idx_restore_int32"].cpu().numpy(), b_ref["rois_idx_restore_int32"])
    for lvl in range(2, 6):
        assert np.array_equal(blobs["rois_fpn%d" % lvl].cpu().numpy(), b_ref["rois_fpn%d" % lvl])


def _level_boundary_rois():
    """Boxes whose sqrt(area) / 224 + 1e-6 (float32) lies within +-64 ulps of 1/2, 1 and 2, the level boundaries 2|3, 3|4, 4|5."""
    out = []
    for t in (0.5, 1.0, 2.0):
        w0 = np.float32((t - 1e-6) * 224)
        ws = w0 + np.arange(-300, 301, dtype=np.float32) * np.spacing(w0)
        hs = w0 + np.arange(-40, 41, dtype=np.float32) * np.spacing(w0) * 7
        W, H = [a.ravel() for a in np.meshgrid(ws, hs)]
        for x1, y1 in ((0.0, 0.0), (17.25, 3.5)):
            r = np.stack([np.full_like(W, x1), np.full_like(W, y1), np.float32(x1) + W - 1, np.float32(y1) + H - 1], 1).astype(np.float32)
            w, h = r[:, 2] - r[:, 0] + 1, r[:, 3] - r[:, 1] + 1
            y = np.sqrt(w * h) / np.float32(224) + np.float32(1e-6)
            out.append(r[np.abs((y - np.float32(t)) / np.spacing(np.float32(t))) <= 64])
    return np.concatenate(out)


def test_level_assignment_at_the_level_boundaries_on_the_device():
    from detectron.pytorch_b200.utils.fpn import map_rois_to_fpn_levels
    from oracle import fpn as OF
    r = _level_boundary_rois()
    ref = OF.map_rois_to_fpn_levels(r.copy(), 2, 5)
    assert set(np.unique(ref).tolist()) == {2.0, 3.0, 4.0, 5.0}
    got = map_rois_to_fpn_levels(dev(r), 2, 5).cpu().numpy()
    bad = np.nonzero(got != ref)[0]
    assert bad.size == 0, "%d of %d levels differ, first %s: device %s oracle %s" % (bad.size, r.shape[0], r[bad[:3]], got[bad[:3]], ref[bad[:3]])
