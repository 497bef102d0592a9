"""Proposal recall: the numpy restatement (oracle/box_proposals.py) against the reference's goldens, the kernel's incremental
column-maximum algorithm against the restatement, the IoU sign sweep, host packing and the C ABI's argument checks on the CPU; the
device evaluation (datasets/json_dataset_evaluator.evaluate_box_proposals, task_evaluation.evaluate_box_proposals,
ops.box_proposal_match_raw) against the goldens and the restatement on the GPU."""
import ctypes
import json
import logging
import os

import numpy as np
import pytest

from oracle import box_proposals as O
from tests import box_proposal_cases as BC

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "box_proposals.npz")
CASES = list(BC.CASES)
FIELDS = ("ar", "recalls", "thresholds", "gt_overlaps", "num_pos")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(a, b, equal_nan=True)


def _configs():
    for tname, thr in BC.THRESHOLD_SETS.items():
        for area in BC.AREA_NAMES:
            for limit in BC.LIMITS:
                yield tname, thr, area, limit


def _check_against_golden(golden, case, evaluate):
    roidb = BC.unpack({k: golden[case + "/in/" + k] for k in ("row_begin", "boxes", "gt_classes", "is_crowd", "seg_areas")})
    raised_somewhere = False
    for tname, thr, area, limit in _configs():
        want = BC.load_golden(golden, case, tname, area, limit)
        if want is None:
            raised_somewhere = True
            with pytest.raises(AssertionError):
                evaluate(roidb, None if thr is None else thr.copy(), area, limit)
            continue
        got = evaluate(roidb, None if thr is None else thr.copy(), area, limit)
        for k in FIELDS:
            assert _same(got[k], want[k]), (case, tname, area, limit, k)
        assert isinstance(got["num_pos"], int) and got["gt_overlaps"].dtype == np.float64
    assert raised_somewhere == (case == "nan_gt")


# ---- CPU: the restatement equals the reference ------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES)
def test_oracle_equals_reference_goldens(golden, case):
    _check_against_golden(golden, case, lambda r, t, a, l: O.evaluate_box_proposals(r, thresholds=t, area=a, limit=l))


def test_goldens_cover_the_listed_cases(golden):
    assert golden["coco_like/in/row_begin"].size == 41
    assert golden["nan_gt/default/raised"].any() and not golden["nan_gt/default/raised"].all()     # limit 0 keeps no proposal
    assert np.isnan(golden["no_positives/default/ar"]).all()
    gt = golden["on_threshold/default/gt_overlaps"]
    assert 0.5 in gt and 0.75 in gt and 1.0 in gt
    areas = golden["area_boundaries/in/seg_areas"]
    for b in BC.AREA_BOUNDS:
        assert np.float32(b) in areas
    assert not golden["nan_proposal/default/raised"].any()


# ---- CPU: the kernel's algorithm ----------------------------------------------------------------------------------------------
def incremental_match(ov):
    """The kernel's greedy assignment on a (P, G) IoU block without NaN: per live column its maximum over the unused proposals and
    the first proposal reaching it; the pick is the live column with the largest maximum (lowest index on ties), and only the
    columns whose argmax was the proposal just taken are recomputed.  Returns the recorded overlap per column (0 if unmatched)."""
    P, G = ov.shape
    rec = np.zeros(G)
    if P == 0 or G == 0:
        return rec
    used = np.zeros(P, np.bool_)
    live = np.ones(G, np.bool_)
    cmax, carg = ov.max(axis=0), ov.argmax(axis=0)
    for _ in range(min(P, G)):
        cand = np.nonzero(live)[0]
        g = cand[np.argmax(cmax[cand])]
        p = carg[g]
        rec[g] = cmax[g]
        live[g] = False
        used[p] = True
        for h in np.nonzero(live & (carg == p))[0]:
            col = np.where(used, -np.inf, ov[:, h])
            carg[h] = int(np.argmax(col))
            cmax[h] = col[carg[h]]
    return rec


def incremental_recall(roidb, area, limit, thresholds=None):
    """evaluate_box_proposals' fields from incremental_match, with the oracle's selection, limits and recall tail."""
    values, num_pos = [np.zeros(0)], 0
    for e in roidb:
        props, pos = O.split_entry(e, area, limit)
        num_pos += len(pos)
        if props is not None:
            values.append(incremental_match(O.overlaps(props, pos).astype(np.float64)))
    thresholds = np.arange(0.5, 0.95 + 1e-5, 0.05) if thresholds is None else thresholds
    return O.recall_summary(np.sort(np.concatenate(values)), num_pos, thresholds)


def _tie_heavy(seed, n_images=25):
    """Integer grid boxes: many exactly equal IoUs, duplicate proposals and duplicate gts."""
    rng = np.random.RandomState(seed)
    roidb = []
    for _ in range(n_images):
        g = rng.randint(0, 15)
        gts = rng.randint(0, 6, (g, 2)) * 10.0
        gts = np.concatenate([gts, gts + rng.choice([9, 19], (g, 1))], 1)
        if g:
            gts = np.concatenate([gts, gts[: rng.randint(0, g + 1)]])
        p = rng.randint(0, 40)
        props = rng.randint(0, 6, (p, 2)) * 10.0
        props = np.concatenate([props, props + rng.choice([9, 19], (p, 1))], 1)
        n = len(gts)
        roidb.append(BC.entry(gts, rng.randint(1, 4, n), rng.uniform(size=n) < 0.1, np.full(n, 150.0), props))
    return roidb


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_incremental_algorithm_equals_oracle(seed):
    sets = [BC.coco_like(seed=100 + seed, n_images=12, max_gt=25, max_props=400), _tie_heavy(seed), BC.ties()]
    for roidb in sets:
        for area in ("all", "small", "medium", "large"):
            for limit in (None, 100, 7, 0, -3):
                want = O.evaluate_box_proposals(roidb, area=area, limit=limit)
                got = incremental_recall(roidb, area, limit)
                for k in FIELDS:
                    assert _same(got[k], want[k]), (seed, area, limit, k)


def test_no_overlap_is_negative_on_degenerate_finite_boxes():
    """Every IoU that is not NaN is >= 0, so masking with -1 equals removing the row and the column."""
    from oracle.targets import bbox_overlaps
    rng = np.random.RandomState(5)
    f32 = np.float32
    base = np.array([0, 1, -1, 0.5, 1e-30, 1e-38, 1e-45, 3e-8, 6e-8, 1e6, 1e10, 1e20, 1e30, 3e38, -1e30, 16777216, 16777217], f32)
    x1 = rng.choice(base, 4000) * rng.choice([1, -1], 4000).astype(f32)
    w = rng.choice(np.array([0, -0.5, -1, -1.5, -2, 1e-7, 1e-30, 1, 10, -10, 1e30, -1e30, 3e38, 6e-8], f32), 4000)
    with np.errstate(over="ignore"):
        boxes = np.stack([x1, x1[::-1], (x1 + w).astype(f32), (x1[::-1] + w[::-1]).astype(f32)], 1).astype(f32)
    boxes = boxes[np.isfinite(boxes).all(1)]
    assert len(boxes) > 3000
    tiny = np.nextafter(f32(100.0), f32(200)) - f32(100.0)
    subulp = np.array([[100, 100, 100 - 1 + tiny, 100 - 1 + tiny], [100, 100, 99, 99], [0, 0, -1, -1], [0, 0, -1 + 6e-8, 5]], f32)
    boxes = np.concatenate([boxes, subulp])
    with np.errstate(all="ignore"):
        for chunk in np.array_split(np.arange(len(boxes)), 8):
            ov = bbox_overlaps(boxes[chunk], boxes)
            assert not (ov[~np.isnan(ov)] < 0).any()
            ov = O.overlaps(boxes[chunk], boxes)
            assert not (ov[~np.isnan(ov)] < 0).any()
        assert np.isinf(bbox_overlaps(boxes, boxes)).sum() == 0


# ---- CPU: host packing and the C ABI -----------------------------------------------------------------------------------------
def test_effective_proposal_counts_follow_python_slicing():
    from detectron.pytorch_b200.datasets import json_dataset_evaluator as J
    n = [0, 1, 2, 3, 7, 100, 1500]
    limits = [None, 1000, 100, 7, 3, 1, 0, -1, -3, -2000]
    got = J.effective_proposal_counts(n, limits)
    assert got.dtype == np.int32 and got.shape == (len(limits), len(n))
    for k, limit in enumerate(limits):
        assert got[k].tolist() == [len(range(p)[:limit]) for p in n]


def test_pack_roidb_selects_as_the_reference():
    from detectron.pytorch_b200.datasets import json_dataset_evaluator as J
    roidb = BC.coco_like(seed=9, n_images=15, max_props=50) + BC.shapes()
    prop_box, prop_begin, gt_box, gt_area, gt_begin = J.pack_roidb(roidb)
    assert prop_box.dtype == np.float32 and gt_box.dtype == np.float32 and gt_area.dtype == np.float64
    for i, e in enumerate(roidb):
        gt = np.where((e["gt_classes"] > 0) & (e["is_crowd"] == 0))[0]
        assert np.array_equal(gt_box[gt_begin[i]:gt_begin[i + 1]], e["boxes"][gt])
        assert np.array_equal(gt_area[gt_begin[i]:gt_begin[i + 1]], e["seg_areas"][gt].astype(np.float64))
        assert np.array_equal(prop_box[prop_begin[i]:prop_begin[i + 1]], e["boxes"][e["gt_classes"] == 0])
    # an image whose proposals are all removed by the limit is evaluated; one without proposals is skipped (P == 0 on the device)
    assert (np.diff(prop_begin) == 0).any()
    assert (J.effective_proposal_counts(np.diff(prop_begin), [0]) == 0).all()


def test_box_proposal_match_abi_checks_arguments():
    from detectron.pytorch_b200 import _lib
    lib = _lib.load()
    fake = ctypes.c_void_p(256)                    # aligned, never dereferenced: every call below returns before any launch
    ranges = (ctypes.c_double * 2)(0.0, 1e10)
    ws = lib.b200_box_proposal_match_workspace_bytes(10, 4, 1, 1)
    assert ws >= 1 * (4 * 8 + 10) and lib.b200_box_proposal_match_workspace_bytes(-1, 4, 1, 1) == 0

    def call(n=2, p=10, g=4, a=1, l=1, t=3, prop=fake, begin=fake, area_host=ranges, workspace=fake, ws_bytes=ws, counts=fake):
        return lib.b200_box_proposal_match(n, p, g, a, l, t, prop, begin, fake, fake, fake, fake, area_host, fake, workspace, ws_bytes,
                                           fake, fake, fake, counts, None)
    for bad in (dict(n=-1), dict(p=-1), dict(g=-1), dict(a=-1), dict(a=9), dict(l=-1), dict(t=-1), dict(prop=None), dict(begin=None),
                dict(area_host=None), dict(counts=None), dict(prop=ctypes.c_void_p(260))):
        assert call(**bad) == -1, bad
    assert call(workspace=None) == -2 and call(ws_bytes=ws - 1) == -2
    for zero in (dict(n=0), dict(a=0), dict(l=0)):
        assert call(**zero, prop=None, begin=None, area_host=None, workspace=None) == 0, zero


def test_task_evaluation_result_layout_and_log(caplog):
    from detectron.pytorch_b200.datasets import task_evaluation as T
    empty = T._empty_box_proposal_results()
    assert list(empty["box_proposal"].keys()) == ["AR@100", "ARs@100", "ARm@100", "ARl@100", "AR@1000", "ARs@1000", "ARm@1000",
                                                  "ARl@1000"]
    res = {"ds": {"box_proposal": dict(empty["box_proposal"], **{"AR@100": 0.51234})}}
    with caplog.at_level(logging.INFO, logger=T.logger.name):
        T.log_box_proposal_results(res)
    assert caplog.messages[0] == "ds" and caplog.messages[1] == "AR@100  : 0.512" and caplog.messages[8] == "ARl@1000: -1.000"


def test_unknown_area_fails_as_the_reference():
    from detectron.pytorch_b200.datasets import json_dataset_evaluator as J
    with pytest.raises(AssertionError, match="Unknown area range: tiny"):
        J.evaluate_box_proposals(None, BC.shapes(), area="tiny")


# ---- GPU: the device evaluation -----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_device_equals_reference_goldens(golden, case):
    from detectron.pytorch_b200.datasets import json_dataset_evaluator as J
    _check_against_golden(golden, case, lambda r, t, a, l: J.evaluate_box_proposals(None, r, thresholds=t, area=a, limit=l))


class _Dataset:
    def __init__(self, name):
        self.name = name


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_task_evaluation_equals_reference_in_one_launch(golden, case):
    from detectron.pytorch_b200 import _lib
    from detectron.pytorch_b200.datasets import task_evaluation as T
    roidb = BC.unpack({k: golden[case + "/in/" + k] for k in ("row_begin", "boxes", "gt_classes", "is_crowd", "seg_areas")})
    if golden[case + "/task/raised"]:
        with pytest.raises(AssertionError):
            T.evaluate_box_proposals(_Dataset(case), roidb)
        return
    before = _lib.launch_count()
    out = T.evaluate_box_proposals(_Dataset(case), roidb)
    assert _lib.launch_count() - before == 1
    assert list(out.keys()) == [case] and list(out[case].keys()) == ["box_proposal"]
    res = out[case]["box_proposal"]
    assert list(res.keys()) == json.loads(golden[case + "/task/keys"].tobytes().decode())
    assert _same(np.asarray(list(res.values()), np.float64), golden[case + "/task/values"])


@pytest.mark.gpu
def test_task_evaluation_kernel_launches_once_per_chunk(monkeypatch):
    import torch
    from detectron.pytorch_b200.datasets import json_dataset_evaluator as J
    from detectron.pytorch_b200.datasets import task_evaluation as T
    roidb = BC.coco_like(seed=4, n_images=30, max_props=300)
    monkeypatch.setattr(J, "BOX_PROPOSAL_CHUNK_IMAGES", 7)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        T.evaluate_box_proposals(_Dataset("d"), roidb)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if "box_proposal_match_kernel" in e.name]
    assert len(names) == 5                          # ceil(30 / 7) chunks


def _scale_roidb():
    """2000 images of 2000 proposals; most have a COCO-like gt count, every 25th 280 .. 600 gts."""
    rng = np.random.RandomState(17)
    roidb = []
    light = BC.scale_set(seed=18, n_images=2000, props=(2000, 2000), gt_mean=7.3)
    for i, e in enumerate(light):
        if i % 25 == 0:
            e = BC.scale_set(seed=1000 + i, n_images=1, props=(2000, 2000), gt_mean=None, max_gt=600)[0]
            if (e["gt_classes"] > 0).sum() < 300:
                g = int(rng.randint(300, 601))
                e = BC.scale_set(seed=2000 + i, n_images=1, props=(2000, 2000), gt_mean=g, max_gt=600)[0]
        roidb.append(e)
    return roidb


@pytest.mark.gpu
def test_device_equals_restatement_at_scale(monkeypatch):
    """All 2000 images against the numpy restatement of the kernel's incremental algorithm (itself checked against the oracle on
    the CPU), with the chunk at its default and small."""
    from detectron.pytorch_b200.datasets import json_dataset_evaluator as J
    roidb = _scale_roidb()
    assert max((e["gt_classes"] > 0).sum() for e in roidb) > 500 and len(roidb) == 2000
    configs = [("all", None), ("medium", 100), ("large", 1000)]
    want = {c: incremental_recall(roidb, *c) for c in configs}
    for chunk in (J.BOX_PROPOSAL_CHUNK_IMAGES, 61):
        monkeypatch.setattr(J, "BOX_PROPOSAL_CHUNK_IMAGES", chunk)
        for area, limit in configs:
            got = J.evaluate_box_proposals(None, roidb, area=area, limit=limit)
            for k in FIELDS:
                assert _same(got[k], want[(area, limit)][k]), (chunk, area, limit, k)


@pytest.mark.gpu
def test_device_equals_oracle_on_large_gt_images(monkeypatch):
    """The reference loop's restatement itself (oracle/box_proposals.py) on the scale set's 80 images of 280 .. 600 gts and 300 of its
    COCO-like ones, so the at-scale check does not rest on the kernel's own algorithm alone."""
    from detectron.pytorch_b200.datasets import json_dataset_evaluator as J
    full = _scale_roidb()
    heavy = [e for i, e in enumerate(full) if i % 25 == 0]
    roidb = heavy + [e for i, e in enumerate(full) if i % 25][:300]
    assert len(heavy) == 80 and min((e["gt_classes"] > 0).sum() for e in heavy) >= 250
    monkeypatch.setattr(J, "BOX_PROPOSAL_CHUNK_IMAGES", 97)
    for area, limit in [("all", None), ("large", 1000), ("medium", 100)]:
        want = O.evaluate_box_proposals(roidb, area=area, limit=limit)
        got = J.evaluate_box_proposals(None, roidb, area=area, limit=limit)
        for k in FIELDS:
            assert _same(got[k], want[k]), (area, limit, k)


@pytest.mark.gpu
def test_raw_entry_converts_dtypes_and_refuses_bad_inputs():
    import torch
    from detectron.pytorch_b200 import ops
    from detectron.pytorch_b200.datasets import json_dataset_evaluator as J
    roidb = BC.coco_like(seed=8, n_images=6, max_props=200)
    prop_box, prop_begin, gt_box, gt_area, gt_begin = J.pack_roidb(roidb)
    counts = J.effective_proposal_counts(np.diff(prop_begin), [None, 7])
    ranges, thr = [J.BOX_PROPOSAL_AREA_RANGES["all"]], J.default_recall_thresholds()
    cuda = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()  # noqa: E731
    want = ops.box_proposal_match_raw(cuda(prop_box), cuda(prop_begin), cuda(gt_box), cuda(gt_area), cuda(gt_begin), cuda(counts),
                                      ranges, thr)
    # int64 offsets / counts (torch.tensor of a list), float64 boxes, float32 areas, a non-contiguous box view
    wide = torch.from_numpy(np.concatenate([prop_box, prop_box], 1).astype(np.float64)).cuda()[:, :4]
    got = ops.box_proposal_match_raw(wide, cuda(prop_begin.astype(np.int64)), cuda(gt_box.astype(np.float64)),
                                     cuda(gt_area.astype(np.float32)), torch.tensor(gt_begin.tolist()).cuda(),
                                     torch.tensor(counts.tolist()).cuda(), ranges, thr)
    for w, g in zip(want, got):
        assert torch.equal(w, g)
    args = [cuda(prop_box), cuda(prop_begin), cuda(gt_box), cuda(gt_area), cuda(gt_begin), cuda(counts)]
    bad = {0: cuda(prop_box[:, :3]), 1: cuda(prop_begin[:-1]), 2: torch.from_numpy(gt_box), 4: cuda(gt_begin[::-1].copy()),
           5: cuda(counts[:, :-1])}
    for k, t in bad.items():
        with pytest.raises(ValueError):
            ops.box_proposal_match_raw(*[t if j == k else a for j, a in enumerate(args)], ranges, thr)


@pytest.mark.gpu
def test_raw_tensors_equal_roidb_path():
    import torch
    from detectron.pytorch_b200 import ops
    from detectron.pytorch_b200.datasets import json_dataset_evaluator as J
    roidb = BC.coco_like(seed=6, n_images=20)
    prop_box, prop_begin, gt_box, gt_area, gt_begin = J.pack_roidb(roidb)
    limits, areas = [None, 100, 7], ["all", "small", "large"]
    ranges = [J.BOX_PROPOSAL_AREA_RANGES[a] for a in areas]
    thr = J.default_recall_thresholds()
    cuda = lambda x: torch.from_numpy(x).cuda()  # noqa: E731
    overlap, excluded, error, counts = ops.box_proposal_match_raw(
        cuda(prop_box), cuda(prop_begin), cuda(gt_box), cuda(gt_area), cuda(gt_begin),
        cuda(J.effective_proposal_counts(np.diff(prop_begin), limits)), ranges, thr)
    assert not error.any()
    for l, limit in enumerate(limits):
        for a, area in enumerate(areas):
            want = J.evaluate_box_proposals(None, roidb, area=area, limit=limit)
            ov = overlap[l, a][~excluded[l, a]].cpu().numpy().astype(np.float64)
            assert _same(np.sort(ov), want["gt_overlaps"])
            assert _same(counts[l, a].cpu().numpy() / float(want["num_pos"]), want["recalls"])


def test_raw_entry_refuses_host_tensors():
    import torch
    from detectron.pytorch_b200 import ops
    z = lambda *shape, dt=torch.int32: torch.zeros(shape, dtype=dt)  # noqa: E731
    with pytest.raises(ValueError, match="CUDA"):
        ops.box_proposal_match_raw(z(1, 4, dt=torch.float32), z(2), z(1, 4, dt=torch.float32), z(1, dt=torch.float64), z(2), z(1, 1),
                                   [(0.0, 1e10)], [0.5])
