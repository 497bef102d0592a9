"""RPN and Fast R-CNN training losses (csrc/losses.cu, ops.rpn_losses / ops.fast_rcnn_losses, modeling/{rpn_heads, FPN,
fast_rcnn_heads}.py) against the reference's own functions (tests/golden/losses.npz, made by make_golden_losses.py) and the float64
restatement in oracle/losses.py.

Tolerances.  The golden values are the reference's float32 results: each element term is a handful of float32 operations (relative
error within a few eps32) and torch sums at most a few thousand such terms in float32 (relative error within log2(n) eps32 for
its pairwise sum).  rtol = 1e-5 covers both with a margin.  A gradient element where softmax - onehot or sigmoid - y cancels
carries the absolute error of its larger operand, so gradients also get GRAD_ULPS eps32 times their largest magnitude.
For the full-size steps the bound on a loss is the one for a float32 sum of n nonnegative terms, each evaluated to within
ELEM_ULPS eps32: |device - oracle| <= (ELEM_ULPS + log2 n) eps32 * sum|term| / divisor + eps32 |loss| (the final float32
division).  Gradients are elementwise: within GRAD_ULPS ulp of the oracle rounded to float32, plus GRAD_ULPS eps32 times the
upstream scale for terms that cancel (sigmoid(x) - y, softmax - onehot).
"""
import math
import sys
import types

import numpy as np
import pytest
import torch

from oracle import losses as O

GOLDEN = "tests/golden/losses.npz"
RPN_CASES = ["fpn_sigmoid", "fpn_softmax", "single_sigmoid", "single_softmax", "single_ignored", "tie", "nonfinite_sigmoid",
             "nonfinite_softmax"]
FRCN_CASES = ["frcn_specific", "frcn_agnostic", "frcn_nonfinite"]
RTOL, ATOL = 1e-5, 1e-9
EPS32 = float(np.finfo(np.float32).eps)
ELEM_ULPS, GRAD_ULPS = 8, 4


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


def _rpn_case(g, case):
    L, softmax, fpn, divisor = (int(v) for v in g[case + "/meta"])
    levels = [tuple(g["%s/%s_%d" % (case, k, l)] for k in ("cls", "bbox", "labels", "targets", "inside", "outside")) for l in range(L)]
    return levels, bool(softmax), bool(fpn), float(divisor)


def _frcn_case(g, case):
    return tuple(g[case + "/" + k] for k in ("cls", "bbox", "labels", "targets", "inside", "outside"))


def _close(actual, expected, what, grad=False):
    """Losses within RTOL; gradients also within GRAD_ULPS eps32 of their largest magnitude (the upstream scale), for the elements
    where softmax - onehot or sigmoid - y cancel."""
    expected = np.asarray(expected, np.float64)
    fin = np.isfinite(expected)
    atol = max(ATOL, GRAD_ULPS * EPS32 * np.abs(expected[fin]).max()) if grad and fin.any() else ATOL
    np.testing.assert_allclose(np.asarray(actual, np.float64), expected, rtol=RTOL, atol=atol, equal_nan=True, err_msg=what)


# ---- CPU: the oracle against the reference ---------------------------------------------------------------------------------
@pytest.mark.parametrize("case", RPN_CASES)
def test_oracle_rpn_matches_golden(golden, case):
    levels, softmax, _, divisor = _rpn_case(golden, case)
    losses, grads = O.rpn_losses(levels, softmax, divisor, grad_coef=golden[case + "/gcoef"])
    _close(losses, golden[case + "/losses"], case + " losses")
    for l, (dc, db) in enumerate(grads):
        _close(dc, golden["%s/d_cls_%d" % (case, l)], "%s d_cls level %d" % (case, l), grad=True)
        _close(db, golden["%s/d_bbox_%d" % (case, l)], "%s d_bbox level %d" % (case, l), grad=True)


@pytest.mark.parametrize("case", FRCN_CASES)
def test_oracle_fast_rcnn_matches_golden(golden, case):
    loss_cls, loss_bbox, acc, d_cls, d_bbox = O.fast_rcnn_losses(*_frcn_case(golden, case), grad_coef=golden[case + "/gcoef"])
    _close([loss_cls, loss_bbox], golden[case + "/losses"][:2], case + " losses")
    assert np.float32(acc) == golden[case + "/losses"][2]
    _close(d_cls, golden[case + "/d_cls"], case + " d_cls", grad=True)
    _close(d_bbox, golden[case + "/d_bbox"], case + " d_bbox", grad=True)


def test_golden_covers_the_special_cases(golden):
    assert golden["fpn_sigmoid/losses"][4, 0] == 0 and np.isnan(golden["fpn_softmax/losses"][4, 0])
    assert np.isnan(golden["single_ignored/losses"][0, 0])
    assert np.isnan(golden["nonfinite_sigmoid/losses"]).all() and np.isnan(golden["nonfinite_softmax/losses"][0, 1])
    i = golden["tie/inside_0"][:, :, :5, :7] * (golden["tie/bbox_0"] - golden["tie/targets_0"][:, :, :5, :7])
    assert (np.abs(i) == O.RPN_BETA).sum() == 6


def test_library_refuses_bad_arguments_before_any_launch():
    import ctypes
    from detectron.pytorch_b200 import _lib
    from detectron.pytorch_b200 import ops
    lib = _lib.load()
    assert lib.b200_loss_workspace_bytes(0) == 0 and lib.b200_loss_workspace_bytes(9) == 0 and lib.b200_loss_workspace_bytes(5) > 0
    descs = (ops._RpnLossLevel * 1)()
    d = descs[0]
    d.num_images, d.num_anchors, d.cls_channels, d.h, d.w, d.hb, d.wb = 1, 3, 3, 4, 4, 4, 4
    d.label_h, d.label_w, d.target_h, d.target_w = 3, 4, 4, 4                        # labels narrower than the logits
    p = ctypes.cast(descs, ctypes.c_void_p)
    assert lib.b200_rpn_loss_forward(1, p, 0, 0.0, None, 0, None, None, None) == -1
    d.label_h = 4                                                                    # now only the pointers are missing
    assert lib.b200_rpn_loss_forward(1, p, 0, 0.0, None, 0, None, None, None) == -1
    assert lib.b200_rpn_loss_forward(0, p, 0, 0.0, None, 0, None, None, None) == -1
    assert lib.b200_rpn_loss_backward(1, p, 2, None, None, None) == -1
    assert lib.b200_fast_rcnn_loss_forward(0, 81, 324, *[None] * 3, 0, *[None] * 4, 0, None, None, None) == -1
    assert lib.b200_fast_rcnn_loss_forward(4, 81, 322, *[None] * 3, 0, *[None] * 4, 0, None, None, None) == -1
    assert lib.b200_fast_rcnn_loss_backward(4, 81, 324, *[None] * 3, 0, *[None] * 6, None) == -1


@pytest.fixture
def no_launch(monkeypatch):
    """CPU tensors stand in for CUDA ones; reaching an autograd Function (the launch) fails the test."""
    from detectron.pytorch_b200 import ops
    monkeypatch.setattr(ops, "_need_cuda_f32", lambda t, name: None)

    def launched(*a, **k):
        raise AssertionError("reached the launch")
    monkeypatch.setattr(ops.RpnLossFunction, "apply", launched)
    monkeypatch.setattr(ops.FastRcnnLossFunction, "apply", launched)
    return ops


def _rpn_blobs(N=2, A=3, h=5, w=7, Hw=8, Ww=8, softmax=False):
    z = lambda *s: torch.zeros(s)  # noqa: E731
    return [z(N, (2 if softmax else 1) * A, h, w), z(N, 4 * A, h, w), torch.zeros((N, A, Hw, Ww), dtype=torch.int32), z(N, 4 * A, Hw, Ww),
            z(N, 4 * A, Hw, Ww), z(N, 4 * A, Hw, Ww)]


def test_argument_errors_are_raised_before_any_launch(no_launch):
    from detectron.pytorch_b200.modeling import FPN, fast_rcnn_heads, rpn_heads
    ops = no_launch
    with pytest.raises(AssertionError, match="reached the launch"):              # well-formed input gets to the launch
        rpn_heads.single_scale_rpn_losses(*_rpn_blobs())
    bad = _rpn_blobs(); bad[2] = torch.zeros((2, 3, 4, 8), dtype=torch.int32)    # a wide blob smaller than the prediction
    with pytest.raises(ValueError, match="narrowed"):
        rpn_heads.single_scale_rpn_losses(*bad)
    bad = _rpn_blobs(); bad[4] = torch.zeros((2, 12, 8, 7))
    with pytest.raises(ValueError, match="narrowed"):
        rpn_heads.single_scale_rpn_losses(*bad)
    bad = _rpn_blobs(); bad[1] = torch.zeros((2, 8, 5, 7))                       # 4A channels
    with pytest.raises(ValueError, match="does not match"):
        rpn_heads.single_scale_rpn_losses(*bad)
    with pytest.raises(ValueError, match="2A channels"):
        rpn_heads.single_scale_rpn_losses(*_rpn_blobs(A=3), cls_activation="softmax")
    with pytest.raises(ValueError, match="CLS_ACTIVATION"):
        rpn_heads.single_scale_rpn_losses(*_rpn_blobs(), cls_activation="relu")
    with pytest.raises(TypeError, match="unknown"):
        rpn_heads.single_scale_rpn_losses(*_rpn_blobs(), beta=1.0)
    with pytest.raises(ValueError, match="missing"):
        FPN.fpn_rpn_losses(rpn_min_level=2, rpn_max_level=3, **{k + "_fpn2": v for k, v in zip(
            ("rpn_cls_logits", "rpn_bbox_pred", "rpn_labels_int32_wide", "rpn_bbox_targets_wide", "rpn_bbox_inside_weights_wide",
             "rpn_bbox_outside_weights_wide"), _rpn_blobs())})
    with pytest.raises(ValueError, match="1 .. 8 levels"):
        ops.rpn_losses([tuple(_rpn_blobs())] * 9)
    R, C = 6, 5
    good = [torch.zeros(R, C), torch.zeros(R, 4 * C), np.arange(R, dtype=np.int32) % C] + [np.zeros((R, 4 * C), np.float32)] * 3
    with pytest.raises(AssertionError, match="reached the launch"):
        fast_rcnn_heads.fast_rcnn_losses(*good)
    for k, v, msg in ((2, np.asarray([0, 1, 2, 3, 4, 5], np.int32), "must lie in"), (2, np.asarray([0, -1, 2, 3, 4, 0]), "must lie in"),
                      (2, np.zeros(5, np.int32), "5 entries"), (2, np.zeros(R, np.float32), "int32 or int64"),
                      (1, torch.zeros(R, 4 * C + 2), "4 C'"), (1, torch.zeros(R + 1, 4 * C), "4 C'"), (3, np.zeros((R, 4), np.float32), "does not match"),
                      (0, torch.zeros(0, C), "4 C'")):
        args = list(good); args[k] = v
        with pytest.raises(ValueError, match=msg):
            fast_rcnn_heads.fast_rcnn_losses(*args)


def test_cpu_tensors_are_refused():
    from detectron.pytorch_b200.modeling import fast_rcnn_heads, rpn_heads
    with pytest.raises(NotImplementedError):
        rpn_heads.single_scale_rpn_losses(*_rpn_blobs())
    with pytest.raises(NotImplementedError):
        fast_rcnn_heads.fast_rcnn_losses(torch.zeros(2, 3), torch.zeros(2, 12), np.zeros(2, np.int32), *[np.zeros((2, 12), np.float32)] * 3)


def test_install_reference_aliases_repoints_the_losses(monkeypatch):
    import detectron.pytorch_b200 as pkg
    from detectron.pytorch_b200.modeling import FPN, fast_rcnn_heads, keypoint_rcnn_heads, mask_rcnn_heads, rpn_heads
    calls = []
    rec = lambda name: (lambda *a, **k: calls.append((name, a, k)) or name)  # noqa: E731
    monkeypatch.setattr(rpn_heads, "single_scale_rpn_losses", rec("rpn"))
    monkeypatch.setattr(FPN, "fpn_rpn_losses", rec("fpn"))
    monkeypatch.setattr(mask_rcnn_heads, "mask_rcnn_losses", rec("mask"))
    monkeypatch.setattr(keypoint_rcnn_heads, "keypoint_losses", rec("kp"))
    parent = types.ModuleType("modeling")
    monkeypatch.setitem(sys.modules, "modeling", parent)
    refs = {}
    for name in ("fast_rcnn_heads", "rpn_heads", "FPN", "mask_rcnn_heads", "keypoint_rcnn_heads"):
        m = types.ModuleType("modeling." + name)
        m.cfg = "cfg-of-" + name
        refs[name] = m
        monkeypatch.setitem(sys.modules, m.__name__, m)
    installed = pkg.install_reference_aliases(losses=True)
    for name in ("fast_rcnn_heads.fast_rcnn_losses", "rpn_heads.single_scale_rpn_losses", "FPN.fpn_rpn_losses",
                 "mask_rcnn_heads.mask_rcnn_losses", "keypoint_rcnn_heads.keypoint_losses"):
        assert "modeling." + name in installed
    assert refs["fast_rcnn_heads"].fast_rcnn_losses is fast_rcnn_heads.fast_rcnn_losses
    refs["rpn_heads"].cfg = "cfg-changed-later"                                   # read at call time
    assert refs["rpn_heads"].single_scale_rpn_losses(1, 2, 3, 4, 5, 6) == "rpn"
    assert calls[-1] == ("rpn", (1, 2, 3, 4, 5, 6), {"cfg": "cfg-changed-later"})
    assert refs["FPN"].fpn_rpn_losses(rpn_cls_logits_fpn2=1) == "fpn"
    assert calls[-1] == ("fpn", (), {"cfg": "cfg-of-FPN", "rpn_cls_logits_fpn2": 1})
    assert refs["mask_rcnn_heads"].mask_rcnn_losses("pred", "m") == "mask"
    assert calls[-1] == ("mask", ("pred", "m"), {"cfg": "cfg-of-mask_rcnn_heads"})
    assert refs["keypoint_rcnn_heads"].keypoint_losses("k", "l", "w", "n") == "kp"
    assert calls[-1] == ("kp", ("k", "l", "w", "n"), {"cfg": "cfg-of-keypoint_rcnn_heads"})
    assert refs["keypoint_rcnn_heads"].keypoint_losses("k", "l", "w") == "kp" and calls[-1][1][3] is None


# ---- GPU -------------------------------------------------------------------------------------------------------------------
def _cuda(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _device_rpn(levels, softmax, divisor, gcoef):
    from detectron.pytorch_b200 import ops
    preds = [(_cuda(lv[0]).requires_grad_(True), _cuda(lv[1]).requires_grad_(True)) for lv in levels]
    losses = ops.rpn_losses([(c, b) + tuple(_cuda(x) for x in lv[2:]) for (c, b), lv in zip(preds, levels)], softmax, divisor)
    (losses * torch.as_tensor(gcoef, dtype=torch.float32, device="cuda")).sum().backward()
    return losses.detach().cpu().numpy(), [(c.grad.cpu().numpy(), b.grad.cpu().numpy()) for c, b in preds]


def _device_frcn(args, gcoef, label_dtype=None):
    from detectron.pytorch_b200.modeling import fast_rcnn_heads
    cs, bp = _cuda(args[0]).requires_grad_(True), _cuda(args[1]).requires_grad_(True)
    lab = _cuda(args[2]) if label_dtype is None else _cuda(args[2]).to(label_dtype)
    lc, lb, acc = fast_rcnn_heads.fast_rcnn_losses(cs, bp, lab, *[_cuda(x) for x in args[3:]])
    assert lc.shape == () and lb.shape == () and acc.shape == () and not acc.requires_grad
    (float(gcoef[0]) * lc + float(gcoef[1]) * lb).backward()
    return np.asarray([lc.item(), lb.item(), acc.item()], np.float32), cs.grad.cpu().numpy(), bp.grad.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("case", RPN_CASES)
def test_device_rpn_matches_golden(golden, case):
    levels, softmax, fpn, divisor = _rpn_case(golden, case)
    losses, grads = _device_rpn(levels, softmax, divisor, golden[case + "/gcoef"])
    _close(losses, golden[case + "/losses"], case + " losses")
    for l, (dc, db) in enumerate(grads):
        _close(dc, golden["%s/d_cls_%d" % (case, l)], "%s d_cls level %d" % (case, l), grad=True)
        _close(db, golden["%s/d_bbox_%d" % (case, l)], "%s d_bbox level %d" % (case, l), grad=True)


@pytest.mark.gpu
@pytest.mark.parametrize("case", FRCN_CASES)
@pytest.mark.parametrize("label_dtype", [None, torch.int64])
def test_device_fast_rcnn_matches_golden(golden, case, label_dtype):
    out, d_cls, d_bbox = _device_frcn(_frcn_case(golden, case), golden[case + "/gcoef"], label_dtype)
    _close(out[:2], golden[case + "/losses"][:2], case + " losses")
    assert out[2] == golden[case + "/losses"][2]
    _close(d_cls, golden[case + "/d_cls"], case + " d_cls", grad=True)
    _close(d_bbox, golden[case + "/d_bbox"], case + " d_bbox", grad=True)


@pytest.mark.gpu
def test_device_reference_names_match_golden(golden):
    """The reference-shaped front doors: fpn_rpn_losses / generic_rpn_losses with cfg-like keywords, per-level 0-d losses."""
    from detectron.pytorch_b200.modeling import FPN, rpn_heads
    levels, softmax, _, _ = _rpn_case(golden, "fpn_softmax")
    kw = {}
    for l, lv in enumerate(levels):
        s = str(2 + l)
        for k, x in zip(("rpn_cls_logits", "rpn_bbox_pred", "rpn_labels_int32_wide", "rpn_bbox_targets_wide",
                         "rpn_bbox_inside_weights_wide", "rpn_bbox_outside_weights_wide"), lv):
            kw[k + "_fpn" + s] = _cuda(x)
    lc, lb = rpn_heads.generic_rpn_losses(fpn_on=True, cls_activation="softmax", **kw)
    assert len(lc) == len(lb) == 5 and all(t.shape == () for t in lc + lb)
    _close(np.stack([[c.item(), b.item()] for c, b in zip(lc, lb)]), golden["fpn_softmax/losses"], "fpn_softmax via generic")
    levels, _, _, _ = _rpn_case(golden, "fpn_sigmoid")
    kw = {"rpn_%s_fpn%d" % (k, 2 + l): _cuda(x) for l, lv in enumerate(levels)
          for k, x in zip(("cls_logits", "bbox_pred", "labels_int32_wide", "bbox_targets_wide", "bbox_inside_weights_wide",
                           "bbox_outside_weights_wide"), lv)}
    lc, lb = FPN.fpn_rpn_losses(rpn_batch_size_per_im=16, ims_per_batch=2, **kw)
    _close(np.stack([[c.item(), b.item()] for c, b in zip(lc, lb)]), golden["fpn_sigmoid/losses"], "fpn_sigmoid via FPN")


# ---- GPU at full size ------------------------------------------------------------------------------------------------------
def _fpn_step(softmax, seed=0, N=2, H=800, W=1344, max_size=1333):
    """Predictions for an N-image FPN P2-P6 step (A = 3) and the wide blobs of roi_data.rpn.rpn_targets on random ground truth."""
    from detectron.pytorch_b200.roi_data import rpn as R
    rng = np.random.RandomState(seed)
    gts = []
    for _ in range(N):
        G = rng.randint(3, 30)
        xy = rng.uniform(0, [W - 200, H - 200], (G, 2))
        wh = rng.uniform(16, 400, (G, 2))
        gts.append(torch.from_numpy(np.hstack([xy, np.minimum(xy + wh, [W - 1, H - 1])]).astype(np.float32)).cuda())
    blobs = R.rpn_targets(gts, np.tile([[H, W, 1.0]], (N, 1)), multilevel_rpn=True, max_size=max_size)
    levels = []
    for lvl in range(2, 7):
        h, w = math.ceil(H / 2 ** lvl), math.ceil(W / 2 ** lvl)
        g = torch.Generator(device="cuda").manual_seed(seed * 10 + lvl)
        cls = torch.randn((N, (6 if softmax else 3), h, w), device="cuda", generator=g) * 3
        bbox = torch.randn((N, 12, h, w), device="cuda", generator=g) * 0.2
        levels.append((cls, bbox) + tuple(blobs[k + "_fpn%d" % lvl] for k in R._NAMES))
    return levels


def _c4_step(softmax, seed=1, N=2, H=800, W=1344):
    """The single-scale RPN at stride 16 with A = 15 (RPN.SIZES 32 .. 512, three aspect ratios)."""
    from detectron.pytorch_b200.roi_data import rpn as R
    rng = np.random.RandomState(seed)
    gts = []
    for _ in range(N):
        G = rng.randint(3, 30)
        xy = rng.uniform(0, [W - 200, H - 200], (G, 2))
        gts.append(torch.from_numpy(np.hstack([xy, xy + rng.uniform(16, 400, (G, 2))]).astype(np.float32)).cuda())
    blobs = R.rpn_targets(gts, np.tile([[H, W, 1.0]], (N, 1)), max_size=1333, rpn_sizes=(32, 64, 128, 256, 512))
    h, w = math.ceil(H / 16), math.ceil(W / 16)
    g = torch.Generator(device="cuda").manual_seed(seed)
    cls = torch.randn((N, 30 if softmax else 15, h, w), device="cuda", generator=g) * 3
    bbox = torch.randn((N, 60, h, w), device="cuda", generator=g) * 0.2
    return [(cls, bbox) + tuple(blobs[k] for k in R._NAMES)]


def _terms_abs_sum(levels, softmax, l):
    """sum |term| of level l's cls and box sums (all terms are nonnegative, so these are the oracle's sums), the numbers of terms
    and the count of labels that are not ignored."""
    x, bp, lab, tg, wi, wo = levels[l]
    h, w = x.shape[2:]
    total, count, _ = (O.rpn_softmax_cls if softmax else O.rpn_sigmoid_cls)(x, lab[:, :, :h, :w])
    box, _ = O.smooth_l1(bp, tg[:, :, :h, :w], wi[:, :, :h, :w], wo[:, :, :h, :w], O.RPN_BETA)
    return total, x.size // (2 if softmax else 1), float(count), box * bp.shape[0], bp.size


def _check_grad(dev, oracle, scale, what):
    o32 = oracle.astype(np.float32)
    ulp = np.spacing(np.abs(o32)).astype(np.float64)
    tol = GRAD_ULPS * ulp + GRAD_ULPS * EPS32 * scale
    err = np.abs(dev.astype(np.float64) - o32.astype(np.float64))
    assert np.array_equal(np.isnan(dev), np.isnan(oracle)), what + ": NaN positions differ"
    fin = ~np.isnan(oracle)
    assert (err[fin] <= tol[fin]).all(), "%s: max error %.3g at tolerance %.3g" % (what, err[fin].max(), tol[fin][np.argmax(err[fin] - tol[fin])])


def _check_full(levels, softmax, divisor):
    from detectron.pytorch_b200 import ops
    L = len(levels)
    gcoef = np.stack([1.0 + 0.25 * np.arange(L), 0.5 + 0.125 * np.arange(L)], axis=1).astype(np.float32)
    preds = [(c.detach().clone().requires_grad_(True), b.detach().clone().requires_grad_(True)) for c, b, *_ in levels]
    losses = ops.rpn_losses([p + tuple(lv[2:]) for p, lv in zip(preds, levels)], softmax, divisor)
    (losses * torch.from_numpy(gcoef).cuda()).sum().backward()
    host = [tuple(t.cpu().numpy() for t in lv) for lv in levels]
    ref, grads = O.rpn_losses(host, softmax, divisor, grad_coef=gcoef)
    dev = losses.detach().cpu().numpy()
    for l in range(L):
        cls_sum, n_cls, count, box_sum, n_box = _terms_abs_sum(host, softmax, l)
        div_cls = divisor if (divisor > 0 and not softmax) else max(count, 1.0)
        for k, (s, n, d) in enumerate(((cls_sum, n_cls, div_cls), (box_sum, n_box, float(host[l][1].shape[0])))):
            if np.isnan(ref[l, k]):                              # softmax at a level without a label: 0 / 0 as in the reference
                assert np.isnan(dev[l, k]), "level %d loss %d: %r, the oracle's is NaN" % (l, k, dev[l, k])
                continue
            bound = (ELEM_ULPS + math.log2(n)) * EPS32 * s / d + EPS32 * abs(ref[l, k])
            assert abs(dev[l, k] - ref[l, k]) <= bound, "level %d loss %d: %r vs %r (bound %.3g)" % (l, k, dev[l, k], ref[l, k], bound)
        gscale_cls = abs(gcoef[l, 0]) / div_cls
        _check_grad(preds[l][0].grad.cpu().numpy(), grads[l][0], gscale_cls, "level %d d_cls" % l)
        _check_grad(preds[l][1].grad.cpu().numpy(), grads[l][1], abs(gcoef[l, 1]) / host[l][1].shape[0], "level %d d_bbox" % l)
    return losses.detach(), [(c.grad, b.grad) for c, b in preds]


@pytest.mark.gpu
@pytest.mark.parametrize("softmax", [False, True])
def test_full_size_fpn_step_matches_oracle(softmax):
    _check_full(_fpn_step(softmax), softmax, 0.0 if softmax else 256.0 * 2)


@pytest.mark.gpu
@pytest.mark.parametrize("softmax", [False, True])
def test_full_size_c4_step_matches_oracle(softmax):
    _check_full(_c4_step(softmax), softmax, 0.0)


def _box_head(agnostic, seed=3, num_classes=81):
    from detectron.pytorch_b200.roi_data import fast_rcnn as FR
    rng = np.random.RandomState(seed)
    per = []
    for i in range(2):
        G = rng.randint(5, 20)
        xy = rng.uniform(0, 900, (G, 2))
        gt = np.hstack([xy, xy + rng.uniform(20, 300, (G, 2))]).astype(np.float32)
        src = rng.randint(0, G, 2000)
        wh = gt[src, 2:] - gt[src, :2]
        props = gt[src] + rng.standard_normal((2000, 4)).astype(np.float32) * np.hstack([wh, wh]) * 0.3
        props[:, 2:] = np.maximum(props[:, 2:], props[:, :2] + 1)
        boxes = torch.from_numpy(np.vstack([gt, props]).astype(np.float32)).cuda()
        per.append(FR.sample_rois(boxes, torch.from_numpy(gt).cuda(), torch.from_numpy(rng.randint(1, num_classes, G).astype(np.int32)).cuda(),
                                  1.0, i, num_classes, cls_agnostic_bbox_reg=agnostic))
    blobs = {k: torch.cat([b[k] for b in per]) for k in ("labels_int32", "bbox_targets", "bbox_inside_weights", "bbox_outside_weights")}
    R = blobs["labels_int32"].numel()
    g = torch.Generator(device="cuda").manual_seed(seed)
    cls = torch.randn((R, num_classes), device="cuda", generator=g)
    bbox = torch.randn((R, blobs["bbox_targets"].shape[1]), device="cuda", generator=g) * 0.5
    return cls, bbox, blobs


@pytest.mark.gpu
@pytest.mark.parametrize("agnostic", [False, True])
def test_box_head_on_sampled_rois_matches_oracle(agnostic):
    from detectron.pytorch_b200.modeling import fast_rcnn_heads
    cls, bbox, b = _box_head(agnostic)
    assert cls.shape == (1024, 81) and bbox.shape[1] == (8 if agnostic else 324)
    cs, bp = cls.clone().requires_grad_(True), bbox.clone().requires_grad_(True)
    lc, lb, acc = fast_rcnn_heads.fast_rcnn_losses(cs, bp, b["labels_int32"], b["bbox_targets"], b["bbox_inside_weights"],
                                                   b["bbox_outside_weights"])
    (0.75 * lc + 1.5 * lb).backward()
    host = [t.cpu().numpy() for t in (cls, bbox, b["labels_int32"], b["bbox_targets"], b["bbox_inside_weights"], b["bbox_outside_weights"])]
    rc, rb, racc, rdc, rdb = O.fast_rcnn_losses(*host, grad_coef=(0.75, 1.5))
    R = host[0].shape[0]
    x = host[0].astype(np.float64)
    ce_terms = -(x - x.max(1, keepdims=True) - np.log(np.exp(x - x.max(1, keepdims=True)).sum(1, keepdims=True)))[np.arange(R), host[2]]
    box_terms, _ = O.smooth_l1(*host[1:2], *host[3:], 1.0)
    for dev, ref, s, n in ((lc.item(), rc, ce_terms.sum(), R), (lb.item(), rb, box_terms * R, host[1].size)):
        assert abs(dev - ref) <= (ELEM_ULPS + math.log2(n)) * EPS32 * s / R + EPS32 * abs(ref), (dev, ref)
    assert acc.item() == np.float32(racc)
    _check_grad(cs.grad.cpu().numpy(), rdc, 0.75 / R, "d cls_score")
    _check_grad(bp.grad.cpu().numpy(), rdb, 1.5 / R, "d bbox_pred")


@pytest.mark.gpu
def test_two_calls_are_bit_identical():
    from detectron.pytorch_b200.modeling import fast_rcnn_heads
    levels = _fpn_step(False, seed=5)
    a = _check_full(levels, False, 512.0)
    b = _check_full(levels, False, 512.0)
    assert torch.equal(a[0], b[0])
    for (c1, b1), (c2, b2) in zip(a[1], b[1]):
        assert torch.equal(c1, c2) and torch.equal(b1, b2)
    cls, bbox, blobs = _box_head(False, seed=6)
    outs = []
    for _ in range(2):
        cs, bp = cls.clone().requires_grad_(True), bbox.clone().requires_grad_(True)
        lc, lb, acc = fast_rcnn_heads.fast_rcnn_losses(cs, bp, blobs["labels_int32"], blobs["bbox_targets"], blobs["bbox_inside_weights"],
                                                       blobs["bbox_outside_weights"])
        (lc + lb).backward()
        outs.append(torch.stack([lc, lb, acc]).detach().cpu().numpy().tobytes() + cs.grad.cpu().numpy().tobytes() + bp.grad.cpu().numpy().tobytes())
    assert outs[0] == outs[1]


@pytest.mark.gpu
def test_forward_and_backward_make_no_host_sync():
    from detectron.pytorch_b200.modeling import FPN, fast_rcnn_heads
    levels = _fpn_step(True, seed=7, H=320, W=480, max_size=480)
    cls, bbox, b = _box_head(True, seed=8)
    kw = {}
    preds = []
    for l, lv in enumerate(levels):
        c, bp = lv[0].clone().requires_grad_(True), lv[1].clone().requires_grad_(True)
        preds += [c, bp]
        for k, x in zip(("rpn_cls_logits", "rpn_bbox_pred", "rpn_labels_int32_wide", "rpn_bbox_targets_wide", "rpn_bbox_inside_weights_wide",
                         "rpn_bbox_outside_weights_wide"), (c, bp) + tuple(lv[2:])):
            kw["%s_fpn%d" % (k, 2 + l)] = x
    cs, bp = cls.clone().requires_grad_(True), bbox.clone().requires_grad_(True)
    for _ in range(2):                                     # the second pass runs with the workspaces already allocated
        torch.cuda.set_sync_debug_mode("error")
        try:
            lc, lb = FPN.fpn_rpn_losses(cls_activation="softmax", **kw)
            c_loss, b_loss, acc = fast_rcnn_heads.fast_rcnn_losses(cs, bp, b["labels_int32"], b["bbox_targets"], b["bbox_inside_weights"],
                                                                   b["bbox_outside_weights"])
            total = sum(x.unsqueeze(0) for x in lc + lb) + c_loss + b_loss
            total.sum().backward()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert all(torch.isfinite(p.grad).all() for p in preds + [cs, bp])


@pytest.mark.gpu
def test_out_of_range_device_label_gives_nan_loss_cls():
    from detectron.pytorch_b200.modeling import fast_rcnn_heads
    cls, bbox, b = _box_head(False, seed=9)
    for bad in (81, -1, 1 << 20):
        labels = b["labels_int32"].clone()
        labels[5] = bad
        lc, lb, acc = fast_rcnn_heads.fast_rcnn_losses(cls, bbox, labels, b["bbox_targets"], b["bbox_inside_weights"], b["bbox_outside_weights"])
        assert math.isnan(lc.item()) and math.isfinite(lb.item()) and math.isfinite(acc.item())
    labels = b["labels_int32"].long().clone()
    labels[0] = 1 << 40
    lc, lb, acc = fast_rcnn_heads.fast_rcnn_losses(cls, bbox, labels, b["bbox_targets"], b["bbox_inside_weights"], b["bbox_outside_weights"])
    assert math.isnan(lc.item()) and math.isfinite(lb.item()) and math.isfinite(acc.item())


@pytest.mark.gpu
def test_chained_training_targets_to_backward_stay_on_device():
    """add_rpn_blobs -> fpn_rpn_losses and the collect training branch -> fast_rcnn_losses -> backward(): every target is a CUDA
    tensor straight from the device loaders, and the losses equal the oracle's."""
    from detectron.pytorch_b200.modeling import FPN, fast_rcnn_heads
    from detectron.pytorch_b200.modeling.collect_and_distribute_fpn_rpn_proposals import CollectAndDistributeFpnRpnProposalsOp
    from detectron.pytorch_b200.roi_data import rpn as R
    rng = np.random.RandomState(11)
    H, W, N, C = 384, 576, 2, 81
    roidb = []
    for _ in range(N):
        G = rng.randint(4, 12)
        xy = rng.uniform(0, [W - 120, H - 120], (G, 2))
        roidb.append(dict(height=H, width=W, boxes=np.hstack([xy, xy + rng.uniform(16, 110, (G, 2))]).astype(np.float32),
                          gt_classes=rng.randint(1, C, G).astype(np.int32), is_crowd=np.zeros(G, bool), seg_areas=np.ones(G, np.float32)))
    blobs = {}
    R.add_rpn_blobs(blobs, [1.0] * N, roidb, multilevel_rpn=True, max_size=W)
    kw, preds = {}, []
    for lvl in range(2, 7):
        h, w = math.ceil(H / 2 ** lvl), math.ceil(W / 2 ** lvl)
        c = (torch.randn((N, 3, h, w), device="cuda") * 2).requires_grad_(True)
        b = (torch.randn((N, 12, h, w), device="cuda") * 0.2).requires_grad_(True)
        preds.append((c, b))
        kw["rpn_cls_logits_fpn%d" % lvl], kw["rpn_bbox_pred_fpn%d" % lvl] = c, b
        for k in R._NAMES:
            t = blobs[k + "_fpn%d" % lvl]
            assert t.is_cuda
            kw[k + "_fpn%d" % lvl] = t
    lc, lb = FPN.fpn_rpn_losses(**kw)
    rois, scores = [], []
    for lvl in range(2, 7):
        n = 200
        i = rng.randint(0, N, n)
        xy = rng.uniform(0, [W - 100, H - 100], (n, 2))
        rois.append(torch.from_numpy(np.hstack([i[:, None], xy, xy + rng.uniform(8, 100, (n, 2))]).astype(np.float32)).cuda())
        scores.append(torch.rand((n, 1), device="cuda"))
    op = CollectAndDistributeFpnRpnProposalsOp(post_nms_topN=2000).train()
    train = dict(BATCH_SIZE_PER_IM=512, FG_FRACTION=0.25, FG_THRESH=0.5, BG_THRESH_HI=0.5, BG_THRESH_LO=0.0, NUM_CLASSES=C,
                 BBOX_REG_WEIGHTS=(10.0, 10.0, 5.0, 5.0), CLS_AGNOSTIC_BBOX_REG=False)
    out = op(rois + scores, roidb, np.asarray([[H, W, 1.0]] * N, np.float32), train=train)
    for k in ("labels_int32", "bbox_targets", "bbox_inside_weights", "bbox_outside_weights"):
        assert out[k].is_cuda
    Rn = out["labels_int32"].numel()
    cs = torch.randn((Rn, C), device="cuda").requires_grad_(True)
    bp = (torch.randn((Rn, 4 * C), device="cuda") * 0.3).requires_grad_(True)
    c_loss, b_loss, acc = fast_rcnn_heads.fast_rcnn_losses(cs, bp, out["labels_int32"], out["bbox_targets"], out["bbox_inside_weights"],
                                                           out["bbox_outside_weights"])
    total = sum(x.unsqueeze(0) for x in lc + lb) + c_loss + b_loss
    total.sum().backward()
    assert all(torch.isfinite(t.grad).all() for p in preds for t in p) and torch.isfinite(cs.grad).all() and torch.isfinite(bp.grad).all()
    host = [(c.detach().cpu().numpy(), b.detach().cpu().numpy()) + tuple(blobs[k + "_fpn%d" % (2 + l)].cpu().numpy() for k in R._NAMES)
            for l, (c, b) in enumerate(preds)]
    ref, _ = O.rpn_losses(host, False, 512.0)
    np.testing.assert_allclose(np.asarray([[c.item(), b.item()] for c, b in zip(lc, lb)]), ref, rtol=1e-5, atol=1e-7)
    rc, rb, racc, _, _ = O.fast_rcnn_losses(*[t.detach().cpu().numpy() for t in (cs, bp, out["labels_int32"], out["bbox_targets"],
                                                                                  out["bbox_inside_weights"], out["bbox_outside_weights"])])
    np.testing.assert_allclose([c_loss.item(), b_loss.item()], [rc, rb], rtol=1e-5, atol=1e-7)
    assert acc.item() == np.float32(racc)
