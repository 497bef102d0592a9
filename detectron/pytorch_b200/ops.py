"""torch.autograd.Function front-ends over the C ABI (new-style, static) + functional helpers.

These are what the reference-shaped shims in `model/` and `modeling/` delegate to.  Every op
  * requires CUDA fp32 tensors (the reference raises NotImplementedError / asserts for CPU input),
  * makes its inputs contiguous (the reference passed raw pointers and silently assumed it),
  * launches on torch's current stream of the tensor's device,
  * allocates outputs with torch.empty (the kernels define every output element; the reference
    needed `.zero_()` passes, functions/roi_align.py:23,39-40).
"""
import ctypes

import numpy as np
import torch
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from . import _lib


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _need_cuda_f32(t, name):
    if not t.is_cuda:
        raise NotImplementedError("%s must be a CUDA tensor (the reference has no CPU path for this op)" % name)
    if t.dtype != torch.float32:
        raise TypeError("%s must be float32, got %s" % (name, t.dtype))


def _rois_ok(rois):
    if rois.dim() != 2 or rois.size(1) != 5:
        raise ValueError("rois must be (R, 5) = [batch_idx, x1, y1, x2, y2], got %s" % (tuple(rois.shape),))


# ------------------------------------------------------------------------------------------------
# RoIAlign (Caffe2-exact, sampling_ratio)
# ------------------------------------------------------------------------------------------------
def roi_align_forward(features, rois, aligned_height, aligned_width, spatial_scale, sampling_ratio):
    _need_cuda_f32(features, "features"); _need_cuda_f32(rois, "rois"); _rois_ok(rois)
    features = features.contiguous(); rois = rois.contiguous()
    N, C, H, W = features.shape
    R = rois.size(0)
    out = torch.empty((R, C, aligned_height, aligned_width), dtype=torch.float32, device=features.device)
    lib = _lib.load()
    ws_bytes = int(lib.b200_roi_align_workspace_bytes(N, R, H, W, aligned_height, aligned_width, sampling_ratio))
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=features.device) if ws_bytes else None   # caching allocator, stream-ordered
    with torch.cuda.device(features.device):
        _lib.check(lib.b200_roi_align_forward_ws(features.data_ptr(), spatial_scale, N, R, H, W, C, aligned_height,
                                                 aligned_width, sampling_ratio, rois.data_ptr(), out.data_ptr(),
                                                 ws.data_ptr() if ws is not None else None, ws_bytes, _stream()),
                   "b200_roi_align_forward_ws")
    return out


def roi_align_backward(grad_output, rois, feature_size, aligned_height, aligned_width, spatial_scale, sampling_ratio):
    _need_cuda_f32(grad_output, "grad_output")
    grad_output = grad_output.contiguous(); rois = rois.contiguous()
    N, C, H, W = feature_size
    grad_input = torch.empty((N, C, H, W), dtype=torch.float32, device=grad_output.device)
    lib = _lib.load()
    ws_bytes = int(lib.b200_roi_align_backward_workspace_bytes(N, rois.size(0), C, H, W, aligned_height, aligned_width,
                                                              sampling_ratio)) if rois.size(0) > 0 else 0
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=grad_output.device) if ws_bytes else None
    with torch.cuda.device(grad_output.device):
        _lib.check(lib.b200_roi_align_backward_ws(grad_output.data_ptr(), spatial_scale, N, rois.size(0), H, W, C,
                                                  aligned_height, aligned_width, sampling_ratio, rois.data_ptr(),
                                                  grad_input.data_ptr(), ws.data_ptr() if ws is not None else None,
                                                  ws_bytes, _stream()),
                   "b200_roi_align_backward_ws")
    return grad_input


class _RoIAlign(Function):
    @staticmethod
    def forward(ctx, features, rois, aligned_height, aligned_width, spatial_scale, sampling_ratio):
        ctx.args = (int(aligned_height), int(aligned_width), float(spatial_scale), int(sampling_ratio))
        ctx.feature_size = tuple(features.shape)
        ctx.save_for_backward(rois)
        return roi_align_forward(features, rois, *ctx.args)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        (rois,) = ctx.saved_tensors
        assert grad_output.is_cuda
        return roi_align_backward(grad_output, rois, ctx.feature_size, *ctx.args), None, None, None, None, None


# ------------------------------------------------------------------------------------------------
# RoIAlign over an FPN pyramid, results written in restored order (SURVEY.md 8f N2)
# ------------------------------------------------------------------------------------------------
class _RoIAlignFPN(Function):
    """One autograd node for the reference's per-level loop + torch.cat + `xform_shuffled[restore_bl]`
    (lib/modeling/model_builder.py:264-303): level l's RoI r is row offset_l + r of the concatenated tensor, which the
    gather moves to every output row j with restore[j] == offset_l + r.  `restore` is a permutation, so each RoI has
    exactly one destination row, and the per-level kernels write it directly (b200_roi_align_forward_indexed); the
    backward reads the gradient rows of the shared tensor in place (b200_roi_align_backward_indexed)."""

    @staticmethod
    def forward(ctx, restore, aligned_height, aligned_width, sampling_ratio, scales, num_levels, *tensors):
        feats, rois = tensors[:num_levels], tensors[num_levels:]
        P = (int(aligned_height), int(aligned_width)); sr = int(sampling_ratio)
        dev = feats[0].device
        counts = [int(r.size(0)) for r in rois]
        total = sum(counts)
        if restore.numel() != total:
            raise ValueError("restore index has %d entries for %d RoIs" % (restore.numel(), total))
        C = feats[0].size(1)
        if restore.is_cuda:
            inv = torch.empty((total,), dtype=torch.int32, device=dev)
            inv[restore.to(dtype=torch.long)] = torch.arange(total, dtype=torch.int32, device=dev)
        else:                                       # the reference's restore index is a host array: invert it there
            inv_h = torch.empty((total,), dtype=torch.int32)
            inv_h[restore.to(dtype=torch.long)] = torch.arange(total, dtype=torch.int32)
            inv = inv_h.to(dev, non_blocking=False)
        out = torch.empty((total, C, P[0], P[1]), dtype=torch.float32, device=dev)
        lib = _lib.load()
        for f, r in zip(feats, rois):
            _need_cuda_f32(f, "features"); _need_cuda_f32(r, "rois"); _rois_ok(r)
            if f.size(1) != C or f.size(0) != feats[0].size(0):
                raise ValueError("every pyramid level must have the same batch size and number of channels")
        kept = [r.contiguous() for r in rois]
        done = False
        if total > 0:
            # one launch sequence over the whole pyramid: levels without RoIs drop out, the rest go level-major
            import ctypes
            live = [l for l in range(num_levels) if counts[l] > 0]
            fl = [feats[l].contiguous() for l in live]
            Lc = len(live)
            N = int(fl[0].size(0))
            hs = (ctypes.c_int * Lc)(*[int(f.size(2)) for f in fl]); wd = (ctypes.c_int * Lc)(*[int(f.size(3)) for f in fl])
            ws_bytes = int(lib.b200_roi_align_fpn_workspace_bytes(Lc, ctypes.cast(hs, ctypes.c_void_p), ctypes.cast(wd, ctypes.c_void_p), N,
                                                                  total, P[0], P[1], sr))
            if ws_bytes > 0:
                ptrs = (ctypes.c_void_p * Lc)(*[f.data_ptr() for f in fl])
                scs = (ctypes.c_float * Lc)(*[float(scales[l]) for l in live])
                begins, acc = [], 0
                for l in live:
                    begins.append(acc); acc += counts[l]
                begins.append(acc)
                bg = (ctypes.c_int * (Lc + 1))(*begins)
                all_rois = torch.cat([kept[l] for l in live], dim=0) if Lc > 1 else kept[live[0]]
                # inv is indexed by the position in the FULL level-major order; empty levels contribute nothing, so it is the same order
                ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
                with torch.cuda.device(dev):
                    _lib.check(lib.b200_roi_align_forward_fpn(Lc, ctypes.cast(ptrs, ctypes.c_void_p), ctypes.cast(hs, ctypes.c_void_p),
                                                              ctypes.cast(wd, ctypes.c_void_p), ctypes.cast(scs, ctypes.c_void_p),
                                                              ctypes.cast(bg, ctypes.c_void_p), N, total, C, P[0], P[1], sr,
                                                              all_rois.data_ptr(), inv.data_ptr(), out.data_ptr(), ws.data_ptr(), ws_bytes,
                                                              _stream()), "b200_roi_align_forward_fpn")
                done = True
        off = 0
        with torch.cuda.device(dev):
            for f, r, sc, n_l in zip(feats, kept, scales, counts):
                if n_l and not done:
                    f = f.contiguous()
                    N, _, H, W = f.shape
                    ws_bytes = int(lib.b200_roi_align_workspace_bytes(N, n_l, H, W, P[0], P[1], sr))
                    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev) if ws_bytes else None
                    rows = inv[off:off + n_l]
                    _lib.check(lib.b200_roi_align_forward_indexed(f.data_ptr(), float(sc), N, n_l, H, W, C, P[0], P[1], sr,
                                                                  r.data_ptr(), rows.data_ptr(), out.data_ptr(),
                                                                  ws.data_ptr() if ws is not None else None, ws_bytes, _stream()),
                               "b200_roi_align_forward_indexed")
                off += n_l
        ctx.meta = (P, sr, [float(sc) for sc in scales], counts, [tuple(f.shape) for f in feats], num_levels)
        ctx.save_for_backward(inv, *kept)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        P, sr, scales, counts, shapes, num_levels = ctx.meta
        inv, rois = ctx.saved_tensors[0], ctx.saved_tensors[1:]
        assert grad_output.is_cuda
        grad_output = grad_output.contiguous()
        dev = grad_output.device
        lib = _lib.load()
        grads = []
        off = 0
        with torch.cuda.device(dev):
            for r, sc, n_l, shape in zip(rois, scales, counts, shapes):
                N, C, H, W = shape
                if n_l == 0:
                    grads.append(torch.zeros(shape, dtype=torch.float32, device=dev))
                    continue
                g = torch.empty(shape, dtype=torch.float32, device=dev)
                ws_bytes = int(lib.b200_roi_align_backward_workspace_bytes(N, n_l, C, H, W, P[0], P[1], sr))
                ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev) if ws_bytes else None
                rows = inv[off:off + n_l]
                _lib.check(lib.b200_roi_align_backward_indexed(grad_output.data_ptr(), rows.data_ptr(), sc, N, n_l, H, W, C,
                                                               P[0], P[1], sr, r.data_ptr(), g.data_ptr(),
                                                               ws.data_ptr() if ws is not None else None, ws_bytes, _stream()),
                           "b200_roi_align_backward_indexed")
                grads.append(g)
                off += n_l
        return (None, None, None, None, None, None) + tuple(grads) + (None,) * num_levels


def roi_align_fpn(features, rois, restore, aligned_height, aligned_width, spatial_scales, sampling_ratio):
    """features: list of (N, C, H_l, W_l) CUDA tensors; rois: list of (R_l, 5) CUDA tensors (same order); restore: the
    reference's `*_idx_restore_int32` (any integer tensor / array of length sum R_l); spatial_scales: one per level.
    Returns (sum R_l, C, PH, PW) in restored order == torch.cat([RoIAlign_l(...)])[restore]."""
    if len(features) != len(rois) or len(features) != len(spatial_scales):
        raise ValueError("features, rois and spatial_scales must have one entry per pyramid level")
    restore = torch.as_tensor(restore)
    return _RoIAlignFPN.apply(restore, aligned_height, aligned_width, sampling_ratio, tuple(spatial_scales), len(features),
                              *features, *rois)


# ------------------------------------------------------------------------------------------------
# RoIAlign (legacy, lattice-corner samples)
# ------------------------------------------------------------------------------------------------
def roi_align_legacy_forward(features, rois, aligned_height, aligned_width, spatial_scale):
    _need_cuda_f32(features, "features"); _need_cuda_f32(rois, "rois"); _rois_ok(rois)
    features = features.contiguous(); rois = rois.contiguous()
    N, C, H, W = features.shape
    R = rois.size(0)
    out = torch.empty((R, C, aligned_height, aligned_width), dtype=torch.float32, device=features.device)
    with torch.cuda.device(features.device):
        _lib.check(_lib.load().b200_roi_align_legacy_forward(features.data_ptr(), spatial_scale, N, R, H, W, C,
                                                             aligned_height, aligned_width, rois.data_ptr(),
                                                             out.data_ptr(), _stream()),
                   "b200_roi_align_legacy_forward")
    return out


def roi_align_legacy_backward(grad_output, rois, feature_size, aligned_height, aligned_width, spatial_scale):
    _need_cuda_f32(grad_output, "grad_output")
    grad_output = grad_output.contiguous(); rois = rois.contiguous()
    N, C, H, W = feature_size
    grad_input = torch.empty((N, C, H, W), dtype=torch.float32, device=grad_output.device)
    with torch.cuda.device(grad_output.device):
        _lib.check(_lib.load().b200_roi_align_legacy_backward(grad_output.data_ptr(), spatial_scale, N, rois.size(0), H, W, C,
                                                              aligned_height, aligned_width, rois.data_ptr(),
                                                              grad_input.data_ptr(), _stream()),
                   "b200_roi_align_legacy_backward")
    return grad_input


class _RoIAlignLegacy(Function):
    @staticmethod
    def forward(ctx, features, rois, aligned_height, aligned_width, spatial_scale):
        ctx.args = (int(aligned_height), int(aligned_width), float(spatial_scale))
        ctx.feature_size = tuple(features.shape)
        ctx.save_for_backward(rois)
        return roi_align_legacy_forward(features, rois, *ctx.args)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        (rois,) = ctx.saved_tensors
        assert grad_output.is_cuda
        return roi_align_legacy_backward(grad_output, rois, ctx.feature_size, *ctx.args), None, None, None, None


# ------------------------------------------------------------------------------------------------
# RoIPool
# ------------------------------------------------------------------------------------------------
def roi_pool_forward(features, rois, pooled_height, pooled_width, spatial_scale):
    _need_cuda_f32(features, "features"); _need_cuda_f32(rois, "rois"); _rois_ok(rois)
    features = features.contiguous(); rois = rois.contiguous()
    N, C, H, W = features.shape
    R = rois.size(0)
    out = torch.empty((R, C, pooled_height, pooled_width), dtype=torch.float32, device=features.device)
    argmax = torch.empty((R, C, pooled_height, pooled_width), dtype=torch.int32, device=features.device)
    with torch.cuda.device(features.device):
        _lib.check(_lib.load().b200_roi_pool_forward(features.data_ptr(), spatial_scale, N, R, H, W, C, pooled_height,
                                                     pooled_width, rois.data_ptr(), out.data_ptr(), argmax.data_ptr(),
                                                     _stream()),
                   "b200_roi_pool_forward")
    return out, argmax


def roi_pool_backward(grad_output, argmax, rois, feature_size, pooled_height, pooled_width, spatial_scale):
    _need_cuda_f32(grad_output, "grad_output")
    grad_output = grad_output.contiguous(); rois = rois.contiguous(); argmax = argmax.contiguous()
    N, C, H, W = feature_size
    grad_input = torch.empty((N, C, H, W), dtype=torch.float32, device=grad_output.device)
    with torch.cuda.device(grad_output.device):
        _lib.check(_lib.load().b200_roi_pool_backward(grad_output.data_ptr(), spatial_scale, N, rois.size(0), H, W, C,
                                                      pooled_height, pooled_width, rois.data_ptr(), grad_input.data_ptr(),
                                                      argmax.data_ptr(), _stream()),
                   "b200_roi_pool_backward")
    return grad_input


class _RoIPool(Function):
    @staticmethod
    def forward(ctx, features, rois, pooled_height, pooled_width, spatial_scale):
        ctx.args = (int(pooled_height), int(pooled_width), float(spatial_scale))
        ctx.feature_size = tuple(features.shape)
        out, argmax = roi_pool_forward(features, rois, *ctx.args)
        ctx.save_for_backward(rois, argmax)
        ctx.mark_non_differentiable(argmax)
        return out, argmax

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output, _grad_argmax):
        rois, argmax = ctx.saved_tensors
        assert grad_output.is_cuda
        return roi_pool_backward(grad_output, argmax, rois, ctx.feature_size, *ctx.args), None, None, None, None


# ------------------------------------------------------------------------------------------------
# RoICrop
# ------------------------------------------------------------------------------------------------
def roi_crop_forward(input1, input2):
    _need_cuda_f32(input1, "input1"); _need_cuda_f32(input2, "input2")
    if input2.dim() != 4 or input2.size(3) != 2:
        raise ValueError("input2 (grid) must be (R, h, w, 2) in (y, x) order, got %s" % (tuple(input2.shape),))
    assert input1.get_device() == input2.get_device(), "input1 and input2 must on the same device"
    input1 = input1.contiguous(); input2 = input2.contiguous()
    N, C, H, W = input1.shape
    R, oh, ow, _ = input2.shape
    out = torch.empty((R, C, oh, ow), dtype=torch.float32, device=input1.device)
    with torch.cuda.device(input1.device):
        _lib.check(_lib.load().b200_roi_crop_forward(input1.data_ptr(), input2.data_ptr(), N, C, H, W, R, oh, ow,
                                                     out.data_ptr(), _stream()),
                   "b200_roi_crop_forward")
    return out


def roi_crop_backward(grad_output, input2, input1_size):
    _need_cuda_f32(grad_output, "grad_output")
    grad_output = grad_output.contiguous(); input2 = input2.contiguous()
    N, C, H, W = input1_size
    R, oh, ow, _ = input2.shape
    grad_input1 = torch.empty((N, C, H, W), dtype=torch.float32, device=grad_output.device)
    grad_input2 = torch.empty_like(input2)
    lib = _lib.load()
    ws_bytes = int(lib.b200_roi_crop_backward_workspace_bytes(N, C, H, W, R, oh, ow))
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=grad_output.device) if ws_bytes else None
    with torch.cuda.device(grad_output.device):
        _lib.check(lib.b200_roi_crop_backward_ws(grad_output.data_ptr(), input2.data_ptr(), N, C, H, W, R, oh, ow,
                                                 grad_input1.data_ptr(), grad_input2.data_ptr(),
                                                 ws.data_ptr() if ws is not None else None, ws_bytes, _stream()),
                   "b200_roi_crop_backward_ws")
    return grad_input1, grad_input2


class _RoICrop(Function):
    @staticmethod
    def forward(ctx, input1, input2):
        ctx.input1_size = tuple(input1.shape)
        ctx.save_for_backward(input2)
        return roi_crop_forward(input1, input2)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        (input2,) = ctx.saved_tensors
        assert grad_output.is_cuda
        return roi_crop_backward(grad_output, input2, ctx.input1_size)


# ------------------------------------------------------------------------------------------------
# NMS
# ------------------------------------------------------------------------------------------------
TOPK_MAX_K = 16384
TOPK_MAX_PROBLEMS = 64


def topk_batched_raw(score_maps, ks):
    """Top-k of several (A, H, W) float32 CUDA score maps in one batched call (b200_topk_batched: radix select + in-CTA sort,
    no host read).  ks: host ints, k_p <= min(A*H*W, 16384); <= 64 problems.  Returns (order int64 (sum k,), scores float32
    (sum k,)): problem p's slice holds, best first, the indices into its (H, W, A) flattening and the scores."""
    import ctypes
    P = len(score_maps)
    if P < 1 or P > TOPK_MAX_PROBLEMS or len(ks) != P:
        raise ValueError("topk_batched_raw: 1..64 problems with one k each")
    maps = []
    for m in score_maps:
        _need_cuda_f32(m, "score map")
        if m.dim() != 3:
            raise ValueError("score maps must be (A, H, W), got %s" % (tuple(m.shape),))
        maps.append(m.contiguous())
    ks = [int(k) for k in ks]
    dev = maps[0].device
    total = sum(ks)
    order = torch.empty((max(total, 1),), dtype=torch.int64, device=dev)
    scores = torch.empty((max(total, 1),), dtype=torch.float32, device=dev)
    lib = _lib.load()
    ptrs = (ctypes.c_void_p * P)(*[m.data_ptr() for m in maps])
    A = (ctypes.c_int * P)(*[m.size(0) for m in maps])
    HW = (ctypes.c_int * P)(*[m.size(1) * m.size(2) for m in maps])
    K = (ctypes.c_int * P)(*ks)
    ws_bytes = int(lib.b200_topk_batched_workspace_bytes(P))
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _lib.check(lib.b200_topk_batched(ctypes.cast(ptrs, ctypes.c_void_p), ctypes.cast(A, ctypes.c_void_p), ctypes.cast(HW, ctypes.c_void_p),
                                         ctypes.cast(K, ctypes.c_void_p), P, order.data_ptr(), scores.data_ptr(), ws.data_ptr(), ws_bytes,
                                         _stream()), "b200_topk_batched")
    return order[:total], scores[:total]


def nms_batched_raw(dets, counts, thresh, cython=False):
    """`len(counts)` independent NMS problems in one pair of launches.  dets: (sum(counts), >=4) rows of the problems back to
    back, each problem score-sorted; counts: host ints.  Returns (keep int32 (sum(counts),), num_out int32 (P,)) on the
    device: problem p's kept indices (relative to its first row) sit at keep[offset_p : offset_p + num_out[p]].
    cython=False: the reference CUDA kernel's IoU test (fused area, IoU > thresh, b200_nms_batched); True: the Cython
    NMS's (separately rounded areas, IoU >= thresh, b200_nms_batched_cython)."""
    import ctypes
    _need_cuda_f32(dets, "dets")
    if dets.dim() != 2 or dets.size(1) < 4:
        raise ValueError("dets must be (N, >=4) = [x1, y1, x2, y2, score], got %s" % (tuple(dets.shape),))
    counts = [int(c) for c in counts]
    if sum(counts) != dets.size(0) or not counts:
        raise ValueError("counts %s do not add up to %d rows" % (counts, dets.size(0)))
    dets = dets.contiguous()
    lib = _lib.load()
    P = len(counts)
    c_arr = (ctypes.c_int * P)(*counts)
    keep = torch.empty((max(dets.size(0), 1),), dtype=torch.int32, device=dets.device)
    num_out = torch.empty((P,), dtype=torch.int32, device=dets.device)
    ws_bytes = int(lib.b200_nms_batched_workspace_bytes(ctypes.cast(c_arr, ctypes.c_void_p), P))
    if ws_bytes == 0:
        raise ValueError("b200_nms_batched: 1..64 problems expected, got %d" % P)
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dets.device)
    with torch.cuda.device(dets.device):
        fn, name = (lib.b200_nms_batched_cython, "b200_nms_batched_cython") if cython else (lib.b200_nms_batched, "b200_nms_batched")
        _lib.check(fn(dets.data_ptr(), ctypes.cast(c_arr, ctypes.c_void_p), P, dets.size(1), float(thresh), keep.data_ptr(), num_out.data_ptr(),
                      ws.data_ptr(), ws_bytes, _stream()), name)
    return keep, num_out


def nms_batched_chunked(dets, counts, thresh, cython=False):
    """nms_batched_raw for any number of problems (b200_nms_batched takes up to 64 per call): same return layout."""
    counts = [int(c) for c in counts]
    if len(counts) <= 64:
        return nms_batched_raw(dets, counts, thresh, cython)
    keeps, nums, off = [], [], 0
    for c0 in range(0, len(counts), 64):
        chunk = counts[c0:c0 + 64]
        n = sum(chunk)
        if n == 0:
            keeps.append(torch.empty((0,), dtype=torch.int32, device=dets.device))
            nums.append(torch.zeros((len(chunk),), dtype=torch.int32, device=dets.device))
        else:
            k, m = nms_batched_raw(dets[off:off + n], chunk, thresh, cython)
            keeps.append(k[:n]); nums.append(m)
        off += n
    return torch.cat(keeps), torch.cat(nums)


def soft_nms_batched(dets, counts, sigma=0.5, overlap_thresh=0.3, score_thresh=0.001, method=1):
    """Soft-NMS (lib/utils/cython_nms.pyx:98-203) on `len(counts)` problems stored back to back in dets (sum(counts), 5).
    Returns (dets_out, inds, num_out): problem p's survivors are dets_out[off_p : off_p + num_out[p]] (decayed scores, the
    reference's output order), inds their original row indices within the problem."""
    import ctypes
    _need_cuda_f32(dets, "dets")
    counts = [int(c) for c in counts]
    if dets.dim() != 2 or dets.size(1) != 5 or sum(counts) != dets.size(0):
        raise ValueError("dets must be (sum(counts), 5)")
    lib = _lib.load()
    out = dets.contiguous().clone()
    P = len(counts)
    inds = torch.empty((max(out.size(0), 1),), dtype=torch.int32, device=dets.device)
    num_out = torch.empty((P,), dtype=torch.int32, device=dets.device)
    offs = 0
    for c0 in range(0, P, 128):
        chunk = counts[c0:c0 + 128]
        n = sum(chunk)
        c_arr = (ctypes.c_int * len(chunk))(*chunk)
        with torch.cuda.device(dets.device):
            _lib.check(lib.b200_soft_nms_batched(out.data_ptr() + offs * 20, ctypes.cast(c_arr, ctypes.c_void_p), len(chunk), float(sigma),
                                                 float(overlap_thresh), float(score_thresh), int(method), inds.data_ptr() + offs * 4,
                                                 num_out.data_ptr() + c0 * 4, _stream()), "b200_soft_nms_batched")
        offs += n
    return out, inds, num_out


def box_voting_batched(top_dets, top_counts, all_dets, all_counts, thresh, scoring=0, beta=1.0):
    """Box voting (lib/utils/boxes.py:268-317) for `len(top_counts)` class problems; returns the refined top_dets."""
    import ctypes
    _need_cuda_f32(top_dets, "top_dets"); _need_cuda_f32(all_dets, "all_dets")
    top_counts = [int(c) for c in top_counts]; all_counts = [int(c) for c in all_counts]
    if len(top_counts) != len(all_counts) or sum(top_counts) != top_dets.size(0) or sum(all_counts) != all_dets.size(0):
        raise ValueError("counts do not match the detection tensors")
    lib = _lib.load()
    top_dets = top_dets.contiguous(); all_dets = all_dets.contiguous()
    out = torch.empty_like(top_dets)
    to = ao = 0
    for c0 in range(0, len(top_counts), 128):
        tc, ac = top_counts[c0:c0 + 128], all_counts[c0:c0 + 128]
        t_arr = (ctypes.c_int * len(tc))(*tc); a_arr = (ctypes.c_int * len(ac))(*ac)
        with torch.cuda.device(top_dets.device):
            _lib.check(lib.b200_box_voting_batched(top_dets.data_ptr() + to * 20, ctypes.cast(t_arr, ctypes.c_void_p),
                                                   all_dets.data_ptr() + ao * 20, ctypes.cast(a_arr, ctypes.c_void_p), len(tc), float(thresh),
                                                   int(scoring), float(beta), out.data_ptr() + to * 20, _stream()), "b200_box_voting_batched")
        to += sum(tc); ao += sum(ac)
    return out


def nms_raw(dets, thresh):
    """Returns (keep int32 (N,), num_out int32 (1,)) on the device, no host sync."""
    _need_cuda_f32(dets, "dets")
    if dets.dim() != 2 or dets.size(1) < 4:
        raise ValueError("dets must be (N, >=4) = [x1, y1, x2, y2, score], got %s" % (tuple(dets.shape),))
    dets = dets.contiguous()
    n, dim = dets.shape
    lib = _lib.load()
    keep = torch.empty((max(n, 1),), dtype=torch.int32, device=dets.device)
    num_out = torch.empty((1,), dtype=torch.int32, device=dets.device)
    ws_bytes = int(lib.b200_nms_workspace_bytes(n))
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dets.device)
    with torch.cuda.device(dets.device):
        _lib.check(lib.b200_nms(dets.data_ptr(), n, dim, float(thresh), keep.data_ptr(), num_out.data_ptr(),
                                ws.data_ptr(), ws_bytes, _stream()),
                   "b200_nms")
    return keep, num_out


# ------------------------------------------------------------------------------------------------
# Test-time mask paste + COCO RLE (SURVEY.md 8f N3, lib/core/test.py:793-847)
# ------------------------------------------------------------------------------------------------
def _segm_inputs(masks, mask_class, boxes, im_h, im_w):
    _need_cuda_f32(masks, "masks"); _need_cuda_f32(boxes, "boxes")
    if masks.dim() != 4 or masks.size(2) != masks.size(3):
        raise ValueError("masks must be (D, Kc, M, M), got %s" % (tuple(masks.shape),))
    D = masks.size(0)
    if boxes.dim() != 2 or boxes.size(0) != D or boxes.size(1) != 4:
        raise ValueError("boxes must be (D, 4) = [x1, y1, x2, y2] with D = %d, got %s" % (D, tuple(boxes.shape)))
    if not torch.is_tensor(mask_class) or mask_class.dim() != 1 or mask_class.numel() != D:
        raise ValueError("mask_class must be a (D,) tensor with D = %d" % D)
    if int(im_h) <= 0 or int(im_w) <= 0:
        raise ValueError("image size must be positive, got %s x %s" % (im_h, im_w))
    mask_class = mask_class.to(device=masks.device, dtype=torch.int32).contiguous()
    return masks.contiguous(), mask_class, boxes.to(masks.device).contiguous(), D, masks.size(1), masks.size(2)


def segm_rle_raw(masks, mask_class, boxes, im_h, im_w, thresh):
    """COCO RLEs of the pasted masks of one image (lib/core/test.py:793-847 per detection, cv2 IPP-off arithmetic).
    masks: float32 CUDA (D, Kc, M, M); mask_class: (D,) channel per detection; boxes: float32 CUDA (D, 4), not expanded.
    Returns device tensors (counts int32, count_offsets int64 (D + 1,), strings uint8, string_offsets int64 (D + 1,)):
    detection d's column-major run lengths are counts[count_offsets[d]:count_offsets[d + 1]], its compressed COCO string
    strings[string_offsets[d]:string_offsets[d + 1]].  Two launches and one host read of the per-detection sizes."""
    masks, mask_class, boxes, D, Kc, M = _segm_inputs(masks, mask_class, boxes, im_h, im_w)
    dev = masks.device
    if D == 0:
        z = torch.zeros((1,), dtype=torch.int64, device=dev)
        return torch.empty((0,), dtype=torch.int32, device=dev), z, torch.empty((0,), dtype=torch.uint8, device=dev), z.clone()
    lib = _lib.load()
    ws_bytes = int(lib.b200_segm_workspace_bytes(D))
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
    sizes = torch.empty((D, 2), dtype=torch.int32, device=dev)
    args = (masks.data_ptr(), mask_class.data_ptr(), boxes.data_ptr(), D, Kc, M, int(im_h), int(im_w), float(thresh))
    with torch.cuda.device(dev):
        _lib.check(lib.b200_segm_rle_sizes(*args, sizes.data_ptr(), ws.data_ptr(), ws_bytes, _stream()), "b200_segm_rle_sizes")
        total = sizes.cpu().to(torch.int64).sum(dim=0)
        counts = torch.empty((int(total[0]),), dtype=torch.int32, device=dev)
        strings = torch.empty((int(total[1]),), dtype=torch.uint8, device=dev)
        count_offs = torch.empty((D + 1,), dtype=torch.int64, device=dev)
        string_offs = torch.empty((D + 1,), dtype=torch.int64, device=dev)
        _lib.check(lib.b200_segm_rle_emit(*args, sizes.data_ptr(), ws.data_ptr(), ws_bytes, counts.data_ptr(), count_offs.data_ptr(),
                                          strings.data_ptr(), string_offs.data_ptr(), _stream()), "b200_segm_rle_emit")
    return counts, count_offs, strings, string_offs


def paste_masks(masks, mask_class, boxes, im_h, im_w, thresh):
    """The full-image binary masks segm_results encodes: uint8 CUDA (D, im_h, im_w), the reference's `im_mask` per detection."""
    masks, mask_class, boxes, D, Kc, M = _segm_inputs(masks, mask_class, boxes, im_h, im_w)
    out = torch.empty((D, int(im_h), int(im_w)), dtype=torch.uint8, device=masks.device)
    if D == 0:
        return out
    with torch.cuda.device(masks.device):
        _lib.check(_lib.load().b200_paste_masks(masks.data_ptr(), mask_class.data_ptr(), boxes.data_ptr(), D, Kc, M, int(im_h), int(im_w),
                                                float(thresh), out.data_ptr(), _stream()), "b200_paste_masks")
    return out


# ------------------------------------------------------------------------------------------------
# Test-time keypoint extraction + OKS NMS (SURVEY.md 8f N3, lib/utils/keypoints.py:103-157, 225-266)
# ------------------------------------------------------------------------------------------------
def _keypoint_rois(rois, D, device):
    _need_cuda_f32(rois, "rois")
    if rois.dim() != 2 or rois.size(0) != D or rois.size(1) < 4:
        raise ValueError("rois must be (D, >=4) = [x1, y1, x2, y2, ...] with D = %d, got %s" % (D, tuple(rois.shape)))
    return rois[:, :4].to(device).contiguous()


def heatmaps_to_keypoints_raw(maps, rois, min_size=0):
    """Keypoints of one image's detections from the keypoint head's logits (lib/utils/keypoints.py:103-157, cv2's float32
    INTER_CUBIC arithmetic).  maps: float32 CUDA (D, K, M, M); rois: float32 CUDA (D, >=4) = [x1, y1, x2, y2];
    min_size: KRCNN.INFERENCE_MIN_SIZE (<= 0: none).  Returns a float32 CUDA (D, 4, K) tensor of rows (x, y, logit, prob).
    One launch, no host sync."""
    _need_cuda_f32(maps, "maps")
    if maps.dim() != 4 or maps.size(2) != maps.size(3):
        raise ValueError("maps must be (D, K, M, M), got %s" % (tuple(maps.shape),))
    D, K, M = maps.size(0), maps.size(1), maps.size(2)
    rois = _keypoint_rois(rois, D, maps.device)
    maps = maps.contiguous()
    out = torch.empty((D, 4, K), dtype=torch.float32, device=maps.device)
    if D == 0:
        return out
    with torch.cuda.device(maps.device):
        _lib.check(_lib.load().b200_heatmaps_to_keypoints(maps.data_ptr(), rois.data_ptr(), D, K, M, int(min_size), out.data_ptr(),
                                                          _stream()),
                   "b200_heatmaps_to_keypoints")
    return out


def rpn_targets_raw(gt_boxes, gt_counts, im_sizes, levels, draw, straddle_thresh=0, positive_overlap=0.7, negative_overlap=0.3):
    """RPN anchor labels and regression targets for N images and all anchor levels (lib/roi_data/rpn.py:115-259).
    gt_boxes: float32 CUDA (sum G, 4), image n's (scaled) ground truth in rows sum(gt_counts[:n]) ...; gt_counts: host ints, each
    >= 1; im_sizes: host (N, 2) = (im_height, im_width); levels: one (field_size, stride, cell_anchors (A, 4) float64) per level.
    draw(counts) is called once with the (N, 3) host array (#fg candidates, #bg candidates, #inside anchors) -- the one host read
    of the call -- and returns, per image, (fg positions to disable, bg positions to enable): int sequences or CUDA tensors.
    Returns one (labels int32 (N, A, F, F), bbox_targets, inside_weights, outside_weights float32 (N, 4A, F, F)) per level."""
    import ctypes
    import numpy as np
    _need_cuda_f32(gt_boxes, "gt_boxes")
    if gt_boxes.dim() != 2 or gt_boxes.size(1) != 4:
        raise ValueError("gt_boxes must be (G, 4) = [x1, y1, x2, y2], got %s" % (tuple(gt_boxes.shape),))
    gt_counts = [int(c) for c in gt_counts]
    N, L = len(gt_counts), len(levels)
    im_sizes = np.ascontiguousarray(im_sizes, dtype=np.float64).reshape(-1, 2)
    if im_sizes.shape[0] != N or sum(gt_counts) != gt_boxes.size(0):
        raise ValueError("rpn_targets_raw: %d images, %d image sizes, %d ground-truth rows for counts %s"
                         % (N, im_sizes.shape[0], gt_boxes.size(0), gt_counts))
    dev = gt_boxes.device
    gt_boxes = gt_boxes.contiguous()
    Fs = [int(F) for F, _, _ in levels]
    cells = [np.asarray(c, dtype=np.float64).reshape(-1, 4) for _, _, c in levels]
    As = [c.shape[0] for c in cells]

    def arr(ctype, vals):
        a = (ctype * max(len(vals), 1))(*vals)
        return ctypes.cast(a, ctypes.c_void_p), a             # the array object keeps the memory alive during the call

    F_p, F_a = arr(ctypes.c_int, Fs)
    A_p, A_a = arr(ctypes.c_int, As)
    S_p, S_a = arr(ctypes.c_double, [float(s) for _, s, _ in levels])
    C_p, C_a = arr(ctypes.c_double, np.concatenate(cells).ravel().tolist() if cells else [])
    I_p, I_a = arr(ctypes.c_double, im_sizes.ravel().tolist())
    G_p, G_a = arr(ctypes.c_int, np.concatenate([[0], np.cumsum(gt_counts)]).astype(int).tolist())
    lib = _lib.load()
    ws_bytes = int(lib.b200_rpn_targets_workspace_bytes(L, F_p, A_p, N, gt_boxes.size(0)))
    if ws_bytes == 0:
        raise ValueError("rpn_targets_raw: unsupported geometry (1..8 levels, <= 32 cell anchors, 1..64 images)")
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
    counts = torch.empty((N, 3), dtype=torch.int32, device=dev)
    common = (L, F_p, A_p, S_p, C_p, N, I_p, G_p, gt_boxes.data_ptr(), float(straddle_thresh))
    with torch.cuda.device(dev):
        _lib.check(lib.b200_rpn_labels(*common, float(positive_overlap), float(negative_overlap), counts.data_ptr(), ws.data_ptr(), ws_bytes,
                                       _stream()), "b200_rpn_labels")
        picks = draw(counts.cpu().numpy())
        dis_parts, en_parts = [], []
        for dis, en in picks:
            dis_parts.append(torch.as_tensor(np.asarray(dis) if not torch.is_tensor(dis) else dis).reshape(-1))
            en_parts.append(torch.as_tensor(np.asarray(en) if not torch.is_tensor(en) else en).reshape(-1))
        if len(dis_parts) != N:
            raise ValueError("draw returned %d entries for %d images" % (len(dis_parts), N))
        D_p, D_a = arr(ctypes.c_int, np.concatenate([[0], np.cumsum([d.numel() for d in dis_parts])]).astype(int).tolist())
        E_p, E_a = arr(ctypes.c_int, np.concatenate([[0], np.cumsum([e.numel() for e in en_parts])]).astype(int).tolist())
        # one int32 device buffer for both draws (a single upload when they come from the host)
        parts = dis_parts + en_parts
        if all(not p.is_cuda for p in parts):
            flat = torch.cat([p.to(torch.int32) for p in parts]).to(dev) if parts else torch.empty((0,), dtype=torch.int32, device=dev)
        else:
            flat = torch.cat([p.to(device=dev, dtype=torch.int32) for p in parts])
        flat = torch.cat([flat, flat.new_zeros((1,))])            # never empty: a valid pointer even without draws
        n_dis = sum(d.numel() for d in dis_parts)
        outs = []
        for F, A in zip(Fs, As):
            outs.append((torch.empty((N, A, F, F), dtype=torch.int32, device=dev),
                         torch.empty((N, 4 * A, F, F), dtype=torch.float32, device=dev),
                         torch.empty((N, 4 * A, F, F), dtype=torch.float32, device=dev),
                         torch.empty((N, 4 * A, F, F), dtype=torch.float32, device=dev)))
        tables = [arr(ctypes.c_void_p, [o[k].data_ptr() for o in outs]) for k in range(4)]
        _lib.check(lib.b200_rpn_emit(*common, counts.data_ptr(), flat.data_ptr(), D_p, flat.data_ptr() + 4 * n_dis, E_p, ws.data_ptr(),
                                     ws_bytes, *[t[0] for t in tables], _stream()), "b200_rpn_emit")
    return outs


MASK_COORD_LIMIT = float(2 ** 20)


def pack_polygons(objects_per_image):
    """Host packer for mask_targets_raw.  objects_per_image: per image, the list of its objects' polygon segmentations (roidb
    `segms` entries: a list of polygons, each a flat [x0, y0, x1, y1, ...] coordinate list).  Returns numpy tables
    (obj_begin (N + 1,), poly_begin (O + 1,), coord_begin (P + 1,) int32; coords (2V,) float32).
    ValueError for an object without polygons, a polygon with fewer than 6 values or an odd count, non-finite coordinates and
    coordinates beyond +-2^20.  The reference's pycocotools frPyObjects dispatches on the first polygon's length: 4 values
    read every polygon of the object as [x, y, w, h] boxes, fewer fail, and an odd count silently drops the last value --
    none of which is a polygon mask, so all are rejected here."""
    import numpy as np
    obj_begin, poly_begin, coord_begin, parts = [0], [0], [0], []
    for objs in objects_per_image:
        for polys in objs:
            if isinstance(polys, dict) or not isinstance(polys, (list, tuple)) or len(polys) == 0:
                raise ValueError("a non-crowd object needs a non-empty list of polygons, got %r" % (type(polys),))
            for p in polys:
                a = np.asarray(p, dtype=np.float64).reshape(-1)
                if a.size < 6 or a.size % 2:
                    raise ValueError("a polygon needs an even number (>= 6) of coordinates, got %d" % a.size)
                if not np.isfinite(a).all():
                    raise ValueError("non-finite polygon coordinate")
                if np.abs(a).max() > MASK_COORD_LIMIT:
                    raise ValueError("polygon coordinate beyond +-2^20")
                parts.append(a.astype(np.float32))
                coord_begin.append(coord_begin[-1] + a.size)
            poly_begin.append(len(coord_begin) - 1)
        obj_begin.append(len(poly_begin) - 1)
    coords = np.concatenate(parts) if parts else np.zeros((0,), np.float32)
    return (np.asarray(obj_begin, np.int32), np.asarray(poly_begin, np.int32), np.asarray(coord_begin, np.int32), coords)


def mask_targets_raw(rois, roi_image, roi_class, packed, resolution, num_classes):
    """Mask R-CNN training mask targets (lib/roi_data/mask_rcnn.py:34-122) for all RoIs of a step in one call (2 launches, no
    device-to-host read).  rois: float32 CUDA (R, 4) unscaled (x1, y1, x2, y2); roi_image: host ints (R,) (image index);
    roi_class: int32 CUDA (R,) -- a class <= 0 gives an all -1 row; packed: pack_polygons' tables; num_classes: 0 for
    class-agnostic masks.  Returns masks_int32 (R, max(num_classes, 1) * M * M) on the device."""
    import ctypes
    import numpy as np
    _need_cuda_f32(rois, "rois")
    if rois.dim() != 2 or rois.size(1) != 4:
        raise ValueError("rois must be (R, 4) = [x1, y1, x2, y2], got %s" % (tuple(rois.shape),))
    if roi_class.dtype != torch.int32 or not roi_class.is_cuda:
        raise TypeError("roi_class must be an int32 CUDA tensor")
    obj_begin, poly_begin, coord_begin, coords = packed
    R, M, K = rois.size(0), int(resolution), int(num_classes)
    roi_image = np.asarray(roi_image, np.int32).reshape(-1)
    if R == 0 or roi_image.size != R or roi_class.numel() != R:
        raise ValueError("mask_targets_raw: %d RoIs, %d image indices, %d classes" % (R, roi_image.size, roi_class.numel()))
    if not 1 <= M <= 64 or K < 0 or not 1 <= obj_begin.size - 1 <= 64:
        raise ValueError("mask_targets_raw: resolution %d (1..64), num_classes %d (>= 0), %d images (1..64)" % (M, K, obj_begin.size - 1))
    dev = rois.device
    rois = rois.contiguous()
    if rois.data_ptr() % 16:
        rois = rois.clone()                                              # the kernel reads a RoI with one 16-byte load
    roi_class = roi_class.contiguous()
    O, P, C = poly_begin.size - 1, coord_begin.size - 1, coords.size
    # one upload: roi_image | poly_begin | coord_begin | coords (as int32 bits)
    host = np.concatenate([roi_image, poly_begin, coord_begin, coords.view(np.int32)])
    buf = torch.from_numpy(host).pin_memory().to(dev, non_blocking=True)
    ptr, i4 = buf.data_ptr(), 4
    boxes = torch.empty((max(O, 1), 4), dtype=torch.float32, device=dev)
    masks = torch.empty((R, max(K, 1) * M * M), dtype=torch.int32, device=dev)
    ob = (ctypes.c_int * obj_begin.size)(*obj_begin.tolist())
    with torch.cuda.device(dev):
        _lib.check(_lib.load().b200_mask_targets(rois.data_ptr(), ptr, roi_class.data_ptr(), R,
                                                 obj_begin.size - 1, ob, P, ptr + i4 * R, C, ptr + i4 * (R + O + 1),
                                                 ptr + i4 * (R + O + P + 2), M, K, boxes.data_ptr(), masks.data_ptr(), _stream()),
                   "b200_mask_targets")
    return masks


def _host_or_device(x, dtype, dev, name):
    """A host array (returned as numpy, for the one upload) or a CUDA tensor of `dtype` (returned as is, contiguous)."""
    import numpy as np
    if torch.is_tensor(x):
        if not x.is_cuda:
            raise NotImplementedError("%s must be a CUDA tensor or a host array, not a CPU tensor" % name)
        return x.to(device=dev, dtype=dtype).reshape(-1).contiguous()
    return np.ascontiguousarray(np.asarray(x).reshape(-1).astype(np.float32 if dtype == torch.float32 else np.int32))


def keypoint_targets_raw(boxes, box_begin, max_overlaps, box_to_gt_ind_map, gt_inds, gt_keypoints, im_scales, fg_rois_per_image, draw,
                         heatmap_size, fg_thresh=0.5, batch_index=None, device=None):
    """Keypoint R-CNN training targets (lib/roi_data/keypoint_rcnn.py:33-82 with lib/utils/keypoints.py:160-211) for N images
    in one call: 2 launches and one host read, the N candidate counts.
    boxes (B, 4) float32, max_overlaps (B,) float32, box_to_gt_ind_map (B,) int32: the merged roidb's (ground truth first, then
    proposals; unscaled), image n's in rows box_begin[n] .. box_begin[n + 1] - 1 (host ints); each a CUDA tensor or a host
    array.  gt_inds: per image, np.where(gt_classes > 0); gt_keypoints: per image (G_n, 3, K) int32 (x, y, v) host arrays.
    im_scales: host (N,); batch_index: host (N,), default 0 .. N - 1.
    draw(counts) is called once with the (N,) host candidate counts and returns, per image, None (the first
    min(fg_rois_per_image, count) candidates in ascending order) or the positions in the candidate list that np.random.choice
    picked (host ints or a CUDA tensor, min(fg_rois_per_image, count) of them).
    A host box_to_gt_ind_map is checked against gt_inds first (numpy's IndexError becomes ValueError); a device one is read
    with the same bounds, an out-of-range entry meaning no person.  Returns (keypoint_rois (R, 5) float32,
    keypoint_locations_int32 (R * K,) int32, keypoint_weights (R * K,) float32, all CUDA; counts (N,) numpy)."""
    import ctypes
    import numpy as np
    box_begin = np.asarray(box_begin, np.int64).reshape(-1)
    N = box_begin.size - 1
    if not 1 <= N <= 64 or box_begin[0] != 0 or (np.diff(box_begin) < 0).any():
        raise ValueError("keypoint_targets_raw: box_begin must start at 0 and not decrease over 1..64 images, got %s" % box_begin.tolist())
    if len(gt_inds) != N or len(gt_keypoints) != N or np.asarray(im_scales).size != N:
        raise ValueError("keypoint_targets_raw: %d images but %d gt_inds, %d gt_keypoints, %d im_scales"
                         % (N, len(gt_inds), len(gt_keypoints), np.asarray(im_scales).size))
    HS, fg = int(heatmap_size), int(fg_rois_per_image)
    kps = [np.asarray(k) for k in gt_keypoints]
    K = kps[0].shape[2] if kps[0].ndim == 3 else -1
    if any(k.ndim != 3 or k.shape[1] != 3 or k.shape[2] != K for k in kps) or not 1 <= K <= 64:
        raise ValueError("gt_keypoints must be (G, 3, K) arrays with the same K in 1..64, got %s" % [k.shape for k in kps])
    if not 1 <= HS <= 4096:
        raise ValueError("heatmap_size %d outside 1..4096" % HS)
    gis = [np.asarray(g, np.int64).reshape(-1) for g in gt_inds]
    for n, (g, k) in enumerate(zip(gis, kps)):
        if g.size and (g.min() < 0 or g.max() >= k.shape[0]):
            raise ValueError("image %d: gt_inds out of range for %d keypoint rows" % (n, k.shape[0]))
    B = int(box_begin[-1])
    dev = device if device is not None else next((t.device for t in (boxes, max_overlaps, box_to_gt_ind_map) if torch.is_tensor(t)),
                                                 torch.device("cuda", torch.cuda.current_device()))
    bx = _host_or_device(boxes, torch.float32, dev, "boxes")
    mo = _host_or_device(max_overlaps, torch.float32, dev, "max_overlaps")
    bm = _host_or_device(box_to_gt_ind_map, torch.int32, dev, "box_to_gt_ind_map")
    def size(a):
        return a.numel() if torch.is_tensor(a) else a.size
    if size(bx) != 4 * B:
        raise ValueError("boxes must be (%d, 4)" % B)
    if size(mo) != B or size(bm) != B:
        raise ValueError("max_overlaps and box_to_gt_ind_map must have %d entries" % B)
    if not torch.is_tensor(bm):
        for n in range(N):
            m, G = bm[box_begin[n]:box_begin[n + 1]], gis[n].size
            if m.size and (m.min() < -G or m.max() >= G):
                raise ValueError("image %d: box_to_gt_ind_map indexes gt_inds of size %d out of range (numpy: IndexError)" % (n, G))
    # one upload: the host-side inputs, gt_inds, the keypoints (float32 as int32 bits), one pad so no part is at the very end
    parts, offs = [], {}

    def put(name, a):
        offs[name] = sum(p.size for p in parts)
        parts.append(a.view(np.int32) if a.dtype == np.float32 else a.astype(np.int32))
    for name, a in (("boxes", bx), ("mo", mo), ("map", bm)):
        if not torch.is_tensor(a):
            put(name, a)
    put("gt_inds", np.concatenate(gis) if any(g.size for g in gis) else np.zeros((0,), np.int32))
    put("kps", np.concatenate([k.astype(np.int32).reshape(-1) for k in kps]))
    parts.append(np.zeros((1,), np.int32))
    buf = torch.from_numpy(np.concatenate(parts)).pin_memory().to(dev, non_blocking=True)
    base = buf.data_ptr()

    def ptr(name, a):
        return a.data_ptr() if torch.is_tensor(a) else base + 4 * offs[name]

    def tab(vals):
        return (ctypes.c_int * len(vals))(*[int(v) for v in vals])
    bb = tab(box_begin)
    gb = tab(np.concatenate([[0], np.cumsum([g.size for g in gis])]))
    pb = tab(np.concatenate([[0], np.cumsum([k.shape[0] for k in kps])]))
    cand =torch.empty((max(B, 1),), dtype=torch.int32, device=dev)
    counts = torch.empty((N,), dtype=torch.int32, device=dev)
    lib = _lib.load()
    with torch.cuda.device(dev):
        _lib.check(lib.b200_keypoint_candidates(ptr("boxes", bx), ptr("mo", mo), ptr("map", bm), N, bb, base + 4 * offs["gt_inds"], gb,
                                                base + 4 * offs["kps"], pb, K, float(fg_thresh), cand.data_ptr(), counts.data_ptr(),
                                                _stream()), "b200_keypoint_candidates")
        counts_h = counts.cpu().numpy()
        picks = list(draw(counts_h))
        if len(picks) != N:
            raise ValueError("draw returned %d entries for %d images" % (len(picks), N))
        sizes = [min(fg, int(c)) for c in counts_h]
        sel = []
        for n, (pk, size) in enumerate(zip(picks, sizes)):
            if pk is None:
                sel.append(torch.arange(size, dtype=torch.int32))
                continue
            pk = pk.reshape(-1) if torch.is_tensor(pk) else torch.from_numpy(np.asarray(pk, np.int64).reshape(-1))
            if pk.numel() != size:
                raise ValueError("image %d: %d keypoint draw positions, the minibatch takes %d" % (n, pk.numel(), size))
            if not pk.is_cuda and size and (int(pk.min()) < 0 or int(pk.max()) >= int(counts_h[n])):
                raise ValueError("image %d: keypoint draw positions outside 0..%d" % (n, int(counts_h[n]) - 1))
            sel.append(pk)
        if all(not p.is_cuda for p in sel):
            flat = torch.cat([p.to(torch.int32) for p in sel] + [torch.zeros((1,), dtype=torch.int32)]).to(dev)
        else:
            flat = torch.cat([p.to(device=dev, dtype=torch.int32) for p in sel] + [torch.zeros((1,), dtype=torch.int32, device=dev)])
        R = sum(sizes)
        rb = tab(np.concatenate([[0], np.cumsum(sizes)]))
        sc = (ctypes.c_float * N)(*[float(np.float32(s)) for s in np.asarray(im_scales).reshape(-1)])
        bi = (ctypes.c_float * N)(*[float(np.float32(b)) for b in (np.arange(N) if batch_index is None else np.asarray(batch_index).reshape(-1))])
        rois = torch.empty((max(R, 1), 5), dtype=torch.float32, device=dev)
        loc = torch.empty((max(R * K, 1),), dtype=torch.int32, device=dev)
        w = torch.empty((max(R * K, 1),), dtype=torch.float32, device=dev)
        _lib.check(lib.b200_keypoint_targets(ptr("boxes", bx), ptr("map", bm), N, bb, base + 4 * offs["gt_inds"], gb, base + 4 * offs["kps"],
                                             pb, K, HS, cand.data_ptr(), counts.data_ptr(), flat.data_ptr(), rb, sc, bi, rois.data_ptr(),
                                             loc.data_ptr(), w.data_ptr(), _stream()), "b200_keypoint_targets")
    return rois[:R], loc[:R * K], w[:R * K], counts_h


def keypoints_to_heatmap_labels_raw(keypoints, rois, heatmap_size):
    """keypoints_to_heatmap_labels (lib/utils/keypoints.py:160-211) for R given RoIs: keypoints (R, 3, K) int32 (host array or
    CUDA tensor), rois CUDA float32 (R, >=4) = [x1, y1, x2, y2].  Returns (heats (R, K) int32 = the reference's result after
    `.astype(np.int32)`, weights (R, K) float32), CUDA.  One launch (the emit of keypoint_targets_raw, each RoI its own
    candidate)."""
    import ctypes
    import numpy as np
    _need_cuda_f32(rois, "rois")
    if rois.dim() != 2 or rois.size(1) < 4:
        raise ValueError("rois must be (R, >=4) = [x1, y1, x2, y2, ...], got %s" % (tuple(rois.shape),))
    dev = rois.device
    kp = keypoints.to(device=dev, dtype=torch.int32) if torch.is_tensor(keypoints) else \
        torch.from_numpy(np.ascontiguousarray(np.asarray(keypoints).astype(np.int32))).to(dev)
    R = rois.size(0)
    if kp.dim() != 3 or kp.size(0) != R or kp.size(1) != 3 or not 1 <= kp.size(2) <= 64:
        raise ValueError("keypoints must be (%d, 3, K) with K in 1..64, got %s" % (R, tuple(kp.shape)))
    K, HS = kp.size(2), int(heatmap_size)
    if not 1 <= HS <= 4096:
        raise ValueError("heatmap_size %d outside 1..4096" % HS)
    if R == 0:
        return torch.empty((0, K), dtype=torch.int32, device=dev), torch.empty((0, K), dtype=torch.float32, device=dev)
    boxes = rois[:, :4].contiguous()
    kp = kp.contiguous()
    ident = torch.arange(R + 1, dtype=torch.int32, device=dev)            # map, gt_inds, candidates and picks; ident[R] = count
    ident[R] = R
    tab = (ctypes.c_int * 2)(0, R)
    one = (ctypes.c_float * 1)(1.0)
    zero = (ctypes.c_float * 1)(0.0)
    rows = torch.empty((R, 5), dtype=torch.float32, device=dev)
    heats = torch.empty((R, K), dtype=torch.int32, device=dev)
    weights = torch.empty((R, K), dtype=torch.float32, device=dev)
    p = ident.data_ptr()
    with torch.cuda.device(dev):
        _lib.check(_lib.load().b200_keypoint_targets(boxes.data_ptr(), p, 1, tab, p, tab, kp.data_ptr(), tab, K, HS, p, p + 4 * R, p, tab, one,
                                                     zero, rows.data_ptr(), heats.data_ptr(), weights.data_ptr(), _stream()),
                   "b200_keypoint_targets")
    return heats, weights


def nms_oks_raw(xy_preds, rois, thresh):
    """Greedy OKS NMS of lib/utils/keypoints.py:225-266 on (D, 4, 17) predictions and their (D, >=4) boxes, float32 CUDA.
    Returns (keep int32 (D,), num_keep int32 (1,)) on the device, no host sync: keep[:num_keep] are the kept indices in
    greedy order (descending mean logit; equal scores the higher index first)."""
    _need_cuda_f32(xy_preds, "xy_preds")
    if xy_preds.dim() != 3 or xy_preds.size(1) != 4:
        raise ValueError("xy_preds must be (D, 4, K), got %s" % (tuple(xy_preds.shape),))
    D, K = xy_preds.size(0), xy_preds.size(2)
    rois = _keypoint_rois(rois, D, xy_preds.device)
    xy_preds = xy_preds.contiguous()
    keep = torch.empty((max(D, 1),), dtype=torch.int32, device=xy_preds.device)
    if D == 0:
        return keep[:0], torch.zeros((1,), dtype=torch.int32, device=xy_preds.device)
    num_keep = torch.empty((1,), dtype=torch.int32, device=xy_preds.device)
    with torch.cuda.device(xy_preds.device):
        _lib.check(_lib.load().b200_nms_oks(xy_preds.data_ptr(), rois.data_ptr(), D, K, float(thresh), keep.data_ptr(), num_keep.data_ptr(),
                                            _stream()),
                   "b200_nms_oks")
    return keep, num_keep


# ------------------------------------------------------------------------------------------------
# Input image blob (lib/utils/blob.py:37-148, lib/roi_data/minibatch.py:47-79)
# ------------------------------------------------------------------------------------------------
# b200_image_blob_desc of include/b200_roi_ops.h
_BLOB_DESC = [("src_offset", "<i8"), ("row_pitch", "<i8"), ("inv_scale", "<f8"), ("height", "<i4"), ("width", "<i4"),
              ("out_h", "<i4"), ("out_w", "<i4"), ("flipped", "<i4"), ("area2x", "<i4"), ("slot", "<i4"), ("reserved", "<i4")]


def pixel_mean_table(pixel_means):
    """(3, 256) float32: channel c of a uint8 value v after the reference's `im = im.astype(np.float32); im -= pixel_means`
    (with the default float64 means, float32(float64(v) - mean)), evaluated by numpy itself."""
    import numpy as np
    t = np.empty((256, 1, 3), np.float32)
    t[...] = np.arange(256, dtype=np.float32).reshape(256, 1, 1)
    t -= np.asarray(pixel_means)
    return np.ascontiguousarray(t.reshape(256, 3).T)


def resized_size(h, w, im_scale):
    """cv2.resize's output size for fx = fy = im_scale: (rint(h * s), rint(w * s)), half to even.  A zero side raises
    ValueError where cv2 raises."""
    import numpy as np
    oh, ow = int(np.rint(h * float(im_scale))), int(np.rint(w * float(im_scale)))
    if oh <= 0 or ow <= 0:
        raise ValueError("resizing a %d x %d image by %r leaves an empty side (cv2.resize raises)" % (h, w, im_scale))
    return oh, ow


def image_blob_raw(images, scales, flipped, pixel_means, stride, out=None):
    """The network's input blob for all images of a call in one launch: image i (uint8 (H, W, 3) BGR, a host array or a CUDA
    tensor) flipped when flipped[i] (im[:, ::-1, :]), minus pixel_means, resized by scales[i] like cv2.resize(fx = fy,
    INTER_LINEAR) with IPP off, zero-padded to the largest resized size (rounded up to a multiple of `stride` when it is not
    None: FPN.COARSEST_STRIDE) and stored NCHW.  Host images go up in one asynchronous copy from one pinned buffer; CUDA
    images are read where they are.  Returns (blob float32 CUDA (N, 3, Hp, Wp), [(h, w) resized size per image]).
    `out`: an optional float32 CUDA tensor of that shape to write into (every element is written)."""
    import numpy as np
    N = len(images)
    if N < 1 or len(scales) != N or len(flipped) != N:
        raise ValueError("image_blob_raw: %d images, %d scales, %d flip flags" % (N, len(scales), len(flipped)))
    dev = next((im.device for im in images if torch.is_tensor(im) and im.is_cuda), torch.device("cuda", torch.cuda.current_device()))
    descs = np.zeros((N,), dtype=_BLOB_DESC)
    host, host_bytes, cuda_ims, sizes = [], 0, [], []
    for i, im in enumerate(images):
        on_dev = torch.is_tensor(im) and im.is_cuda
        if not on_dev:
            im = np.ascontiguousarray(im.numpy() if torch.is_tensor(im) else im)
        dtype_ok = im.dtype == torch.uint8 if on_dev else im.dtype == np.uint8
        if not dtype_ok or len(im.shape) != 3 or im.shape[2] != 3 or im.shape[0] < 1 or im.shape[1] < 1:
            raise ValueError("image %d must be a uint8 (H, W, 3) image, got %s %s" % (i, im.dtype, tuple(im.shape)))
        if on_dev:
            if im.device != dev:
                raise ValueError("image_blob_raw: images on %s and %s" % (dev, im.device))
            if im.stride(2) != 1 or im.stride(1) != 3:
                im = im.contiguous()
            cuda_ims.append((i, im))
        else:
            host.append((i, im, host_bytes))
            host_bytes += (im.nbytes + 15) & ~15
        H, W = int(im.shape[0]), int(im.shape[1])
        s = float(scales[i])
        oh, ow = resized_size(H, W, s)
        d = descs[i]
        d["height"], d["width"], d["out_h"], d["out_w"] = H, W, oh, ow
        d["row_pitch"] = im.stride(0) if on_dev else im.strides[0]
        d["inv_scale"] = 1.0 if (oh, ow) == (H, W) else 1.0 / s          # an unchanged size is a copy in cv2
        d["area2x"] = int(1.0 / s == 2.0)
        d["flipped"] = int(bool(flipped[i]))
        d["slot"] = i
        sizes.append((oh, ow))
    Hp, Wp = max(h for h, _ in sizes), max(w for _, w in sizes)
    if stride:
        Hp, Wp = int(np.ceil(Hp / float(stride)) * stride), int(np.ceil(Wp / float(stride)) * stride)
    if out is None:
        out = torch.empty((N, 3, Hp, Wp), dtype=torch.float32, device=dev)
    elif not (out.is_cuda and out.dtype == torch.float32 and out.is_contiguous() and tuple(out.shape) == (N, 3, Hp, Wp) and out.device == dev):
        raise ValueError("out must be a contiguous float32 CUDA tensor of shape %s on %s" % ((N, 3, Hp, Wp), dev))
    # one pinned staging buffer -- descriptors | mean table | host images, 16-byte aligned -- and one H2D copy into `buf`;
    # CUDA images are addressed relative to buf's base
    table = pixel_mean_table(pixel_means)
    head = descs.nbytes + table.nbytes
    buf = torch.empty((head + host_bytes,), dtype=torch.uint8, device=dev)
    base = buf.data_ptr()
    for i, im, off in host:
        descs[i]["src_offset"] = head + off
    for i, im in cuda_ims:
        descs[i]["src_offset"] = im.data_ptr() - base
    staging = torch.empty((head + host_bytes,), dtype=torch.uint8, pin_memory=True)
    st = staging.numpy()
    st[:descs.nbytes] = descs.view(np.uint8)
    st[descs.nbytes:head] = table.view(np.uint8).reshape(-1)
    for i, im, off in host:
        st[head + off:head + off + im.nbytes] = im.reshape(-1)
    with torch.cuda.device(dev):
        # Asynchronous: torch's pinned-memory allocator records this copy on the stream and does not hand `staging` out again
        # before it has completed, so dropping the last reference on return is safe.
        buf.copy_(staging, non_blocking=True)
        _lib.check(_lib.load().b200_image_blob(base, base, N, base + descs.nbytes, Hp, Wp, out.data_ptr(), _stream()),
                   "b200_image_blob")
    return out, sizes


# ------------------------------------------------------------------------------------------------
# COCO evaluation stages (pycocotools COCOeval.evaluate / accumulate; datasets/coco_eval.py drives them)
# ------------------------------------------------------------------------------------------------
def _ptr(t):
    return 0 if t is None else t.data_ptr()


def coco_rank_raw(pair_det_begin, pair_entry_begin, det_score, num_entries):
    """Stable descending-score rank per (image, category) pair, cut to each pair's entry count (COCOeval.computeIoU /
    evaluateImg's mergesort on -score and [0:maxDets[-1]]).  Returns (entry_det int32, entry_rank int32, entry_score f64)."""
    dev = det_score.device
    P = pair_det_begin.numel() - 1
    entry_det = torch.empty((max(num_entries, 1),), dtype=torch.int32, device=dev)
    entry_rank = torch.empty_like(entry_det)
    entry_score = torch.empty((max(num_entries, 1),), dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.load().b200_coco_rank(P, pair_det_begin.data_ptr(), pair_entry_begin.data_ptr(), det_score.data_ptr(),
                                              entry_det.data_ptr(), entry_rank.data_ptr(), entry_score.data_ptr(), _stream()),
                   "b200_coco_rank")
    return entry_det, entry_rank, entry_score


def coco_bbox_iou_raw(pair_gt_begin, pair_entry_begin, pair_iou_begin, entry_det, det_box, gt_box, gt_flags, ious):
    """computeIoU for iouType 'bbox' (maskApi bbIou) of every pair into `ious` (float64, rows = entries)."""
    with torch.cuda.device(ious.device):
        _lib.check(_lib.load().b200_coco_bbox_iou(pair_gt_begin.numel() - 1, pair_gt_begin.data_ptr(), pair_entry_begin.data_ptr(),
                                                  pair_iou_begin.data_ptr(), entry_det.data_ptr(), det_box.data_ptr(), gt_box.data_ptr(),
                                                  gt_flags.data_ptr(), ious.data_ptr(), _stream()), "b200_coco_bbox_iou")


def coco_oks_raw(vars, pair_gt_begin, pair_entry_begin, pair_iou_begin, entry_det, det_kp, gt_kp, gt_box, gt_area, ious):
    """computeOks of every pair into `ious`; vars = (sigmas * 2) ** 2 as a host float64 array of 17."""
    import ctypes
    import numpy as np
    v = np.ascontiguousarray(vars, np.float64)
    if v.size != 17:
        raise ValueError("OKS needs 17 keypoint variances, got %d" % v.size)
    with torch.cuda.device(ious.device):
        _lib.check(_lib.load().b200_coco_oks(pair_gt_begin.numel() - 1, v.ctypes.data_as(ctypes.c_void_p), pair_gt_begin.data_ptr(),
                                             pair_entry_begin.data_ptr(), pair_iou_begin.data_ptr(), entry_det.data_ptr(), det_kp.data_ptr(),
                                             gt_kp.data_ptr(), gt_box.data_ptr(), gt_area.data_ptr(), ious.data_ptr(), _stream()),
                   "b200_coco_oks")


def coco_masks_raw(words, slot_word, slot_hw, strings, counts, polys, mask_slot_begin, mask_area, mask_range):
    """Mask bitmaps (annToRLE: rleFrString, uncompressed counts, rleFrPoly + merge) into `words`.  strings / counts / polys are
    (slot, begin, data) triples of device tensors, or None; polys' begin is per-polygon vertex offsets and data float64 x, y."""
    def parts(x):
        return (0, None, None, None) if x is None else (x[0].numel(), x[0], x[1], x[2])
    ns, ss, sb, sd = parts(strings)
    nc, cs, cb, cd = parts(counts)
    npl, ps, pb, pd = parts(polys)
    with torch.cuda.device(words.device):
        _lib.check(_lib.load().b200_coco_masks(words.data_ptr(), words.numel(), slot_hw.size(0), slot_word.data_ptr(), slot_hw.data_ptr(),
                                               ns, _ptr(ss), _ptr(sb), _ptr(sd), nc, _ptr(cs), _ptr(cb), _ptr(cd),
                                               npl, 0 if pd is None else pd.numel() // 2, _ptr(ps), _ptr(pb), _ptr(pd),
                                               mask_slot_begin.numel() - 1, mask_slot_begin.data_ptr(), mask_area.data_ptr(),
                                               mask_range.data_ptr(), _stream()), "b200_coco_masks")


def coco_segm_iou_raw(pair_begin, num_pairs, pair_gt_begin, pair_entry_begin, pair_iou_begin, entry_det, det0, gt0, gt_mask0,
                      mask_slot_begin, slot_word, slot_hw, words, mask_area, mask_range, gt_flags, ious):
    """computeIoU for iouType 'segm' (rleIou) of pairs pair_begin .. + num_pairs - 1 on the bitmaps of one coco_masks_raw call."""
    with torch.cuda.device(ious.device):
        _lib.check(_lib.load().b200_coco_segm_iou(pair_begin, num_pairs, pair_gt_begin.data_ptr(), pair_entry_begin.data_ptr(),
                                                  pair_iou_begin.data_ptr(), entry_det.data_ptr(), det0, gt0, gt_mask0,
                                                  mask_slot_begin.data_ptr(), slot_word.data_ptr(), slot_hw.data_ptr(), words.data_ptr(),
                                                  mask_area.data_ptr(), mask_range.data_ptr(), gt_flags.data_ptr(), ious.data_ptr(),
                                                  _stream()), "b200_coco_segm_iou")


def coco_match_raw(iou_thrs, area_rng, max_gt, num_cats, pair_gt_begin, pair_entry_begin, pair_iou_begin, pair_cat, entry_det, det_area,
                   gt_area, gt_flags, ious, num_entries):
    """evaluateImg at maxDets[-1] for every pair and area range.  Returns (entry_flags (A, E) uint32 as int32 bits, npig (K, A))."""
    import ctypes
    import numpy as np
    thr = np.ascontiguousarray(iou_thrs, np.float64)
    rng = np.ascontiguousarray(area_rng, np.float64).reshape(-1)
    A, dev = rng.size // 2, ious.device
    flags = torch.zeros((A, max(num_entries, 1)), dtype=torch.int32, device=dev)
    npig = torch.zeros((num_cats, A), dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.load().b200_coco_match(pair_gt_begin.numel() - 1, thr.size, thr.ctypes.data_as(ctypes.c_void_p), A,
                                               rng.ctypes.data_as(ctypes.c_void_p), int(max_gt), pair_gt_begin.data_ptr(),
                                               pair_entry_begin.data_ptr(), pair_iou_begin.data_ptr(), pair_cat.data_ptr(), entry_det.data_ptr(),
                                               det_area.data_ptr(), gt_area.data_ptr(), gt_flags.data_ptr(), ious.data_ptr(), num_entries,
                                               flags.data_ptr(), npig.data_ptr(), _stream()), "b200_coco_match")
    return flags, npig


def coco_accumulate_raw(max_dets, cat_entry_begin, cat_pairs, order, entry_rank, entry_score, entry_flags, npig, rec_thrs, T, num_entries,
                        max_cat_entries):
    """accumulate(): precision / scores (T, R, K, A, M) and recall (T, K, A, M) float64 on the device, -1 where COCOeval skips.
    max_cat_entries: the largest category's entry count (host int, < 2^21)."""
    import ctypes
    import numpy as np
    md = np.ascontiguousarray(max_dets, np.int32)
    K, A = npig.shape
    M, R, dev = md.size, rec_thrs.numel(), npig.device
    precision = torch.full((T, R, K, A, M), -1.0, dtype=torch.float64, device=dev)
    scores = torch.full((T, R, K, A, M), -1.0, dtype=torch.float64, device=dev)
    recall = torch.full((T, K, A, M), -1.0, dtype=torch.float64, device=dev)
    ws_bytes = A * M * num_entries * 20
    ws = torch.empty((max(ws_bytes // 8, 1),), dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.load().b200_coco_accumulate(K, A, M, T, R, md.ctypes.data_as(ctypes.c_void_p), cat_entry_begin.data_ptr(),
                                                    cat_pairs.data_ptr(), order.data_ptr(), entry_rank.data_ptr(), entry_score.data_ptr(),
                                                    entry_flags.data_ptr(), num_entries, int(max_cat_entries), npig.data_ptr(), rec_thrs.data_ptr(), ws.data_ptr(),
                                                    ws_bytes, precision.data_ptr(), recall.data_ptr(), scores.data_ptr(), _stream()),
                   "b200_coco_accumulate")
    return precision, recall, scores


# ------------------------------------------------------------------------------------------------
# PASCAL VOC evaluation (the reference's voc_eval loop; datasets/voc_eval.py drives it)
# ------------------------------------------------------------------------------------------------
def voc_match_raw(pair_gt_begin, gt_box, gt_difficult, det_pair, det_box, ovthresh):
    """tp / fp / neither of every detection (uint8 1 / 0 / 2), detections in rank order within each class.  pair_gt_begin
    (P + 1) int32, gt_box (G, 4) float64, gt_difficult (G,) uint8, det_pair (D,) int32, det_box (D, 4) float64, all on one device."""
    D, G, dev = det_pair.numel(), gt_difficult.numel(), det_pair.device
    outcome = torch.empty((max(D, 1),), dtype=torch.uint8, device=dev)
    ws = torch.empty((max(G, 1),), dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.load().b200_voc_match(D, pair_gt_begin.numel() - 1, G, float(ovthresh), pair_gt_begin.data_ptr(), gt_box.data_ptr(),
                                              gt_difficult.data_ptr(), det_pair.data_ptr(), det_box.data_ptr(), ws.data_ptr(),
                                              outcome.data_ptr(), _stream()), "b200_voc_match")
    return outcome[:D]


# ------------------------------------------------------------------------------------------------
# Proposal recall (the reference's evaluate_box_proposals; datasets/json_dataset_evaluator.py drives it)
# ------------------------------------------------------------------------------------------------
def _offsets_ok(begin, rows):
    b = begin.cpu()
    return b.numel() >= 1 and int(b[0]) == 0 and int(b[-1]) == rows and bool((b[1:] >= b[:-1]).all())


def box_proposal_match_raw(prop_box, prop_begin, gt_box, gt_area, gt_begin, prop_count, area_ranges, thresholds):
    """The greedy proposal-to-gt assignment of every (limit, area range, image) in one launch.
    prop_box (P, 4) and prop_begin (N + 1): each image's proposals in the reference's order (e.g. GenerateProposalsOp's
    rois[:, 1:] / im_scale); gt_box (G, 4), gt_area (G,) and gt_begin (N + 1): each image's non-crowd foreground gt boxes and
    seg_areas; prop_count (L, N): the proposals each limit keeps (json_dataset_evaluator.effective_proposal_counts).  All are CUDA
    tensors on one device; boxes are evaluated as float32, gt_area as float64 and the offsets and counts as int32 (other dtypes are
    converted, as the reference casts its boxes with astype(np.float32)).  The offsets must start at 0, not decrease and end at P / G.
    area_ranges: A <= 8 host pairs [lo, hi]; thresholds: T float64 values (host sequence or device tensor).
    Returns overlap (L, A, G) float32 (the recorded IoU, 0 if unmatched), excluded (L, A, G) bool (not part of gt_overlaps: out of range
    or image without proposals), error (L, A, N) bool (a NaN IoU fails the reference's assert) and counts (L, A, T) int64 (counted gts
    whose float64 overlap is >= each threshold, over the images without error)."""
    named = (("prop_box", prop_box), ("prop_begin", prop_begin), ("gt_box", gt_box), ("gt_area", gt_area), ("gt_begin", gt_begin),
             ("prop_count", prop_count))
    for name, t in named:
        if not isinstance(t, torch.Tensor) or not t.is_cuda:
            raise ValueError("box_proposal_match_raw: %s must be a CUDA tensor" % name)
    dev = prop_begin.device
    if any(t.device != dev for _, t in named):
        raise ValueError("box_proposal_match_raw: all tensors must be on one device, got %s" % ([str(t.device) for _, t in named],))
    prop_box = prop_box.to(torch.float32).contiguous()
    gt_box = gt_box.to(torch.float32).contiguous()
    gt_area = gt_area.to(torch.float64).contiguous()
    prop_begin, gt_begin, prop_count = (t.to(torch.int32).contiguous() for t in (prop_begin, gt_begin, prop_count))
    if prop_box.dim() != 2 or prop_box.shape[1] != 4 or gt_box.dim() != 2 or gt_box.shape[1] != 4:
        raise ValueError("box_proposal_match_raw: prop_box and gt_box must be (rows, 4), got %s and %s"
                         % (tuple(prop_box.shape), tuple(gt_box.shape)))
    N, P, G = prop_begin.numel() - 1, prop_box.shape[0], gt_box.shape[0]
    if prop_begin.dim() != 1 or gt_begin.shape != prop_begin.shape or gt_area.shape != (G,):
        raise ValueError("box_proposal_match_raw: prop_begin and gt_begin must both be (N + 1,) and gt_area (G,)")
    if prop_count.dim() != 2 or prop_count.shape[1] != N:
        raise ValueError("box_proposal_match_raw: prop_count must be (L, %d), got %s" % (N, tuple(prop_count.shape)))
    if not _offsets_ok(prop_begin, P) or not _offsets_ok(gt_begin, G):
        raise ValueError("box_proposal_match_raw: row offsets must start at 0, not decrease and end at the row count")
    L = prop_count.shape[0]
    ranges = np.ascontiguousarray(np.asarray(area_ranges, np.float64).reshape(-1, 2))
    A = ranges.shape[0]
    thr = torch.as_tensor(thresholds, dtype=torch.float64, device=dev).reshape(-1).contiguous()
    T = thr.numel()
    overlap = torch.empty((L, A, G), dtype=torch.float32, device=dev)
    excluded = torch.empty((L, A, G), dtype=torch.uint8, device=dev)
    error = torch.empty((L, A, N), dtype=torch.uint8, device=dev)
    counts = torch.zeros((L, A, T), dtype=torch.int64, device=dev)
    lib = _lib.load()
    ws = torch.empty((lib.b200_box_proposal_match_workspace_bytes(P, G, A, L),), dtype=torch.uint8, device=dev)
    ptr = lambda t: t.data_ptr() if t.numel() else None  # noqa: E731
    with torch.cuda.device(dev):
        _lib.check(lib.b200_box_proposal_match(N, P, G, A, L, T, ptr(prop_box), prop_begin.data_ptr(), ptr(gt_box), ptr(gt_area),
                                               gt_begin.data_ptr(), prop_count.data_ptr(), ranges.ctypes.data, ptr(thr), ws.data_ptr(),
                                               ws.numel(), ptr(overlap), ptr(excluded), error.data_ptr(), ptr(counts), _stream()),
                   "b200_box_proposal_match")
    return overlap, excluded.bool(), error.bool(), counts


# ------------------------------------------------------------------------------------------------
# Training losses: RPN (single-scale and FPN) and Fast R-CNN, forward and backward in one launch each
# ------------------------------------------------------------------------------------------------
class _RpnLossLevel(ctypes.Structure):
    _fields_ = [(n, ctypes.c_void_p) for n in ("cls_logits", "bbox_pred", "labels_wide", "bbox_targets_wide", "bbox_inside_wide",
                                               "bbox_outside_wide", "cls_grad", "bbox_grad")] + \
               [(n, ctypes.c_int) for n in ("num_images", "num_anchors", "cls_channels", "h", "w", "hb", "wb", "label_h", "label_w",
                                            "target_h", "target_w")]


RPN_LOSS_MAX_LEVELS = 8
_loss_workspaces = {}


def _loss_workspace(dev, num_levels):
    """The zero-filled workspace of the loss kernels, one per (device, stream): the kernels leave it zero after every call, and
    calls on one stream never overlap."""
    key = (dev.index, _stream())
    need = int(_lib.load().b200_loss_workspace_bytes(num_levels))
    ws = _loss_workspaces.get(key)
    if ws is None or ws.numel() < need:
        ws = torch.zeros((max(need, int(_lib.load().b200_loss_workspace_bytes(RPN_LOSS_MAX_LEVELS))),), dtype=torch.uint8, device=dev)
        _loss_workspaces[key] = ws
    return ws


def _target(x, dtype, dev, name):
    """A target blob on `dev` in `dtype` (numpy arrays are uploaded); predictions are never converted."""
    t = torch.as_tensor(x)
    if t.device != dev or t.dtype != dtype:
        t = t.to(device=dev, dtype=dtype)
    return t.contiguous()


def _rpn_levels_desc(cls, bbox, targets, softmax, grads=None):
    descs = (_RpnLossLevel * len(cls))()
    for l, (c, b, (lab, tg, wi, wo)) in enumerate(zip(cls, bbox, targets)):
        d = descs[l]
        d.cls_logits, d.bbox_pred, d.labels_wide = c.data_ptr(), b.data_ptr(), lab.data_ptr()
        d.bbox_targets_wide, d.bbox_inside_wide, d.bbox_outside_wide = tg.data_ptr(), wi.data_ptr(), wo.data_ptr()
        if grads is not None:
            d.cls_grad, d.bbox_grad = grads[0][l].data_ptr(), grads[1][l].data_ptr()
        d.num_images, d.cls_channels, d.h, d.w = c.shape
        d.num_anchors = c.shape[1] // 2 if softmax else c.shape[1]
        d.hb, d.wb = b.shape[2], b.shape[3]
        d.label_h, d.label_w = lab.shape[2], lab.shape[3]
        d.target_h, d.target_w = tg.shape[2], tg.shape[3]
    return descs


class RpnLossFunction(Function):
    """losses (L, 2) = per level (loss_cls, loss_bbox), and the per-level cls divisor (not differentiable).
    apply(L, softmax, fixed_divisor, *cls_logits, *bbox_pred, *(labels, targets, inside, outside) per level)."""

    @staticmethod
    def forward(ctx, L, softmax, fixed_divisor, *tensors):
        cls, bbox = tensors[:L], tensors[L:2 * L]
        targets = [tensors[2 * L + 4 * l:2 * L + 4 * l + 4] for l in range(L)]
        dev = cls[0].device
        descs = _rpn_levels_desc(cls, bbox, targets, softmax)
        losses = torch.empty((L, 2), dtype=torch.float32, device=dev)
        divisor = torch.empty((L,), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            ws = _loss_workspace(dev, L)
            _lib.check(_lib.load().b200_rpn_loss_forward(L, ctypes.cast(descs, ctypes.c_void_p), int(softmax), float(fixed_divisor),
                                                         ws.data_ptr(), ws.numel(), losses.data_ptr(), divisor.data_ptr(), _stream()),
                       "b200_rpn_loss_forward")
        ctx.mark_non_differentiable(divisor)
        ctx.L, ctx.softmax = L, softmax
        ctx.save_for_backward(divisor, *tensors)
        return losses, divisor

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_losses, _grad_divisor):
        divisor, *tensors = ctx.saved_tensors
        L = ctx.L
        cls, bbox = tensors[:L], tensors[L:2 * L]
        targets = [tensors[2 * L + 4 * l:2 * L + 4 * l + 4] for l in range(L)]
        grads = ([torch.empty_like(c) for c in cls], [torch.empty_like(b) for b in bbox])
        descs = _rpn_levels_desc(cls, bbox, targets, ctx.softmax, grads)
        g = grad_losses.to(torch.float32).contiguous()
        with torch.cuda.device(g.device):
            _lib.check(_lib.load().b200_rpn_loss_backward(L, ctypes.cast(descs, ctypes.c_void_p), int(ctx.softmax), g.data_ptr(),
                                                          divisor.data_ptr(), _stream()), "b200_rpn_loss_backward")
        return (None, None, None) + tuple(grads[0]) + tuple(grads[1]) + (None,) * (4 * L)


def _shape4(t, name):
    if t.dim() != 4:
        raise ValueError("%s must be 4-D (N, C, H, W), got %s" % (name, tuple(t.shape)))
    return tuple(t.shape)


def rpn_losses(levels, softmax=False, fixed_divisor=0.0):
    """The RPN losses of every level in one launch (and one for the backward).  levels: per level (rpn_cls_logits, rpn_bbox_pred,
    labels_int32_wide, bbox_targets_wide, bbox_inside_weights_wide, bbox_outside_weights_wide): float32 CUDA predictions
    (N, A or 2A (softmax), h, w) and (N, 4A, hb, wb); the wide target blobs (N, A, >= h, >= w) and (N, 4A, >= hb, >= wb), tensors or
    numpy arrays, read in their [:h, :w] window in place.  fixed_divisor > 0 (sigmoid only) divides every level's cls sum by it
    instead of by its count of labels >= 0.  Returns the (L, 2) tensor of (loss_cls, loss_bbox) per level."""
    L = len(levels)
    if not 1 <= L <= RPN_LOSS_MAX_LEVELS:
        raise ValueError("rpn_losses takes 1 .. %d levels, got %d" % (RPN_LOSS_MAX_LEVELS, L))
    cls, bbox, targets = [], [], []
    dev = None
    for l, lv in enumerate(levels):
        if len(lv) != 6:
            raise ValueError("level %d: expected (cls_logits, bbox_pred, labels, targets, inside, outside)" % l)
        c, b = lv[0], lv[1]
        _need_cuda_f32(c, "rpn_cls_logits"); _need_cuda_f32(b, "rpn_bbox_pred")
        dev = c.device if dev is None else dev
        if c.device != dev or b.device != dev:
            raise ValueError("level %d: every prediction must be on %s" % (l, dev))
        N, Cc, h, w = _shape4(c, "rpn_cls_logits")
        Nb, Cb, hb, wb = _shape4(b, "rpn_bbox_pred")
        if softmax and Cc % 2:
            raise ValueError("level %d: softmax rpn_cls_logits needs 2A channels, got %d" % (l, Cc))
        A = Cc // 2 if softmax else Cc
        if Nb != N or Cb != 4 * A:
            raise ValueError("level %d: rpn_bbox_pred %s does not match rpn_cls_logits %s (expected (%d, %d, h, w))"
                             % (l, (Nb, Cb, hb, wb), (N, Cc, h, w), N, 4 * A))
        lab = _target(lv[2], torch.int32, dev, "rpn_labels_int32_wide")
        t3 = [_target(x, torch.float32, dev, "rpn_bbox_*_wide") for x in lv[3:]]
        Nl, Al, Hl, Wl = _shape4(lab, "rpn_labels_int32_wide")
        if Nl != N or Al != A or Hl < h or Wl < w:
            raise ValueError("level %d: rpn_labels_int32_wide %s cannot be narrowed to (%d, %d, %d, %d)" % (l, (Nl, Al, Hl, Wl), N, A, h, w))
        ts = _shape4(t3[0], "rpn_bbox_targets_wide")
        if any(tuple(x.shape) != ts for x in t3) or ts[0] != N or ts[1] != 4 * A or ts[2] < hb or ts[3] < wb:
            raise ValueError("level %d: the bbox target / weight blobs %s cannot be narrowed to (%d, %d, %d, %d)"
                             % (l, [tuple(x.shape) for x in t3], N, 4 * A, hb, wb))
        if N * Cc * h * w >= 2 ** 31 or N * 4 * A * hb * wb >= 2 ** 31:
            raise ValueError("level %d: more than 2^31 - 1 prediction elements" % l)
        cls.append(c.contiguous()); bbox.append(b.contiguous())
        targets += [lab] + t3
    losses, _ = RpnLossFunction.apply(L, bool(softmax), float(fixed_divisor), *cls, *bbox, *targets)
    return losses


class FastRcnnLossFunction(Function):
    """apply(cls_score, bbox_pred, labels, targets, inside, outside) -> (losses (2,) = (loss_cls, loss_bbox), accuracy ())."""

    @staticmethod
    def forward(ctx, cls_score, bbox_pred, labels, targets, inside, outside):
        dev = cls_score.device
        R, C = cls_score.shape
        B = bbox_pred.shape[1]
        losses = torch.empty((2,), dtype=torch.float32, device=dev)
        accuracy = torch.empty((), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            ws = _loss_workspace(dev, 1)
            _lib.check(_lib.load().b200_fast_rcnn_loss_forward(R, C, B, cls_score.data_ptr(), bbox_pred.data_ptr(), labels.data_ptr(),
                                                               int(labels.dtype == torch.int64), targets.data_ptr(), inside.data_ptr(),
                                                               outside.data_ptr(), ws.data_ptr(), ws.numel(), losses.data_ptr(),
                                                               accuracy.data_ptr(), _stream()), "b200_fast_rcnn_loss_forward")
        ctx.mark_non_differentiable(accuracy)
        ctx.save_for_backward(cls_score, bbox_pred, labels, targets, inside, outside)
        return losses, accuracy

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_losses, _grad_accuracy):
        cls_score, bbox_pred, labels, targets, inside, outside = ctx.saved_tensors
        R, C = cls_score.shape
        B = bbox_pred.shape[1]
        d_cls = torch.empty_like(cls_score) if ctx.needs_input_grad[0] else None
        d_bbox = torch.empty_like(bbox_pred) if ctx.needs_input_grad[1] else None
        if d_cls is None and d_bbox is None:
            return None, None, None, None, None, None
        g = grad_losses.to(torch.float32).contiguous()
        with torch.cuda.device(g.device):
            _lib.check(_lib.load().b200_fast_rcnn_loss_backward(R, C, B, cls_score.data_ptr(), bbox_pred.data_ptr(), labels.data_ptr(),
                                                                int(labels.dtype == torch.int64), targets.data_ptr(), inside.data_ptr(),
                                                                outside.data_ptr(), g.data_ptr(), d_cls.data_ptr() if d_cls is not None else None,
                                                                d_bbox.data_ptr() if d_bbox is not None else None, _stream()),
                       "b200_fast_rcnn_loss_backward")
        return d_cls, d_bbox, None, None, None, None


def fast_rcnn_losses(cls_score, bbox_pred, label_int32, bbox_targets, bbox_inside_weights, bbox_outside_weights):
    """(loss_cls, loss_bbox, accuracy_cls) as 0-d CUDA tensors, in one launch (one more for the backward).  cls_score (R, C) and
    bbox_pred (R, B) float32 CUDA; labels (R,) int32 / int64 and the three (R, B) blobs as tensors or numpy arrays (uploaded).
    Host labels outside [0, C) raise ValueError; a device label outside [0, C) gives a NaN loss_cls."""
    _need_cuda_f32(cls_score, "cls_score"); _need_cuda_f32(bbox_pred, "bbox_pred")
    dev = cls_score.device
    if bbox_pred.device != dev:
        raise ValueError("cls_score and bbox_pred must be on the same device")
    if (cls_score.dim() != 2 or bbox_pred.dim() != 2 or bbox_pred.shape[0] != cls_score.shape[0] or bbox_pred.shape[1] % 4
            or bbox_pred.shape[1] == 0):
        raise ValueError("cls_score must be (R, C) and bbox_pred (R, 4 C'), got %s and %s" % (tuple(cls_score.shape), tuple(bbox_pred.shape)))
    R, C = cls_score.shape
    if R == 0 or C == 0:
        raise ValueError("fast_rcnn_losses needs at least one RoI and one class, got cls_score %s" % (tuple(cls_score.shape),))
    if not torch.is_tensor(label_int32):
        lab_h = np.asarray(label_int32)
        if lab_h.size and (lab_h.min() < 0 or lab_h.max() >= C):
            raise ValueError("label_int32 must lie in [0, %d), got [%d, %d]" % (C, lab_h.min(), lab_h.max()))
    labels = torch.as_tensor(label_int32)
    if labels.dtype not in (torch.int32, torch.int64):
        raise ValueError("label_int32 must be int32 or int64, got %s" % labels.dtype)
    labels = _target(labels, labels.dtype, dev, "label_int32").reshape(-1)
    if labels.numel() != R:
        raise ValueError("label_int32 has %d entries for %d RoIs" % (labels.numel(), R))
    blobs = [_target(x, torch.float32, dev, n) for x, n in ((bbox_targets, "bbox_targets"), (bbox_inside_weights, "bbox_inside_weights"),
                                                           (bbox_outside_weights, "bbox_outside_weights"))]
    for t, n in zip(blobs, ("bbox_targets", "bbox_inside_weights", "bbox_outside_weights")):
        if tuple(t.shape) != tuple(bbox_pred.shape):
            raise ValueError("%s %s does not match bbox_pred %s" % (n, tuple(t.shape), tuple(bbox_pred.shape)))
    losses, accuracy = FastRcnnLossFunction.apply(cls_score.contiguous(), bbox_pred.contiguous(), labels, *blobs)
    loss_cls, loss_bbox = losses.unbind(0)
    return loss_cls, loss_bbox, accuracy
