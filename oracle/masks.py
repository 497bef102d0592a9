"""TEST INFRASTRUCTURE (CPU oracle, never imported by the product): the Mask R-CNN training mask targets
(lib/roi_data/mask_rcnn.py:34-122 with lib/utils/segms.py:93-131), restated in numpy, and the polygon rasteriser they call.

The rasteriser is pycocotools' published algorithm (maskApi.c rleFrPoly + rleDecode, BSD), restated step by step:

  vertices   x[j] = (int)(5 * xy[2j] + .5), C truncation toward zero; the ring is closed (x[k] = x[0])
  walk       every edge upsampled to integer points, start and end swapped when `flip`, interpolated coordinate
             (int)(ys + s * t + .5) in double with separate roundings; all edges appended (shared vertices appear twice)
  crossings  consecutive walk points whose u differs give a column xd = (min-side u + .5) / 5 - .5, kept when it is an
             integer in [0, w - 1]; its row yd = ceil(clamp((min(v) + .5) / 5 - .5, 0, h))
  RLE        toggles at column-major positions xd * h + yd, a sentinel at h * w, sorted, differenced, zero runs merged
  decode     runs alternate 0 / 1 starting with 0, column-major

A degenerate edge (dx = dy = 0) divides 0 by 0; its v is what x86's cvttsd2si gives for NaN, INT_MIN, and the crossing logic
never reads it (its u equals its neighbours' wherever a crossing could be kept).

Pinned by tests/golden/mask_targets.npz, produced by the UNMODIFIED reference add_mask_rcnn_blobs with this module's
frPyObjects / decode in place of pycocotools.mask (tests/golden/make_golden_masks.py), and by hand-derived known answers.
"""
import numpy as np

f32 = np.float32
SCALE = 5.0
INT_MIN = -2 ** 31


def _trunc_int(a):
    return np.trunc(a).astype(np.int64)


def upsampled_walk(xy):
    """The (u, v) walk of one polygon (float64 flat [x0, y0, x1, y1, ...]); int64 arrays."""
    xy = np.asarray(xy, dtype=np.float64)
    k = xy.size // 2
    x = np.empty(k + 1, np.int64); y = np.empty(k + 1, np.int64)
    x[:k] = _trunc_int(SCALE * xy[0:2 * k:2] + .5); x[k] = x[0]
    y[:k] = _trunc_int(SCALE * xy[1:2 * k:2] + .5); y[k] = y[0]
    us, vs = [], []
    for j in range(k):
        xs, xe, ys, ye = int(x[j]), int(x[j + 1]), int(y[j]), int(y[j + 1])
        dx, dy = abs(xe - xs), abs(ys - ye)
        flip = (dx >= dy and xs > xe) or (dx < dy and ys > ye)
        if flip:
            xs, xe = xe, xs
            ys, ye = ye, ys
        if dx >= dy:
            d = np.arange(dx + 1, dtype=np.int64)
            t = dx - d if flip else d
            u = t + xs
            if dx == 0:
                v = np.full(1, INT_MIN, np.int64)                       # (int)(ys + NaN * 0 + .5) on x86
            else:
                s = float(ye - ys) / dx
                v = _trunc_int((float(ys) + s * t.astype(np.float64)) + .5)
        else:
            d = np.arange(dy + 1, dtype=np.int64)
            t = dy - d if flip else d
            v = t + ys
            s = float(xe - xs) / dy
            u = _trunc_int((float(xs) + s * t.astype(np.float64)) + .5)
        us.append(u); vs.append(v)
    if not us:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    return np.concatenate(us), np.concatenate(vs)


def toggles(xy, h, w):
    """Column-major toggle positions of one polygon (crossings only, no sentinel), in walk order."""
    u, v = upsampled_walk(xy)
    if u.size < 2:
        return np.zeros(0, np.int64)
    u0, u1, v0, v1 = u[:-1], u[1:], v[:-1], v[1:]
    sel = u1 != u0
    u0, u1, v0, v1 = u0[sel], u1[sel], v0[sel], v1[sel]
    xd = np.where(u1 < u0, u1, u1 - 1).astype(np.float64)
    xd = (xd + .5) / SCALE - .5
    keep = (np.floor(xd) == xd) & (xd >= 0) & (xd <= w - 1)
    xd, v0, v1 = xd[keep], v0[keep], v1[keep]
    yd = np.minimum(v0, v1).astype(np.float64)
    yd = (yd + .5) / SCALE - .5
    yd = np.ceil(np.clip(yd, 0, h))
    return xd.astype(np.int64) * h + yd.astype(np.int64)


def rle_fr_poly(xy, h, w):
    """rleFrPoly: uncompressed RLE counts (uint32) of one polygon on an h x w grid."""
    a = np.sort(np.concatenate([toggles(xy, h, w), [h * w]]))
    a = np.diff(np.concatenate([[0], a]))
    b = [int(a[0])]
    j = 1
    while j < a.size:
        if a[j] > 0:
            b.append(int(a[j])); j += 1
        else:
            j += 1
            if j < a.size:
                b[-1] += int(a[j]); j += 1
    return np.asarray(b, np.uint32)


def rle_decode(counts, h, w):
    """rleDecode: (h, w) uint8 from alternating 0 / 1 runs, column-major."""
    flat = np.zeros(h * w, np.uint8)
    p, val = 0, 0
    for c in counts:
        flat[p:p + int(c)] = val
        p += int(c); val = 1 - val
    return flat.reshape(w, h).T


def frPyObjects(pyobj, h, w):
    """pycocotools.mask.frPyObjects for a list of polygons (the only form add_mask_rcnn_blobs passes): one RLE per polygon."""
    if not isinstance(pyobj, list) or not pyobj or len(pyobj[0]) <= 4:
        raise NotImplementedError("only lists of polygons with more than 4 values are restated")
    return [{"size": [h, w], "counts": rle_fr_poly(np.asarray(p, np.float64), h, w)} for p in pyobj]


def decode(rles):
    """pycocotools.mask.decode: (h, w, n) uint8 for a list of RLEs, (h, w) for one."""
    if isinstance(rles, list):
        return np.stack([rle_decode(r["counts"], *r["size"]) for r in rles], axis=2)
    return rle_decode(rles["counts"], *rles["size"])


def polys_to_boxes(polys):
    """segms.polys_to_boxes: tight float32 box of each object's polygons."""
    out = np.zeros((len(polys), 4), f32)
    for i, poly in enumerate(polys):
        out[i] = [min(min(p[::2]) for p in poly), min(min(p[1::2]) for p in poly), max(max(p[::2]) for p in poly),
                  max(max(p[1::2]) for p in poly)]
    return out


def normalise(poly, box, M):
    """segms.polys_to_mask_wrt_box's float32 normalisation of one polygon to the box."""
    box = np.asarray(box, f32)
    w = np.maximum(box[2] - box[0], f32(1)); h = np.maximum(box[3] - box[1], f32(1))
    p = np.array(poly, dtype=f32)
    p[0::2] = (p[0::2] - box[0]) * f32(M) / w
    p[1::2] = (p[1::2] - box[1]) * f32(M) / h
    return p


def polys_to_mask_wrt_box(polygons, box, M):
    """(M, M) uint8 union of the object's polygons rasterised relative to the box, [y][x]."""
    m = decode(frPyObjects([normalise(p, box, M) for p in polygons], M, M))
    return (np.sum(m, axis=2) > 0).astype(np.uint8)


def add_mask_rcnn_blobs(blobs, sampled_boxes, roidb, im_scale, batch_idx, M=14, cls_specific=True, num_classes=81):
    """mask_rcnn.add_mask_rcnn_blobs for one image; adds mask_rois, roi_has_mask_int32, masks_int32 (numpy) to `blobs`."""
    from oracle.targets import bbox_overlaps
    inds = np.where((np.asarray(roidb["gt_classes"]) > 0) & (np.asarray(roidb["is_crowd"]) == 0))[0]
    polys_gt = [roidb["segms"][i] for i in inds]
    labels = np.asarray(blobs["labels_int32"])
    fg = np.where(labels > 0)[0]
    roi_has_mask = labels.copy()
    roi_has_mask[roi_has_mask > 0] = 1
    sampled_boxes = np.asarray(sampled_boxes, f32)
    if fg.size > 0:
        cls = labels[fg]
        rois = sampled_boxes[fg]
        ov = bbox_overlaps(rois, polys_to_boxes(polys_gt))
        if ov.shape[1] == 0:
            raise ValueError("fg RoIs but no non-crowd polygon (np.argmax of an empty row)")
        arg = np.argmax(ov, axis=1)
        masks = np.zeros((fg.size, M * M), np.int32)
        for i in range(fg.size):
            masks[i] = polys_to_mask_wrt_box(polys_gt[arg[i]], rois[i], M).reshape(-1)
    else:
        bg = np.where(labels == 0)[0]
        if bg.size == 0:
            raise ValueError("no RoI at all")
        rois = sampled_boxes[bg[0]].reshape(1, -1).copy()
        masks = -np.ones((1, M * M), np.int32)
        cls = np.zeros(1, np.int32)
        roi_has_mask[0] = 1
    if cls_specific:
        out = -np.ones((masks.shape[0], num_classes * M * M), np.int32)
        for i in range(masks.shape[0]):
            c = int(cls[i])
            if c > 0:
                out[i, c * M * M:(c + 1) * M * M] = masks[i]
        masks = out
    rois = rois * f32(im_scale)
    blobs["mask_rois"] = np.hstack([np.full((rois.shape[0], 1), batch_idx, f32), rois]).astype(f32)
    blobs["roi_has_mask_int32"] = roi_has_mask.astype(np.int32)
    blobs["masks_int32"] = masks
    return blobs
