"""COCOeval's evaluate() and accumulate() on the device, with its summarize() on the host.

`evaluate(coco_gt_dataset, dets, iou_type)` takes the ground truth as the annotation-file dict and the detections as the
reference's results writers would produce them (json_dataset_evaluator.py here converts all_boxes / all_segms / all_keyps),
and returns a `CocoEvalResult` shaped like pycocotools' COCOeval after accumulate(): `.params`, `.eval` ('precision',
'recall', 'scores' as float64 numpy arrays) and, after `.summarize()`, `.stats`.

The host packs detections and ground truth per (image, category) pair, image-major, and uploads them once (masks once per chunk
of images).  The device ranks, scores, matches and accumulates (csrc/coco_eval.cu); the ordering of the accumulation is one
pair of stable torch sorts.  Differences from pycocotools, all on inputs pycocotools rejects or mishandles: an empty results list
is evaluated as no detections (loadRes raises on it), and a mask whose size is not its image's is refused (rleIou scores it -1).
"""
import numpy as np
import torch

from .. import ops

KPT_OKS_SIGMAS = np.array([.26, .25, .25, .35, .35, .79, .79, .72, .72, .62, .62, 1.07, 1.07, .87, .87, .89, .89]) / 10.0
MASK_CHUNK_WORDS = 1 << 28                                               # at most 1 GiB of mask bitmaps per chunk of images
MASK_COORD_LIMIT = float(2 ** 20)


class Params:
    """pycocotools' Params for one iouType (useCats = 1)."""

    def __init__(self, iouType="segm"):
        self.imgIds, self.catIds = [], []
        self.iouThrs = np.linspace(.5, 0.95, int(np.round((0.95 - .5) / .05)) + 1, endpoint=True)
        self.recThrs = np.linspace(.0, 1.00, int(np.round((1.00 - .0) / .01)) + 1, endpoint=True)
        if iouType == "keypoints":
            self.maxDets = [20]
            self.areaRng = [[0 ** 2, 1e5 ** 2], [32 ** 2, 96 ** 2], [96 ** 2, 1e5 ** 2]]
            self.areaRngLbl = ["all", "medium", "large"]
        else:
            self.maxDets = [1, 10, 100]
            self.areaRng = [[0 ** 2, 1e5 ** 2], [0 ** 2, 32 ** 2], [32 ** 2, 96 ** 2], [96 ** 2, 1e5 ** 2]]
            self.areaRngLbl = ["all", "small", "medium", "large"]
        self.useCats = 1
        self.kpt_oks_sigmas = KPT_OKS_SIGMAS.copy()
        self.iouType = iouType
        self.useSegm = None


def summarize(ev, p, out=print):
    """COCOeval.summarize on the accumulated arrays: 12 stats (bbox, segm) or 10 (keypoints), each the mean over s > -1."""
    def _summarize(ap=1, iouThr=None, areaRng="all", maxDets=100):
        iStr = " {:<18} {} @[ IoU={:<9} | area={:>6s} | maxDets={:>3d} ] = {:0.3f}"
        titleStr = "Average Precision" if ap == 1 else "Average Recall"
        typeStr = "(AP)" if ap == 1 else "(AR)"
        iouStr = "{:0.2f}:{:0.2f}".format(p.iouThrs[0], p.iouThrs[-1]) if iouThr is None else "{:0.2f}".format(iouThr)
        aind = [i for i, aRng in enumerate(p.areaRngLbl) if aRng == areaRng]
        mind = [i for i, mDet in enumerate(p.maxDets) if mDet == maxDets]
        s = ev["precision"] if ap == 1 else ev["recall"]
        if iouThr is not None:
            s = s[np.where(iouThr == p.iouThrs)[0]]
        s = s[:, :, :, aind, mind] if ap == 1 else s[:, :, aind, mind]
        mean_s = -1 if len(s[s > -1]) == 0 else np.mean(s[s > -1])
        if out is not None:
            out(iStr.format(titleStr, typeStr, iouStr, areaRng, maxDets, mean_s))
        return mean_s

    if p.iouType == "keypoints":
        kinds = [(1, {}), (1, {"iouThr": .5}), (1, {"iouThr": .75}), (1, {"areaRng": "medium"}), (1, {"areaRng": "large"}),
                 (0, {}), (0, {"iouThr": .5}), (0, {"iouThr": .75}), (0, {"areaRng": "medium"}), (0, {"areaRng": "large"})]
        return np.array([_summarize(ap, maxDets=20, **kw) for ap, kw in kinds], dtype=np.float64)
    md = p.maxDets
    stats = np.zeros((12,))
    stats[0] = _summarize(1)
    stats[1] = _summarize(1, iouThr=.5, maxDets=md[2])
    stats[2] = _summarize(1, iouThr=.75, maxDets=md[2])
    stats[3] = _summarize(1, areaRng="small", maxDets=md[2])
    stats[4] = _summarize(1, areaRng="medium", maxDets=md[2])
    stats[5] = _summarize(1, areaRng="large", maxDets=md[2])
    stats[6] = _summarize(0, maxDets=md[0])
    stats[7] = _summarize(0, maxDets=md[1])
    stats[8] = _summarize(0, maxDets=md[2])
    stats[9] = _summarize(0, areaRng="small", maxDets=md[2])
    stats[10] = _summarize(0, areaRng="medium", maxDets=md[2])
    stats[11] = _summarize(0, areaRng="large", maxDets=md[2])
    return stats


class CocoEvalResult:
    """What the reference reads from a COCOeval after accumulate() and summarize(): params, eval, stats."""

    def __init__(self, params, ev):
        self.params = params
        self.eval = ev
        self.stats = []

    def summarize(self, out=print):
        self.stats = summarize(self.eval, self.params, out)


class Detections:
    """The results list as arrays, in results order: image id, category id, score (float64) and one of
    box (n, 4) float64 xywh / strings (list of (bytes, (h, w))) / keypoints (n, 17, 3) float64."""

    def __init__(self, image_id, category_id, score, box=None, strings=None, keypoints=None):
        self.image_id = np.asarray(image_id, np.int64).reshape(-1)
        self.category_id = np.asarray(category_id, np.int64).reshape(-1)
        self.score = np.asarray(score, np.float64).reshape(-1)
        self.box, self.strings, self.keypoints = box, strings, keypoints


def _upload(arrays, dev):
    """One pinned host buffer, one host-to-device copy; returns device tensors viewing it (16-byte aligned each).  An empty
    array comes back as one zero element, so that every table the kernels receive has an address."""
    arrays = [a if a.size else np.zeros((1,) + a.shape[1:], a.dtype) for a in arrays]
    offs, total = [], 0
    for a in arrays:
        offs.append(total)
        total += (a.nbytes + 15) // 16 * 16
    host = torch.empty((max(total, 16),), dtype=torch.uint8, pin_memory=True)
    hv = host.numpy()
    for a, o in zip(arrays, offs):
        hv[o:o + a.nbytes] = np.ascontiguousarray(a).view(np.uint8).reshape(-1)
    buf = host.to(dev, non_blocking=True)
    out = []
    for a, o in zip(arrays, offs):
        t = torch.from_numpy(np.zeros(0, a.dtype)).dtype
        out.append(buf[o:o + a.nbytes].view(t).reshape(a.shape))
    return out, buf, host


def _group(img_idx, cat_idx, K):
    key = img_idx.astype(np.int64) * K + cat_idx
    order = np.argsort(key, kind="stable")
    return key, order


def evaluate(dataset, dets, iou_type, device=None):
    """COCOeval(cocoGt, cocoDt, iou_type).evaluate() + accumulate() on the device.  dataset: the annotation-file dict;
    dets: Detections.  Returns a CocoEvalResult (call .summarize() for stats)."""
    if iou_type not in ("bbox", "segm", "keypoints"):
        raise ValueError("iou_type must be bbox, segm or keypoints, got %r" % (iou_type,))
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    p = Params(iou_type)
    images = {img["id"]: img for img in dataset.get("images", [])}
    p.imgIds = sorted(images)
    p.catIds = sorted(c["id"] for c in dataset.get("categories", []))
    I, K = len(p.imgIds), len(p.catIds)
    T, R, A, M = len(p.iouThrs), len(p.recThrs), len(p.areaRng), len(p.maxDets)
    img_index = {i: n for n, i in enumerate(p.imgIds)}
    cat_index = {c: n for n, c in enumerate(p.catIds)}
    if K == 0 or I == 0:
        raise ValueError("the dataset needs at least one image and one category")

    # ground truth of the evaluated images and categories, annotation order within an image
    anns = [a for a in dataset.get("annotations", []) if a["image_id"] in img_index and a["category_id"] in cat_index]
    g_img = np.array([img_index[a["image_id"]] for a in anns], np.int64)
    g_cat = np.array([cat_index[a["category_id"]] for a in anns], np.int64)
    g_key, g_ord = _group(g_img, g_cat, K)
    anns = [anns[i] for i in g_ord]
    g_key = g_key[g_ord]
    crowd = np.array([int(a["iscrowd"]) for a in anns], np.int32)
    ignore = np.array([1 if ("iscrowd" in a and a["iscrowd"]) else 0 for a in anns], np.int32)
    if iou_type == "keypoints":
        ignore |= np.array([1 if a["num_keypoints"] == 0 else 0 for a in anns], np.int32)
    gt_flags = ((crowd != 0) * 1 | ignore * 2 | np.array([4 if a["id"] != 0 else 0 for a in anns], np.int32)).astype(np.int32)
    gt_area = np.array([a["area"] for a in anns], np.float64)

    # detections, grouped per pair in results order
    for i in np.unique(dets.image_id):
        if int(i) not in img_index:
            raise ValueError("Results do not correspond to current coco set")
    keep = np.array([c in cat_index for c in dets.category_id.tolist()], bool) if dets.category_id.size else np.zeros(0, bool)
    d_img = np.array([img_index[int(i)] for i in dets.image_id[keep]], np.int64)
    d_cat = np.array([cat_index[int(c)] for c in dets.category_id[keep]], np.int64)
    d_sel = np.flatnonzero(keep)
    d_key, d_ord = _group(d_img, d_cat, K)
    d_sel = d_sel[d_ord]
    d_key = d_key[d_ord]
    score = dets.score[d_sel]
    if not np.isfinite(score).all():
        raise ValueError("detection scores must be finite")

    pair_key = np.union1d(d_key, g_key).astype(np.int64)
    P = pair_key.size
    pair_det_begin = np.searchsorted(d_key, pair_key, side="left").astype(np.int32)
    pair_det_begin = np.append(pair_det_begin, d_key.size).astype(np.int32)
    pair_gt_begin = np.append(np.searchsorted(g_key, pair_key, side="left"), g_key.size).astype(np.int32)
    nd = np.diff(pair_det_begin)
    ng = np.diff(pair_gt_begin)
    ne = np.minimum(nd, p.maxDets[-1])
    pair_entry_begin = np.concatenate([[0], np.cumsum(ne)]).astype(np.int32)
    E = int(pair_entry_begin[-1])
    niou = np.where(ng > 0, ne * ng, 0)
    pair_iou_begin = np.concatenate([[0], np.cumsum(niou)]).astype(np.int64)
    pair_cat = (pair_key % K).astype(np.int32)
    pair_img = (pair_key // K).astype(np.int64)
    entry_cat = np.repeat(pair_cat, ne)
    cat_entries = np.bincount(entry_cat, minlength=K)
    cat_entry_begin = np.concatenate([[0], np.cumsum(cat_entries)]).astype(np.int32)
    cat_pairs = np.bincount(pair_cat, minlength=K).astype(np.int32)

    if iou_type == "bbox":
        det_box = np.ascontiguousarray(dets.box[d_sel], np.float64).reshape(-1, 4)
        det_area = det_box[:, 2] * det_box[:, 3]                         # loadRes: bb[2] * bb[3]
        gt_box = np.array([a["bbox"] for a in anns], np.float64).reshape(-1, 4)
        extra = [det_box, gt_box]
    elif iou_type == "keypoints":
        kp = np.ascontiguousarray(dets.keypoints[d_sel], np.float64).reshape(-1, 17, 3)
        x0, x1 = kp[:, :, 0].min(axis=1), kp[:, :, 0].max(axis=1)
        y0, y1 = kp[:, :, 1].min(axis=1), kp[:, :, 1].max(axis=1)
        det_area = (x1 - x0) * (y1 - y0)                                 # loadRes: the keypoints' extent
        gt_kp = np.array([a["keypoints"] for a in anns], np.float64).reshape(-1, 17, 3)
        gt_box = np.array([a["bbox"] for a in anns], np.float64).reshape(-1, 4)
        extra = [kp, gt_kp, gt_box]
    else:
        det_area = np.zeros(d_sel.size, np.float64)                      # the RLE's pixel count, from the device
        extra = []
    host = [pair_det_begin, pair_gt_begin, pair_entry_begin, pair_iou_begin, pair_cat, cat_entry_begin, cat_pairs,
            np.ascontiguousarray(score), np.ascontiguousarray(det_area), gt_area, gt_flags, entry_cat.astype(np.int32),
            p.recThrs.astype(np.float64)] + extra
    dv, _buf, _host = _upload(host, dev)
    (t_pdb, t_pgb, t_peb, t_pib, t_pcat, t_ceb, t_cp, t_score, t_darea, t_garea, t_gflags, t_ecat, t_rec) = dv[:13]
    with torch.cuda.device(dev):
        entry_det, entry_rank, entry_score = ops.coco_rank_raw(t_pdb, t_peb, t_score, E)
        ious = torch.empty((max(int(pair_iou_begin[-1]), 1),), dtype=torch.float64, device=dev)
        if iou_type == "bbox":
            ops.coco_bbox_iou_raw(t_pgb, t_peb, t_pib, entry_det, dv[13], dv[14], t_gflags, ious)
        elif iou_type == "keypoints":
            ops.coco_oks_raw((p.kpt_oks_sigmas * 2) ** 2, t_pgb, t_peb, t_pib, entry_det, dv[13], dv[14], dv[15], t_garea, ious)
        else:
            _segm_ious(dets, d_sel, anns, images, p.imgIds, pair_img, pair_det_begin, pair_gt_begin, t_pgb, t_peb, t_pib, entry_det,
                       t_gflags, t_darea, ious, dev)
        flags, npig = ops.coco_match_raw(p.iouThrs, p.areaRng, int(ng.max()) if P else 0, K, t_pgb, t_peb, t_pib, t_pcat, entry_det,
                                         t_darea, t_garea, t_gflags, ious, E)
        # accumulate()'s order: category, then descending score, ties in (image, rank) order -- two stable sorts
        if E:
            o1 = torch.sort(-entry_score[:E], stable=True).indices
            o2 = torch.sort(t_ecat[o1], stable=True).indices
            order = o1[o2].to(torch.int32)
        else:
            order = torch.zeros((1,), dtype=torch.int32, device=dev)
        precision, recall, scores = ops.coco_accumulate_raw(p.maxDets, t_ceb, t_cp, order, entry_rank, entry_score, flags, npig, t_rec,
                                                            T, E, int(cat_entries.max()))
        out = torch.cat([precision.reshape(-1), recall.reshape(-1), scores.reshape(-1)]).cpu().numpy()
    n1, n2 = T * R * K * A * M, T * K * A * M
    ev = {"params": p, "counts": [T, R, K, A, M], "precision": out[:n1].reshape(T, R, K, A, M),
          "recall": out[n1:n1 + n2].reshape(T, K, A, M), "scores": out[n1 + n2:].reshape(T, R, K, A, M)}
    return CocoEvalResult(p, ev)


def _gt_mask_parts(ann, h, w):
    """annToRLE's input: ('poly', [float64 arrays]) / ('string', bytes) / ('counts', uint32)."""
    segm = ann["segmentation"]
    if isinstance(segm, list):
        polys = []
        for q in segm:
            a = np.asarray(q, np.float64).reshape(-1)
            if a.size < 6 or a.size % 2:
                raise ValueError("a polygon needs an even number (>= 6) of coordinates, got %d" % a.size)
            if not np.isfinite(a).all() or np.abs(a).max() > MASK_COORD_LIMIT:
                raise ValueError("polygon coordinates must be finite and within +-2^20")
            polys.append(a)
        if not polys:
            raise ValueError("an object without polygons")
        return "poly", polys
    if list(segm["size"]) != [h, w]:
        raise ValueError("a ground-truth RLE of size %s on a %d x %d image" % (segm["size"], h, w))
    c = segm["counts"]
    if isinstance(c, list):
        return "counts", np.asarray(c, np.uint32)
    return "string", c.encode("ascii") if isinstance(c, str) else bytes(c)


def _segm_ious(dets, d_sel, anns, images, img_ids, pair_img, pair_det_begin, pair_gt_begin, t_pgb, t_peb, t_pib, entry_det, t_gflags,
               t_darea, ious, dev):
    """Mask IoUs chunk by chunk of images: bitmaps of every detection and ground-truth object, then rleIou per pair."""
    P = pair_img.size
    hw_img = np.array([[images[i]["height"], images[i]["width"]] for i in img_ids], np.int64)
    words_img = (hw_img[:, 0] * hw_img[:, 1] + 31) // 32
    det_strings = [dets.strings[i] for i in d_sel]
    # bitmap words of each pair: one bitmap per detection, one per ground-truth polygon or RLE, at its image's size
    gt_slots = np.array([len(a["segmentation"]) if isinstance(a["segmentation"], list) else 1 for a in anns], np.int64)
    gt_slot_cum = np.concatenate([[0], np.cumsum(gt_slots)])
    pair_slots = np.diff(pair_det_begin).astype(np.int64) + gt_slot_cum[pair_gt_begin[1:]] - gt_slot_cum[pair_gt_begin[:-1]]
    pair_words = pair_slots * words_img[pair_img]
    # chunks of whole images, each within MASK_CHUNK_WORDS unless one image alone needs more
    starts = np.flatnonzero(np.concatenate([[True], pair_img[1:] != pair_img[:-1]])) if P else np.zeros(0, np.int64)
    bounds = np.append(starts, P)
    img_words = np.add.reduceat(pair_words, starts) if P else np.zeros(0, np.int64)
    c0, words = 0, 0
    for n in range(starts.size):
        if n > c0 and words + int(img_words[n]) > MASK_CHUNK_WORDS:
            _segm_chunk(int(bounds[c0]), int(bounds[n]), det_strings, anns, hw_img, words_img, pair_img, pair_det_begin, pair_gt_begin,
                        t_pgb, t_peb, t_pib, entry_det, t_gflags, t_darea, ious, dev)
            c0, words = n, 0
        words += int(img_words[n])
    if starts.size:
        _segm_chunk(int(bounds[c0]), P, det_strings, anns, hw_img, words_img, pair_img, pair_det_begin, pair_gt_begin, t_pgb, t_peb,
                    t_pib, entry_det, t_gflags, t_darea, ious, dev)


def _segm_chunk(p0, p1, det_strings, anns, hw_img, words_img, p_img, pair_det_begin, pair_gt_begin, t_pgb, t_peb, t_pib,
                entry_det, t_gflags, t_darea, ious, dev):
    d0, d1 = int(pair_det_begin[p0]), int(pair_det_begin[p1])
    g0, g1 = int(pair_gt_begin[p0]), int(pair_gt_begin[p1])
    det_img = np.repeat(p_img[p0:p1], np.diff(pair_det_begin[p0:p1 + 1]))
    gt_img = np.repeat(p_img[p0:p1], np.diff(pair_gt_begin[p0:p1 + 1]))
    slot_img, mask_first = [], []
    str_slot, str_parts, cnt_slot, cnt_parts, poly_slot, poly_parts = [], [], [], [], [], []
    for j in range(d1 - d0):
        s, (h, w) = det_strings[d0 + j]
        i = det_img[j]
        if (h, w) != tuple(hw_img[i]):
            raise ValueError("a detection mask of size (%d, %d) on a %d x %d image" % (h, w, hw_img[i][0], hw_img[i][1]))
        mask_first.append(len(slot_img)); slot_img.append(i)
        str_slot.append(len(slot_img) - 1); str_parts.append(s)
    for j in range(g1 - g0):
        i = gt_img[j]
        kind, data = _gt_mask_parts(anns[g0 + j], int(hw_img[i][0]), int(hw_img[i][1]))
        mask_first.append(len(slot_img))
        if kind == "poly":
            for q in data:
                poly_slot.append(len(slot_img)); poly_parts.append(q); slot_img.append(i)
        elif kind == "counts":
            cnt_slot.append(len(slot_img)); cnt_parts.append(data); slot_img.append(i)
        else:
            str_slot.append(len(slot_img)); str_parts.append(data); slot_img.append(i)
    mask_first.append(len(slot_img))
    slot_img = np.asarray(slot_img, np.int64)
    slot_word = np.concatenate([[0], np.cumsum(words_img[slot_img])]).astype(np.int64)
    slot_hw = np.ascontiguousarray(hw_img[slot_img].astype(np.int32))
    str_bytes = np.frombuffer(b"".join(str_parts), np.uint8) if str_parts else np.zeros(0, np.uint8)
    str_begin = np.concatenate([[0], np.cumsum([len(s) for s in str_parts])]).astype(np.int64)
    cnt_data = np.concatenate(cnt_parts).astype(np.uint32) if cnt_parts else np.zeros(0, np.uint32)
    cnt_begin = np.concatenate([[0], np.cumsum([c.size for c in cnt_parts])]).astype(np.int64)
    xy = np.concatenate(poly_parts) if poly_parts else np.zeros(0, np.float64)
    vtx_begin = np.concatenate([[0], np.cumsum([q.size // 2 for q in poly_parts])]).astype(np.int32)
    host = [slot_word, slot_hw, np.asarray(str_slot, np.int32), str_begin, str_bytes, np.asarray(cnt_slot, np.int32), cnt_begin, cnt_data,
            np.asarray(poly_slot, np.int32), vtx_begin, xy, np.asarray(mask_first, np.int32)]
    (t_sw, t_shw, t_ss, t_sb, t_sd, t_cs, t_cb, t_cd, t_ps, t_pb, t_pd, t_msb), _buf, _host = _upload(host, dev)
    n_masks = len(mask_first) - 1
    words = torch.empty((max(int(slot_word[-1]), 1),), dtype=torch.int32, device=dev)
    area = torch.empty((max(n_masks, 1),), dtype=torch.int64, device=dev)
    rng = torch.empty((max(n_masks, 1), 2), dtype=torch.int32, device=dev)
    ops.coco_masks_raw(words, t_sw, t_shw, (t_ss, t_sb, t_sd) if str_slot else None, (t_cs, t_cb, t_cd) if cnt_slot else None,
                       (t_ps, t_pb, t_pd) if poly_slot else None, t_msb, area, rng)
    if d1 > d0:
        t_darea[d0:d1] = area[:d1 - d0].to(torch.float64)
    ops.coco_segm_iou_raw(p0, p1 - p0, t_pgb, t_peb, t_pib, entry_det, d0, g0, d1 - d0, t_msb, t_sw, t_shw, words, area, rng, t_gflags, ious)
