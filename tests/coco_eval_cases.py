"""Seeded synthetic COCO evaluation sets (tests/test_coco_eval.py, tools/coco_eval_probe.py).

make_set() builds an annotation dict and the per-class results lists the reference's test_net hands to evaluate_all:
all_boxes[cls][img] float32 (N, 5), all_segms[cls][img] lists of compressed RLE dicts, all_keyps[cls][img] lists of
(4, 17) float32 arrays (x, y, logit, prob).  Ground truth mixes polygon objects (1-3 polygons of 20-200 vertices),
crowd objects as uncompressed RLEs, a compressed-RLE object, categories without ground truth, images without ground truth
and an image with only crowd ground truth.  results() restates the reference's results writers for the oracle.
"""
import json

import numpy as np

from oracle import segms as OS


def star(rng, cx, cy, rx, ry, k):
    a = np.sort(rng.uniform(0, 2 * np.pi, k))
    r = rng.uniform(0.5, 1.0, k)
    return [float(v) for xy in zip(cx + rx * r * np.cos(a), cy + ry * r * np.sin(a)) for v in xy]


def _rect_counts(h, w, x0, y0, x1, y1):
    m = np.zeros((h, w), np.uint8)
    m[y0:y1, x0:x1] = 1
    return OS.rle_counts(m)


def make_set(seed=0, n_images=12, n_cats=6, gt_per_image=7, dets_per_image=40, size=(120, 200), keypoints=False, masks=True,
             vertices=(20, 60), det_masks=None):
    """det_masks (default: masks): give each detection a rectangle mask as a compressed RLE."""
    det_masks = masks if det_masks is None else det_masks
    rng = np.random.RandomState(seed)
    cat_ids = sorted(rng.choice(np.arange(1, 3 * n_cats + 1), n_cats, replace=False).tolist())
    cats = [{"id": int(c), "name": "cat%d" % c} for c in cat_ids]
    img_ids = rng.choice(np.arange(1, 10 * n_images + 1), n_images, replace=False).tolist()
    images, anns = [], []
    aid = 1
    for n, iid in enumerate(img_ids):
        h, w = int(rng.randint(size[0], size[1] + 1)), int(rng.randint(size[0], size[1] + 1))
        images.append({"id": int(iid), "height": h, "width": w})
        if n == 1:
            continue                                                     # an image without ground truth
        only_crowd = n == 2
        for j in range(gt_per_image if not only_crowd else 2):
            c = cat_ids[int(rng.randint(0, max(n_cats - 1, 1)))]         # the last category never has ground truth
            if keypoints:
                c = cat_ids[0]
            crowd = only_crowd or rng.rand() < 0.08
            cx, cy = rng.uniform(0.15 * w, 0.85 * w), rng.uniform(0.15 * h, 0.85 * h)
            rx, ry = rng.uniform(4, 0.3 * w), rng.uniform(4, 0.3 * h)
            x0, y0 = max(int(cx - rx), 0), max(int(cy - ry), 0)
            x1, y1 = min(int(cx + rx) + 1, w), min(int(cy + ry) + 1, h)
            ann = {"id": aid, "image_id": int(iid), "category_id": int(c), "iscrowd": int(crowd),
                   "bbox": [float(x0), float(y0), float(x1 - x0), float(y1 - y0)]}
            if crowd:
                ann["segmentation"] = {"size": [h, w], "counts": [int(v) for v in _rect_counts(h, w, x0, y0, x1, y1)]}
            elif masks and rng.rand() < 0.1:
                ann["segmentation"] = {"size": [h, w], "counts": OS.rle_string(_rect_counts(h, w, x0, y0, x1, y1)).decode()}
            else:
                ann["segmentation"] = [star(rng, cx + rng.uniform(-rx, rx) * .3, cy + rng.uniform(-ry, ry) * .3, rx, ry,
                                            int(rng.randint(vertices[0], vertices[1] + 1))) for _ in range(int(rng.randint(1, 4)))]
            ann["area"] = float(rng.uniform(0.5, 1.0) * (x1 - x0) * (y1 - y0))
            if rng.rand() < 0.1:
                ann["area"] = float(rng.choice([32 ** 2, 96 ** 2, 31.5 ** 2, 100.0]))  # on and near the area range edges
            if keypoints:
                v = rng.choice([0, 1, 2], 17, p=[0.3, 0.3, 0.4])
                if rng.rand() < 0.15:
                    v[:] = 0
                kx = rng.uniform(x0, x1, 17); ky = rng.uniform(y0, y1, 17)
                ann["keypoints"] = [float(t) for xyv in zip(np.round(kx), np.round(ky), v) for t in xyv]
                ann["num_keypoints"] = int(np.count_nonzero(v))
            anns.append(ann)
            aid += 1
    dataset = {"images": images, "annotations": anns, "categories": cats}
    # detections: near ground truth of the image (any category), plus background ones, with tied scores
    K = n_cats + 1
    all_boxes = [[[] for _ in img_ids] for _ in range(K)]
    all_segms = [[[] for _ in img_ids] for _ in range(K)]
    all_keyps = [[[] for _ in img_ids] for _ in range(K)]
    sorted_ids = sorted(img_ids)
    by_img = {}
    for a in anns:
        by_img.setdefault(a["image_id"], []).append(a)
    by_id = {im["id"]: im for im in images}
    for i, iid in enumerate(sorted_ids):
        h, w = by_id[iid]["height"], by_id[iid]["width"]
        gts = by_img.get(iid, [])
        per_cls, src = {}, {}
        for _ in range(dets_per_image if i != 3 else 0):                 # image 3 (sorted order) has no detections
            g = None
            if gts and rng.rand() < 0.75:
                g = gts[int(rng.randint(0, len(gts)))]
                x, y, bw, bh = g["bbox"]
                b = np.array([x, y, x + bw - 1, y + bh - 1]) + rng.standard_normal(4) * rng.choice([0.5, 3, 10])
                cls = cat_ids.index(g["category_id"]) + 1 if rng.rand() < 0.85 else int(rng.randint(1, K))
            else:
                x, y = rng.uniform(0, w - 5), rng.uniform(0, h - 5)
                b = np.array([x, y, x + rng.uniform(2, w / 2), y + rng.uniform(2, h / 2)])
                cls = int(rng.randint(1, K))
            if keypoints:
                cls = 1
            s = np.float32(rng.choice([0.5, 0.25, rng.uniform(0.05, 1.0)]))
            per_cls.setdefault(cls, []).append(np.append(b, s))
            src.setdefault(cls, []).append(g)
        for cls, rows in per_cls.items():
            dets = np.asarray(rows, np.float32)
            all_boxes[cls][i] = dets
            if det_masks:
                rles = []
                for r in dets:
                    x0, y0 = int(np.clip(r[0], 0, w)), int(np.clip(r[1], 0, h))
                    x1, y1 = int(np.clip(r[2], 0, w)), int(np.clip(r[3], 0, h))
                    rles.append({"size": [h, w], "counts": OS.rle_string(_rect_counts(h, w, x0, y0, x1 + 1, y1 + 1)).decode()})
                all_segms[cls][i] = rles
            if keypoints:
                kl = []
                for r, g in zip(dets, src[cls]):
                    kp = np.zeros((4, 17), np.float32)
                    if g is not None and rng.rand() < 0.8:                # near the person's keypoints: OKS spread over (0, 1]
                        gk = np.asarray(g["keypoints"]).reshape(17, 3)
                        sd = rng.choice([0.5, 2.0, 6.0])
                        kp[0] = gk[:, 0] + rng.standard_normal(17) * sd; kp[1] = gk[:, 1] + rng.standard_normal(17) * sd
                    else:
                        kp[0] = rng.uniform(r[0], r[2], 17); kp[1] = rng.uniform(r[1], r[3], 17)
                    kp[2] = rng.standard_normal(17) * 3; kp[3] = rng.uniform(0, 1, 17)
                    kl.append(kp)
                all_keyps[cls][i] = kl
    return dataset, all_boxes, all_segms, all_keyps


def results(dataset, all_boxes, all_segms=None, all_keyps=None, iou_type="bbox", keypoint_confidence="bbox"):
    """The reference's results writers (json_dataset_evaluator.py), restated: the list json.dump would write."""
    cats = sorted(dataset["categories"], key=lambda c: c["id"])
    image_ids = sorted(im["id"] for im in dataset["images"])
    out = []
    for cls_ind, cat in enumerate(cats, start=1):
        if cls_ind >= len(all_boxes):
            break
        for i, image_id in enumerate(image_ids):
            dets = all_boxes[cls_ind][i]
            if isinstance(dets, list) and len(dets) == 0:
                continue
            dets = np.asarray(dets).astype(np.float64)
            if iou_type == "bbox":
                xywh = np.hstack((dets[:, 0:2], dets[:, 2:4] - dets[:, 0:2] + 1))
                out += [{"image_id": image_id, "category_id": cat["id"], "bbox": [float(v) for v in xywh[k]], "score": float(dets[k, -1])}
                        for k in range(dets.shape[0])]
            elif iou_type == "segm":
                out += [{"image_id": image_id, "category_id": cat["id"], "segmentation": all_segms[cls_ind][i][k],
                         "score": float(dets[k, -1])} for k in range(dets.shape[0])]
            else:
                for j, kd in enumerate(all_keyps[cls_ind][i]):
                    xy = []
                    for k in range(kd.shape[1]):
                        xy += [float(kd[0, k]), float(kd[1, k]), 1]
                    if keypoint_confidence == "bbox":
                        s = float(dets[j, -1])
                    else:
                        s = 0.0
                        for v in kd[2 if keypoint_confidence == "logit" else 3].astype(np.float64):
                            s += v
                        s /= kd.shape[1]
                    out.append({"image_id": image_id, "category_id": cat["id"], "keypoints": xy, "score": float(s)})
    return out


def oracle_eval(dataset, res, iou_type):
    """oracle/cocoeval.py's COCOeval.  Like pycocotools it rewrites the annotations it reads: the ground truth is copied, the
    results list `res` is consumed."""
    from oracle import cocoeval as C
    ds = dict(dataset, annotations=[dict(a) for a in dataset["annotations"]])   # 'segmentation' is replaced by its RLE
    gt = C.COCO(ds)
    dt = gt.loadRes(res) if res else C.COCO({"images": dataset["images"], "annotations": [],
                                                             "categories": dataset["categories"]})
    ev = C.COCOeval(gt, dt, iou_type)
    ev.evaluate()
    ev.accumulate()
    ev.stats = C.summarize(ev.eval, ev.params, out=None)
    return ev


def coco_scale_set(seed=2024, n_images=5000, n_cats=80):
    """COCO-val scale: 5 000 images, 80 categories, ~7 objects per image (1-3 polygons of 20-200 vertices, some crowd RLEs),
    100 detections per image with masks pasted and encoded on the device (ops.segm_rle_raw)."""
    import torch
    from detectron.pytorch_b200 import ops
    ds, ab, _, _ = make_set(seed, n_images=n_images, n_cats=n_cats, dets_per_image=100, size=(240, 480), masks=True,
                               vertices=(20, 200), keypoints=False, det_masks=False)
    sorted_ids = sorted(im["id"] for im in ds["images"])
    hw = {im["id"]: (im["height"], im["width"]) for im in ds["images"]}
    rng = np.random.RandomState(seed)
    asg = [[[] for _ in sorted_ids] for _ in ab]
    for i, iid in enumerate(sorted_ids):
        h, w = hw[iid]
        rows = [(c, k) for c in range(1, len(ab)) if len(ab[c][i]) for k in range(len(ab[c][i]))]
        if not rows:
            continue
        boxes = np.stack([ab[c][i][k][:4] for c, k in rows]).astype(np.float32)
        masks = rng.uniform(0, 1, (len(rows), 1, 28, 28)).astype(np.float32)
        counts, coffs, strings, soffs = ops.segm_rle_raw(torch.from_numpy(masks).cuda(), torch.zeros(len(rows), dtype=torch.int32).cuda(),
                                                         torch.from_numpy(boxes).cuda(), h, w, 0.5)
        s, so = strings.cpu().numpy().tobytes(), soffs.cpu().numpy()
        for j, (c, k) in enumerate(rows):
            if not asg[c][i]:
                asg[c][i] = []
            asg[c][i].append({"size": [h, w], "counts": s[so[j]:so[j + 1]].decode()})
    return ds, ab, asg


def load_golden(gold, name):
    """(dataset, all_boxes, all_segms, all_keyps, iou_type, confidence, expected) of one case of
    tests/golden/coco_eval.npz (tests/golden/make_golden_coco_eval.py)."""
    g = name + "/"
    ds = json.loads(gold[g + "dataset"].tobytes())
    K, I = int(gold[g + "num_classes"]), int(gold[g + "num_images"])

    def unflatten(rows, slots):
        out = [[[] for _ in range(I)] for _ in range(K)]
        for r, (c, i) in zip(rows, slots):
            out[c][i].append(r)
        return out
    ab = unflatten(gold[g + "boxes"], gold[g + "box_slot"])
    ab = [[np.asarray(v, np.float32) if v else [] for v in imgs] for imgs in ab]
    asg = json.loads(gold[g + "segms"].tobytes()) if g + "segms" in gold else None
    ak = unflatten(gold[g + "keypoints"], gold[g + "kp_slot"]) if g + "keypoints" in gold else None
    expected = {k: gold[g + k] for k in ("precision", "recall", "scores", "stats")}
    expected["results"] = json.loads(gold[g + "results"].tobytes())
    return ds, ab, asg, ak, str(gold[g + "iou_type"]), str(gold[g + "confidence"]) or None, expected
