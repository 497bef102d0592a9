"""TEST INFRASTRUCTURE (CPU oracle, never imported by the product): COCO evaluation restated in numpy.

pycocotools is not installed, so its published algorithm (pycocotools 2.0: coco.py COCO.loadRes / annToRLE, cocoeval.py
COCOeval.evaluate / accumulate / summarize, maskApi.c bbIou / rleIou / rleArea / rleToBbox / rleMerge / rleFrString) is
restated here step for step.  Parity with pycocotools' own binary is unpinned: this module is pinned by hand-derived known
answers (tests/test_coco_eval.py) and, with the reference's writers around it, by tests/golden/coco_eval.npz.

Masks are handled as run-length intervals rather than by maskApi's run merge; the integer intersection and union they give
are the same.  The polygon rasteriser is oracle/masks.py's rleFrPoly, vectorised over the walk (rle_fr_poly below equals
oracle.masks.rle_fr_poly).  The class names follow pycocotools, so the golden generator can put this module in place of
pycocotools.coco / pycocotools.cocoeval.
"""
import copy
import json
from collections import defaultdict

import numpy as np

from oracle import masks as _masks

SPACING1 = np.spacing(1)
KPT_OKS_SIGMAS = np.array([.26, .25, .25, .35, .35, .79, .79, .72, .72, .62, .62, 1.07, 1.07, .87, .87, .89, .89]) / 10.0


# ---- maskApi ---------------------------------------------------------------------------------------------------------------
def rle_fr_string(s):
    """rleFrString, vectorised: compressed COCO counts (bytes or str) -> int64 counts."""
    if isinstance(s, str):
        s = s.encode("ascii")
    c = np.frombuffer(bytes(s), np.uint8).astype(np.int64) - 48
    if c.size == 0:
        return np.zeros(0, np.int64)
    ends = np.flatnonzero((c & 0x20) == 0)
    starts = np.concatenate([[0], ends[:-1] + 1])
    lens = ends - starts + 1
    k = np.arange(c.size) - np.repeat(starts, lens)
    x = np.add.reduceat((c & 0x1f) << (5 * k), starts)
    neg = (c[ends] & 0x10) != 0
    x[neg] |= (np.int64(-1) << (5 * lens[neg]))
    cnts = x.copy()
    cnts[1::2] = np.cumsum(x[1::2])
    cnts[2::2] = np.cumsum(x[2::2])
    return cnts & 0xffffffff                                            # cnts[m] = (uint) x


def counts_of(rle):
    c = rle["counts"]
    if isinstance(c, (bytes, str)):
        return rle_fr_string(c)
    return np.asarray(c, np.int64)


def ones_intervals(counts):
    """(starts, ends) of the runs of ones of column-major counts, zero-length runs dropped."""
    b = np.concatenate([[0], np.cumsum(np.asarray(counts, np.int64))])
    s, e = b[1:-1:2], b[2::2]
    n = min(s.size, e.size)
    s, e = s[:n], e[:n]
    keep = e > s
    return s[keep], e[keep]


def _ones_before(s, e, p):
    """Number of one-pixels of the disjoint sorted intervals (s, e) at positions < p (p an array)."""
    cum = np.concatenate([[0], np.cumsum(e - s)])
    j = np.searchsorted(e, p, side="right")                             # intervals ending at or before p
    jj = np.minimum(j, s.size - 1)
    return cum[j] + np.where((j < s.size) & (s[jj] < p), p - s[jj], 0)


def intersection(a, b):
    (sa, ea), (sb, eb) = a, b
    if sa.size == 0 or sb.size == 0:
        return 0
    return int(np.sum(_ones_before(sb, eb, ea) - _ones_before(sb, eb, sa)))


def union_intervals(parts):
    """rleMerge(intersect = 0) as intervals: the union of several masks."""
    s = np.concatenate([p[0] for p in parts]); e = np.concatenate([p[1] for p in parts])
    if s.size == 0:
        return s, e
    o = np.argsort(s, kind="stable"); s, e = s[o], e[o]
    run_max = np.maximum.accumulate(e)
    idx = np.flatnonzero(np.concatenate([[True], s[1:] > run_max[:-1]]))
    return s[idx], np.maximum.reduceat(e, idx)


def intervals_to_counts(iv, n):
    s, e = iv
    b = np.concatenate([[0], np.stack([s, e], 1).reshape(-1), [n]])
    return np.diff(b).astype(np.int64)


def rle_fr_poly(xy, h, w):
    """rleFrPoly (oracle/masks.py), vectorised over the upsampled walk.  Returns int64 counts."""
    xy = np.asarray(xy, np.float64)
    k = xy.size // 2
    x = np.trunc(5.0 * xy[0:2 * k:2] + .5).astype(np.int64); x = np.append(x, x[0])
    y = np.trunc(5.0 * xy[1:2 * k:2] + .5).astype(np.int64); y = np.append(y, y[0])
    xs, xe, ys, ye = x[:-1], x[1:], y[:-1], y[1:]
    dx, dy = np.abs(xe - xs), np.abs(ys - ye)
    shallow = dx >= dy
    flip = (shallow & (xs > xe)) | (~shallow & (ys > ye))
    xs2, xe2 = np.where(flip, xe, xs), np.where(flip, xs, xe)
    ys2, ye2 = np.where(flip, ye, ys), np.where(flip, ys, ye)
    n = np.where(shallow, dx, dy)
    rep = n + 1
    edge = np.repeat(np.arange(k), rep)
    d = np.arange(rep.sum()) - np.repeat(np.cumsum(rep) - rep, rep)
    t = np.where(flip[edge], n[edge] - d, d)
    with np.errstate(divide="ignore", invalid="ignore"):
        s = np.where(shallow, (ye2 - ys2) / np.where(dx == 0, 1, dx).astype(np.float64),
                     (xe2 - xs2) / np.where(dy == 0, 1, dy).astype(np.float64))
    tf = t.astype(np.float64)
    sh = shallow[edge]
    u = np.where(sh, t + xs2[edge], np.trunc((xs2[edge].astype(np.float64) + s[edge] * tf) + .5).astype(np.int64))
    v = np.where(sh, np.trunc((ys2[edge].astype(np.float64) + s[edge] * tf) + .5).astype(np.int64), t + ys2[edge])
    v = np.where(sh & (dx[edge] == 0), _masks.INT_MIN, v)
    if u.size < 2:
        tog = np.zeros(0, np.int64)
    else:
        u0, u1, v0, v1 = u[:-1], u[1:], v[:-1], v[1:]
        sel = u1 != u0
        u0, u1, v0, v1 = u0[sel], u1[sel], v0[sel], v1[sel]
        xd = (np.where(u1 < u0, u1, u1 - 1).astype(np.float64) + .5) / 5.0 - .5
        keep = (np.floor(xd) == xd) & (xd >= 0) & (xd <= w - 1)
        xd, v0, v1 = xd[keep], v0[keep], v1[keep]
        yd = np.ceil(np.clip((np.minimum(v0, v1).astype(np.float64) + .5) / 5.0 - .5, 0, h))
        tog = xd.astype(np.int64) * h + yd.astype(np.int64)
    # toggles -> intervals: a position toggled an odd number of times flips the value (rleFrPoly's zero-run merge)
    pos, cnt = np.unique(tog[tog < h * w], return_counts=True)
    pos = pos[cnt % 2 == 1]
    b = np.concatenate([pos, [h * w]]) if pos.size % 2 else pos
    return intervals_to_counts((b[0::2], b[1::2]), h * w)


def area(rle):
    c = counts_of(rle)
    return int(np.sum(c[1::2]))


def to_bbox(rle):
    """rleToBbox."""
    h, w = rle["size"]
    c = counts_of(rle)
    m = (c.size // 2) * 2
    if m == 0:
        return np.zeros(4)
    cc = np.cumsum(c[:m])
    j = np.arange(m)
    tpos = cc - (j % 2)
    yy, xx = tpos % h, tpos // h
    xs, xe, ys, ye = xx.min(), xx.max(), yy.min(), yy.max()
    if np.any(xx[0::2] < xx[1::2]):
        ys, ye = 0, h - 1
    return np.array([xs, ys, xe - xs + 1, ye - ys + 1], np.float64)


def bb_iou(dt, gt, iscrowd):
    """bbIou in double: dt (m, 4), gt (n, 4) xywh -> (m, n)."""
    dt = np.asarray(dt, np.float64).reshape(-1, 4); gt = np.asarray(gt, np.float64).reshape(-1, 4)
    da = dt[:, 2] * dt[:, 3]; ga = gt[:, 2] * gt[:, 3]
    w = np.minimum((dt[:, 0] + dt[:, 2])[:, None], (gt[:, 0] + gt[:, 2])[None]) - np.maximum(dt[:, 0][:, None], gt[:, 0][None])
    h = np.minimum((dt[:, 1] + dt[:, 3])[:, None], (gt[:, 1] + gt[:, 3])[None]) - np.maximum(dt[:, 1][:, None], gt[:, 1][None])
    i = w * h
    crowd = np.asarray(iscrowd, bool)[None]
    u = np.where(crowd, da[:, None], (da[:, None] + ga[None]) - i)
    with np.errstate(divide="ignore", invalid="ignore"):
        o = i / u
    return np.where((w <= 0) | (h <= 0), 0.0, o)


def rle_iou(dt, gt, iscrowd):
    """rleIou: dt, gt lists of RLE dicts of one image size -> (m, n) float64."""
    o = np.zeros((len(dt), len(gt)))
    di = [ones_intervals(counts_of(r)) for r in dt]
    gi = [ones_intervals(counts_of(r)) for r in gt]
    da = [int(np.sum(e - s)) for s, e in di]
    ga = [int(np.sum(e - s)) for s, e in gi]
    for g in range(len(gt)):
        if gi[g][0].size == 0:
            continue
        glo, ghi = gi[g][0][0], gi[g][1][-1]
        for d in range(len(dt)):
            if di[d][0].size == 0 or di[d][0][0] >= ghi or di[d][1][-1] <= glo:
                continue
            i = intersection(di[d], gi[g])
            if i == 0:
                continue
            u = da[d] if iscrowd[g] else da[d] + ga[g] - i
            o[d, g] = float(i) / float(u)
    return o


class mask:  # noqa: N801 -- the pycocotools.mask names the restated COCO / COCOeval call
    @staticmethod
    def frPyObjects(pyobj, h, w):
        if isinstance(pyobj, list):
            return [{"size": [h, w], "counts": rle_fr_poly(p, h, w)} for p in pyobj]
        return {"size": [h, w], "counts": np.asarray(pyobj["counts"], np.int64)}

    @staticmethod
    def merge(rles):
        h, w = rles[0]["size"]
        return {"size": [h, w], "counts": intervals_to_counts(union_intervals([ones_intervals(counts_of(r)) for r in rles]), h * w)}

    @staticmethod
    def area(rle):
        return area(rle)

    @staticmethod
    def toBbox(rle):
        return to_bbox(rle)


# ---- pycocotools.coco ----------------------------------------------------------------------------------------------------
class COCO:
    def __init__(self, annotation_file=None):
        self.dataset, self.anns, self.cats, self.imgs = {}, {}, {}, {}
        self.imgToAnns, self.catToImgs = defaultdict(list), defaultdict(list)
        if annotation_file is not None:
            if isinstance(annotation_file, dict):
                self.dataset = annotation_file
            else:
                with open(annotation_file) as f:
                    self.dataset = json.load(f)
            self.createIndex()

    def createIndex(self):
        self.anns, self.cats, self.imgs = {}, {}, {}
        self.imgToAnns, self.catToImgs = defaultdict(list), defaultdict(list)
        for ann in self.dataset.get("annotations", []):
            self.imgToAnns[ann["image_id"]].append(ann)
            self.anns[ann["id"]] = ann
        for img in self.dataset.get("images", []):
            self.imgs[img["id"]] = img
        for cat in self.dataset.get("categories", []):
            self.cats[cat["id"]] = cat
        for ann in self.dataset.get("annotations", []):
            self.catToImgs[ann["category_id"]].append(ann["image_id"])

    def getAnnIds(self, imgIds=(), catIds=()):
        imgIds = imgIds if isinstance(imgIds, (list, tuple, np.ndarray)) else [imgIds]
        catIds = catIds if isinstance(catIds, (list, tuple, np.ndarray)) else [catIds]
        if len(imgIds) == 0:
            anns = self.dataset.get("annotations", [])
        else:
            anns = [a for i in imgIds if i in self.imgToAnns for a in self.imgToAnns[i]]
        if len(catIds):
            cs = set(catIds)
            anns = [a for a in anns if a["category_id"] in cs]
        return [a["id"] for a in anns]

    def getCatIds(self):
        return [c["id"] for c in self.dataset.get("categories", [])]

    def getImgIds(self):
        return list(self.imgs.keys())

    def loadAnns(self, ids):
        return [self.anns[i] for i in ids]

    def loadCats(self, ids):
        return [self.cats[i] for i in ids]

    def loadRes(self, resFile):
        res = COCO()
        res.dataset["images"] = [img for img in self.dataset["images"]]
        if isinstance(resFile, str):
            with open(resFile) as f:
                anns = json.load(f)
        else:
            anns = resFile
        assert isinstance(anns, list), "results is not an array of objects"
        annsImgIds = [ann["image_id"] for ann in anns]
        assert set(annsImgIds) == (set(annsImgIds) & set(self.getImgIds())), \
            "Results do not correspond to current coco set"
        if anns and "bbox" in anns[0] and anns[0]["bbox"] != []:
            res.dataset["categories"] = copy.deepcopy(self.dataset["categories"])
            for id, ann in enumerate(anns):
                bb = ann["bbox"]
                x1, x2, y1, y2 = [bb[0], bb[0] + bb[2], bb[1], bb[1] + bb[3]]
                if "segmentation" not in ann:
                    ann["segmentation"] = [[x1, y1, x1, y2, x2, y2, x2, y1]]
                ann["area"] = bb[2] * bb[3]
                ann["id"] = id + 1
                ann["iscrowd"] = 0
        elif anns and "segmentation" in anns[0]:
            res.dataset["categories"] = copy.deepcopy(self.dataset["categories"])
            for id, ann in enumerate(anns):
                ann["area"] = area(ann["segmentation"])
                if "bbox" not in ann:
                    ann["bbox"] = to_bbox(ann["segmentation"])
                ann["id"] = id + 1
                ann["iscrowd"] = 0
        elif anns and "keypoints" in anns[0]:
            res.dataset["categories"] = copy.deepcopy(self.dataset["categories"])
            for id, ann in enumerate(anns):
                s = ann["keypoints"]
                x, y = s[0::3], s[1::3]
                x0, x1, y0, y1 = np.min(x), np.max(x), np.min(y), np.max(y)
                ann["area"] = (x1 - x0) * (y1 - y0)
                ann["id"] = id + 1
                ann["bbox"] = [x0, y0, x1 - x0, y1 - y0]
        res.dataset["annotations"] = anns
        res.createIndex()
        return res

    def annToRLE(self, ann):
        t = self.imgs[ann["image_id"]]
        h, w = t["height"], t["width"]
        segm = ann["segmentation"]
        if isinstance(segm, list):
            return mask.merge(mask.frPyObjects(segm, h, w))
        if isinstance(segm["counts"], list):
            return mask.frPyObjects(segm, h, w)
        return segm


# ---- pycocotools.cocoeval ------------------------------------------------------------------------------------------------
class Params:
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


def oks(dts, gts, sigmas=KPT_OKS_SIGMAS):
    """computeOks for one (image, category): dts / gts annotation dicts (dts already sorted and cut)."""
    vars = (sigmas * 2) ** 2
    k = len(sigmas)
    ious = np.zeros((len(dts), len(gts)))
    for j, gt in enumerate(gts):
        g = np.array(gt["keypoints"])
        xg, yg, vg = g[0::3], g[1::3], g[2::3]
        k1 = np.count_nonzero(vg > 0)
        bb = gt["bbox"]
        x0 = bb[0] - bb[2]; x1 = bb[0] + bb[2] * 2
        y0 = bb[1] - bb[3]; y1 = bb[1] + bb[3] * 2
        for i, dt in enumerate(dts):
            d = np.array(dt["keypoints"])
            xd, yd = d[0::3], d[1::3]
            if k1 > 0:
                dx = xd - xg; dy = yd - yg
            else:
                z = np.zeros((k))
                dx = np.max((z, x0 - xd), axis=0) + np.max((z, xd - x1), axis=0)
                dy = np.max((z, y0 - yd), axis=0) + np.max((z, yd - y1), axis=0)
            e = (dx ** 2 + dy ** 2) / vars / (gt["area"] + np.spacing(1)) / 2
            if k1 > 0:
                e = e[vg > 0]
            ious[i, j] = np.sum(np.exp(-e)) / e.shape[0]
    return ious


class COCOeval:
    def __init__(self, cocoGt=None, cocoDt=None, iouType="segm"):
        self.cocoGt, self.cocoDt = cocoGt, cocoDt
        self.evalImgs = defaultdict(list)
        self.eval = {}
        self._gts, self._dts = defaultdict(list), defaultdict(list)
        self.params = Params(iouType=iouType)
        self._paramsEval = {}
        self.stats = []
        self.ious = {}
        if cocoGt is not None:
            self.params.imgIds = sorted(cocoGt.getImgIds())
            self.params.catIds = sorted(cocoGt.getCatIds())

    def _prepare(self):
        p = self.params
        gts = self.cocoGt.loadAnns(self.cocoGt.getAnnIds(imgIds=p.imgIds, catIds=p.catIds))
        dts = self.cocoDt.loadAnns(self.cocoDt.getAnnIds(imgIds=p.imgIds, catIds=p.catIds))
        if p.iouType == "segm":
            for anns, coco in ((gts, self.cocoGt), (dts, self.cocoDt)):
                for ann in anns:
                    ann["segmentation"] = coco.annToRLE(ann)
        for gt in gts:
            gt["ignore"] = gt["ignore"] if "ignore" in gt else 0
            gt["ignore"] = "iscrowd" in gt and gt["iscrowd"]
            if p.iouType == "keypoints":
                gt["ignore"] = (gt["num_keypoints"] == 0) or gt["ignore"]
        self._gts, self._dts = defaultdict(list), defaultdict(list)
        for gt in gts:
            self._gts[gt["image_id"], gt["category_id"]].append(gt)
        for dt in dts:
            self._dts[dt["image_id"], dt["category_id"]].append(dt)
        self.evalImgs = defaultdict(list)
        self.eval = {}

    def evaluate(self):
        p = self.params
        p.imgIds = list(np.unique(p.imgIds))
        p.catIds = list(np.unique(p.catIds))
        p.maxDets = sorted(p.maxDets)
        self.params = p
        self._prepare()
        computeIoU = self.computeOks if p.iouType == "keypoints" else self.computeIoU
        self.ious = {(imgId, catId): computeIoU(imgId, catId) for imgId in p.imgIds for catId in p.catIds}
        maxDet = p.maxDets[-1]
        self.evalImgs = [self.evaluateImg(imgId, catId, areaRng, maxDet)
                         for catId in p.catIds for areaRng in p.areaRng for imgId in p.imgIds]
        self._paramsEval = copy.deepcopy(self.params)

    def _sorted_dt(self, imgId, catId):
        dt = self._dts[imgId, catId]
        inds = np.argsort([-d["score"] for d in dt], kind="mergesort")
        dt = [dt[i] for i in inds]
        return dt[0:self.params.maxDets[-1]]

    def computeIoU(self, imgId, catId):
        p = self.params
        gt = self._gts[imgId, catId]
        dt = self._dts[imgId, catId]
        if len(gt) == 0 and len(dt) == 0:
            return []
        dt = self._sorted_dt(imgId, catId)
        if len(gt) == 0 or len(dt) == 0:
            return []
        iscrowd = [int(o["iscrowd"]) for o in gt]
        if p.iouType == "segm":
            return rle_iou([d["segmentation"] for d in dt], [g["segmentation"] for g in gt], iscrowd)
        return bb_iou([d["bbox"] for d in dt], [g["bbox"] for g in gt], iscrowd)

    def computeOks(self, imgId, catId):
        gts = self._gts[imgId, catId]
        dts = self._sorted_dt(imgId, catId)
        if len(gts) == 0 or len(dts) == 0:
            return []
        return oks(dts, gts, self.params.kpt_oks_sigmas)

    def evaluateImg(self, imgId, catId, aRng, maxDet):
        p = self.params
        gt = self._gts[imgId, catId]
        dt = self._dts[imgId, catId]
        if len(gt) == 0 and len(dt) == 0:
            return None
        for g in gt:
            g["_ignore"] = 1 if (g["ignore"] or (g["area"] < aRng[0] or g["area"] > aRng[1])) else 0
        gtind = np.argsort([g["_ignore"] for g in gt], kind="mergesort")
        gt = [gt[i] for i in gtind]
        dtind = np.argsort([-d["score"] for d in dt], kind="mergesort")
        dt = [dt[i] for i in dtind[0:maxDet]]
        iscrowd = [int(o["iscrowd"]) for o in gt]
        ious = self.ious[imgId, catId][:, gtind] if len(self.ious[imgId, catId]) > 0 else self.ious[imgId, catId]
        T, G, D = len(p.iouThrs), len(gt), len(dt)
        gtm = np.zeros((T, G)); dtm = np.zeros((T, D))
        gtIg = np.array([g["_ignore"] for g in gt]); dtIg = np.zeros((T, D))
        if len(ious) != 0:
            iou_rows = [list(map(float, r)) for r in ious]
            gig = [int(x) for x in gtIg]
            for tind, t in enumerate(p.iouThrs):
                gm = [0] * G
                for dind, d in enumerate(dt):
                    iou = min([t, 1 - 1e-10])
                    m = -1
                    row = iou_rows[dind]
                    for gind in range(G):
                        if gm[gind] > 0 and not iscrowd[gind]:
                            continue
                        if m > -1 and gig[m] == 0 and gig[gind] == 1:
                            break
                        if row[gind] < iou:
                            continue
                        iou = row[gind]
                        m = gind
                    if m == -1:
                        continue
                    dtIg[tind, dind] = gig[m]
                    dtm[tind, dind] = gt[m]["id"]
                    gm[m] = d["id"]
                gtm[tind] = gm
        a = np.array([d["area"] < aRng[0] or d["area"] > aRng[1] for d in dt]).reshape((1, len(dt)))
        dtIg = np.logical_or(dtIg, np.logical_and(dtm == 0, np.repeat(a, T, 0)))
        return {"image_id": imgId, "category_id": catId, "aRng": aRng, "maxDet": maxDet,
                "dtIds": [d["id"] for d in dt], "gtIds": [g["id"] for g in gt], "dtMatches": dtm, "gtMatches": gtm,
                "dtScores": [d["score"] for d in dt], "gtIgnore": gtIg, "dtIgnore": dtIg}

    def accumulate(self, p=None):
        if p is None:
            p = self.params
        p.catIds = p.catIds if p.useCats == 1 else [-1]
        T, R, K, A, M = len(p.iouThrs), len(p.recThrs), len(p.catIds), len(p.areaRng), len(p.maxDets)
        precision = -np.ones((T, R, K, A, M))
        recall = -np.ones((T, K, A, M))
        scores = -np.ones((T, R, K, A, M))
        _pe = self._paramsEval
        setK, setA, setM, setI = set(_pe.catIds), set(map(tuple, _pe.areaRng)), set(_pe.maxDets), set(_pe.imgIds)
        k_list = [n for n, k in enumerate(p.catIds) if k in setK]
        m_list = [m for n, m in enumerate(p.maxDets) if m in setM]
        a_list = [n for n, a in enumerate(map(lambda x: tuple(x), p.areaRng)) if a in setA]
        i_list = [n for n, i in enumerate(p.imgIds) if i in setI]
        I0, A0 = len(_pe.imgIds), len(_pe.areaRng)
        for k, k0 in enumerate(k_list):
            Nk = k0 * A0 * I0
            for a, a0 in enumerate(a_list):
                Na = a0 * I0
                for m, maxDet in enumerate(m_list):
                    E = [self.evalImgs[Nk + Na + i] for i in i_list]
                    E = [e for e in E if e is not None]
                    if len(E) == 0:
                        continue
                    dtScores = np.concatenate([e["dtScores"][0:maxDet] for e in E])
                    inds = np.argsort(-dtScores, kind="mergesort")
                    dtScoresSorted = dtScores[inds]
                    dtm = np.concatenate([e["dtMatches"][:, 0:maxDet] for e in E], axis=1)[:, inds]
                    dtIg = np.concatenate([e["dtIgnore"][:, 0:maxDet] for e in E], axis=1)[:, inds]
                    gtIg = np.concatenate([e["gtIgnore"] for e in E])
                    npig = np.count_nonzero(gtIg == 0)
                    if npig == 0:
                        continue
                    tps = np.logical_and(dtm, np.logical_not(dtIg))
                    fps = np.logical_and(np.logical_not(dtm), np.logical_not(dtIg))
                    tp_sum = np.cumsum(tps, axis=1).astype(dtype=np.float64)
                    fp_sum = np.cumsum(fps, axis=1).astype(dtype=np.float64)
                    for t, (tp, fp) in enumerate(zip(tp_sum, fp_sum)):
                        tp = np.array(tp); fp = np.array(fp)
                        nd = len(tp)
                        rc = tp / npig
                        pr = tp / (fp + tp + np.spacing(1))
                        q = np.zeros((R,)); ss = np.zeros((R,))
                        recall[t, k, a, m] = rc[-1] if nd else 0
                        pr = pr.tolist(); q = q.tolist()
                        for i in range(nd - 1, 0, -1):
                            if pr[i] > pr[i - 1]:
                                pr[i - 1] = pr[i]
                        inds = np.searchsorted(rc, p.recThrs, side="left")
                        try:
                            for ri, pi in enumerate(inds):
                                q[ri] = pr[pi]
                                ss[ri] = dtScoresSorted[pi]
                        except IndexError:
                            pass
                        precision[t, :, k, a, m] = np.array(q)
                        scores[t, :, k, a, m] = np.array(ss)
        self.eval = {"params": p, "counts": [T, R, K, A, M], "precision": precision, "recall": recall, "scores": scores}

    def summarize(self):
        self.stats = summarize(self.eval, self.params)

    def __str__(self):
        self.summarize()
        return ""


def summarize(ev, p, out=print):
    """COCOeval.summarize: the 12 (bbox, segm) or 10 (keypoints) stats, printing the table through `out`."""
    def _summarize(ap=1, iouThr=None, areaRng="all", maxDets=100):
        iStr = " {:<18} {} @[ IoU={:<9} | area={:>6s} | maxDets={:>3d} ] = {:0.3f}"
        titleStr = "Average Precision" if ap == 1 else "Average Recall"
        typeStr = "(AP)" if ap == 1 else "(AR)"
        iouStr = "{:0.2f}:{:0.2f}".format(p.iouThrs[0], p.iouThrs[-1]) if iouThr is None else "{:0.2f}".format(iouThr)
        aind = [i for i, aRng in enumerate(p.areaRngLbl) if aRng == areaRng]
        mind = [i for i, mDet in enumerate(p.maxDets) if mDet == maxDets]
        if ap == 1:
            s = ev["precision"]
            if iouThr is not None:
                s = s[np.where(iouThr == p.iouThrs)[0]]
            s = s[:, :, :, aind, mind]
        else:
            s = ev["recall"]
            if iouThr is not None:
                s = s[np.where(iouThr == p.iouThrs)[0]]
            s = s[:, :, aind, mind]
        mean_s = -1 if len(s[s > -1]) == 0 else np.mean(s[s > -1])
        if out is not None:
            out(iStr.format(titleStr, typeStr, iouStr, areaRng, maxDets, mean_s))
        return mean_s

    if p.iouType == "keypoints":
        stats = np.zeros((10,))
        for i, (ap, kw) in enumerate([(1, {}), (1, {"iouThr": .5}), (1, {"iouThr": .75}), (1, {"areaRng": "medium"}),
                                      (1, {"areaRng": "large"}), (0, {}), (0, {"iouThr": .5}), (0, {"iouThr": .75}),
                                      (0, {"areaRng": "medium"}), (0, {"areaRng": "large"})]):
            stats[i] = _summarize(ap, maxDets=20, **kw)
        return stats
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
