"""Seeded synthetic PASCAL VOC evaluation sets (tests/test_voc_eval.py, tests/golden/make_golden_voc_eval.py, tools/voc_eval_probe.py).

make_set() gives (classes, image names, recs, all_boxes): recs {name: objects as parse_rec returns them}, all_boxes[cls][img] float32
(n, 5) arrays or [] as the reference's test_net hands them to evaluate_boxes (class 0 is __background__).  Ground truth has integer
boxes, some difficult, images without objects and all-difficult images.  Detections lie near ground truth of the image (mostly of
their class) or anywhere, some on coordinates that round half-way in the writer's '{:.1f}'.  Scores are distinct within a class
(k / 1000) unless `ties`, where they come from four values.  edge_set() adds hand-placed cases.  write_devkit() lays a set out as a
VOCdevkit directory.
"""
import json
import os

import numpy as np

CLASSES20 = ["aeroplane", "bicycle", "bird", "boat", "bottle", "bus", "car", "cat", "chair", "cow", "diningtable", "dog", "horse",
             "motorbike", "person", "pottedplant", "sheep", "sofa", "train", "tvmonitor"]


def _obj(name, box, difficult=0, truncated=0, pose="Unspecified"):
    return {"name": name, "pose": pose, "truncated": int(truncated), "difficult": int(difficult), "bbox": [int(v) for v in box]}


def make_set(seed=0, n_images=12, n_classes=4, objs_per_image=3.0, dets_per_image=20, difficult_rate=0.15, ties=False, size=(500, 375)):
    rng = np.random.RandomState(seed)
    classes = CLASSES20[:n_classes] if n_classes <= 20 else ["class%d" % k for k in range(n_classes)]
    names = ["%06d" % v for v in np.sort(rng.choice(np.arange(1, 20 * n_images + 1), n_images, replace=False))]
    W, H = size
    recs = {}
    for n, name in enumerate(names):
        objs = []
        if n != 1:                                                       # image 1 has no objects
            for _ in range(max(int(rng.poisson(objs_per_image)), 1)):
                x1, y1 = int(rng.randint(0, W - 20)), int(rng.randint(0, H - 20))
                x2, y2 = min(x1 + int(rng.randint(8, 200)), W - 1), min(y1 + int(rng.randint(8, 200)), H - 1)
                difficult = n == 2 or rng.rand() < difficult_rate           # image 2: all difficult
                objs.append(_obj(classes[int(rng.randint(0, n_classes))], (x1, y1, x2, y2), difficult, rng.rand() < 0.3,
                                 rng.choice(["Left", "Right", "Frontal", "Unspecified"])))
        recs[name] = objs
    all_boxes = [[[] for _ in names] for _ in range(n_classes + 1)]
    rows = [[[] for _ in names] for _ in range(n_classes + 1)]
    for i, name in enumerate(names):
        objs = recs[name]
        for _ in range(dets_per_image):
            if objs and rng.rand() < 0.7:
                o = objs[int(rng.randint(0, len(objs)))]
                b = np.asarray(o["bbox"], np.float64) - 1 + rng.standard_normal(4) * rng.choice([0.5, 3, 12])
                cls = classes.index(o["name"]) + 1 if rng.rand() < 0.85 else int(rng.randint(1, n_classes + 1))
            else:
                x, y = rng.uniform(0, W - 10), rng.uniform(0, H - 10)
                b = np.array([x, y, x + rng.uniform(2, W / 3), y + rng.uniform(2, H / 3)])
                cls = int(rng.randint(1, n_classes + 1))
            if rng.rand() < 0.2:
                b = np.round(b * 20) / 20                                # multiples of 0.05: half-way cases of '{:.1f}'
            rows[cls][i].append(b)
    for c in range(1, n_classes + 1):
        n_c = sum(len(r) for r in rows[c])
        if ties:
            scores = rng.choice([0.25, 0.5, 0.75, 0.9], n_c)
        else:
            assert n_c < 1000
            scores = (rng.choice(np.arange(1, 1000), n_c, replace=False)) / 1000.0
        k = 0
        for i in range(len(names)):
            if rows[c][i]:
                n = len(rows[c][i])
                all_boxes[c][i] = np.column_stack([np.asarray(rows[c][i]), scores[k:k + n]]).astype(np.float32)
                k += n
    return ["__background__"] + classes, names, recs, all_boxes


def edge_set(seed=5):
    """make_set plus hand-placed cases: IoU exactly 0.5, a detection on a difficult box, several detections on one box, zero-width
    and inverted boxes after rounding, a zero-area ground-truth box under a zero-width detection (IoU 0 / 0 = NaN), detections on
    an image without ground truth of their class, and a class whose only objects are difficult (npos = 0)."""
    classes, names, recs, ab = make_set(seed, n_images=8, n_classes=3, dets_per_image=10)
    c1, c2, c3 = classes[1], classes[2], classes[3]
    recs[names[4]] = [_obj(c1, (10, 10, 29, 29)), _obj(c1, (100, 100, 139, 139), difficult=1), _obj(c2, (200, 50, 260, 120)),
                      _obj(c2, (300, 200, 299, 240))]
    recs[names[5]] = [_obj(c3, (50, 50, 90, 90), difficult=1)]
    for name in names:                                                   # c3 only as difficult objects
        recs[name] = [o if o["name"] != c3 else dict(o, difficult=1) for o in recs[name]]

    def put(cls, img, rows):
        old = ab[cls][img]
        new = np.asarray(rows, np.float32)
        ab[cls][img] = new if isinstance(old, list) else np.concatenate([old, new])

    put(1, 4, [[9, 9, 28, 18, .991],                                     # file box (10, 10, 29, 19): IoU 200 / 400 = 0.5 -> fp
               [99, 99, 138, 138, .992],                                 # on the difficult box: neither
               [9, 9, 28, 28, .995], [9.04, 9, 28.04, 28, .994], [10, 9, 28, 28, .993],   # three on one box: tp, fp, fp
               [30.04, 5, 29.04, 40, .990],                              # rounds to x1 31.0, x2 30.0: zero width
               [60, 60, 40, 40, .989]])                                  # inverted
    put(2, 4, [[299, 199, 298, 239, .996],                               # zero width on the zero-width box: 0 / 0
               [199, 49, 259, 119, .997]])
    put(2, 1, [[5, 5, 50, 50, .998]])                                    # image 1 has no objects
    put(3, 5, [[49, 49, 89, 89, .999], [10, 10, 40, 40, .988]])          # class 3: npos = 0
    for c in range(1, len(classes)):                                     # keep scores distinct within each class
        vals = np.concatenate([a[:, -1] for a in ab[c] if not isinstance(a, list)])
        assert np.unique(np.round(vals.astype(np.float64), 3)).size == vals.size, c
    return classes, names, recs, ab


def xml_text(name, objects):
    parts = ["<annotation>", "  <folder>VOC</folder>", "  <filename>%s.jpg</filename>" % name]
    for o in objects:
        b = o["bbox"]
        parts += ["  <object>", "    <name>%s</name>" % o["name"], "    <pose>%s</pose>" % o["pose"],
                  "    <truncated>%d</truncated>" % o["truncated"], "    <difficult>%d</difficult>" % o["difficult"],
                  "    <bndbox>", "      <xmin>%d</xmin>" % b[0], "      <ymin>%d</ymin>" % b[1], "      <xmax>%d</xmax>" % b[2],
                  "      <ymax>%d</ymax>" % b[3], "    </bndbox>", "  </object>"]
    return "\n".join(parts + ["</annotation>", ""])


def write_devkit(root, dataset_name, names, xml_texts):
    """VOC<year>/Annotations/<name>.xml and VOC<year>/ImageSets/Main/<image set>.txt under root, for a `voc_<year>_<image set>`
    dataset name; also the empty results directory the reference's writer expects."""
    year, image_set = dataset_name[4:8], dataset_name[9:]
    base = os.path.join(root, "VOC" + year)
    for d in ("Annotations", os.path.join("ImageSets", "Main")):
        os.makedirs(os.path.join(base, d), exist_ok=True)
    os.makedirs(os.path.join(root, "results", "VOC" + year, "Main"), exist_ok=True)
    for name, text in zip(names, xml_texts):
        with open(os.path.join(base, "Annotations", name + ".xml"), "w") as f:
            f.write(text)
    with open(os.path.join(base, "ImageSets", "Main", image_set + ".txt"), "w") as f:
        f.write("".join(n + "\n" for n in names))
    return root


def dataset_dict(classes, names):
    """The annotation-file dict of a VOC set converted to COCO json: image ids in image-set order, categories in class order."""
    return {"images": [{"id": i + 1, "file_name": n + ".jpg", "height": 375, "width": 500} for i, n in enumerate(names)],
            "annotations": [], "categories": [{"id": k, "name": c} for k, c in enumerate(classes) if k > 0]}


def load_golden(gold, case):
    """(dataset name, classes, names, xml texts, all_boxes, expected) of one case of tests/golden/voc_eval.npz; expected holds
    'lines' {cls: written text}, 'recs' {name: objects} and per class (rec, prec, ap)."""
    g = case + "/"
    text = lambda k: json.loads(gold[g + k].tobytes())                   # noqa: E731
    classes, names, xmls = text("classes"), text("names"), text("xml")
    ab = [[[] for _ in names] for _ in classes]
    for r, (c, i) in zip(gold[g + "boxes"], gold[g + "box_slot"]):
        ab[c][i].append(r)
    ab = [[np.asarray(v, np.float32) if len(v) else [] for v in imgs] for imgs in ab]
    off = gold[g + "curve_begin"]
    curves = {c: (gold[g + "rec"][off[k]:off[k + 1]], gold[g + "prec"][off[k]:off[k + 1]], gold[g + "ap"][k])
              for k, c in enumerate(classes[1:])}
    expected = {"lines": text("lines"), "recs": text("recs"), "curves": curves}
    return str(gold[g + "dataset_name"]), classes, names, xmls, ab, expected


def scale_set(seed=2007, n_images=4952):
    """VOC2007-test scale: 4 952 images, 20 classes, about 3 objects per image (some difficult), 100 detections per image."""
    return make_set(seed, n_images=n_images, n_classes=20, objs_per_image=2.4, dets_per_image=100, ties=True)
