"""detectron.pytorch_b200 -- H100-native (sm_90a) RoIAlign / RoIPool / RoICrop / NMS for
Detectron.pytorch, behind the reference's own Python surface.

    from detectron.pytorch_b200.modeling.roi_xfrom.roi_align.functions.roi_align import RoIAlignFunction
    from detectron.pytorch_b200.model.roi_pooling.functions.roi_pool import RoIPoolFunction
    from detectron.pytorch_b200.model.roi_crop.functions.roi_crop import RoICropFunction
    from detectron.pytorch_b200.model.nms.nms_gpu import nms_gpu

or, to make an unmodified checkout of the reference pick these up under ITS import paths
(`model.*`, `modeling.roi_xfrom.*`), call :func:`install_reference_aliases` before importing
`modeling.model_builder`.
"""
__version__ = "0.1.0"


def install_reference_aliases(overwrite=True, proposals=False, nms=False, segms=False, keypoints=False, voc=False, losses=False,
                              test_aug=False, bbox=False):
    """Register this package's op modules in sys.modules under the reference's import paths.

    After this, `from modeling.roi_xfrom.roi_align.functions.roi_align import RoIAlignFunction`
    (lib/modeling/model_builder.py:13), `from model.roi_pooling.functions.roi_pool import
    RoIPoolFunction` (:11), `from model.roi_crop.functions.roi_crop import RoICropFunction` (:12) and
    `from model.nms.nms_gpu import nms_gpu` resolve to the sm_90a implementations.
    Parent packages that already exist (e.g. the reference's own `modeling`) are left alone; only the
    op sub-packages are injected.  `proposals=True` additionally routes `modeling.generate_proposals` (the RPN proposal
    layer, rpn_heads.py / FPN.py import it) and `modeling.collect_and_distribute_fpn_rpn_proposals` to the device
    implementations (SURVEY.md 8f N1); the latter only implements the inference path, hence opt-in.
    `nms=True` re-points the reference's `utils.boxes.nms` (lib/utils/boxes.py:320-324; called from
    generate_proposals.py:161 and core/test.py:764 with numpy arrays) at the device NMS (`utils/boxes.py` here); the
    reference's `utils.boxes` must be importable for that.
    `segms=True` re-points the reference's `core.test.segm_results` (lib/core/test.py:793-847, called from im_detect_all)
    at the device mask paste + RLE (`core/test.py` here), which needs no pycocotools; the reference's `core.test` must be
    importable for that.
    `keypoints=True` re-points the reference's `core.test.keypoint_results` (lib/core/test.py:850-866, called from
    im_detect_all) at the device keypoint extraction and OKS NMS (`core/test.py` here), reading the reference's `cfg`
    at call time; the reference's `core.test` must be importable for that.
    `voc=True` re-points the reference's `datasets.voc_eval.voc_eval` (lib/datasets/voc_eval.py:86-223) and the copy of that name
    bound in `datasets.voc_dataset_evaluator` at the device evaluation (`datasets/voc_eval.py` here), which reads and writes the
    annotation cache in binary mode, so the reference's VOC evaluator runs on Python 3; both reference modules must be importable.
    `losses=True` re-points the reference's training losses at the device ones that take the device target blobs:
    `modeling.fast_rcnn_heads.fast_rcnn_losses`, `modeling.rpn_heads.single_scale_rpn_losses` (which the reference's
    generic_rpn_losses calls), `modeling.FPN.fpn_rpn_losses`, `modeling.mask_rcnn_heads.mask_rcnn_losses` and
    `modeling.keypoint_rcnn_heads.keypoint_losses` (`modeling/` here), each reading its reference module's `cfg` at call time;
    those reference modules must be importable.
    `test_aug=True` re-points the reference's `core.test` im_detect_mask(_aug) and im_detect_keypoints(_aug) (and, with them,
    segm_results and keypoint_results) at the device test-time augmentation (`core/test.py` here).
    `bbox=True` re-points the reference's `core.test` im_detect_bbox, im_detect_bbox_aug, im_detect_bbox_hflip,
    im_detect_bbox_scale, im_detect_bbox_aspect_ratio and box_results_with_nms_and_limit (whose inputs are then CUDA tensors)
    at the device box decode and combine (`core/test.py` here).  Each reads the reference's `cfg` at call time; with
    `bbox=True, test_aug=True` the reference's im_detect_all runs unmodified with no head output leaving the device.
    """
    import importlib
    import sys
    names = [
        "model.roi_align", "model.roi_align.functions", "model.roi_align.functions.roi_align",
        "model.roi_align.modules", "model.roi_align.modules.roi_align",
        "model.roi_pooling", "model.roi_pooling.functions", "model.roi_pooling.functions.roi_pool",
        "model.roi_pooling.modules", "model.roi_pooling.modules.roi_pool",
        "model.roi_crop", "model.roi_crop.functions", "model.roi_crop.functions.roi_crop",
        "model.roi_crop.modules", "model.roi_crop.modules.roi_crop",
        "model.roi_crop.functions.gridgen", "model.roi_crop.functions.crop_resize", "model.roi_crop.modules.gridgen",
        "model.nms", "model.nms.nms_gpu", "model.nms.nms_wrapper",
        "modeling.roi_xfrom", "modeling.roi_xfrom.roi_align", "modeling.roi_xfrom.roi_align.functions",
        "modeling.roi_xfrom.roi_align.functions.roi_align", "modeling.roi_xfrom.roi_align.modules",
        "modeling.roi_xfrom.roi_align.modules.roi_align", "modeling.roi_xfrom.roi_align.functions.roi_align_fpn",
    ]
    if proposals:
        names += ["modeling.generate_proposals", "modeling.collect_and_distribute_fpn_rpn_proposals"]
    installed = []
    for top in ("model", "modeling"):
        if top not in sys.modules:
            try:
                importlib.import_module(top)            # the reference's own package, if on sys.path
            except ImportError:
                sys.modules[top] = importlib.import_module(__name__ + "." + top)
                installed.append(top)
    for name in names:
        if name in sys.modules and not overwrite:
            continue
        mod = importlib.import_module(__name__ + "." + name)
        sys.modules[name] = mod
        parent, _, child = name.rpartition(".")
        if parent in sys.modules:
            setattr(sys.modules[parent], child, mod)
        installed.append(name)
    if nms:
        ref_boxes = importlib.import_module("utils.boxes")          # the reference's module
        ref_boxes.nms = importlib.import_module(__name__ + ".utils.boxes").nms
        installed.append("utils.boxes.nms")
    segms = segms or test_aug
    keypoints = keypoints or test_aug
    if test_aug:
        ref_test = importlib.import_module("core.test")              # the reference's module
        ours_test = importlib.import_module(__name__ + ".core.test")
        for name in ("im_detect_mask", "im_detect_mask_aug", "im_detect_keypoints", "im_detect_keypoints_aug"):
            setattr(ref_test, name, (lambda f: lambda *a: f(*a, cfg=ref_test.cfg))(getattr(ours_test, name)))
            installed.append("core.test." + name)
    if bbox:
        ref_test = importlib.import_module("core.test")              # the reference's module
        ours_test = importlib.import_module(__name__ + ".core.test")
        for name in ("im_detect_bbox", "im_detect_bbox_aug", "im_detect_bbox_hflip", "im_detect_bbox_scale",
                     "im_detect_bbox_aspect_ratio", "box_results_with_nms_and_limit"):
            setattr(ref_test, name, (lambda f: lambda *a, **k: f(*a, cfg=ref_test.cfg, **k))(getattr(ours_test, name)))
            installed.append("core.test." + name)
    if segms:
        ref_test = importlib.import_module("core.test")              # the reference's module
        ours = importlib.import_module(__name__ + ".core.test").segm_results
        ref_test.segm_results = lambda cls_boxes, masks, ref_boxes, im_h, im_w: ours(cls_boxes, masks, ref_boxes, im_h, im_w,
                                                                                     cfg=ref_test.cfg)
        installed.append("core.test.segm_results")
    if keypoints:
        ref_test = importlib.import_module("core.test")              # the reference's module
        ours_kp = importlib.import_module(__name__ + ".core.test").keypoint_results
        ref_test.keypoint_results = lambda cls_boxes, pred_heatmaps, ref_boxes: ours_kp(cls_boxes, pred_heatmaps, ref_boxes,
                                                                                         cfg=ref_test.cfg)
        installed.append("core.test.keypoint_results")
    if voc:
        ours_voc = importlib.import_module(__name__ + ".datasets.voc_eval").voc_eval
        for name in ("datasets.voc_eval", "datasets.voc_dataset_evaluator"):      # the reference's modules
            importlib.import_module(name).voc_eval = ours_voc
            installed.append(name + ".voc_eval")
    if losses:
        ours = __name__ + ".modeling."
        ref = importlib.import_module("modeling.fast_rcnn_heads")                  # the reference's modules
        ref.fast_rcnn_losses = importlib.import_module(ours + "fast_rcnn_heads").fast_rcnn_losses
        ref_rpn = importlib.import_module("modeling.rpn_heads")
        ours_rpn = importlib.import_module(ours + "rpn_heads").single_scale_rpn_losses
        ref_rpn.single_scale_rpn_losses = lambda *a, **k: ours_rpn(*a, cfg=ref_rpn.cfg, **k)
        ref_fpn = importlib.import_module("modeling.FPN")
        ours_fpn = importlib.import_module(ours + "FPN").fpn_rpn_losses
        ref_fpn.fpn_rpn_losses = lambda **k: ours_fpn(cfg=ref_fpn.cfg, **k)
        ref_mask = importlib.import_module("modeling.mask_rcnn_heads")
        ours_mask = importlib.import_module(ours + "mask_rcnn_heads").mask_rcnn_losses
        ref_mask.mask_rcnn_losses = lambda masks_pred, masks_int32: ours_mask(masks_pred, masks_int32, cfg=ref_mask.cfg)
        ref_kp = importlib.import_module("modeling.keypoint_rcnn_heads")
        ours_kp_loss = importlib.import_module(ours + "keypoint_rcnn_heads").keypoint_losses
        ref_kp.keypoint_losses = lambda kps_pred, loc, w, norm=None: ours_kp_loss(kps_pred, loc, w, norm, cfg=ref_kp.cfg)
        installed += ["modeling.fast_rcnn_heads.fast_rcnn_losses", "modeling.rpn_heads.single_scale_rpn_losses",
                      "modeling.FPN.fpn_rpn_losses", "modeling.mask_rcnn_heads.mask_rcnn_losses",
                      "modeling.keypoint_rcnn_heads.keypoint_losses"]
    return installed
