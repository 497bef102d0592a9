"""COCO evaluation of detections, masks and keypoints (lib/datasets/json_dataset_evaluator.py, task_evaluation.py) and PASCAL
VOC detection AP (lib/datasets/voc_dataset_evaluator.py, voc_eval.py)."""
