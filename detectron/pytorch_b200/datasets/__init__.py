"""COCO evaluation of detections, masks and keypoints (lib/datasets/json_dataset_evaluator.py, task_evaluation.py)."""
