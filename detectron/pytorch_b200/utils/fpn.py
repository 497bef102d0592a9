"""FPN level assignment on tensors (any device); mirrors lib/utils/fpn.py:11-28 (reference, numpy).

`map_rois_to_fpn_levels` is Eqn. (1) of the FPN paper as the reference evaluates it: float32 areas with the `+ 1`
box convention (utils/boxes.py:58-69; negative areas are zeroed), s = sqrt(area),
level = clip(floor(k0 + log2(s / s0 + 1e-6)), k_min, k_max).
"""
import torch


def map_rois_to_fpn_levels(rois, k_min, k_max, canonical_scale=224, canonical_level=4):
    """rois (R, 4) [x1, y1, x2, y2] float32 -> (R,) float32 levels in [k_min, k_max]."""
    w = rois[:, 2] - rois[:, 0] + 1
    h = rois[:, 3] - rois[:, 1] + 1
    areas = w * h
    areas = torch.where(areas < 0, torch.zeros_like(areas), areas)
    s = torch.sqrt(areas)
    # At a level boundary floor() turns a last-bit difference into a level, so both roundings are pinned to numpy's: a true
    # float32 division by a tensor (a Python-number divisor may be applied as a multiplication by its rounded reciprocal on
    # CUDA) and log2 rounded once from float64 (CUDA's float32 log2 is not correctly rounded).  Without this, 161 of 182 232
    # boxes within 64 ulps of a boundary got another level than the reference's numpy on an H100.
    y = torch.div(s, torch.full((), float(canonical_scale), dtype=s.dtype, device=s.device)) + 1e-6
    lvls = torch.floor(canonical_level + torch.log2(y.double()).to(s.dtype))
    return torch.clamp(lvls, k_min, k_max)
