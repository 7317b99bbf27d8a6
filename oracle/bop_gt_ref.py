"""oracle/bop_gt_ref.py -- the per-gt loop bodies of the BOP toolkit's scripts/calc_gt_info.py and scripts/calc_gt_masks.py
restated in numpy (test infrastructure).

One ground-truth instance at a time, whole images as numpy arrays, from the same depth images the device gets: the test
depth as raw uint16 with its depth_scale, and the instance's render alone on the enlarged canvas (3h x 3w, principal point
shifted by (w, h)) in METRES.  Units as include/mpx.h: mpx_bop_gt_info states them (test depth in mm = fp32(raw) *
fp32(scale), rendered depth in mm = fp32(metres * 1000)).  scene_gt_info follows calc_gt_info.py (distance images by
misc.depth_im_to_dist_im_fast), the masks follow calc_gt_masks.py (misc.depth_im_to_dist_im, rounded differently).  The
product's megapose6d_b200/bop_dataset.py is checked against this module, and this module against the stored outputs of
the toolkit's own functions (tests/golden/reference/bop_gt_info_toolkit.npz).
"""
from __future__ import annotations

import numpy as np

from oracle.bop_ref import dist_image as dist_image_fast  # misc.depth_im_to_dist_im_fast
from oracle.bop_ref import visib_mask  # visibility.estimate_visib_mask_gt, bop19 mode


def dist_image(depth: np.ndarray, K: np.ndarray) -> np.ndarray:
    """misc.depth_im_to_dist_im: X d = ((x - cx) d) (1 / fx) in float64, then the norm with the depth."""
    h, w = depth.shape
    xs, ys = np.meshgrid(np.arange(w), np.arange(h))
    Xs = np.multiply(xs - K[0, 2], depth) * (1.0 / K[0, 0])
    Ys = np.multiply(ys - K[1, 2], depth) * (1.0 / K[1, 1])
    return np.sqrt(Xs.astype(np.float64) ** 2 + Ys.astype(np.float64) ** 2 + depth.astype(np.float64) ** 2)


def calc_2d_bbox(xs, ys) -> list:
    """misc.calc_2d_bbox without clipping: (x_min, y_min, x_max - x_min, y_max - y_min)."""
    return [int(xs.min()), int(ys.min()), int(xs.max() - xs.min()), int(ys.max() - ys.min())]


def test_depth_mm(raw: np.ndarray, depth_scale: float) -> np.ndarray:
    return raw.astype(np.float32) * np.float32(depth_scale)


def render_mm(depth_m: np.ndarray) -> np.ndarray:
    return (np.asarray(depth_m, np.float32) * np.float32(1000.0)).astype(np.float32)


def gt_info(depth_mm: np.ndarray, depth_gt_large_mm: np.ndarray, K: np.ndarray, delta) -> dict:
    """calc_gt_info.py:126-191 for one gt: depth_mm [h, w] float32 test depth, depth_gt_large_mm [3h, 3w] float32."""
    h, w = depth_mm.shape
    depth_gt = depth_gt_large_mm[h:2 * h, w:2 * w]
    dist_gt = dist_image_fast(depth_gt, K)
    dist_im = dist_image_fast(depth_mm, K)
    visib_gt = visib_mask(dist_im, dist_gt, delta)
    obj_mask_gt_large = depth_gt_large_mm > 0
    obj_mask_gt = dist_gt > 0
    px_count_all = int(np.sum(obj_mask_gt_large))
    px_count_valid = int(np.sum(dist_im[obj_mask_gt] > 0))
    px_count_visib = int(visib_gt.sum())
    visib_fract = px_count_visib / float(px_count_all) if px_count_all > 0 else 0.0
    bbox, bbox_visib = [-1, -1, -1, -1], [-1, -1, -1, -1]
    if px_count_visib > 0:
        ys, xs = obj_mask_gt_large.nonzero()
        bbox = calc_2d_bbox(xs - w, ys - h)
        ys, xs = visib_gt.nonzero()
        bbox_visib = calc_2d_bbox(xs, ys)
    return dict(px_count_all=px_count_all, px_count_valid=px_count_valid, px_count_visib=px_count_visib,
                visib_fract=float(visib_fract), bbox_obj=bbox, bbox_visib=bbox_visib)


def gt_masks(depth_mm: np.ndarray, depth_gt_mm: np.ndarray, K: np.ndarray, delta):
    """calc_gt_masks.py:105-127 for one gt: (mask, mask_visib) bool [h, w] from the render in the image window."""
    dist_im = dist_image(depth_mm, K)
    dist_gt = dist_image(depth_gt_mm, K)
    return dist_gt > 0, visib_mask(dist_im, dist_gt, delta)


def annotate(raw: np.ndarray, depth_scale: float, K: np.ndarray, depth_gt_large_m: np.ndarray, delta):
    """(scene_gt_info entry, mask, mask_visib) of one gt from the device's inputs: raw uint16 test depth, metre canvas."""
    h, w = raw.shape
    dt = test_depth_mm(raw, depth_scale)
    large = render_mm(depth_gt_large_m)
    mask, mask_visib = gt_masks(dt, large[h:2 * h, w:2 * w], K, delta)
    return gt_info(dt, large, K, delta), mask, mask_visib
