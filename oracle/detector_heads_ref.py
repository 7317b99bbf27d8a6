"""float64 oracle of the detector engine's RoI heads (megapose6d_b200/detector_engine.py RoiHeadsEngine,
csrc/detector_heads.cu), in the form of oracle/detector_ref.py: torchvision's CUDA fp32 MultiScaleRoIAlign for the
pooling, the pooled features rounded once to act16, every layer evaluated in float64 with act16 weights and fp32 biases
and its output rounded once to act16 after bias and ReLU; the fp32 outputs are exact conversions."""
from __future__ import annotations

from typing import Tuple

import torch
import torch.nn.functional as F

from .detector_ref import _conv, q


@torch.no_grad()
def roi_heads_box(model, features, proposals, image_sizes) -> Tuple[torch.Tensor, torch.Tensor]:
    """float64 (class_logits [P, C], box_regression [P, 4C]) of the engine's box branch: torchvision's CUDA fp32
    MultiScaleRoIAlign, the pooled features rounded once to act16, then fc6, fc7 (ReLU) and the predictor in float64
    with act16 weights and fp32 biases, each output rounded once to act16.  features: the OrderedDict of fp32 levels."""
    rh = model.roi_heads
    x = q(rh.box_roi_pool(features, proposals, image_sizes).double()).flatten(1)
    for fc in (rh.box_head.fc6, rh.box_head.fc7):
        x = q(F.relu(F.linear(x, q(fc.weight.double()), fc.bias.float().double())))
    pred = rh.box_predictor
    return (q(F.linear(x, q(pred.cls_score.weight.double()), pred.cls_score.bias.float().double())),
            q(F.linear(x, q(pred.bbox_pred.weight.double()), pred.bbox_pred.bias.float().double())))


@torch.no_grad()
def roi_heads_mask(model, features, boxes, image_sizes) -> torch.Tensor:
    """float64 mask logits [N, C, 2s, 2s] of the engine's mask branch: torchvision's CUDA fp32 MultiScaleRoIAlign
    rounded once to act16, the four 3x3 convolutions (ReLU), the 2x2/s2 deconvolution (ReLU) and the logits, each in
    float64 with act16 weights and fp32 biases and rounded once to act16."""
    rh = model.roi_heads
    x = q(rh.mask_roi_pool(features, boxes, image_sizes).double())
    for block in rh.mask_head:
        x = _conv(x, block[0], relu=True)
    conv5 = rh.mask_predictor.conv5_mask
    x = q(F.relu(F.conv_transpose2d(x, q(conv5.weight.double()), conv5.bias.float().double(), stride=2)))
    return _conv(x, rh.mask_predictor.mask_fcn_logits)


# Stated bounds (DESIGN §4) of the RoI heads with Gaussian weights, in units of each output tensor's largest magnitude.
# The oracle is the engine's function; the engine differs from it by the fp32 summation order inside each layer, which
# moves an output by at most one act16 step where the two sums straddle a rounding boundary.  Through the three box
# layers or the six mask layers such steps add like the roundings of the backbone's bound: a few u = 2^-11.
HEADS_VS_ORACLE = 2.0 ** -7
