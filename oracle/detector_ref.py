"""float64 oracle of the detector engine's ResNet-50 FPN + RPN head plan (megapose6d_b200/detector_engine.py,
csrc/detector_net.cu), written against torchvision's modules: the function the engine computes, with its quantisation
points and nothing else.

  * the input batch rounded to act16 (the engine's space-to-depth conversion);
  * every FrozenBatchNorm2d folded into the convolution before it in float64 with the module's eps, the folded weights
    rounded to act16 and the biases to fp32, as the engine stores them;
  * each convolution evaluated in float64 and its output rounded ONCE to act16 after bias, residual and ReLU -- the
    bottleneck's identity / downsample residual and the FPN's nearest-upsampled top-down term are added before that
    rounding, as the engine adds them in its fp32 epilogue;
  * max-pool, nearest upsampling and the pool level's [::2, ::2] are exact.
Only the fp32 summation order inside a convolution differs from the engine.  act16 is fp16; conversions saturate at
+-65504.
"""
from __future__ import annotations

from typing import List, Tuple

import torch
import torch.nn.functional as F

F16_MAX = 65504.0


def q(t: torch.Tensor) -> torch.Tensor:
    """Round to fp16 (through fp32, saturating), back to float64."""
    return t.to(torch.float32).clamp(-F16_MAX, F16_MAX).to(torch.float16).to(torch.float64)


def _folded(conv, bn) -> Tuple[torch.Tensor, torch.Tensor]:
    scale = bn.weight.double() / torch.sqrt(bn.running_var.double() + bn.eps)
    w = conv.weight.double() * scale.view(-1, 1, 1, 1)
    b = bn.bias.double() - bn.running_mean.double() * scale
    return q(w), b.float().double()


def _conv(x, conv, bn=None, residual=None, relu=False, round_out=True):
    if bn is not None:
        w, b = _folded(conv, bn)
    else:
        w, b = q(conv.weight.double()), conv.bias.float().double()
    y = F.conv2d(x, w.to(x.device), b.to(x.device), stride=conv.stride, padding=conv.padding)
    if residual is not None:
        y = y + residual
    if relu:
        y = F.relu(y)
    return q(y) if round_out else y


@torch.no_grad()
def forward(model, images: torch.Tensor) -> Tuple[List[torch.Tensor], List[torch.Tensor], List[torch.Tensor]]:
    """images: the padded fp32 batch [n, 3, h, w] (ImageList.tensors) -> float64 (features, objectness, deltas), five
    levels each, as torchvision's backbone and RPN head return them."""
    body, fpn, head = model.backbone.body, model.backbone.fpn, model.rpn.head
    x = q(images.double())
    x = _conv(x, body.conv1, body.bn1, relu=True)
    x = F.max_pool2d(x, kernel_size=3, stride=2, padding=1)
    c = []
    for li in range(1, 5):
        for blk in getattr(body, f"layer{li}"):
            identity = x
            t = _conv(x, blk.conv1, blk.bn1, relu=True)
            t = _conv(t, blk.conv2, blk.bn2, relu=True)
            if blk.downsample is not None:
                identity = _conv(x, blk.downsample[0], blk.downsample[1])
            x = _conv(t, blk.conv3, blk.bn3, residual=identity, relu=True)
        c.append(x)
    inner = _conv(c[3], fpn.inner_blocks[3][0])
    feats = [_conv(inner, fpn.layer_blocks[3][0])]
    for i in (2, 1, 0):
        lateral = _conv(c[i], fpn.inner_blocks[i][0], round_out=False)
        top_down = F.interpolate(inner, size=lateral.shape[-2:], mode="nearest")
        inner = q(lateral + top_down)
        feats.insert(0, _conv(inner, fpn.layer_blocks[i][0]))
    feats.append(feats[-1][:, :, ::2, ::2])
    objectness, deltas = [], []
    for f in feats:
        t = _conv(f, head.conv[0][0], relu=True)
        objectness.append(_conv(t, head.cls_logits))
        deltas.append(_conv(t, head.bbox_pred))
    return feats, objectness, deltas


# Stated bounds (DESIGN §4), per output tensor and in units of that tensor's largest magnitude.
# The oracle against torchvision's fp32 backbone + RPN head (TF32 off): every act16 rounding adds a relative error of at
# most u = 2^-11 to its element, about 60 of them lie on the deepest path (stem, 48 bottleneck convolutions, FPN, RPN),
# and through weights of Gaussian scale they add like a random walk: a few u * sqrt(depth / 8) of the tensor's scale.
# Observed on the seeded workload: at most 3.3 u at 64x96; the bound is 16 u.
ORACLE_VS_FP32 = 2.0 ** -7
# The engine against this oracle: only the fp32 summation order differs, so a convolution output can differ by one act16
# rounding step (u of its magnitude) where the two sums straddle a rounding boundary, and those differences propagate
# through the rest of the plan like the roundings above: the same form and the same 16 u.  Observed on an H100: 5.1 u
# at 1x480x640, 3.9 u at 2x256x320 (and 4.9 u / 4.0 u for the engine against torchvision fp32, bound 32 u).
ENGINE_VS_ORACLE = 2.0 ** -7
