"""Seeded Mask R-CNN detectors for the detector engine's tests and benchmark (no trained checkpoint is available).

`make_detector` builds what `megapose6d_b200.detector.create_model_detector` builds -- torchvision's Mask R-CNN on a
ResNet-50 FPN, three aspect ratios per anchor size -- with seeded weights and seeded FrozenBatchNorm2d statistics, so
that the float64 fold does real work.  The residual branches' last norm is scaled down (as trained ResNets' are small)
so that activations stay well inside the fp16 range through the 16 bottlenecks.

`spread_scores` multiplies the RPN objectness layer and the box predictor's class scores: with torchvision's
initialisation (std 0.01) every class score of a random model sits near 1 / n_classes, under the default 0.05 score
threshold, and the model detects nothing.  Spread scores give detections whose ranks and thresholds are well separated.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch

ANCHOR_SIZES = ((32,), (64,), (128,), (256,), (512,))


def detector_cfg(input_resize: Tuple[int, int] = (480, 640), n_classes: int = 21):
    """A detector run configuration in the layout `detector.load_detector` reads (training/detector_models_cfg.py)."""
    return dict(input_resize=list(input_resize), backbone_str="resnet50-fpn", anchor_sizes=[list(s) for s in ANCHOR_SIZES],
                train_ds_names=[["ycbv.pbr", 1]],
                label_to_category_id={"background": 0, **{f"obj_{i:06d}": i for i in range(1, n_classes + 1)}})


@torch.no_grad()
def seed_weights(model: torch.nn.Module, seed: int = 0, spread_scores: Optional[float] = None,
                 residual_scale: float = 0.2) -> torch.nn.Module:
    """Seeded parameters and FrozenBatchNorm2d statistics, in place."""
    from torchvision.ops.misc import FrozenBatchNorm2d

    g = torch.Generator().manual_seed(seed)
    for name, m in model.named_modules():
        if isinstance(m, torch.nn.Conv2d):
            fan_in = m.in_channels * m.kernel_size[0] * m.kernel_size[1]
            m.weight.copy_(torch.randn(m.weight.shape, generator=g) * (2.0 / fan_in) ** 0.5)
            if m.bias is not None:
                m.bias.copy_(torch.randn(m.bias.shape, generator=g) * 0.05)
        elif isinstance(m, FrozenBatchNorm2d):
            c = m.weight.numel()
            scale = residual_scale if name.endswith("bn3") or name.endswith("downsample.1") else 1.0
            m.weight.copy_((0.75 + 0.5 * torch.rand(c, generator=g)) * scale)
            m.bias.copy_(torch.randn(c, generator=g) * 0.1)
            m.running_mean.copy_(torch.randn(c, generator=g) * 0.1)
            m.running_var.copy_(0.5 + torch.rand(c, generator=g))
        elif isinstance(m, torch.nn.Linear):
            m.weight.copy_(torch.randn(m.weight.shape, generator=g) * (1.0 / m.in_features) ** 0.5)
            m.bias.copy_(torch.randn(m.bias.shape, generator=g) * 0.01)
    # the score layers read ReLU outputs (all >= 0): zero-sum weight rows keep one class from winning every box
    cls = model.roi_heads.box_predictor.cls_score.weight
    cls.sub_(cls.mean(dim=1, keepdim=True))
    if spread_scores:
        model.rpn.head.cls_logits.weight.mul_(spread_scores)
        cls.mul_(spread_scores)
    return model


def make_detector(input_resize: Tuple[int, int] = (480, 640), n_classes: int = 21, seed: int = 0,
                  spread_scores: Optional[float] = None, device: str = "cuda") -> torch.nn.Module:
    """Seeded torchvision MaskRCNN (n_classes objects + background), eval mode, on `device`, with `.config` / `.cfg` as
    `detector.load_detector` sets them."""
    from megapose6d_b200.detector import check_update_config_detector, create_model_detector
    from megapose6d_b200.load_model import Cfg

    cfg = check_update_config_detector(Cfg(**detector_cfg(input_resize, n_classes)))
    torch.manual_seed(seed)
    model = create_model_detector(cfg, len(cfg.label_to_category_id))
    seed_weights(model, seed, spread_scores)
    model = model.to(device).eval()
    model.cfg = cfg
    model.config = cfg
    return model


def write_detector_run(root, run_id: str, input_resize: Tuple[int, int] = (480, 640), n_classes: int = 21, seed: int = 0,
                       spread_scores: Optional[float] = None, background_bias: float = 0.0) -> None:
    """`<root>/<run_id>/{config.yaml, checkpoint.pth.tar}` of a seeded detector, the layout `load_detector` reads.
    `background_bias` is added to the background class logit: fewer boxes pass the score threshold."""
    from pathlib import Path

    import yaml

    model = make_detector(input_resize, n_classes, seed, spread_scores, device="cpu")
    with torch.no_grad():
        model.roi_heads.box_predictor.cls_score.bias[0] += background_bias
    run = Path(root) / run_id
    run.mkdir(parents=True, exist_ok=True)
    (run / "config.yaml").write_text(yaml.safe_dump(detector_cfg(input_resize, n_classes)))
    torch.save({"state_dict": model.state_dict()}, run / "checkpoint.pth.tar")



@torch.no_grad()
def integer_weights(model: torch.nn.Module, seed: int = 0, nnz: int = 2) -> torch.nn.Module:
    """In place: every convolution of the backbone and the RPN head gets `nnz` weights of +-1 per output channel (the rest
    zero) and an integer bias in -2..2; every FrozenBatchNorm2d is the identity plus an integer shift (eps 0).  With
    small-integer images every product and every fp32 partial sum of the plan is an integer below 2^24 -- each sum has
    at most nnz terms of at most 65504 plus the bias and one residual -- so fp32 accumulation is exact in any order and
    only the one rounding per convolution remains."""
    from torchvision.ops.misc import FrozenBatchNorm2d

    g = torch.Generator().manual_seed(seed)
    for m in list(model.backbone.modules()) + list(model.rpn.head.modules()):
        if isinstance(m, torch.nn.Conv2d):
            co = m.out_channels
            k = m.weight[0].numel()
            w = torch.zeros(co, k)
            idx = torch.stack([torch.randperm(k, generator=g)[:nnz] for _ in range(co)])
            w.scatter_(1, idx, (torch.randint(0, 2, (co, nnz), generator=g) * 2 - 1).float())
            m.weight.copy_(w.view_as(m.weight))
            if m.bias is not None:
                m.bias.copy_(torch.randint(-2, 3, (co,), generator=g).float())
        elif isinstance(m, FrozenBatchNorm2d):
            m.weight.fill_(1.0)
            m.bias.copy_(torch.randint(-2, 3, m.bias.shape, generator=g).float())
            m.running_mean.zero_()
            m.running_var.fill_(1.0)
            m.eps = 0.0
    return model


@torch.no_grad()
def integer_roi_heads_weights(model: torch.nn.Module, seed: int = 0, nnz: int = 2) -> torch.nn.Module:
    """In place: every layer of the RoI heads (fc6, fc7, cls_score, bbox_pred, the mask head's convolutions,
    conv5_mask and mask_fcn_logits) gets `nnz` weights of +-1 per output row (the rest zero) and an integer bias in
    -2..2.  Each output is then a sum of nnz act16 inputs and an integer, which fp32 accumulates exactly in any order
    for inputs of small dynamic range, so only the one rounding per layer remains between the engine and the float64
    oracle (oracle/detector_heads_ref.py)."""
    rh = model.roi_heads
    g = torch.Generator().manual_seed(seed)
    layers = [rh.box_head.fc6, rh.box_head.fc7, rh.box_predictor.cls_score, rh.box_predictor.bbox_pred,
              *[block[0] for block in rh.mask_head], rh.mask_predictor.mask_fcn_logits]
    for m in layers:
        co = m.weight.shape[0]
        k = m.weight[0].numel()
        w = torch.zeros(co, k)
        idx = torch.stack([torch.randperm(k, generator=g)[:nnz] for _ in range(co)])
        w.scatter_(1, idx, (torch.randint(0, 2, (co, nnz), generator=g) * 2 - 1).float())
        m.weight.copy_(w.view_as(m.weight))
        m.bias.copy_(torch.randint(-2, 3, (co,), generator=g).float())
    conv5 = rh.mask_predictor.conv5_mask  # weight [in, out, 2, 2]: nnz input channels per (output channel, tap)
    ci, co = conv5.weight.shape[:2]
    w = torch.zeros(co * 4, ci)
    idx = torch.stack([torch.randperm(ci, generator=g)[:nnz] for _ in range(co * 4)])
    w.scatter_(1, idx, (torch.randint(0, 2, (co * 4, nnz), generator=g) * 2 - 1).float())
    conv5.weight.copy_(w.view(co, 2, 2, ci).permute(3, 0, 1, 2))
    conv5.bias.copy_(torch.randint(-2, 3, (co,), generator=g).float())
    return model
