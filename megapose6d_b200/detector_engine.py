"""The Mask R-CNN detector's ResNet-50 FPN backbone and RPN head on the engine's wgmma convolutions.

`engine_model(model)` takes a torchvision `MaskRCNN` (what `detector.create_model_detector` builds, the reference's
models/mask_rcnn.py:23-46) and returns a module that is called like it (`module(list_of_images)` in eval mode) and returns
the same kind of detections.  The backbone (body + FPN) and `rpn.head` run as one `mpx_fpn_forward` (include/mpx.h,
csrc/detector_net.cu); everything else is the model's own torchvision objects, run unchanged: the transform, the anchor
generator, proposal decoding and filtering, the RoI heads and the postprocessing.  The model itself is not modified.

Weights are repacked once:
  * FrozenBatchNorm2d folded into the convolution before it, in float64 with the module's eps (`backbone._fold`);
  * the 7x7/s2 stem rewritten as the 4x4 convolution over the space-to-depth input (`backbone._stem_s2d`, c_pad 16);
  * `cls_logits` (A rows) and `bbox_pred` (4A rows) merged into one 1x1 convolution of 64 rows, the rest zero;
  * every matrix rounded once to the library's 16-bit type, saturating.

With `device_paste=True` the module runs the RoI heads' stages one by one (the model's box RoI pool, box head, box predictor,
postprocess_detections, mask RoI pool, mask head and mask predictor, unchanged) and then, instead of maskrcnn_inference
and GeneralizedRCNNTransform.postprocess, one `mpx_mask_paste` (include/mpx.h) for the whole batch: sigmoid, the label's
channel, resize_boxes and paste_masks_in_image on the device.  torchvision pastes the masks in a Python loop with several
host synchronisations per detection; the device paste has none, so the number of synchronisations per call no longer
grows with the number of detections.  Boxes, labels and scores are those of `device_paste=False`; the probabilities differ
from torchvision's by a few ulps at most (see `mask_paste`).
"""
from __future__ import annotations

import ctypes
from collections import OrderedDict
from typing import Dict, List, NamedTuple, Optional, Tuple

import torch
from torch import nn

from . import _abi
from .backbone import _fold, _pack, _stem_s2d

C_PAD = 16  # space-to-depth channels per sub-pixel: 3 colour channels, zero-padded
LAYERS = [3, 4, 6, 3]
WIDTHS = [64, 128, 256, 512]
FPN_IN = [256, 512, 1024, 2048]
FPN_CHANNELS = 256
HEAD_ROWS = 64  # merged RPN 1x1: A objectness rows + 4A delta rows, zero-padded
MAX_ANCHORS = HEAD_ROWS // 5
LEVELS = ["0", "1", "2", "3", "pool"]


class PlanConv(NamedTuple):
    """One convolution of the plan, as the engine runs it (stem: as the torchvision 7x7 module it replaces)."""
    modules: Tuple[str, ...]  # Conv2d module name(s); two for the merged RPN 1x1
    norm: Optional[str]       # FrozenBatchNorm2d folded into it, or None (the convolution has its own bias)
    kernel: int
    stride: int
    padding: int
    c_in: int
    c_out: int


def weight_plan(n_anchors: int) -> List[PlanConv]:
    """The 63 convolutions in the order mpx_fpn_create takes them (include/mpx.h)."""
    body = "backbone.body"
    plan = [PlanConv((f"{body}.conv1",), f"{body}.bn1", 7, 2, 3, 3, 64)]
    c_in = 64
    for li, (nb, width) in enumerate(zip(LAYERS, WIDTHS)):
        for bi in range(nb):
            p = f"{body}.layer{li + 1}.{bi}"
            stride = 2 if bi == 0 and li > 0 else 1
            plan.append(PlanConv((p + ".conv1",), p + ".bn1", 1, 1, 0, c_in, width))
            plan.append(PlanConv((p + ".conv2",), p + ".bn2", 3, stride, 1, width, width))
            if bi == 0:
                plan.append(PlanConv((p + ".downsample.0",), p + ".downsample.1", 1, stride, 0, c_in, 4 * width))
            plan.append(PlanConv((p + ".conv3",), p + ".bn3", 1, 1, 0, width, 4 * width))
            c_in = 4 * width
    for i, c in enumerate(FPN_IN):
        plan.append(PlanConv((f"backbone.fpn.inner_blocks.{i}.0",), None, 1, 1, 0, c, FPN_CHANNELS))
    for i in range(4):
        plan.append(PlanConv((f"backbone.fpn.layer_blocks.{i}.0",), None, 3, 1, 1, FPN_CHANNELS, FPN_CHANNELS))
    plan.append(PlanConv(("rpn.head.conv.0.0",), None, 3, 1, 1, FPN_CHANNELS, FPN_CHANNELS))
    plan.append(PlanConv(("rpn.head.cls_logits", "rpn.head.bbox_pred"), None, 1, 1, 0, FPN_CHANNELS, 5 * n_anchors))
    return plan


def _refuse(what: str) -> None:
    raise NotImplementedError(f"engine_model: {what} is not served by the engine's ResNet-50 FPN plan")


def check_supported(model: nn.Module) -> int:
    """Raises NotImplementedError for a structure the plan does not serve; returns the anchors per location."""
    from torchvision.models.detection.backbone_utils import BackboneWithFPN
    from torchvision.models.detection.generalized_rcnn import GeneralizedRCNN
    from torchvision.models.resnet import Bottleneck
    from torchvision.ops.feature_pyramid_network import LastLevelMaxPool
    from torchvision.ops.misc import FrozenBatchNorm2d

    if not isinstance(model, GeneralizedRCNN) or not hasattr(model, "rpn"):
        _refuse(f"a {type(model).__name__}")
    if getattr(model.transform, "size_divisible", None) != 32:
        _refuse(f"size_divisible={getattr(model.transform, 'size_divisible', None)}")
    bb = model.backbone
    if not isinstance(bb, BackboneWithFPN):
        _refuse(f"the backbone {type(bb).__name__}")
    body = bb.body
    if dict(body.return_layers) != {"layer1": "0", "layer2": "1", "layer3": "2", "layer4": "3"}:
        _refuse(f"returned layers {dict(body.return_layers)}")
    for li, nb in enumerate(LAYERS):
        layer = getattr(body, f"layer{li + 1}", None)
        if layer is None or len(layer) != nb or not all(isinstance(b, Bottleneck) for b in layer):
            _refuse(f"layer{li + 1} (the ResNet-50 body has [3, 4, 6, 3] Bottleneck blocks)")
    if not isinstance(bb.fpn.extra_blocks, LastLevelMaxPool):
        _refuse(f"the FPN extra block {type(bb.fpn.extra_blocks).__name__}")
    if bb.out_channels != FPN_CHANNELS:
        _refuse(f"an FPN of {bb.out_channels} channels")
    for blocks in (bb.fpn.inner_blocks, bb.fpn.layer_blocks):
        if len(blocks) != 4 or any(len(b) != 1 for b in blocks):
            _refuse("an FPN with a norm layer or other than four levels")
    head = model.rpn.head
    if len(head.conv) != 1:
        _refuse(f"an RPN head with conv_depth={len(head.conv)}")
    n_anchors = head.cls_logits.out_channels
    if n_anchors > MAX_ANCHORS or head.bbox_pred.out_channels != 4 * n_anchors:
        _refuse(f"{n_anchors} anchors per location (at most {MAX_ANCHORS})")
    mods = dict(model.named_modules())
    for pc in weight_plan(n_anchors):
        if pc.norm is not None and type(mods.get(pc.norm)) is not FrozenBatchNorm2d:
            _refuse(f"the norm {type(mods.get(pc.norm)).__name__} at {pc.norm} (FrozenBatchNorm2d only)")
        for name in pc.modules:
            conv = mods.get(name)
            if not isinstance(conv, nn.Conv2d):
                _refuse(f"{name} (not a Conv2d)")
            if conv.dilation != (1, 1) or conv.groups != 1:
                _refuse(f"dilation {conv.dilation} / groups {conv.groups} at {name}")
            k = pc.kernel
            if (conv.kernel_size != (k, k) or conv.stride != (pc.stride, pc.stride) or conv.padding != (pc.padding,) * 2
                    or conv.in_channels != pc.c_in or (len(pc.modules) == 1 and conv.out_channels != pc.c_out)
                    or (conv.bias is None) != (pc.norm is not None)):
                _refuse(f"the convolution {name} {tuple(conv.weight.shape)} stride {conv.stride} padding {conv.padding}")
    mp = body.maxpool
    if (mp.kernel_size, mp.stride, mp.padding) != (3, 2, 1):
        _refuse("the stem max-pool")
    return n_anchors


def fold_plan(model: nn.Module, n_anchors: int) -> List[Tuple[torch.Tensor, torch.Tensor]]:
    """float64 (weight OIHW, bias) per plan entry: norms folded, the RPN 1x1 merged and zero-padded to 64 rows."""
    sd = model.state_dict()
    mods = dict(model.named_modules())
    out = []
    for pc in weight_plan(n_anchors):
        if pc.norm is not None:
            out.append(_fold(sd, pc.modules[0], pc.norm, eps=mods[pc.norm].eps))
            continue
        w = torch.cat([sd[m + ".weight"].detach().double().cpu() for m in pc.modules])
        b = torch.cat([sd[m + ".bias"].detach().double().cpu() for m in pc.modules])
        if len(pc.modules) > 1:
            w = torch.cat([w, w.new_zeros(HEAD_ROWS - w.shape[0], *w.shape[1:])])
            b = torch.cat([b, b.new_zeros(HEAD_ROWS - b.shape[0])])
        out.append((w, b))
    return out


def to_act16(t: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """float -> the 16-bit type, round-to-nearest-even through fp32, saturating at the type's largest finite value."""
    lim = float(torch.finfo(dtype).max)
    return t.to(torch.float32).clamp(-lim, lim).to(dtype)


def level_sizes(h: int, w: int) -> List[Tuple[int, int]]:
    """(h_l, w_l) of the levels '0', '1', '2', '3', 'pool' for a padded batch of h x w (multiples of 32)."""
    sizes = [(h >> l, w >> l) for l in range(2, 6)]
    return sizes + [((sizes[-1][0] + 1) // 2, (sizes[-1][1] + 1) // 2)]


MASK_MAX_RESOLUTION = 64  # mpx_mask_paste's largest m (Mask R-CNN: 28)
MASK_MAX_IMAGES = 64      # images per mpx_mask_paste call


def check_supported_device_paste(model: nn.Module) -> None:
    """Raises NotImplementedError for RoI heads whose masks `device_paste=True` cannot paste on the device."""
    from torchvision.models.detection.transform import GeneralizedRCNNTransform

    if type(model.transform) is not GeneralizedRCNNTransform:
        _refuse(f"the transform {type(model.transform).__name__}")
    rh = model.roi_heads
    if rh.mask_roi_pool is None or rh.mask_head is None or rh.mask_predictor is None:
        _refuse("RoI heads without a mask branch (device_paste=True pastes masks)")
    if rh.keypoint_roi_pool is not None or rh.keypoint_head is not None or rh.keypoint_predictor is not None:
        _refuse("a keypoint branch")
    size = rh.mask_roi_pool.output_size
    size = (size, size) if isinstance(size, int) else tuple(size)
    conv5 = getattr(rh.mask_predictor, "conv5_mask", None)
    if (size[0] != size[1] or not isinstance(conv5, nn.ConvTranspose2d) or conv5.stride != (2, 2)
            or conv5.kernel_size != (2, 2) or 2 * size[0] > MASK_MAX_RESOLUTION):
        _refuse(f"a mask predictor of {size} RoIs (square pools and a 2x2/2 ConvTranspose2d to at most "
                f"{MASK_MAX_RESOLUTION}x{MASK_MAX_RESOLUTION} masks)")


def mask_paste(mask_logits: torch.Tensor, labels: torch.Tensor, boxes: torch.Tensor, counts: List[int],
               image_sizes: List[Tuple[int, int]], original_sizes: List[Tuple[int, int]]
               ) -> Tuple[List[torch.Tensor], List[torch.Tensor]]:
    """maskrcnn_inference + resize_boxes + paste_masks_in_image on the device, in one launch for the batch.
    mask_logits [N, classes, m, m] fp32, labels [N] int64, boxes [N, 4] fp32 in the transformed images' coordinates,
    counts: detections per image (the rows of image 0 first).  Returns per image the resized boxes [count, 4] and the
    fp32 masks [count, 1, H, W] at the original size."""
    n_images = len(counts)
    if not 1 <= n_images <= MASK_MAX_IMAGES:
        raise ValueError(f"mask_paste: {n_images} images, must be 1..{MASK_MAX_IMAGES}")
    n, n_classes, m, m2 = mask_logits.shape
    if m != m2 or labels.shape != (n,) or boxes.shape != (n, 4) or sum(counts) != n:
        raise ValueError(f"mask_paste: logits {tuple(mask_logits.shape)}, labels {tuple(labels.shape)}, boxes "
                         f"{tuple(boxes.shape)}, counts {counts}")
    device = mask_logits.device
    logits = mask_logits.to(torch.float32).contiguous()
    labels = labels.to(torch.int64).contiguous()
    boxes = boxes.to(torch.float32).contiguous()
    boxes_out = torch.empty_like(boxes)
    masks = [torch.empty(c, 1, H, W, device=device) for c, (H, W) in zip(counts, original_sizes)]
    sizes = [v for (h, w), (H, W) in zip(image_sizes, original_sizes) for v in (h, w, H, W)]
    c_counts = (ctypes.c_int32 * n_images)(*counts)
    c_sizes = (ctypes.c_int32 * (4 * n_images))(*sizes)
    c_masks = (ctypes.c_void_p * n_images)(*[t.data_ptr() if t.numel() else None for t in masks])
    _abi.check(_abi.lib().mpx_mask_paste(logits.data_ptr(), labels.data_ptr(), boxes.data_ptr(), n, n_classes, m,
                                         n_images, c_counts, c_sizes, boxes_out.data_ptr(), c_masks,
                                         _abi.stream_ptr()))
    return list(boxes_out.split(counts)), masks


ROI_LEVELS = ["0", "1", "2", "3"]
ROI_CHANNELS = 256
BOX_POOL = 7
MAX_ROWS = 2048  # conv_forward's largest C_out


def _rows(n: int) -> int:
    return (n + 63) // 64 * 64


def check_supported_roi_heads(model: nn.Module) -> None:
    """Raises NotImplementedError for RoI heads `engine_roi_heads=True` does not serve (and for whatever
    check_supported_device_paste refuses)."""
    from torchvision.models.detection.faster_rcnn import FastRCNNPredictor, TwoMLPHead
    from torchvision.models.detection.mask_rcnn import MaskRCNNHeads, MaskRCNNPredictor
    from torchvision.ops import MultiScaleRoIAlign

    check_supported_device_paste(model)
    rh = model.roi_heads
    for name in ("box_roi_pool", "mask_roi_pool"):
        pool = getattr(rh, name)
        if type(pool) is not MultiScaleRoIAlign or list(pool.featmap_names) != ROI_LEVELS:
            _refuse(f"the {name} {type(pool).__name__} (MultiScaleRoIAlign on '0'..'3' only)")
        if not isinstance(pool.sampling_ratio, int) or pool.sampling_ratio < 1 or pool.sampling_ratio > 16:
            _refuse(f"the {name} sampling_ratio {pool.sampling_ratio} (a fixed ratio 1..16)")
        if not isinstance(pool.canonical_scale, int) or not isinstance(pool.canonical_level, int):
            _refuse(f"the {name} canonical scale / level {pool.canonical_scale} / {pool.canonical_level}")
    if tuple(rh.box_roi_pool.output_size) != (BOX_POOL, BOX_POOL):
        _refuse(f"a box pool of {tuple(rh.box_roi_pool.output_size)} (7x7 only)")
    head = rh.box_head
    if type(head) is not TwoMLPHead or head.fc6.in_features != ROI_CHANNELS * BOX_POOL * BOX_POOL:
        _refuse(f"the box head {type(head).__name__} (TwoMLPHead on 256x7x7 only)")
    hidden = head.fc6.out_features
    if (hidden % 64 or hidden > MAX_ROWS or head.fc7.in_features != hidden or head.fc7.out_features != hidden
            or head.fc6.bias is None or head.fc7.bias is None):
        _refuse(f"a box head of representation size {hidden} (a multiple of 64 up to {MAX_ROWS}, with biases)")
    pred = rh.box_predictor
    if type(pred) is not FastRCNNPredictor or pred.cls_score.in_features != hidden:
        _refuse(f"the box predictor {type(pred).__name__} (FastRCNNPredictor only)")
    n_classes = pred.cls_score.out_features
    if pred.bbox_pred.out_features != 4 * n_classes or _rows(5 * n_classes) > MAX_ROWS:
        _refuse(f"a box predictor of {n_classes} classes (5 x classes rounded up to 64 at most {MAX_ROWS})")
    mh = rh.mask_head
    if type(mh) is not MaskRCNNHeads or len(mh) != 4:
        _refuse(f"the mask head {type(mh).__name__} (MaskRCNNHeads with four layers only)")
    for i, block in enumerate(mh):
        conv = block[0] if isinstance(block, nn.Sequential) else None
        if (not isinstance(conv, nn.Conv2d) or len(block) != 2 or not isinstance(block[1], nn.ReLU)
                or conv.kernel_size != (3, 3) or conv.stride != (1, 1) or conv.padding != (1, 1)
                or conv.dilation != (1, 1) or conv.groups != 1 or conv.in_channels != ROI_CHANNELS
                or conv.out_channels != ROI_CHANNELS or conv.bias is None):
            _refuse(f"mask head layer {i} (3x3 convolutions of 256 channels with bias and ReLU, no norm)")
    mp = rh.mask_predictor
    conv5, logits = getattr(mp, "conv5_mask", None), getattr(mp, "mask_fcn_logits", None)
    if (type(mp) is not MaskRCNNPredictor or conv5.in_channels != ROI_CHANNELS or conv5.out_channels != ROI_CHANNELS
            or conv5.padding != (0, 0) or conv5.output_padding != (0, 0) or conv5.groups != 1
            or conv5.dilation != (1, 1) or conv5.bias is None or not isinstance(logits, nn.Conv2d)
            or logits.kernel_size != (1, 1) or logits.out_channels != n_classes or logits.bias is None):
        _refuse(f"the mask predictor {type(mp).__name__} (MaskRCNNPredictor, 256 channels, one logit per class)")


def roi_heads_plan(model: nn.Module) -> List[Tuple[torch.Tensor, torch.Tensor]]:
    """float64 (weight [C_out, R*S*C_in] with k = (r, s, c), bias [C_out]) of the nine convolutions mpx_roi_heads_create
    takes: fc6 as a 7x7 convolution, fc7, the merged predictor, the four mask-head 3x3, conv5_mask as a 1x1 convolution
    to the four sub-pixels, mask_fcn_logits.  The predictors are zero-padded to a multiple of 64 rows."""
    rh = model.roi_heads
    d = lambda t: t.detach().double().cpu()  # noqa: E731

    def pad(w, b):
        rows = _rows(w.shape[0])
        return (torch.cat([w, w.new_zeros(rows - w.shape[0], w.shape[1])]),
                torch.cat([b, b.new_zeros(rows - b.shape[0])]))

    fc6, fc7 = rh.box_head.fc6, rh.box_head.fc7
    hidden = fc6.out_features
    plan = [(_pack(d(fc6.weight).view(hidden, ROI_CHANNELS, BOX_POOL, BOX_POOL)), d(fc6.bias)),
            (d(fc7.weight), d(fc7.bias))]
    pred = rh.box_predictor
    plan.append(pad(torch.cat([d(pred.cls_score.weight), d(pred.bbox_pred.weight)]),
                    torch.cat([d(pred.cls_score.bias), d(pred.bbox_pred.bias)])))
    plan += [(_pack(d(block[0].weight)), d(block[0].bias)) for block in rh.mask_head]
    conv5, logits = rh.mask_predictor.conv5_mask, rh.mask_predictor.mask_fcn_logits
    # ConvTranspose2d weight [in, out, dy, dx] -> row (dy * 2 + dx) * out + o, column = input channel
    plan.append((d(conv5.weight).permute(2, 3, 1, 0).reshape(4 * ROI_CHANNELS, ROI_CHANNELS), d(conv5.bias).repeat(4)))
    plan.append(pad(d(logits.weight).flatten(1), d(logits.bias)))
    return plan


def pool_args(pool: nn.Module, features: List[torch.Tensor], image_sizes: List[Tuple[int, int]]):
    """(scales, canonical_scale, canonical_level, sampling_ratio) as MultiScaleRoIAlign computes them for these features
    and images (torchvision.ops.poolers._setup_scales), without caching them in the module."""
    from torchvision.ops.poolers import _setup_scales

    scales, _ = _setup_scales(features, image_sizes, pool.canonical_scale, pool.canonical_level)
    return (ctypes.c_float * 4)(*scales), pool.canonical_scale, pool.canonical_level, pool.sampling_ratio


class RoiHeadsEngine:
    """Owns the repacked device weights of the RoI heads and the mpx_roi_heads handle (include/mpx.h)."""

    def __init__(self, model: nn.Module, device="cuda"):
        check_supported_roi_heads(model)
        rh = model.roi_heads
        self.device = torch.device(device)
        self.n_classes = rh.box_predictor.cls_score.out_features
        self.hidden = rh.box_head.fc6.out_features
        self.mask_pool = int(rh.mask_roi_pool.output_size[0])
        self._box_pool, self._mask_pool = rh.box_roi_pool, rh.mask_roi_pool
        act = _abi.act_dtype()
        plan = roi_heads_plan(model)
        self._weights = [to_act16(w, act).to(self.device).contiguous() for w, _ in plan]
        self._biases = [b.to(torch.float32).to(self.device).contiguous() for _, b in plan]
        n = len(self._weights)
        wp = (ctypes.c_void_p * n)(*[t.data_ptr() for t in self._weights])
        bp = (ctypes.c_void_p * n)(*[t.data_ptr() for t in self._biases])
        handle = ctypes.c_void_p()
        _abi.check(_abi.lib().mpx_roi_heads_create(wp, bp, n, self.n_classes, self.hidden, ctypes.byref(handle)))
        self._handle = handle
        self._workspace: Optional[torch.Tensor] = None

    def __del__(self):
        try:
            if getattr(self, "_handle", None) is not None:
                _abi.lib().mpx_roi_heads_destroy(self._handle)
        except Exception:  # noqa: BLE001
            pass

    def _ws(self, n_box: int, n_mask: int) -> torch.Tensor:
        need = _abi.lib().mpx_roi_heads_workspace_bytes(self._handle, n_box, n_mask, self.mask_pool)
        if self._workspace is None or self._workspace.numel() < need:
            self._workspace = None
            self._workspace = torch.empty(max(need, 256), dtype=torch.uint8, device=self.device)
        return self._workspace

    def _features(self, features, n_images: int, batch_hw: Tuple[int, int]) -> Tuple[List[torch.Tensor], "ctypes.Array"]:
        """The levels '0'..'3', checked against the shapes the kernels derive from the batch size and count."""
        feats = [features[k] for k in ROI_LEVELS]
        for l, f in enumerate(feats):
            want = (n_images, ROI_CHANNELS, batch_hw[0] >> (l + 2), batch_hw[1] >> (l + 2))
            if f.dtype != torch.float32 or not f.is_contiguous() or tuple(f.shape) != want or not f.is_cuda:
                raise ValueError(f"RoiHeadsEngine: level {l} must be a contiguous fp32 CUDA tensor {list(want)}, "
                                 f"got {f.dtype} {tuple(f.shape)} on {f.device}")
        return feats, (ctypes.c_void_p * 4)(*[f.data_ptr() for f in feats])

    def _boxes(self, boxes: torch.Tensor, n: int) -> torch.Tensor:
        if tuple(boxes.shape) != (n, 4) or not boxes.is_cuda:
            raise ValueError(f"RoiHeadsEngine: boxes must be a CUDA tensor [{n}, 4], got {tuple(boxes.shape)} on "
                             f"{boxes.device}")
        return boxes.to(torch.float32).contiguous()

    def box(self, features, boxes: torch.Tensor, counts: List[int], batch_hw: Tuple[int, int],
            image_sizes: List[Tuple[int, int]]) -> Tuple[torch.Tensor, torch.Tensor]:
        """box_roi_pool + box_head + box_predictor: fp32 class_logits [P, C] and box_regression [P, 4C] of the RoIs
        `boxes` [P, 4] (counts: RoIs per image)."""
        feats, fp = self._features(features, len(counts), batch_hw)
        n = int(sum(counts))
        boxes = self._boxes(boxes, n)
        logits = torch.empty(n, self.n_classes, device=self.device)
        deltas = torch.empty(n, 4 * self.n_classes, device=self.device)
        ws = self._ws(n, 0)
        _abi.check(_abi.lib().mpx_roi_box_forward(
            self._handle, fp, len(counts), batch_hw[0], batch_hw[1], *pool_args(self._box_pool, feats, image_sizes),
            boxes.data_ptr(), (ctypes.c_int32 * len(counts))(*counts), logits.data_ptr(), deltas.data_ptr(),
            ws.data_ptr(), ws.numel(), _abi.stream_ptr()))
        return logits, deltas

    def mask(self, features, boxes: torch.Tensor, counts: List[int], batch_hw: Tuple[int, int],
             image_sizes: List[Tuple[int, int]]) -> torch.Tensor:
        """mask_roi_pool + mask_head + mask_predictor: fp32 mask logits [N, C, 2s, 2s] of the boxes [N, 4]."""
        feats, fp = self._features(features, len(counts), batch_hw)
        n = int(sum(counts))
        m = 2 * self.mask_pool
        boxes = self._boxes(boxes, n)
        out = torch.empty(n, self.n_classes, m, m, device=self.device)
        ws = self._ws(0, n)
        _abi.check(_abi.lib().mpx_roi_mask_forward(
            self._handle, fp, len(counts), batch_hw[0], batch_hw[1], *pool_args(self._mask_pool, feats, image_sizes),
            self.mask_pool, boxes.data_ptr(), (ctypes.c_int32 * len(counts))(*counts), out.data_ptr(), ws.data_ptr(),
            ws.numel(), _abi.stream_ptr()))
        return out


class FpnEngine:
    """Owns the repacked device weights and the mpx_fpn handle.  `run(images)` returns the FPN features, objectness and
    deltas of a padded fp32 batch [n, 3, h, w] as lists of five fp32 NCHW tensors.  The tensors are the engine's own
    output buffers, one set per shape, overwritten by the next call of that shape."""

    def __init__(self, model: nn.Module, device="cuda"):
        self.n_anchors = check_supported(model)
        self.device = torch.device(device)
        act = _abi.act_dtype()
        self._weights: List[torch.Tensor] = []
        self._biases: List[torch.Tensor] = []
        for i, (w, b) in enumerate(fold_plan(model, self.n_anchors)):
            wmat = _stem_s2d(w, C_PAD) if i == 0 else _pack(w)
            self._weights.append(to_act16(wmat, act).to(self.device).contiguous())
            self._biases.append(b.to(torch.float32).to(self.device).contiguous())
        n = len(self._weights)
        wp = (ctypes.c_void_p * n)(*[t.data_ptr() for t in self._weights])
        bp = (ctypes.c_void_p * n)(*[t.data_ptr() for t in self._biases])
        handle = ctypes.c_void_p()
        _abi.check(_abi.lib().mpx_fpn_create(wp, bp, n, self.n_anchors, ctypes.byref(handle)))
        self._handle = handle
        self._workspace: Optional[torch.Tensor] = None
        self._outputs: Dict[Tuple[int, int, int], Tuple[List[torch.Tensor], ...]] = {}

    def __del__(self):
        try:
            if getattr(self, "_handle", None) is not None:
                _abi.lib().mpx_fpn_destroy(self._handle)
        except Exception:  # noqa: BLE001
            pass

    def run(self, images: torch.Tensor) -> Tuple[List[torch.Tensor], List[torch.Tensor], List[torch.Tensor]]:
        n, c, h, w = images.shape
        if c != 3 or images.dtype != torch.float32:
            raise ValueError(f"FpnEngine.run: expected fp32 [n, 3, h, w], got {images.dtype} {tuple(images.shape)}")
        images = images.contiguous()
        need = _abi.lib().mpx_fpn_workspace_bytes(n, h, w)
        if need and (self._workspace is None or self._workspace.numel() < need):
            self._workspace = None
            self._workspace = torch.empty(need, dtype=torch.uint8, device=self.device)
        outs = self._outputs.get((n, h, w))
        if outs is None:
            sizes = level_sizes(h, w)
            A = self.n_anchors

            def alloc(ch):
                return [torch.empty(n, ch, hl, wl, device=self.device) for hl, wl in sizes]

            outs = self._outputs[(n, h, w)] = (alloc(FPN_CHANNELS), alloc(A), alloc(4 * A))
        arrays = [(ctypes.c_void_p * 5)(*[t.data_ptr() for t in ts]) for ts in outs]
        ws = self._workspace
        _abi.check(_abi.lib().mpx_fpn_forward(self._handle, _abi.ptr(images), n, h, w, *arrays,
                                              None if ws is None else ws.data_ptr(), 0 if ws is None else ws.numel(),
                                              _abi.stream_ptr()))
        return outs


class EngineMaskRCNN(nn.Module):
    """Called like torchvision's GeneralizedRCNN in eval mode: `module(images)` -> list of dicts(boxes, labels, scores,
    masks).  Holds the model's transform, RPN and RoI heads by reference (not as submodules: it does not own them)."""

    def __init__(self, model: nn.Module, device="cuda", device_paste: bool = False, engine_roi_heads: bool = False):
        super().__init__()
        device_paste = device_paste or engine_roi_heads
        if engine_roi_heads:
            check_supported_roi_heads(model)
        elif device_paste:
            check_supported_device_paste(model)
        self.device_paste = device_paste
        self.engine_roi_heads = engine_roi_heads
        self.engine = FpnEngine(model, device)
        self.roi_engine = RoiHeadsEngine(model, device) if engine_roi_heads else None
        self._stages = (model.transform, model.rpn, model.roi_heads)
        for attr in ("config", "cfg"):
            if hasattr(model, attr):
                setattr(self, attr, getattr(model, attr))
        self.train(False)

    def train(self, mode: bool = True):
        if mode:
            raise NotImplementedError("the engine detector runs inference only")
        return super().train(False)

    def heads(self, image_list) -> Tuple["OrderedDict[str, torch.Tensor]", List[torch.Tensor], List[torch.Tensor]]:
        """The backbone's feature OrderedDict and the RPN head's objectness / deltas of a transformed ImageList."""
        feats, objectness, deltas = self.engine.run(image_list.tensors)
        return OrderedDict(zip(LEVELS, feats)), objectness, deltas

    def proposals(self, image_list, features, objectness, deltas) -> List[torch.Tensor]:
        """RegionProposalNetwork.forward (eval) from the head's outputs: the model's anchor generator, box coder and
        proposal filter."""
        from torchvision.models.detection.rpn import concat_box_prediction_layers

        rpn = self._stages[1]
        anchors = rpn.anchor_generator(image_list, list(features.values()))
        num_anchors_per_level = [o[0].numel() for o in objectness]
        objectness, pred_bbox_deltas = concat_box_prediction_layers(objectness, deltas)
        proposals = rpn.box_coder.decode(pred_bbox_deltas.detach(), anchors).view(len(anchors), -1, 4)
        boxes, _ = rpn.filter_proposals(proposals, objectness, image_list.image_sizes, num_anchors_per_level)
        return boxes

    @torch.no_grad()
    def forward(self, images: List[torch.Tensor], targets=None):
        if targets is not None:
            raise NotImplementedError("the engine detector runs inference only")
        transform, _, roi_heads = self._stages
        original_image_sizes = [(int(img.shape[-2]), int(img.shape[-1])) for img in images]
        image_list, _ = transform(images)
        features, objectness, deltas = self.heads(image_list)
        proposals = self.proposals(image_list, features, objectness, deltas)
        if not self.device_paste:
            detections, _ = roi_heads(features, proposals, image_list.image_sizes)
            return transform.postprocess(detections, image_list.image_sizes, original_image_sizes)
        if self.engine_roi_heads:
            return self.detect_engine(features, proposals, tuple(image_list.tensors.shape[-2:]), image_list.image_sizes,
                                      original_image_sizes)
        return self.detect(features, proposals, image_list.image_sizes, original_image_sizes)

    def detect(self, features, proposals, image_sizes, original_image_sizes) -> List[Dict[str, torch.Tensor]]:
        """RoIHeads.forward (eval) up to the mask logits with the model's modules, then `mask_paste` in place of
        maskrcnn_inference and GeneralizedRCNNTransform.postprocess."""
        rh = self._stages[2]
        box_features = rh.box_head(rh.box_roi_pool(features, proposals, image_sizes))
        class_logits, box_regression = rh.box_predictor(box_features)
        boxes, scores, labels = rh.postprocess_detections(class_logits, box_regression, proposals, image_sizes)
        mask_logits = rh.mask_predictor(rh.mask_head(rh.mask_roi_pool(features, boxes, image_sizes)))
        counts = [int(b.shape[0]) for b in boxes]
        boxes, masks = mask_paste(mask_logits, torch.cat(labels), torch.cat(boxes), counts, image_sizes,
                                  original_image_sizes)
        return [dict(boxes=b, labels=l, scores=s, masks=m) for b, l, s, m in zip(boxes, labels, scores, masks)]


    def detect_engine(self, features, proposals, batch_hw, image_sizes, original_image_sizes
                      ) -> List[Dict[str, torch.Tensor]]:
        """`detect` with the box and mask branches on the engine (`RoiHeadsEngine`) and the model's
        postprocess_detections between them."""
        rh = self._stages[2]
        counts = [int(p.shape[0]) for p in proposals]
        class_logits, box_regression = self.roi_engine.box(features, torch.cat(proposals), counts, batch_hw, image_sizes)
        boxes, scores, labels = rh.postprocess_detections(class_logits, box_regression, proposals, image_sizes)
        counts = [int(b.shape[0]) for b in boxes]
        boxes_cat = torch.cat(boxes)
        mask_logits = self.roi_engine.mask(features, boxes_cat, counts, batch_hw, image_sizes)
        boxes, masks = mask_paste(mask_logits, torch.cat(labels), boxes_cat, counts, image_sizes, original_image_sizes)
        return [dict(boxes=b, labels=l, scores=s, masks=m) for b, l, s, m in zip(boxes, labels, scores, masks)]


def engine_model(model: nn.Module, device="cuda", device_paste: bool = False,
                 engine_roi_heads: bool = False) -> EngineMaskRCNN:
    """`model` (a torchvision MaskRCNN on `device`, in eval mode) with its backbone and RPN head on the engine.  Raises
    NotImplementedError, before any device work, for a structure the plan does not serve: a backbone other than the
    ResNet-50 body with FPN (returned layers 1-4, 256 channels, LastLevelMaxPool), a norm other than FrozenBatchNorm2d,
    dilation, an RPN head with conv_depth != 1 or more than 12 anchors per location, size_divisible != 32.
    `device_paste=True` also pastes the masks on the device (`mask_paste`) and refuses, likewise, RoI heads without a mask
    branch or with a keypoint branch, non-square mask pools, a mask predictor other than a 2x2/2 ConvTranspose2d and
    masks larger than 64x64, and a transform other than GeneralizedRCNNTransform.  `engine_roi_heads=True` implies
    `device_paste=True` and runs the box and mask branches on the engine (`RoiHeadsEngine`); it refuses as well pools
    other than MultiScaleRoIAlign on '0'..'3' with a fixed sampling ratio, a box pool other than 7x7, a box head other
    than TwoMLPHead on 256x7x7, a box predictor other than FastRCNNPredictor or with 5 x classes above 2048 rows, a mask
    head other than MaskRCNNHeads (four 3x3 convolutions of 256 channels, no norm, ReLU) and a mask predictor other than
    MaskRCNNPredictor."""
    return EngineMaskRCNN(model, device, device_paste, engine_roi_heads)
