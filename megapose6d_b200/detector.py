"""Detector front-end: 2D detections (boxes, labels, scores, masks) for PoseEstimator(detector_model=...).

Drop-in for the reference's `Detector` (src/megapose/inference/detector.py:34-142) and `load_detector`
(src/megapose/inference/utils.py:57-70, training/detector_models_cfg.py:24-38, models/mask_rcnn.py:23-46): same
constructor, `image_tensor_from_numpy`, `get_detections(observation, detection_th, output_masks, mask_th,
one_instance_per_class)` / `__call__`, and the same collection comes back (infos columns `batch_im_id`, `label`, `score`,
`instance_id`; `bboxes` float32 [N, 4]; optional bool `masks` [N, H, W]).

The network itself is, as in the reference, torchvision's Mask R-CNN (a library model, not part of the render-and-compare
hot path; `create_model_detector` builds it when torchvision is importable).  What is re-done here is the wrapper: the
reference walks every detection in Python with one `.item()` (a device synchronisation) per score and per label and
stacks per-object box / mask slices; this version concatenates the per-image outputs on the device, reads scores and
category ids back with ONE copy, and thresholds all masks in one launch.  Row order and values are identical
(tests/test_detector.py compares with the reference class loaded by path).

One deliberate difference: with no detection at all the reference allocates `masks` as [0, 3, H] (it reads the shape of
the [B, 3, H, W] batch at the wrong positions, detector.py:113); here the empty mask tensor is [0, H, W].
"""
from __future__ import annotations

from pathlib import Path
from typing import Any, Optional

import numpy as np
import pandas as pd
import torch

from .pose_estimator import add_instance_id, filter_detections
from .tensor_collection import PandasTensorCollection
from .types import DetectionsType, ObservationTensor

RGB_DIMS = [0, 1, 2]


class Detector(torch.nn.Module):
    def __init__(self, model: torch.nn.Module) -> None:
        super().__init__()
        self.model = model
        self.model.eval()
        self.config = model.config
        self.category_id_to_label = {v: k for k, v in self.config.label_to_category_id.items()}

    def image_tensor_from_numpy(self, rgb: np.ndarray) -> torch.Tensor:
        """[H, W, 3] uint8 -> [3, H, W] float in [0, 1] (detector.py:42-62)."""
        assert rgb.dtype == np.uint8
        rgb_tensor = torch.as_tensor(rgb).float() / 255
        if rgb_tensor.shape[-1] == 3:
            rgb_tensor = rgb_tensor.permute(2, 0, 1)
        return rgb_tensor

    @torch.no_grad()
    def get_detections(self, observation: ObservationTensor, detection_th: Optional[float] = None,
                       output_masks: bool = False, mask_th: float = 0.8,
                       one_instance_per_class: bool = False) -> DetectionsType:
        """detector.py:64-139.  `detection_th`: keep detections scoring above it; `mask_th`: probability threshold of the
        instance masks; `one_instance_per_class`: keep the best detection of every (image, label)."""
        images = observation.images[:, RGB_DIMS]
        device = images.device
        outputs_ = self.model([image_n for image_n in images])

        counts = [int(o["boxes"].shape[0]) for o in outputs_]
        n_total = sum(counts)
        if n_total > 0:
            bboxes = torch.cat([torch.as_tensor(o["boxes"]).reshape(-1, 4) for o in outputs_]).to(device).float()
            # scores and category ids of every image in one device -> host copy
            packed = torch.cat([torch.stack([torch.as_tensor(o["scores"]).double().reshape(-1),
                                             torch.as_tensor(o["labels"]).double().reshape(-1)], dim=1)
                                for o in outputs_]).cpu().numpy()
            scores = packed[:, 0]  # float64 holds a float32 score exactly: the value `.item()` gives in the reference
            labels = [self.category_id_to_label[int(c)] for c in packed[:, 1]]
            infos = pd.DataFrame(dict(batch_im_id=np.repeat(np.arange(len(counts)), counts), label=labels, score=scores))
            masks = None
            if output_masks:
                masks = (torch.cat([torch.as_tensor(o["masks"])[:, 0] for o in outputs_]) > mask_th).to(device)
        else:
            infos = pd.DataFrame(dict(score=[], label=[], batch_im_id=[]))
            bboxes = torch.empty(0, 4, device=device).float()
            masks = torch.empty(0, images.shape[2], images.shape[3], dtype=torch.bool, device=device)

        outputs = PandasTensorCollection(infos=infos, bboxes=bboxes)
        if output_masks:
            outputs.register_tensor("masks", masks)
        if detection_th is not None:
            keep = np.where(outputs.infos["score"] > detection_th)[0]
            outputs = outputs[keep]
        if one_instance_per_class:
            outputs = filter_detections(outputs, one_instance_per_class=True)
        return add_instance_id(outputs)

    def __call__(self, *args: Any, **kwargs: Any) -> DetectionsType:
        return self.get_detections(*args, **kwargs)


def check_update_config_detector(cfg):
    """training/detector_models_cfg.py:24-27: category names get the dataset prefix of the first training set."""
    obj_prefix = cfg.train_ds_names[0][0].split(".")[0]
    cfg.label_to_category_id = {f"{obj_prefix}-{k}": v for k, v in cfg.label_to_category_id.items()}
    return cfg


def create_model_detector(cfg, n_classes: int) -> torch.nn.Module:
    """training/detector_models_cfg.py:30-37 + models/mask_rcnn.py:23-46: torchvision Mask R-CNN on a ResNet-50 FPN,
    three aspect ratios per anchor size, input resized to `cfg.input_resize`."""
    try:
        from torchvision.models.detection.backbone_utils import resnet_fpn_backbone
        from torchvision.models.detection.mask_rcnn import MaskRCNN
        from torchvision.models.detection.rpn import AnchorGenerator
    except ImportError as exc:  # pragma: no cover -- torchvision is part of the image
        raise RuntimeError("the Mask R-CNN detector needs torchvision (the reference uses it as well)") from exc
    assert cfg.backbone_str == "resnet50-fpn"
    anchor_sizes = tuple(tuple(s) for s in cfg.anchor_sizes)
    backbone = resnet_fpn_backbone(backbone_name="resnet50", weights=None)
    return MaskRCNN(backbone=backbone, num_classes=n_classes,
                    rpn_anchor_generator=AnchorGenerator(anchor_sizes, ((0.5, 1.0, 2.0),) * len(anchor_sizes)),
                    max_size=max(cfg.input_resize), min_size=min(cfg.input_resize))


def load_detector(run_id: str, models_root: Optional[Path] = None, device: str = "cuda", engine: bool = False,
                  device_paste: bool = False, engine_roi_heads: bool = False) -> Detector:
    """inference/utils.py:57-70: `<models_root>/<run_id>/{config.yaml, checkpoint.pth.tar}` -> Detector.  `engine=True`
    runs the Mask R-CNN's ResNet-50 FPN backbone and RPN head on the engine's wgmma convolutions
    (`detector_engine.engine_model`; the rest of the model stays torchvision's); with `device_paste=True` as well, the
    mask logits are turned into image-sized masks on the device (`engine_model(..., device_paste=True)`) instead of by
    torchvision's per-detection loop; with `engine_roi_heads=True` (implying `device_paste`) the RoI heads' box and mask
    branches run on the engine too (`engine_model(..., engine_roi_heads=True)`); the default is torchvision's model
    throughout, as in the reference."""
    for name, on in (("device_paste", device_paste), ("engine_roi_heads", engine_roi_heads)):
        if on and not engine:
            raise ValueError(f"load_detector: {name}=True needs engine=True")
    from . import load_model

    run_dir = Path(models_root if models_root is not None else load_model.LOCAL_DATA_DIR / "experiments") / run_id  # EXP_DIR
    cfg = check_update_config_detector(load_model.load_cfg(run_dir / "config.yaml"))
    model = create_model_detector(cfg, len(cfg.label_to_category_id))
    ckpt = torch.load(run_dir / "checkpoint.pth.tar", map_location="cpu", weights_only=False)
    model.load_state_dict(ckpt["state_dict"])
    model = model.to(device).eval()
    model.cfg = cfg
    model.config = cfg
    if engine:
        from .detector_engine import engine_model

        model = engine_model(model, device, device_paste=device_paste, engine_roi_heads=engine_roi_heads)
    return Detector(model)
