"""Engine detector with device_paste=True, host side: the RoI-head structures it refuses before any device work, and the
options that select it."""
import pytest
import torch

pytest.importorskip("torchvision")

from megapose6d_b200 import _abi, detector as D, detector_engine as E, prediction_runner  # noqa: E402
from workloads import detector as W  # noqa: E402


def _variants():
    from torchvision.models.detection.backbone_utils import resnet_fpn_backbone
    from torchvision.models.detection.faster_rcnn import FasterRCNN
    from torchvision.models.detection.keypoint_rcnn import KeypointRCNNHeads, KeypointRCNNPredictor
    from torchvision.models.detection.mask_rcnn import MaskRCNN, MaskRCNNPredictor
    from torchvision.models.detection.transform import GeneralizedRCNNTransform
    from torchvision.ops import MultiScaleRoIAlign

    def bb():
        return resnet_fpn_backbone(backbone_name="resnet50", weights=None)

    def keypoints():
        m = MaskRCNN(bb(), num_classes=3)
        m.roi_heads.keypoint_roi_pool = MultiScaleRoIAlign(["0", "1", "2", "3"], 14, 2)
        m.roi_heads.keypoint_head = KeypointRCNNHeads(256, (512,) * 8)
        m.roi_heads.keypoint_predictor = KeypointRCNNPredictor(512, 17)
        return m

    def mask_predictor():
        m = MaskRCNN(bb(), num_classes=3)
        m.roi_heads.mask_predictor = torch.nn.Sequential(MaskRCNNPredictor(256, 256, 3))
        return m

    class Transform(GeneralizedRCNNTransform):
        pass

    def transform():
        m = MaskRCNN(bb(), num_classes=3)
        t = m.transform
        m.transform = Transform(t.min_size, t.max_size, t.image_mean, t.image_std)
        return m

    return {
        "no_mask_branch": lambda: FasterRCNN(bb(), num_classes=3),
        "keypoints": keypoints,
        "mask_pool_33": lambda: MaskRCNN(bb(), num_classes=3,
                                         mask_roi_pool=MultiScaleRoIAlign(["0", "1", "2", "3"], 33, 2)),
        "mask_pool_not_square": lambda: MaskRCNN(bb(), num_classes=3,
                                                 mask_roi_pool=MultiScaleRoIAlign(["0", "1", "2", "3"], (14, 7), 2)),
        "mask_predictor": mask_predictor,
        "transform": transform,
    }


@pytest.mark.parametrize("variant", sorted(_variants()))
def test_roi_heads_mode_refuses_unserved_structures(variant):
    m = _variants()[variant]().eval()
    launches = _abi.lib().mpx_launch_count()
    with pytest.raises(NotImplementedError):
        E.engine_model(m, device="cpu", device_paste=True)
    assert _abi.lib().mpx_launch_count() == launches


def test_seeded_detector_is_served():
    E.check_supported_device_paste(W.make_detector((64, 96), seed=0, device="cpu"))


def test_load_detector_refuses_device_paste_without_the_engine(tmp_path):
    with pytest.raises(ValueError, match="needs engine=True"):
        D.load_detector("no-such-run", models_root=tmp_path, device_paste=True)


def test_device_paste_flag_needs_a_detector(tmp_path, capsys):
    with pytest.raises(SystemExit):
        prediction_runner.main([str(tmp_path), "--save-dir", str(tmp_path / "out"), "--detector-device-paste"])
    assert "--detector-engine needs --detector" in capsys.readouterr().err
