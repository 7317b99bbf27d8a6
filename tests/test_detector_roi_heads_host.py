"""Engine detector with engine_roi_heads=True, host side: the weight repacking of the RoI heads, the structures it refuses
before any device work, the options that select it, and the float64 oracle against torchvision's fp32 RoI heads."""
import pytest
import torch
import torch.nn.functional as F

pytest.importorskip("torchvision")

from megapose6d_b200 import _abi, detector as D, detector_engine as E, prediction_runner  # noqa: E402
from oracle import detector_heads_ref as R  # noqa: E402
from workloads import detector as W  # noqa: E402


@pytest.fixture(scope="module")
def model():
    return W.make_detector((64, 96), n_classes=5, seed=3, device="cpu")


def test_fc6_as_7x7_convolution_matches_linear(model):
    g = torch.Generator().manual_seed(0)
    plan = E.roi_heads_plan(model)
    fc6 = model.roi_heads.box_head.fc6
    x = torch.randn(5, 256, 7, 7, generator=g, dtype=torch.float64)
    want = F.linear(x.flatten(1), fc6.weight.double(), fc6.bias.double())
    w, b = plan[0]
    assert w.shape == (fc6.out_features, 7 * 7 * 256)
    got = x.permute(0, 2, 3, 1).reshape(5, -1) @ w.T + b  # NHWC rows, k = (y, x, c)
    torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)


def test_merged_predictor_rows(model):
    w, b = E.roi_heads_plan(model)[2]
    pred = model.roi_heads.box_predictor
    c = pred.cls_score.out_features
    assert w.shape[0] == 64 and b.shape[0] == 64  # 5 x 6 classes = 30 rows, padded
    assert torch.equal(w[:c], pred.cls_score.weight.double()) and torch.equal(w[c:5 * c], pred.bbox_pred.weight.double())
    assert not w[5 * c:].any() and not b[5 * c:].any()


def test_deconvolution_as_1x1_and_depth_to_space(model):
    g = torch.Generator().manual_seed(1)
    conv5 = model.roi_heads.mask_predictor.conv5_mask
    x = torch.randn(3, 256, 14, 14, generator=g, dtype=torch.float64)
    want = F.conv_transpose2d(x, conv5.weight.double(), conv5.bias.double(), stride=2)
    w, b = E.roi_heads_plan(model)[7]
    y = torch.einsum("nchw,oc->nhwo", x, w) + b  # [n, 14, 14, (dy, dx, o)]
    got = y.view(3, 14, 14, 2, 2, 256).permute(0, 5, 1, 3, 2, 4).reshape(3, 256, 28, 28)
    torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)


def test_mask_layers_repacked(model):
    plan = E.roi_heads_plan(model)
    g = torch.Generator().manual_seed(2)
    x = torch.randn(2, 256, 14, 14, generator=g, dtype=torch.float64)
    conv = model.roi_heads.mask_head[0][0]
    want = F.conv2d(x, conv.weight.double(), conv.bias.double(), padding=1)
    w, b = plan[3]
    got = F.conv2d(x, w.view(256, 3, 3, 256).permute(0, 3, 1, 2), b, padding=1)
    torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)
    logits = model.roi_heads.mask_predictor.mask_fcn_logits
    w, b = plan[8]
    assert w.shape == (64, 256) and torch.equal(w[:6], logits.weight.double().flatten(1)) and not w[6:].any()


def _variants():
    from torchvision.models.detection.backbone_utils import resnet_fpn_backbone
    from torchvision.models.detection.faster_rcnn import FastRCNNPredictor, TwoMLPHead
    from torchvision.models.detection.keypoint_rcnn import KeypointRCNNHeads, KeypointRCNNPredictor
    from torchvision.models.detection.mask_rcnn import MaskRCNN, MaskRCNNHeads
    from torchvision.ops import MultiScaleRoIAlign

    def bb():
        return resnet_fpn_backbone(backbone_name="resnet50", weights=None)

    def mrcnn(**kw):
        return MaskRCNN(bb(), num_classes=3, **kw)

    def edit(fn):
        def make():
            m = mrcnn()
            fn(m.roi_heads)
            return m
        return make

    def keypoints(rh):
        rh.keypoint_roi_pool = MultiScaleRoIAlign(["0", "1", "2", "3"], 14, 2)
        rh.keypoint_head = KeypointRCNNHeads(256, (512,) * 8)
        rh.keypoint_predictor = KeypointRCNNPredictor(512, 17)

    class Pool(MultiScaleRoIAlign):
        pass

    return {
        "box_pool_adaptive_sampling": lambda: mrcnn(box_roi_pool=MultiScaleRoIAlign(["0", "1", "2", "3"], 7, 0)),
        "box_pool_levels": lambda: mrcnn(box_roi_pool=MultiScaleRoIAlign(["0", "1", "2"], 7, 2)),
        "box_pool_subclass": lambda: mrcnn(box_roi_pool=Pool(["0", "1", "2", "3"], 7, 2)),
        "mask_pool_levels": lambda: mrcnn(mask_roi_pool=MultiScaleRoIAlign(["0", "1", "2", "3", "pool"], 14, 2)),
        "box_pool_size": edit(lambda rh: setattr(rh, "box_roi_pool", MultiScaleRoIAlign(["0", "1", "2", "3"], 5, 2))),
        "box_head": edit(lambda rh: setattr(rh, "box_head", torch.nn.Sequential(TwoMLPHead(256 * 49, 1024)))),
        "box_head_size": edit(lambda rh: setattr(rh, "box_head", TwoMLPHead(256 * 49, 1000))),
        "box_predictor": edit(lambda rh: setattr(rh, "box_predictor", torch.nn.Sequential(FastRCNNPredictor(1024, 3)))),
        "too_many_classes": lambda: MaskRCNN(bb(), num_classes=410),
        "mask_head_norm": edit(lambda rh: setattr(rh, "mask_head",
                                                  MaskRCNNHeads(256, (256,) * 4, 1, norm_layer=torch.nn.BatchNorm2d))),
        "mask_head_dilation": edit(lambda rh: setattr(rh, "mask_head", MaskRCNNHeads(256, (256,) * 4, 2))),
        "mask_head_depth": edit(lambda rh: setattr(rh, "mask_head", MaskRCNNHeads(256, (256,) * 3, 1))),
        "keypoints": edit(keypoints),
        "no_mask_branch": edit(lambda rh: setattr(rh, "mask_head", None)),
    }


@pytest.mark.parametrize("variant", sorted(_variants()))
def test_engine_roi_heads_refuses_unserved_structures(variant):
    m = _variants()[variant]().eval()
    launches = _abi.lib().mpx_launch_count()
    with pytest.raises(NotImplementedError):
        E.engine_model(m, device="cpu", engine_roi_heads=True)
    assert _abi.lib().mpx_launch_count() == launches


def test_seeded_detectors_are_served(model):
    E.check_supported_roi_heads(model)
    E.check_supported_roi_heads(W.make_detector((64, 96), n_classes=90, seed=0, device="cpu"))


def test_load_detector_refuses_roi_heads_without_the_engine(tmp_path):
    with pytest.raises(ValueError, match="engine_roi_heads=True needs engine=True"):
        D.load_detector("no-such-run", models_root=tmp_path, engine_roi_heads=True)


def test_roi_heads_flag_implies_the_engine(tmp_path, capsys):
    with pytest.raises(SystemExit):
        prediction_runner.main([str(tmp_path), "--save-dir", str(tmp_path / "out"), "--detector-engine-roi-heads"])
    assert "--detector-engine needs --detector" in capsys.readouterr().err


def test_oracle_against_torchvision_fp32(model):
    """The float64 oracle (act16 roundings) against torchvision's fp32 RoI heads on the same pooled features: within
    R.HEADS_VS_ORACLE of each output's largest magnitude."""
    g = torch.Generator().manual_seed(5)
    feats = {k: torch.randn(2, 256, 64 // s, 96 // s, generator=g) for k, s in zip(["0", "1", "2", "3"], (4, 8, 16, 32))}
    xy = torch.rand(40, 2, generator=g) * torch.tensor([80.0, 50.0])
    wh = 2 + torch.rand(40, 2, generator=g) * 40
    boxes = torch.cat([xy, xy + wh], 1)
    proposals = [boxes[:25], boxes[25:]]
    sizes = [(64, 96), (60, 90)]
    rh = model.roi_heads
    with torch.no_grad():
        x = rh.box_head(rh.box_roi_pool(feats, proposals, sizes))
        logits, deltas = rh.box_predictor(x)
        masks = rh.mask_predictor(rh.mask_head(rh.mask_roi_pool(feats, proposals, sizes)))
    o_logits, o_deltas = R.roi_heads_box(model, feats, proposals, sizes)
    o_masks = R.roi_heads_mask(model, feats, proposals, sizes)
    for got, want in ((o_logits, logits), (o_deltas, deltas), (o_masks, masks)):
        err = (got - want.double()).abs().max() / want.abs().max()
        assert err <= R.HEADS_VS_ORACLE, float(err)
