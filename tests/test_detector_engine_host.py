"""Detector engine, host side: the weight plan and its float64 transformations against torchvision's own modules, the
float64 oracle, and the structures engine_model refuses."""
import copy

import pytest
import torch
import torch.nn.functional as F

pytest.importorskip("torchvision")

from megapose6d_b200 import _abi, backbone, detector_engine as E  # noqa: E402
from oracle import detector_ref as R  # noqa: E402
from workloads import detector as W  # noqa: E402


@pytest.fixture(scope="module")
def model():
    return W.make_detector((64, 96), seed=0, device="cpu")


def test_frozen_bn_fold_equals_conv_then_frozen_bn(model):
    mods = dict(model.named_modules())
    g = torch.Generator().manual_seed(0)
    for pc, (w, b) in zip(E.weight_plan(3), E.fold_plan(model, 3)):
        if pc.norm is None:
            continue
        conv, bn = mods[pc.modules[0]], mods[pc.norm]
        x = torch.randn(2, pc.c_in, 9, 9, generator=g, dtype=torch.float64)
        want = copy.deepcopy(bn).double()(F.conv2d(x, conv.weight.double(), None, conv.stride, conv.padding))
        got = F.conv2d(x, w, b, conv.stride, conv.padding)
        assert ((got - want).abs().max() / want.abs().max()).item() < 1e-12, pc.modules[0]


def test_stem_s2d_equals_the_7x7_stride_2_convolution(model):
    w, b = E.fold_plan(model, 3)[0]
    x = torch.randn(2, 3, 32, 48, dtype=torch.float64, generator=torch.Generator().manual_seed(1))
    want = F.conv2d(x, w, b, stride=2, padding=3)
    xs = torch.zeros(2, E.C_PAD, 32, 48, dtype=torch.float64)
    xs[:, :3] = x
    xs = xs.view(2, E.C_PAD, 16, 2, 24, 2).permute(0, 1, 3, 5, 2, 4).reshape(2, E.C_PAD, 2, 2, 16, 24)
    xs = xs.permute(0, 2, 3, 1, 4, 5).reshape(2, 4 * E.C_PAD, 16, 24)  # channel (dy*2+dx)*c_pad + c
    w2 = backbone._stem_s2d(w, E.C_PAD).view(64, 4, 4, 4 * E.C_PAD).permute(0, 3, 1, 2)
    got = F.conv2d(F.pad(xs, (2, 1, 2, 1)), w2, b)
    assert got.shape == want.shape and (got - want).abs().max().item() < 1e-12


def test_merged_rpn_1x1_equals_the_two_torchvision_convolutions(model):
    w, b = E.fold_plan(model, 3)[-1]
    assert w.shape == (E.HEAD_ROWS, 256, 1, 1) and not w[15:].any() and not b[15:].any()
    head = copy.deepcopy(model.rpn.head).double()
    t = torch.randn(2, 256, 5, 7, dtype=torch.float64, generator=torch.Generator().manual_seed(2))
    y = F.conv2d(t, w, b)
    assert torch.allclose(y[:, :3], head.cls_logits(t), rtol=0, atol=1e-12)
    assert torch.allclose(y[:, 3:15], head.bbox_pred(t), rtol=0, atol=1e-12)


def test_weight_plan_covers_backbone_and_rpn_head_convolutions_once(model):
    plan = E.weight_plan(3)
    assert len(plan) == 63
    names = [m for pc in plan for m in pc.modules]
    assert len(names) == len(set(names))
    convs = {n: m for n, m in model.named_modules() if isinstance(m, torch.nn.Conv2d)}
    served = {n for n in convs if n.startswith("backbone.") or n.startswith("rpn.head.")}
    assert set(names) == served
    assert not any(n.startswith("roi_heads.") for n in names)
    for pc in plan:
        for n in pc.modules:
            m = convs[n]
            assert m.kernel_size == (pc.kernel,) * 2 and m.stride == (pc.stride,) * 2 and m.padding == (pc.padding,) * 2
            assert m.in_channels == pc.c_in
        assert sum(convs[n].out_channels for n in pc.modules) == pc.c_out


@torch.no_grad()
def test_oracle_tracks_torchvision_fp32_within_its_bound(model):
    x = torch.randn(2, 3, 64, 96, generator=torch.Generator().manual_seed(3))
    f, o, d = R.forward(model, x)
    tf = model.backbone(x)
    to, td = model.rpn.head(list(tf.values()))
    for got, want in zip(f + o + d, list(tf.values()) + to + td):
        assert got.shape == want.shape
        err = (got - want.double()).abs().max().item()
        assert err <= R.ORACLE_VS_FP32 * want.abs().max().item()


@torch.no_grad()
def test_oracle_equals_exact_float64_on_integer_operands(model):
    m = W.integer_weights(copy.deepcopy(model), seed=1, nnz=1)  # every value stays an fp16-exact integer
    x = torch.randint(0, 4, (2, 3, 64, 96), generator=torch.Generator().manual_seed(4)).float()
    f, o, d = R.forward(m, x)
    md = copy.deepcopy(m).double()
    tf = md.backbone(x.double())
    to, td = md.rpn.head(list(tf.values()))
    for got, want in zip(f + o + d, list(tf.values()) + to + td):
        assert torch.equal(got, want)
    assert max(t.abs().max().item() for t in f) > 8


def _variants():
    from torchvision.models.detection.backbone_utils import resnet_fpn_backbone
    from torchvision.models.detection.mask_rcnn import MaskRCNN
    from torchvision.models.detection.rpn import AnchorGenerator, RPNHead

    def mrcnn(bb=None, **kw):
        return MaskRCNN(bb or resnet_fpn_backbone(backbone_name="resnet50", weights=None), num_classes=3, **kw)

    def dilated():
        m = mrcnn()
        m.backbone.body.layer4[0].conv2.dilation = (2, 2)
        return m

    def many_anchors():
        ag = AnchorGenerator(((32,), (64,), (128,), (256,), (512,)), ((0.25, 0.5, 1.0, 2.0, 4.0, 8.0, 0.125),) * 5)
        return mrcnn(rpn_anchor_generator=ag, rpn_head=RPNHead(256, 13))

    return {
        "resnet34": lambda: mrcnn(resnet_fpn_backbone(backbone_name="resnet34", weights=None)),
        "returned_layers": lambda: mrcnn(resnet_fpn_backbone(backbone_name="resnet50", weights=None,
                                                             returned_layers=[2, 3, 4])),
        "batchnorm": lambda: mrcnn(resnet_fpn_backbone(backbone_name="resnet50", weights=None,
                                                       norm_layer=torch.nn.BatchNorm2d)),
        "dilation": dilated,
        "rpn_conv_depth": lambda: mrcnn(rpn_head=RPNHead(256, 3, conv_depth=2)),
        "anchors_13": many_anchors,
        "size_divisible": lambda: mrcnn(size_divisible=64),
    }


@pytest.mark.parametrize("variant", sorted(_variants()))
def test_engine_model_refuses_unserved_structures(variant):
    m = _variants()[variant]().eval()
    launches = _abi.lib().mpx_launch_count()
    with pytest.raises(NotImplementedError):
        E.engine_model(m, device="cpu")
    assert _abi.lib().mpx_launch_count() == launches


def test_seeded_detector_is_served(model):
    assert E.check_supported(model) == 3
