"""Detector engine on the device (csrc/detector_net.cu: mpx_fpn_forward): bit-exact against the float64 oracle on integer
operands at every size and batch, graph replay, the stated bounds on Gaussian weights, the wiring into torchvision's
stages, detections end to end, ABI refusals, the pose pipeline and the command line."""
from __future__ import annotations

import copy
import ctypes

import numpy as np
import pytest
import torch

pytest.importorskip("torchvision")

from megapose6d_b200 import _abi, detector as D, detector_engine as E  # noqa: E402
from oracle import detector_ref as R  # noqa: E402
from workloads import detector as W  # noqa: E402

pytestmark = pytest.mark.gpu

# fp32 means fp32: torchvision's side of every comparison runs without TF32
torch.backends.cuda.matmul.allow_tf32 = False
torch.backends.cudnn.allow_tf32 = False


def _outputs(engine, images):
    return [t.clone() for ts in engine.run(images) for t in ts]


def _set_graphs(on: bool):
    _abi.lib().mpx_net_set_graphs(1 if on else 0)


@pytest.fixture(scope="module")
def integer_model():
    return W.integer_weights(W.make_detector((480, 640), seed=0, device="cuda"), seed=3, nnz=2)


@pytest.fixture(scope="module")
def integer_engine(integer_model):
    return E.FpnEngine(integer_model)


_oracle_cache = {}


@pytest.mark.parametrize("graphs", [False, True], ids=["eager", "graphs"])
# padded batch sizes of input_resize (480, 640), (240, 320) and (540, 720): GeneralizedRCNNTransform pads to multiples of 32
@pytest.mark.parametrize("hw", [(480, 640), (256, 320), (544, 736)], ids=lambda s: f"{s[0]}x{s[1]}")
@pytest.mark.parametrize("n", [1, 3])
def test_bit_exact_against_the_oracle_on_integer_operands(integer_model, integer_engine, n, hw, graphs):
    key = (n, hw)
    g = torch.Generator().manual_seed(n * 1000 + hw[0])
    images = torch.randint(0, 4, (n, 3, *hw), generator=g).float().cuda()
    if key not in _oracle_cache:
        _oracle_cache.clear()
        _oracle_cache[key] = [t.float() for ts in R.forward(integer_model, images) for t in ts]
    want = _oracle_cache[key]
    _set_graphs(graphs)
    try:
        for _ in range(3 if graphs else 1):  # eager first sight, capture, replay
            got = _outputs(integer_engine, images)
    finally:
        _set_graphs(True)
    assert len(got) == 15
    for i, (a, b) in enumerate(zip(got, want)):
        assert a.shape == b.shape, i
        assert torch.equal(a, b), f"output {i}: {(a != b).sum().item()} elements differ, max {(a - b).abs().max().item()}"
    assert max(t.abs().max().item() for t in want[:5]) > 2048  # roundings (and saturation) were exercised


def test_graph_replay_equals_eager_and_caches_a_graph_per_shape(integer_engine):
    a = torch.randint(0, 4, (2, 3, 256, 320), generator=torch.Generator().manual_seed(1)).float().cuda()
    b = torch.randint(0, 4, (1, 3, 320, 448), generator=torch.Generator().manual_seed(2)).float().cuda()
    _set_graphs(False)
    eager_a, eager_b = _outputs(integer_engine, a), _outputs(integer_engine, b)
    _set_graphs(True)
    for _ in range(3):
        replay_a = _outputs(integer_engine, a)
    l0 = _abi.lib().mpx_launch_count()
    replay_a = _outputs(integer_engine, a)
    assert _abi.lib().mpx_launch_count() - l0 == 78  # a replay counts the graph's launches
    for _ in range(3):
        replay_b = _outputs(integer_engine, b)
    again_a = _outputs(integer_engine, a)
    for x, y in zip(replay_a + again_a, eager_a + eager_a):
        assert torch.equal(x, y)
    for x, y in zip(replay_b, eager_b):
        assert torch.equal(x, y)


@pytest.fixture(scope="module")
def gaussian_model():
    return W.make_detector((480, 640), seed=1, device="cuda")


@pytest.mark.parametrize("n,hw", [(1, (480, 640)), (2, (256, 320))], ids=["1x480x640", "2x256x320"])
def test_gaussian_weights_within_the_stated_bounds(gaussian_model, n, hw):
    images = torch.randn(n, 3, *hw, generator=torch.Generator().manual_seed(5)).cuda()
    got = _outputs(E.FpnEngine(gaussian_model), images)
    oracle = [t for ts in R.forward(gaussian_model, images) for t in ts]
    with torch.no_grad():
        feats = gaussian_model.backbone(images)
        obj, dl = gaussian_model.rpn.head(list(feats.values()))
    tv = list(feats.values()) + obj + dl
    worst_o, worst_t = 0.0, 0.0
    for i, (a, o, t) in enumerate(zip(got, oracle, tv)):
        eo = (a.double() - o).abs().max().item() / o.abs().max().item()
        et = (a.double() - t.double()).abs().max().item() / t.abs().max().item()
        worst_o, worst_t = max(worst_o, eo), max(worst_t, et)
        assert eo <= R.ENGINE_VS_ORACLE, (i, eo)
        assert et <= R.ORACLE_VS_FP32 + R.ENGINE_VS_ORACLE, (i, et)
    print(f"engine vs oracle {worst_o * 2 ** 11:.2f} u, vs torchvision fp32 {worst_t * 2 ** 11:.2f} u (u = 2^-11)")


class _GivenHead(torch.nn.Module):
    """Stands in for RPNHead in a copy of the model's RPN: returns the given objectness and deltas."""

    def __init__(self, objectness, deltas):
        super().__init__()
        self.out = (objectness, deltas)

    def forward(self, features):
        return self.out


def test_wiring_equals_torchvision_stages_fed_the_engine_tensors(gaussian_model):
    sd_before = {k: v.clone() for k, v in gaussian_model.state_dict().items()}
    images = [torch.rand(3, 480, 640, generator=torch.Generator().manual_seed(s)).cuda() for s in (6, 7)]
    with torch.backends.cudnn.flags(enabled=True, benchmark=False, deterministic=True, allow_tf32=False):
        before = gaussian_model(images)
        module = E.engine_model(gaussian_model)
        after = gaussian_model(images)
    for x, y in zip(before, after):
        for k in x:
            assert torch.equal(x[k], y[k]), k
    sd = gaussian_model.state_dict()
    assert sd.keys() == sd_before.keys() and all(torch.equal(sd[k], v) for k, v in sd_before.items())
    got = module(images)
    with torch.no_grad():
        image_list, _ = gaussian_model.transform(images)
        features, objectness, deltas = module.heads(image_list)
        rpn = copy.copy(gaussian_model.rpn)
        rpn._modules = dict(rpn._modules)
        rpn.head = _GivenHead(objectness, deltas)
        proposals, _ = rpn(image_list, features)
        dets, _ = gaussian_model.roi_heads(features, proposals, image_list.image_sizes)
        want = gaussian_model.transform.postprocess(dets, image_list.image_sizes, [(480, 640)] * 2)
    assert gaussian_model.rpn.head is not rpn.head and isinstance(gaussian_model.rpn.head, torch.nn.Module)
    for x, y in zip(got, want):
        assert x.keys() == y.keys()
        for k in x:
            assert torch.equal(x[k], y[k]), k


def _iou(a, b):
    lt = torch.maximum(a[:, None, :2], b[None, :, :2])
    rb = torch.minimum(a[:, None, 2:], b[None, :, 2:])
    inter = (rb - lt).clamp(min=0).prod(-1)
    area = lambda t: (t[:, 2:] - t[:, :2]).prod(-1)  # noqa: E731
    return inter / (area(a)[:, None] + area(b)[None, :] - inter)


def _partners(src, dst, tau, thresh):
    """Every detection of `src` clear of the threshold and of its rank neighbours by more than tau has a partner in dst."""
    s = src["scores"]
    checked = 0
    iou = _iou(src["boxes"], dst["boxes"]) if len(dst["boxes"]) else None
    for i in range(len(s)):
        near = [abs(s[i] - thresh)] + [abs(s[i] - s[j]) for j in (i - 1, i + 1) if 0 <= j < len(s)]
        if min(float(v) for v in near) <= tau:
            continue
        checked += 1
        assert iou is not None, f"detection {i} (score {float(s[i]):.4f}) has no partner"
        ok = (dst["labels"] == src["labels"][i]) & (iou[i] >= 0.9) & ((dst["scores"] - s[i]).abs() <= tau)
        assert bool(ok.any()), f"detection {i} (score {float(s[i]):.4f}) has no partner"
    return checked


def test_detections_end_to_end_match_torchvision_fp32():
    model = W.make_detector((480, 640), seed=4, spread_scores=3.0, device="cuda")
    images = [torch.rand(3, 480, 640, generator=torch.Generator().manual_seed(s)).cuda() for s in (8, 9)]
    module = E.engine_model(model)
    with torch.no_grad():
        image_list, _ = model.transform(images)
        feats = model.backbone(image_list.tensors)
        obj, _ = model.rpn.head(list(feats.values()))
        e_feats, e_obj, _ = module.heads(image_list)
        e_feat = max((a - b).abs().max().item() / b.abs().max().item() for a, b in zip(e_feats.values(), feats.values()))
        want = model(images)
    got = module(images)
    # tau: the box head sees RoI-pooled features carrying a relative error e_feat; through the two-layer MLP and the
    # class logits (|logit| <= ~8 with spread scores) a softmax score moves by at most a quarter of the logit change:
    # 8 * e_feat * 8 / 4 = 16 e_feat, and never less than 0.01
    tau = max(0.01, 16 * e_feat)
    checked = 0
    for w, g in zip(want, got):
        thresh = model.roi_heads.score_thresh
        if len(w["scores"]) == model.roi_heads.detections_per_img:
            thresh = max(thresh, float(w["scores"][-1]))
        checked += _partners(w, g, tau, thresh) + _partners(g, w, tau, thresh)
    print(f"e_feat {e_feat:.2e}, tau {tau:.3f}, {checked} detections matched, "
          f"counts {[len(w['scores']) for w in want]} / {[len(g['scores']) for g in got]}")
    assert checked > 0


def test_abi_refusals_launch_nothing(integer_engine):
    lib = _abi.lib()
    n, h, w = 1, 256, 320
    images = torch.zeros(n, 3, h, w, device="cuda")
    sizes = E.level_sizes(h, w)
    outs = [[torch.empty(n, c, a, b, device="cuda") for a, b in sizes] for c in (256, 3, 12)]
    ws = torch.empty(lib.mpx_fpn_workspace_bytes(n, h, w), dtype=torch.uint8, device="cuda")
    host_ws = torch.empty(16, dtype=torch.uint8)

    def arr(ts, bad=None):
        p = [t.data_ptr() for t in ts]
        if bad is not None:
            p[2] = bad
        return (ctypes.c_void_p * 5)(*p)

    ok = [arr(o) for o in outs]
    cases = [
        ("size", dict(h=250), "multiples of 32"),
        ("batch", dict(n=0), "need n >= 1"),
        ("null_handle", dict(handle=None), "fpn is NULL"),
        ("null_images", dict(images=None), "d_images is NULL"),
        ("null_feature", dict(arrays=[arr(outs[0], bad=0)] + ok[1:]), "level 2 is NULL or not device memory"),
        ("host_delta", dict(arrays=ok[:2] + [arr(outs[2], bad=host_ws.data_ptr())]), "not device memory"),
        ("null_array", dict(arrays=[None] + ok[1:]), "h_features is NULL"),
        ("host_workspace", dict(ws=(host_ws.data_ptr(), ws.numel())), "d_workspace is not device memory"),
        ("short_workspace", dict(ws=(ws.data_ptr(), ws.numel() - 256)), "workspace of"),
    ]
    for name, kw, msg in cases:
        args = dict(handle=integer_engine._handle, images=images.data_ptr(), n=n, h=h, w=w, arrays=ok,
                    ws=(ws.data_ptr(), ws.numel()))
        args.update(kw)
        before = lib.mpx_launch_count()
        rc = lib.mpx_fpn_forward(args["handle"], args["images"], args["n"], args["h"], args["w"], *args["arrays"],
                                 args["ws"][0], args["ws"][1], _abi.stream_ptr())
        assert rc != 0, name
        assert msg in lib.mpx_last_error().decode(), (name, lib.mpx_last_error())
        assert lib.mpx_launch_count() == before, name
    handle = ctypes.c_void_p()
    wp = (ctypes.c_void_p * 63)(*([None] * 63))
    assert lib.mpx_fpn_create(wp, wp, 63, 3, ctypes.byref(handle)) != 0
    assert lib.mpx_fpn_create(wp, wp, 62, 3, ctypes.byref(handle)) != 0
    assert "expected 63" in lib.mpx_last_error().decode()
    w_ok = (ctypes.c_void_p * 63)(*[t.data_ptr() for t in integer_engine._weights])
    b_ok = (ctypes.c_void_p * 63)(*[t.data_ptr() for t in integer_engine._biases])
    assert lib.mpx_fpn_create(w_ok, b_ok, 63, 13, ctypes.byref(handle)) != 0
    assert "1..12" in lib.mpx_last_error().decode()
    torch.cuda.synchronize()


def test_pipeline_with_engine_detector_equals_passing_its_detections(tmp_path):
    from megapose6d_b200 import load_model
    from megapose6d_b200.types import ObservationTensor
    from tests import helpers

    ds, images, K = helpers.make_scene(2, seed=6)
    load_model.write_run(tmp_path, "coarse-rgb-906902141", helpers.make_state_dict(helpers.COARSE_CFG, 5))
    load_model.write_run(tmp_path, "refiner-rgb-653307694", helpers.make_state_dict(helpers.REFINER_CFG, 6))
    est = load_model.load_named_model("megapose-1.0-RGB", ds, models_root=tmp_path)
    est.load_SO3_grid(72)
    labels = [o.label for o in ds.list_objects]
    W.write_detector_run(tmp_path, "detector-engine-test", input_resize=tuple(images.shape[-2:]), n_classes=len(labels),
                         seed=7, spread_scores=3.0)
    det = D.load_detector("detector-engine-test", models_root=tmp_path, engine=True)
    assert isinstance(det.model, E.EngineMaskRCNN)
    det.category_id_to_label = {i + 1: l for i, l in enumerate(labels)}
    obs = ObservationTensor(images[:, :3].contiguous(), K.clone()).cuda()
    est.detector_model = det
    detections = det.get_detections(obs)
    assert len(detections) > 0
    a, _ = est.run_inference_pipeline(obs, run_detector=True, n_refiner_iterations=2)
    b, _ = est.run_inference_pipeline(obs, detections=detections, n_refiner_iterations=2)
    assert list(a.infos["label"]) == list(b.infos["label"]) and torch.equal(a.poses, b.poses)
    assert np.array_equal(a.infos["pose_score"].to_numpy(), b.infos["pose_score"].to_numpy())


from tests.test_gpu_bop_gt_info import split  # noqa: E402,F401  (the written BOP split fixture)


def test_prediction_runner_with_the_engine_detector_writes_its_csv(split, tmp_path, capsys):
    from megapose6d_b200 import bop_dataset, load_model, prediction_runner
    from tests import helpers

    if not (split / "test" / "000001" / "scene_gt_info.json").exists():
        bop_dataset.compute_gt_info(split, "test")
    ckpt = tmp_path / "ckpt"
    load_model.write_run(ckpt, "coarse-rgb-906902141", helpers.make_state_dict(helpers.COARSE_CFG, 5))
    load_model.write_run(ckpt, "refiner-rgb-653307694", helpers.make_state_dict(helpers.REFINER_CFG, 6))
    W.write_detector_run(ckpt, "detector-bop", input_resize=(480, 640), n_classes=3, seed=2, background_bias=4.0)
    prediction_runner.main(["--bop-dataset", str(split), "--label-format", "ycbv-{label}", "--model", "megapose-1.0-RGB",
                            "--models-root", str(ckpt), "--detector", "detector-bop", "--detector-engine",
                            "--save-dir", str(tmp_path / "out")])
    rows = prediction_runner.load_bop_results(tmp_path / "out" / "bop_refiner_final.csv")
    assert len(rows) > 0 and {r["obj_id"] for r in rows} <= {1, 2, 3}
    print(f"{len(rows)} poses from the engine detector's detections")
