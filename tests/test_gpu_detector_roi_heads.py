"""The detector's RoI heads on the engine (engine_roi_heads=True, include/mpx.h mpx_roi_*, csrc/detector_heads.cu):
the level assignment and pooled values bit for bit against torchvision's MultiScaleRoIAlign, both branches bit for bit
against the float64 oracle on integer operands and within the stated bound with Gaussian weights, the ABI's refusals, and the whole detector against
torchvision fp32 and against device_paste=True."""
import ctypes

import pytest
import torch

pytest.importorskip("torchvision")

from megapose6d_b200 import _abi, detector_engine as E  # noqa: E402
from oracle import detector_heads_ref as R  # noqa: E402
from tests.test_gpu_detector_engine import _partners  # noqa: E402
from workloads import detector as W  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
LEVELS = ["0", "1", "2", "3"]


def _features(n, h, w, seed, integer=False):
    g = torch.Generator().manual_seed(seed)
    out = {}
    for k, s in zip(LEVELS, (4, 8, 16, 32)):
        t = torch.randint(-8, 9, (n, 256, h // s, w // s), generator=g).float() if integer else \
            torch.randn(n, 256, h // s, w // s, generator=g)
        out[k] = t.to(DEV).contiguous()
    return out


def _boxes(count, h, w, seed):
    """Boxes across the image edges, sub-pixel boxes and boxes of every level, in one shuffled list."""
    g = torch.Generator().manual_seed(seed)
    xy = torch.rand(count, 2, generator=g) * torch.tensor([w * 1.2, h * 1.2]) - torch.tensor([w * 0.1, h * 0.1])
    side = torch.exp(torch.rand(count, 1, generator=g) * 7.0 - 1.5)  # 0.2 .. 245 px
    aspect = torch.exp(torch.randn(count, 1, generator=g) * 0.4)
    wh = torch.cat([side * aspect, side / aspect], 1)
    return torch.cat([xy, xy + wh], 1)


def _boundary_boxes(h, w):
    """Squares whose sqrt(area) sits on LevelMapper's boundaries 112, 224 and 448 px (and the floats either side)."""
    out = []
    for s in (112.0, 224.0, 448.0):
        for side in (torch.tensor(s).nextafter(torch.tensor(0.0)), torch.tensor(s), torch.tensor(s).nextafter(torch.tensor(1e9))):
            x0 = float(w) / 4
            out.append([x0, 10.0, x0 + float(side), 10.0 + float(side)])
    out += [[5.0, 5.0, 5.0, 5.0], [w - 0.3, h - 0.2, w + 40.0, h + 30.0], [-50.0, -60.0, 3.0, 2.5], [10.0, 10.0, 10.4, 10.7],
            [40.0, 30.0, 20.0, 60.0]]  # negative area: a NaN level, which torchvision pools on no level (zeros)
    return torch.tensor(out)


def _pool_call(feats, boxes, counts, hw, image_sizes, pool, levels=None):
    fl = [feats[k] for k in LEVELS]
    out = torch.full((boxes.shape[0], *pool.output_size, 256), float("nan"), device=DEV)
    lv = torch.full((boxes.shape[0],), -1, dtype=torch.int32, device=DEV)
    _abi.check(_abi.lib().mpx_roi_pool((ctypes.c_void_p * 4)(*[f.data_ptr() for f in fl]), len(counts), hw[0], hw[1],
                                       *E.pool_args(pool, fl, image_sizes), boxes.data_ptr(),
                                       (ctypes.c_int32 * len(counts))(*counts), pool.output_size[0], out.data_ptr(),
                                       lv.data_ptr(), _abi.stream_ptr()))
    return out.permute(0, 3, 1, 2), lv


@pytest.mark.parametrize("output_size,sampling", [(7, 2), (14, 2), (7, 1), (5, 3)])
def test_levels_and_pooling_bit_identical_to_torchvision(output_size, sampling):
    from torchvision.ops import MultiScaleRoIAlign

    h, w = 480, 640
    feats = _features(2, h, w, seed=1)
    boxes = [torch.cat([_boundary_boxes(h, w), _boxes(300, h, w, 2)]), _boxes(200, 448, 608, 3)]
    image_sizes = [(h, w), (448, 608)]
    pool = MultiScaleRoIAlign(LEVELS, output_size, sampling)
    cat = torch.cat(boxes).to(DEV).contiguous()
    got, levels = _pool_call(feats, cat, [b.shape[0] for b in boxes], (h, w), image_sizes, pool)
    want = pool(feats, [b.to(DEV) for b in boxes], image_sizes)
    want_levels = pool.map_levels([b.to(DEV) for b in boxes]).to(torch.int32)
    assert torch.equal(levels, want_levels)
    assert set(levels.tolist()) >= {0, 1, 2, 3}
    assert torch.equal(got, want)


@pytest.mark.parametrize("n,h,w", [(1, 480, 640), (3, 480, 640), (1, 256, 320), (3, 256, 320)])
def test_branches_bit_exact_on_integer_operands(n, h, w):
    model = W.make_detector((h, w), n_classes=21, seed=5, device="cpu")
    W.integer_roi_heads_weights(model, seed=6)
    model = model.to(DEV).eval()
    engine = E.RoiHeadsEngine(model, DEV)
    feats = _features(n, h, w, seed=7, integer=True)
    counts = [400, 0, 137][:n]
    proposals = [_boxes(c, h, w, 10 + i).to(DEV) for i, c in enumerate(counts)]
    image_sizes = [(h, w)] * n
    logits, deltas = engine.box(feats, torch.cat(proposals), counts, (h, w), image_sizes)
    o_logits, o_deltas = R.roi_heads_box(model, feats, proposals, image_sizes)
    assert torch.equal(logits, o_logits.float()) and torch.equal(deltas, o_deltas.float())
    det = [p[: c // 4] for p, c in zip(proposals, counts)]
    dcounts = [d.shape[0] for d in det]
    masks = engine.mask(feats, torch.cat(det), dcounts, (h, w), image_sizes)
    o_masks = R.roi_heads_mask(model, feats, det, image_sizes)
    assert masks.shape == (sum(dcounts), 22, 28, 28)  # 21 objects and the background
    assert torch.equal(masks, o_masks.float())


def test_branches_gaussian_weights_within_bound():
    h, w = 480, 640
    model = W.make_detector((h, w), n_classes=21, seed=8, spread_scores=3.0, device=DEV)
    engine = E.RoiHeadsEngine(model, DEV)
    feats = _features(2, h, w, seed=9)
    counts = [500, 300]
    proposals = [_boxes(c, h, w, 20 + i).to(DEV) for i, c in enumerate(counts)]
    sizes = [(h, w)] * 2
    logits, deltas = engine.box(feats, torch.cat(proposals), counts, (h, w), sizes)
    o_logits, o_deltas = R.roi_heads_box(model, feats, proposals, sizes)
    masks = engine.mask(feats, torch.cat(proposals), counts, (h, w), sizes)
    o_masks = R.roi_heads_mask(model, feats, proposals, sizes)
    for got, want in ((logits, o_logits), (deltas, o_deltas), (masks, o_masks)):
        err = float((got.double() - want).abs().max() / want.abs().max())
        print(f"engine vs oracle {err / 2 ** -11:.2f} u")
        assert err <= R.HEADS_VS_ORACLE


def test_zero_rois_launch_nothing():
    h, w = 256, 320
    model = W.make_detector((h, w), n_classes=21, seed=5, device=DEV)
    engine = E.RoiHeadsEngine(model, DEV)
    feats = _features(2, h, w, seed=1)
    launches = _abi.lib().mpx_launch_count()
    logits, deltas = engine.box(feats, torch.empty(0, 4, device=DEV), [0, 0], (h, w), [(h, w)] * 2)
    masks = engine.mask(feats, torch.empty(0, 4, device=DEV), [0, 0], (h, w), [(h, w)] * 2)
    assert _abi.lib().mpx_launch_count() == launches
    assert logits.shape == (0, 22) and deltas.shape == (0, 88) and masks.shape == (0, 22, 28, 28)


def test_abi_refusals_launch_nothing():
    h, w = 256, 320
    model = W.make_detector((h, w), n_classes=21, seed=5, device=DEV)
    engine = E.RoiHeadsEngine(model, DEV)
    lib = _abi.lib()
    feats = [f for f in _features(1, h, w, seed=1).values()]
    boxes = _boxes(10, h, w, 1).to(DEV)
    logits = torch.empty(10, 22, device=DEV)
    deltas = torch.empty(10, 88, device=DEV)
    ws = torch.empty(lib.mpx_roi_heads_workspace_bytes(engine._handle, 10, 0, 14), dtype=torch.uint8, device=DEV)
    host = torch.empty(16)
    good = dict(handle=engine._handle, feats=[f.data_ptr() for f in feats], n=1, h=h, w=w, scales=[0.25, 0.125, 0.0625, 0.03125],
                sampling=2, boxes=boxes.data_ptr(), counts=[10], logits=logits.data_ptr(), deltas=deltas.data_ptr(),
                ws=ws.data_ptr(), ws_bytes=ws.numel())

    def call(**kw):
        a = {**good, **kw}
        return lib.mpx_roi_box_forward(a["handle"], (ctypes.c_void_p * 4)(*a["feats"]), a["n"], a["h"], a["w"],
                                       (ctypes.c_float * 4)(*a["scales"]), 224, 4, a["sampling"], a["boxes"],
                                       (ctypes.c_int32 * len(a["counts"]))(*a["counts"]), a["logits"], a["deltas"],
                                       a["ws"], a["ws_bytes"], None)

    cases = [
        (dict(handle=None), "heads is NULL"),
        (dict(h=250), "multiples of 32"),
        (dict(n=0, counts=[]), "n_images=0"),
        (dict(counts=[-1]), "has -1 RoIs"),
        (dict(sampling=0), "sampling_ratio=0"),
        (dict(scales=[0.25, 0.125, 0.0625, 0.03]), "scales"),
        (dict(feats=[feats[0].data_ptr(), 0, feats[2].data_ptr(), feats[3].data_ptr()]), "level 1 is NULL"),
        (dict(boxes=host.data_ptr()), "d_boxes is NULL or not device memory"),
        (dict(logits=None), "d_class_logits is NULL"),
        (dict(deltas=host.data_ptr()), "not device memory"),
        (dict(ws_bytes=ws.numel() - 1), "workspace of"),
        (dict(ws=ws.data_ptr() + 16, ws_bytes=ws.numel() - 16), "256-B aligned"),
    ]
    launches = lib.mpx_launch_count()
    for kw, msg in cases:
        rc = call(**kw)
        assert rc != 0, kw
        assert msg in lib.mpx_last_error().decode(), (kw, lib.mpx_last_error())
    assert lib.mpx_launch_count() == launches
    assert call() == 0, lib.mpx_last_error()
    torch.cuda.synchronize()


def test_detections_end_to_end():
    """engine_roi_heads=True against torchvision fp32 and against device_paste=True, with the partner criterion of
    test_gpu_detector_engine (tau from the FPN features' relative error)."""
    model = W.make_detector((480, 640), seed=4, spread_scores=3.0, device=DEV)
    images = [torch.rand(3, 480, 640, generator=torch.Generator().manual_seed(s)).to(DEV) for s in (8, 9)]
    heads = E.engine_model(model, engine_roi_heads=True)
    paste = E.engine_model(model, device_paste=True)
    with torch.no_grad():
        image_list, _ = model.transform(images)
        feats = model.backbone(image_list.tensors)
        e_feats, _, _ = heads.heads(image_list)
        e_feat = max((a - b).abs().max().item() / b.abs().max().item() for a, b in zip(e_feats.values(), feats.values()))
        want = model(images)
    got = heads(images)
    ref = paste(images)
    tau = max(0.01, 16 * e_feat)
    checked = 0
    thresh = model.roi_heads.score_thresh
    for w, g, p in zip(want, got, ref):
        assert g["boxes"].dtype == torch.float32 and g["labels"].dtype == torch.int64 and g["masks"].dtype == torch.float32
        assert g["masks"].shape[1:] == (1, 480, 640)
        t = max(thresh, float(w["scores"][-1])) if len(w["scores"]) == model.roi_heads.detections_per_img else thresh
        checked += _partners(w, g, tau, t) + _partners(g, w, tau, t)
        checked += _partners(p, g, tau, t) + _partners(g, p, tau, t)
    print(f"e_feat {e_feat:.2e}, tau {tau:.3f}, {checked} detections matched")
    assert checked > 0


def test_no_detection_gives_torchvision_empty_shapes():
    model = W.make_detector((256, 320), seed=4, spread_scores=3.0, device=DEV)
    with torch.no_grad():
        model.roi_heads.box_predictor.cls_score.bias[0] += 1e4  # background wins every box
    heads = E.engine_model(model, engine_roi_heads=True)
    images = [torch.rand(3, 256, 320, generator=torch.Generator().manual_seed(1)).to(DEV)]
    got = heads(images)
    with torch.no_grad():
        want = model(images)
    for k in ("boxes", "labels", "scores", "masks"):
        assert got[0][k].shape == want[0][k].shape and got[0][k].dtype == want[0][k].dtype, k


def test_pool_mask_and_create_refusals_launch_nothing():
    h, w = 256, 320
    model = W.make_detector((h, w), n_classes=21, seed=5, device=DEV)
    engine = E.RoiHeadsEngine(model, DEV)
    lib = _abi.lib()
    feats = [f for f in _features(1, h, w, seed=1).values()]
    fp = (ctypes.c_void_p * 4)(*[f.data_ptr() for f in feats])
    scales = (ctypes.c_float * 4)(0.25, 0.125, 0.0625, 0.03125)
    boxes = _boxes(10, h, w, 1).to(DEV)
    counts = (ctypes.c_int32 * 1)(10)
    pooled = torch.empty(10, 7, 7, 256, device=DEV)
    masks = torch.empty(10, 22, 28, 28, device=DEV)
    ws = torch.empty(lib.mpx_roi_heads_workspace_bytes(engine._handle, 0, 10, 14), dtype=torch.uint8, device=DEV)
    host = torch.empty(16)
    big = (ctypes.c_int32 * 1)(600000)

    def pool(out_size=7, out=pooled.data_ptr(), levels=None, b=boxes.data_ptr(), c=counts):
        return lib.mpx_roi_pool(fp, 1, h, w, scales, 224, 4, 2, b, c, out_size, out, levels, None)

    def mask(mask_pool=14, out=masks.data_ptr(), c=counts, wsb=ws.numel()):
        return lib.mpx_roi_mask_forward(engine._handle, fp, 1, h, w, scales, 224, 4, 2, mask_pool, boxes.data_ptr(), c,
                                        out, ws.data_ptr(), wsb, None)

    def create(n=9, classes=22, hidden=1024, bad=None):
        wp = [t.data_ptr() for t in engine._weights]
        if bad is not None:
            wp[bad] = host.data_ptr()
        out = ctypes.c_void_p()
        return lib.mpx_roi_heads_create((ctypes.c_void_p * 9)(*wp), (ctypes.c_void_p * 9)(*[t.data_ptr() for t in engine._biases]),
                                        n, classes, hidden, ctypes.byref(out))

    cases = [
        (lambda: pool(out_size=0), "output size 0"),
        (lambda: pool(out_size=33), "output size 33"),
        (lambda: pool(out=None), "d_pooled is NULL"),
        (lambda: pool(levels=host.data_ptr()), "d_levels is not device memory"),
        (lambda: pool(b=host.data_ptr()), "d_boxes is NULL or not device memory"),
        (lambda: mask(mask_pool=0), "mask pool 0"),
        (lambda: mask(mask_pool=32, c=big), "must be below 2^31"),
        (lambda: mask(out=host.data_ptr()), "d_mask_logits is not device memory"),
        (lambda: mask(wsb=ws.numel() - 1), "workspace of"),
        (lambda: create(n=8), "expected 9 conv tensors"),
        (lambda: create(classes=410), "410 classes"),
        (lambda: create(hidden=1000), "representation size 1000"),
        (lambda: create(bad=4), "conv 4 has a NULL or non-device tensor"),
    ]
    launches = lib.mpx_launch_count()
    for fn, msg in cases:
        assert fn() != 0, msg
        assert msg in lib.mpx_last_error().decode(), (msg, lib.mpx_last_error())
    assert lib.mpx_launch_count() == launches
    assert lib.mpx_roi_heads_workspace_bytes(engine._handle, 0, 600000, 32) == 0
    assert pool() == 0 and mask() == 0, lib.mpx_last_error()
    torch.cuda.synchronize()


def test_engine_refuses_features_of_another_shape():
    h, w = 256, 320
    model = W.make_detector((h, w), n_classes=21, seed=5, device=DEV)
    engine = E.RoiHeadsEngine(model, DEV)
    feats = _features(2, h, w, seed=1)
    boxes = _boxes(4, h, w, 1).to(DEV)
    with pytest.raises(ValueError, match="level 0"):
        engine.box(feats, boxes, [4], (h, w), [(h, w)])  # two images' features, one count
    with pytest.raises(ValueError, match="level 0"):
        engine.box(feats, boxes, [2, 2], (h + 32, w), [(h, w)] * 2)
    with pytest.raises(ValueError, match="boxes must be"):
        engine.mask(feats, boxes, [2, 1], (h, w), [(h, w)] * 2)


def test_pipeline_with_the_roi_heads_detector_equals_passing_its_detections(tmp_path):
    import numpy as np

    from megapose6d_b200 import detector as D, load_model
    from megapose6d_b200.types import ObservationTensor
    from tests import helpers

    ds, images, K = helpers.make_scene(2, seed=6)
    load_model.write_run(tmp_path, "coarse-rgb-906902141", helpers.make_state_dict(helpers.COARSE_CFG, 5))
    load_model.write_run(tmp_path, "refiner-rgb-653307694", helpers.make_state_dict(helpers.REFINER_CFG, 6))
    est = load_model.load_named_model("megapose-1.0-RGB", ds, models_root=tmp_path)
    est.load_SO3_grid(72)
    labels = [o.label for o in ds.list_objects]
    W.write_detector_run(tmp_path, "detector-heads-test", input_resize=tuple(images.shape[-2:]), n_classes=len(labels),
                         seed=7, spread_scores=3.0)
    det = D.load_detector("detector-heads-test", models_root=tmp_path, engine=True, engine_roi_heads=True)
    assert isinstance(det.model, E.EngineMaskRCNN) and det.model.roi_engine is not None
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


def test_prediction_runner_with_the_roi_heads_detector_writes_its_csv(split, tmp_path):
    from megapose6d_b200 import bop_dataset, load_model, prediction_runner
    from tests import helpers

    if not (split / "test" / "000001" / "scene_gt_info.json").exists():
        bop_dataset.compute_gt_info(split, "test")
    ckpt = tmp_path / "ckpt"
    load_model.write_run(ckpt, "coarse-rgb-906902141", helpers.make_state_dict(helpers.COARSE_CFG, 5))
    load_model.write_run(ckpt, "refiner-rgb-653307694", helpers.make_state_dict(helpers.REFINER_CFG, 6))
    W.write_detector_run(ckpt, "detector-bop", input_resize=(480, 640), n_classes=3, seed=2, background_bias=4.0)
    prediction_runner.main(["--bop-dataset", str(split), "--label-format", "ycbv-{label}", "--model", "megapose-1.0-RGB",
                            "--models-root", str(ckpt), "--detector", "detector-bop", "--detector-engine-roi-heads",
                            "--save-dir", str(tmp_path / "out")])
    rows = prediction_runner.load_bop_results(tmp_path / "out" / "bop_refiner_final.csv")
    assert len(rows) > 0 and {r["obj_id"] for r in rows} <= {1, 2, 3}
