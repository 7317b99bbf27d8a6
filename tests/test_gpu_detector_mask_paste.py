"""Mask inference and pasting on the device (csrc/detector_net.cu: mpx_mask_paste) against torchvision's
maskrcnn_inference, resize_boxes and paste_masks_in_image fed the same tensors: boxes bit for bit, probabilities within
MAX_ULPS, edge, outside and sub-pixel boxes; the engine detector with device_paste=True end to end, its host
synchronisations, ABI refusals, the pose pipeline and the command line."""
from __future__ import annotations

import copy
import ctypes
import warnings

import numpy as np
import pytest
import torch

pytest.importorskip("torchvision")

from torchvision.models.detection.roi_heads import maskrcnn_inference, paste_masks_in_image  # noqa: E402
from torchvision.models.detection.transform import resize_boxes  # noqa: E402

from megapose6d_b200 import _abi, detector as D, detector_engine as E  # noqa: E402
from workloads import detector as W  # noqa: E402

pytestmark = pytest.mark.gpu

# The probabilities are torchvision's fp32 expressions (sigmoid, the bilinear weights and sums of upsample_bilinear2d);
# only the compiler's contraction of those sums into FMAs may differ from ATen's build: a few ulps at most.
MAX_ULPS = 4


def _ulps(a: torch.Tensor, b: torch.Tensor) -> int:
    """Largest distance in units in the last place between two tensors of non-negative fp32 values."""
    assert (a >= 0).all() and (b >= 0).all()
    return int((a.contiguous().view(torch.int32).long() - b.contiguous().view(torch.int32).long()).abs().max().item())


def _torchvision(logits, labels, boxes, counts, image_sizes, original_sizes):
    probs = maskrcnn_inference(logits, list(labels.split(counts)))
    out_boxes, out_masks = [], []
    for p, b, s, o in zip(probs, boxes.split(counts), image_sizes, original_sizes):
        rb = resize_boxes(b, s, o)
        out_boxes.append(rb)
        out_masks.append(paste_masks_in_image(p, rb, o))
    return out_boxes, out_masks


def _compare(got, want, what=""):
    (gb, gm), (wb, wm) = got, want
    worst = 0
    for i, (a, b) in enumerate(zip(gb, wb)):
        assert torch.equal(a, b), f"{what} boxes of image {i}"
    for i, (a, b) in enumerate(zip(gm, wm)):
        assert a.shape == b.shape and a.dtype == b.dtype, (what, i, a.shape, b.shape)
        if a.numel():
            worst = max(worst, _ulps(a, b))
            away = (b - 0.5).abs() > 1e-5
            assert torch.equal((a > 0.5)[away], (b > 0.5)[away]), f"{what} thresholded masks of image {i}"
    assert worst <= MAX_ULPS, f"{what}: {worst} ulps"
    return worst


def _case(seed, counts, image_sizes, n_classes=22, m=28):
    """Logits and labels at random; boxes inside each transformed image (as postprocess_detections clips them), a few
    of them sub-pixel and a few on the image's edges."""
    g = torch.Generator().manual_seed(seed)
    n = sum(counts)
    logits = torch.randn(n, n_classes, m, m, generator=g) * 4
    labels = torch.randint(1, n_classes, (n,), generator=g)
    boxes = []
    for c, (h, w) in zip(counts, image_sizes):
        xy = torch.rand(c, 2, generator=g) * torch.tensor([w, h])
        wh = torch.rand(c, 2, generator=g) * torch.tensor([w, h]) * 0.6
        wh[: c // 5] = torch.rand(c // 5, 2, generator=g) * 0.9 + 0.01  # narrower than one pixel
        b = torch.cat([xy, xy + wh], 1)
        b[c // 5: 2 * c // 5, 0] = 0.0                                  # on the left / top edge
        b[c // 5: 2 * c // 5, 1] = 0.0
        b[2 * c // 5: 3 * c // 5, 2] = float(w)                        # on the right / bottom edge
        b[2 * c // 5: 3 * c // 5, 3] = float(h)
        b[:, 0::2] = b[:, 0::2].clamp(0, w)
        b[:, 1::2] = b[:, 1::2].clamp(0, h)
        boxes.append(b)
    return logits.cuda(), labels.cuda(), torch.cat(boxes).cuda()


@pytest.mark.parametrize("counts,image_sizes,original_sizes", [
    ([40], [(480, 640)], [(480, 640)]),
    ([25, 0, 37], [(480, 640)] * 3, [(480, 640)] * 3),
    ([30, 20], [(240, 320), (224, 320)], [(480, 640), (448, 640)]),   # input_resize (240, 320) of 480x640 / 448x640 frames
    ([12], [(800, 1066)], [(540, 720)]),                               # an upscaling transform
], ids=["one", "empty_image", "downscaled", "upscaled"])
def test_paste_equals_torchvision(counts, image_sizes, original_sizes):
    logits, labels, boxes = _case(sum(counts) + len(counts), counts, image_sizes)
    got = E.mask_paste(logits, labels, boxes, counts, image_sizes, original_sizes)
    want = _torchvision(logits, labels, boxes, counts, image_sizes, original_sizes)
    worst = _compare(got, want)
    print(f"{sum(counts)} masks, worst {worst} ulps")


def test_boxes_partly_and_wholly_outside_the_image():
    h, w = 100, 120
    boxes = torch.tensor([[-30.0, -20.0, 40.0, 30.0],    # across the top-left corner
                          [90.0, 80.0, 150.0, 130.0],    # across the bottom-right corner
                          [-0.4, 10.0, 0.2, 10.5],       # sub-pixel, on the left edge
                          [119.6, 99.7, 120.0, 100.0],   # sub-pixel, in the bottom-right corner
                          [-80.0, -60.0, -30.0, -20.0],  # wholly outside, above and left
                          [200.0, 10.0, 260.0, 40.0]])   # wholly outside, right
    g = torch.Generator().manual_seed(11)
    logits = (torch.randn(6, 3, 28, 28, generator=g) * 4).cuda()
    labels = torch.tensor([1, 2, 1, 2, 1, 2]).cuda()
    got_b, got_m = E.mask_paste(logits, labels, boxes.cuda(), [6], [(h, w)], [(h, w)])
    want_b, want_m = _torchvision(logits[:4], labels[:4], boxes[:4].cuda(), [4], [(h, w)], [(h, w)])
    _compare(([got_b[0][:4]], [got_m[0][:4]]), (want_b, want_m), "partly outside")
    # torchvision's slicing does not serve boxes wholly outside the image; nothing of them is in the image
    assert torch.equal(got_b[0][4:], boxes[4:].cuda())
    assert not got_m[0][4:].any()


def test_labels_outside_the_classes_paste_nothing():
    logits, labels, boxes = _case(3, [4], [(64, 64)], n_classes=3)
    labels = torch.tensor([-1, 3, 1, 2]).cuda()
    got_b, got_m = E.mask_paste(logits, labels, boxes, [4], [(64, 64)], [(64, 64)])
    assert not got_m[0][:2].any()
    want = _torchvision(logits[2:], labels[2:], boxes[2:], [2], [(64, 64)], [(64, 64)])
    _compare(([got_b[0][2:]], [got_m[0][2:]]), want)


def test_abi_refusals_launch_nothing():
    lib = _abi.lib()
    logits, labels, boxes = _case(5, [3], [(64, 64)])
    out_b = torch.empty_like(boxes)
    masks = torch.empty(3, 1, 64, 64, device="cuda")
    host = torch.empty(3 * 22 * 28 * 28)
    ok = dict(logits=logits.data_ptr(), labels=labels.data_ptr(), boxes=boxes.data_ptr(), n=3, classes=22, m=28,
              images=1, counts=[3], sizes=[64, 64, 64, 64], out=out_b.data_ptr(), masks=[masks.data_ptr()])
    cases = [
        ("no_images", dict(images=0, counts=[], sizes=[], masks=[]), "n_images=0"),
        ("mask_size", dict(m=65), "m=65"),
        ("classes", dict(classes=0), "n_classes=0"),
        ("count_sum", dict(n=4), "add up to 3"),
        ("negative_count", dict(counts=[-1], n=-1), "n_masks=-1"),
        ("size", dict(sizes=[64, 64, 0, 64]), "must be positive"),
        ("null_masks", dict(masks=[None]), "NULL or not device memory"),
        ("host_logits", dict(logits=host.data_ptr()), "d_logits is not device memory"),
        ("null_boxes_out", dict(out=None), "d_boxes_out is NULL"),
    ]
    for name, kw, msg in cases:
        a = dict(ok)
        a.update(kw)
        k = a["images"]
        before = lib.mpx_launch_count()
        rc = lib.mpx_mask_paste(a["logits"], a["labels"], a["boxes"], a["n"], a["classes"], a["m"], k,
                                (ctypes.c_int32 * max(k, 1))(*a["counts"]), (ctypes.c_int32 * max(4 * k, 1))(*a["sizes"]),
                                a["out"], (ctypes.c_void_p * max(k, 1))(*a["masks"]), _abi.stream_ptr())
        assert rc != 0, name
        assert msg in lib.mpx_last_error().decode(), (name, lib.mpx_last_error())
        assert lib.mpx_launch_count() == before, name
    torch.cuda.synchronize()


@pytest.fixture(scope="module")
def spread_model():
    return W.make_detector((480, 640), seed=4, spread_scores=3.0, device="cuda")


def _images(seeds, hw=(480, 640)):
    return [torch.rand(3, *hw, generator=torch.Generator().manual_seed(s)).cuda() for s in seeds]


def test_paste_module_equals_the_engine_module_with_its_masks_pasted_on_the_device(spread_model):
    """device_paste=True changes nothing but the mask pasting: boxes, labels and scores are the device_paste=False module's,
    bit for bit, and masks within MAX_ULPS; two images of different sizes in one batch get their own sizes."""
    base, paste = E.engine_model(spread_model), E.engine_model(spread_model, device_paste=True)
    images = _images((8,)) + _images((9,), (448, 600))
    with torch.no_grad():
        want = base(images)
    got = paste(images)
    counts = [len(w["scores"]) for w in want]
    assert sum(counts) > 0
    for g, w, img in zip(got, want, images):
        assert g.keys() == w.keys()
        for k in ("boxes", "labels", "scores"):
            assert torch.equal(g[k], w[k]), k
        assert g["masks"].shape == (len(w["scores"]), 1, *img.shape[-2:])
    worst = _compare(([g["boxes"] for g in got], [g["masks"] for g in got]),
                     ([w["boxes"] for w in want], [w["masks"] for w in want]), "end to end")
    print(f"detections {counts}, worst {worst} ulps")


def test_an_image_without_detections_gives_torchvision_empty_shapes(spread_model):
    quiet = copy.deepcopy(spread_model)
    with torch.no_grad():
        quiet.roi_heads.box_predictor.cls_score.bias[0] += 50.0
        want = quiet(_images((8,)))
    got = E.engine_model(quiet, device_paste=True)(_images((8,)))
    assert len(want[0]["scores"]) == 0
    for k in want[0]:
        assert got[0][k].shape == want[0][k].shape and got[0][k].dtype == want[0][k].dtype, k


def _syncs(fn) -> int:
    """Synchronising CUDA calls torch makes during fn() (torch.cuda.set_sync_debug_mode)."""
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    return sum("synchroniz" in str(w.message) for w in rec)


def test_synchronisations_do_not_grow_with_the_detections(spread_model):
    """Up to 100 or at most 5 detections per image: the same synchronising calls with device_paste=True (torchvision's
    stages before the paste synchronise per image and per level, not per detection); torchvision's paste adds several per
    detection.  Without any detection torchvision's RoI pooling skips a little work: no more calls."""
    few = copy.deepcopy(spread_model)
    few.roi_heads.detections_per_img = 5
    quiet = copy.deepcopy(spread_model)
    with torch.no_grad():
        quiet.roi_heads.box_predictor.cls_score.bias[0] += 50.0
    images = _images((8, 9))
    counts, syncs = {}, {}
    for name, model in (("many", spread_model), ("few", few), ("none", quiet)):
        for device_paste in (False, True):
            module = E.engine_model(model, device_paste=device_paste)
            out = module(images)  # warm-up: first sight of the shape, graph capture
            module(images)
            counts[name] = sum(len(o["scores"]) for o in out)
            syncs[name, device_paste] = _syncs(lambda: module(images))
    print(f"detections {counts}, synchronising calls {syncs}")
    assert counts["many"] > counts["few"] > 0 and counts["none"] == 0
    assert syncs["many", True] == syncs["few", True] >= syncs["none", True]
    assert syncs["many", False] >= syncs["few", False] + counts["many"] - counts["few"]


def test_pipeline_with_the_device_paste_detector_equals_passing_its_detections(tmp_path):
    from megapose6d_b200 import load_model
    from megapose6d_b200.types import ObservationTensor
    from tests import helpers

    ds, images, K = helpers.make_scene(2, seed=6)
    load_model.write_run(tmp_path, "coarse-rgb-906902141", helpers.make_state_dict(helpers.COARSE_CFG, 5))
    load_model.write_run(tmp_path, "refiner-rgb-653307694", helpers.make_state_dict(helpers.REFINER_CFG, 6))
    est = load_model.load_named_model("megapose-1.0-RGB", ds, models_root=tmp_path)
    est.load_SO3_grid(72)
    labels = [o.label for o in ds.list_objects]
    W.write_detector_run(tmp_path, "detector-paste-test", input_resize=tuple(images.shape[-2:]), n_classes=len(labels),
                         seed=7, spread_scores=3.0)
    det = D.load_detector("detector-paste-test", models_root=tmp_path, engine=True, device_paste=True)
    assert isinstance(det.model, E.EngineMaskRCNN) and det.model.device_paste
    det.category_id_to_label = {i + 1: l for i, l in enumerate(labels)}
    obs = ObservationTensor(images[:, :3].contiguous(), K.clone()).cuda()
    est.detector_model = det
    detections = det.get_detections(obs, output_masks=True)
    assert len(detections) > 0 and detections.masks.shape[0] == len(detections)
    a, _ = est.run_inference_pipeline(obs, run_detector=True, n_refiner_iterations=2)
    b, _ = est.run_inference_pipeline(obs, detections=detections, n_refiner_iterations=2)
    assert list(a.infos["label"]) == list(b.infos["label"]) and torch.equal(a.poses, b.poses)
    assert np.array_equal(a.infos["pose_score"].to_numpy(), b.infos["pose_score"].to_numpy())


from tests.test_gpu_bop_gt_info import split  # noqa: E402,F401  (the written BOP split fixture)


def test_prediction_runner_with_the_device_paste_detector_writes_its_csv(split, tmp_path):
    from megapose6d_b200 import bop_dataset, load_model, prediction_runner
    from tests import helpers

    if not (split / "test" / "000001" / "scene_gt_info.json").exists():
        bop_dataset.compute_gt_info(split, "test")
    ckpt = tmp_path / "ckpt"
    load_model.write_run(ckpt, "coarse-rgb-906902141", helpers.make_state_dict(helpers.COARSE_CFG, 5))
    load_model.write_run(ckpt, "refiner-rgb-653307694", helpers.make_state_dict(helpers.REFINER_CFG, 6))
    W.write_detector_run(ckpt, "detector-bop", input_resize=(480, 640), n_classes=3, seed=2, background_bias=4.0)
    prediction_runner.main(["--bop-dataset", str(split), "--label-format", "ycbv-{label}", "--model", "megapose-1.0-RGB",
                            "--models-root", str(ckpt), "--detector", "detector-bop", "--detector-device-paste",
                            "--save-dir", str(tmp_path / "out")])
    rows = prediction_runner.load_bop_results(tmp_path / "out" / "bop_refiner_final.csv")
    assert len(rows) > 0 and {r["obj_id"] for r in rows} <= {1, 2, 3}
