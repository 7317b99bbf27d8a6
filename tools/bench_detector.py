"""Time the Mask R-CNN detector with its ResNet-50 FPN backbone and RPN head on the engine against torchvision.

Workload: the seeded detector of `workloads.detector.make_detector` (no trained checkpoint is available), 480x640 images,
batch 1 and 8, with `input_resize` (480, 640) and the reference default (240, 320).  Arms:
  engine     backbone + RPN head as one mpx_fpn_forward (detector_engine.engine_model), the rest torchvision fp32
  engine_paste  as engine, and the masks pasted on the device (engine_model(..., device_paste=True): one mpx_mask_paste)
  engine_heads  as engine_paste, and the RoI heads' box and mask branches on the engine (engine_model(...,
             engine_roi_heads=True): mpx_roi_box_forward, torchvision's postprocess_detections, mpx_roi_mask_forward)
  fp32       torchvision, TF32 off
  tf32       torchvision with torch's defaults (cuDNN convolutions in TF32)
  fp16_cl    torchvision under fp16 autocast, channels_last
Stages: `heads` = backbone + RPN head (one mpx_fpn_forward for the engine), `rest` = anchors, proposals, RoI heads and
postprocessing from those outputs, `detector` = the whole `Detector.get_detections`.  `rest` is split, on the engine's
head outputs, into torchvision's `proposals` (anchors, decoding, filter_proposals), `box` (box RoI pool, box head, box
predictor, postprocess_detections), `mask` (mask RoI pool, mask head, mask predictor) and `paste` (maskrcnn_inference and
GeneralizedRCNNTransform.postprocess), next to the engine's `box_engine` (mpx_roi_box_forward and the same
postprocess_detections), `mask_engine` (mpx_roi_mask_forward) and `paste_engine` (mpx_mask_paste).  After a warm-up, every window times
each arm in turn (CUDA events, `--calls` calls) and the medians over `--windows` windows are reported, with the engine's
convolution TFLOP/s (mpx_profile_enable: events around every convolution, FLOPs from the shapes), the largest per-level
relative error of each arm's head outputs against fp32, the device name and its power limit, as one JSON line.

    python tools/bench_detector.py [--windows 5] [--calls 5]
"""
from __future__ import annotations

import argparse
import contextlib
import copy
import ctypes
import json
import statistics
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from torchvision.models.detection.roi_heads import maskrcnn_inference  # noqa: E402

from megapose6d_b200 import _abi, detector_engine as E  # noqa: E402
from megapose6d_b200.detector import Detector  # noqa: E402
from megapose6d_b200.types import ObservationTensor  # noqa: E402
from tools.bench_teaserpp import gpu_info  # noqa: E402
from workloads.detector import make_detector  # noqa: E402


def timed(fn, calls: int) -> float:
    """Milliseconds per call between CUDA events."""
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(calls):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / calls


def arm_context(arm: str):
    if arm == "tf32":
        return torch.backends.cudnn.flags(enabled=True, allow_tf32=True)
    if arm == "fp16_cl":
        return torch.autocast("cuda", dtype=torch.float16)
    return contextlib.nullcontext()


def split_stages(model, engine, roi, image_list, batch: int):
    """torchvision's stages after the RPN head, one by one, each fed the previous stage's outputs computed once from the
    engine's head outputs; and the device paste on the same inputs."""
    rh, sizes, orig = model.roi_heads, image_list.image_sizes, [(480, 640)] * batch
    with torch.no_grad():
        feats, o, d = engine.heads(image_list)
        props = engine.proposals(image_list, feats, o, d)
        cls, reg = rh.box_predictor(rh.box_head(rh.box_roi_pool(feats, props, sizes)))
        boxes, scores, labels = rh.postprocess_detections(cls, reg, props, sizes)
        logits = rh.mask_predictor(rh.mask_head(rh.mask_roi_pool(feats, boxes, sizes)))
    counts = [int(b.shape[0]) for b in boxes]

    def proposals():
        with torch.no_grad():
            return engine.proposals(image_list, feats, o, d)

    def box():
        with torch.no_grad():
            c, r = rh.box_predictor(rh.box_head(rh.box_roi_pool(feats, props, sizes)))
            return rh.postprocess_detections(c, r, props, sizes)

    def mask():
        with torch.no_grad():
            return rh.mask_predictor(rh.mask_head(rh.mask_roi_pool(feats, boxes, sizes)))

    def paste():
        with torch.no_grad():
            dets = [dict(boxes=b, labels=l, scores=s, masks=p)
                    for b, l, s, p in zip(boxes, labels, scores, maskrcnn_inference(logits, labels))]
            return model.transform.postprocess(dets, sizes, orig)

    def paste_engine():
        return E.mask_paste(logits, torch.cat(labels), torch.cat(boxes), counts, sizes, orig)

    hw = tuple(image_list.tensors.shape[-2:])
    n_props = [int(p.shape[0]) for p in props]
    props_cat, boxes_cat = torch.cat(props), torch.cat(boxes)

    def box_engine():
        with torch.no_grad():
            c, r = roi.box(feats, props_cat, n_props, hw, sizes)
            return rh.postprocess_detections(c, r, props, sizes)

    def mask_engine():
        return roi.mask(feats, boxes_cat, counts, hw, sizes)

    return dict(proposals=proposals, box=box, mask=mask, paste=paste, box_engine=box_engine, mask_engine=mask_engine,
                paste_engine=paste_engine), counts


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--calls", type=int, default=5)
    args = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    out = dict(gpu_info(), windows=args.windows, calls=args.calls, cases=[])
    lib = _abi.lib()
    for resize in ((480, 640), (240, 320)):
        model = make_detector(resize, seed=0, device="cuda")
        cl = copy.deepcopy(model).to(memory_format=torch.channels_last)
        engine = E.engine_model(model)
        engine_paste = E.engine_model(model, device_paste=True)
        engine_heads = E.engine_model(model, engine_roi_heads=True)
        tv = {"fp32": model, "tf32": model, "fp16_cl": cl}
        for batch in (1, 8):
            g = torch.Generator().manual_seed(batch)
            images = torch.rand(batch, 3, 480, 640, generator=g).cuda()
            obs = ObservationTensor(images, torch.eye(3).repeat(batch, 1, 1).cuda())
            image_list, _ = model.transform(list(images))
            arms = ["engine", "engine_paste", "engine_heads", "fp32", "tf32", "fp16_cl"]
            heads_out, fns = {}, {}
            for arm in arms:
                m = {"engine": engine, "engine_paste": engine_paste, "engine_heads": engine_heads}.get(arm) or tv[arm]
                det = Detector(m)

                def heads(arm=arm):
                    with arm_context(arm), torch.no_grad():
                        if arm.startswith("engine"):
                            f, o, d = engine.heads(image_list)
                            return list(f.values()), o, d
                        x = image_list.tensors
                        if arm == "fp16_cl":
                            x = x.to(memory_format=torch.channels_last)
                        feats = tv[arm].backbone(x)
                        o, d = tv[arm].rpn.head(list(feats.values()))
                        return list(feats.values()), o, d

                f, o, d = heads()
                heads_out[arm] = [t.float().clone() for t in f + o + d]
                feats = dict(zip(E.LEVELS, f))

                def rest(arm=arm, feats=feats, o=o, d=d):
                    with arm_context(arm), torch.no_grad():
                        props = engine.proposals(image_list, feats, o, d)
                        if arm == "engine_paste":
                            return engine_paste.detect(feats, props, image_list.image_sizes, [(480, 640)] * batch)
                        if arm == "engine_heads":
                            return engine_heads.detect_engine(feats, props, tuple(image_list.tensors.shape[-2:]),
                                                              image_list.image_sizes, [(480, 640)] * batch)
                        r = tv[arm] if not arm.startswith("engine") else model
                        dets, _ = r.roi_heads(feats, props, image_list.image_sizes)
                        return r.transform.postprocess(dets, image_list.image_sizes, [(480, 640)] * batch)

                def whole(arm=arm, det=det):
                    with arm_context(arm):
                        return det.get_detections(obs)

                fns[arm] = dict(heads=heads, rest=rest, detector=whole)
            fns["split"], counts = split_stages(model, engine, engine_heads.roi_engine, image_list, batch)
            for arm in arms:  # warm-up: algorithm selection, graph capture
                for fn in fns[arm].values():
                    for _ in range(3):
                        fn()
            for fn in fns["split"].values():
                for _ in range(3):
                    fn()
            times = {arm: {s: [] for s in fns[arm]} for arm in arms + ["split"]}
            for _ in range(args.windows):
                for arm in arms + ["split"]:
                    for stage, fn in fns[arm].items():
                        times[arm][stage].append(timed(fn, args.calls))
            med = {arm: {s: statistics.median(v) for s, v in st.items()} for arm, st in times.items()}
            lib.mpx_profile_enable(1)
            engine.engine.run(image_list.tensors)
            ms, fl, n = ctypes.c_double(), ctypes.c_double(), ctypes.c_longlong()
            _abi.check(lib.mpx_profile_summary(ctypes.byref(ms), ctypes.byref(fl), ctypes.byref(n)))
            lib.mpx_profile_enable(0)
            ref = heads_out["fp32"]
            err = {arm: max((a - b).abs().max().item() / b.abs().max().item() for a, b in zip(heads_out[arm], ref))
                   for arm in arms if arm != "fp32"}
            case = dict(input_resize=list(resize), batch=batch, padded=list(image_list.tensors.shape[-2:]), ms=med,
                        engine_conv_ms=ms.value, engine_conv_tflops=fl.value / ms.value / 1e9,
                        engine_conv_launches=n.value, max_rel_err_vs_fp32=err,
                        heads_speedup_vs_fp32=med["fp32"]["heads"] / med["engine"]["heads"],
                        heads_speedup_vs_tf32=med["tf32"]["heads"] / med["engine"]["heads"],
                        heads_speedup_vs_fp16_cl=med["fp16_cl"]["heads"] / med["engine"]["heads"],
                        detector_speedup_vs_fp32=med["fp32"]["detector"] / med["engine"]["detector"],
                        detector_speedup_paste_vs_engine=med["engine"]["detector"] / med["engine_paste"]["detector"],
                        detector_speedup_heads_vs_paste=med["engine_paste"]["detector"] / med["engine_heads"]["detector"],
                        detections=counts)
            out["cases"].append(case)
            print(json.dumps(case), file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
