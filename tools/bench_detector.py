"""Time the Mask R-CNN detector with its ResNet-50 FPN backbone and RPN head on the engine against torchvision.

Workload: the seeded detector of `workloads.detector.make_detector` (no trained checkpoint is available), 480x640 images,
batch 1 and 8, with `input_resize` (480, 640) and the reference default (240, 320).  Arms:
  engine     backbone + RPN head as one mpx_fpn_forward (detector_engine.engine_model), the rest torchvision fp32
  fp32       torchvision, TF32 off
  tf32       torchvision with torch's defaults (cuDNN convolutions in TF32)
  fp16_cl    torchvision under fp16 autocast, channels_last
Stages: `heads` = backbone + RPN head (one mpx_fpn_forward for the engine), `rest` = anchors, proposals, RoI heads and
postprocessing from those outputs, `detector` = the whole `Detector.get_detections`.  After a warm-up, every window times
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
        tv = {"fp32": model, "tf32": model, "fp16_cl": cl}
        for batch in (1, 8):
            g = torch.Generator().manual_seed(batch)
            images = torch.rand(batch, 3, 480, 640, generator=g).cuda()
            obs = ObservationTensor(images, torch.eye(3).repeat(batch, 1, 1).cuda())
            image_list, _ = model.transform(list(images))
            arms = ["engine", "fp32", "tf32", "fp16_cl"]
            heads_out, fns = {}, {}
            for arm in arms:
                m = engine if arm == "engine" else tv[arm]
                det = Detector(m)

                def heads(arm=arm):
                    with arm_context(arm), torch.no_grad():
                        if arm == "engine":
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
                        r = tv[arm] if arm != "engine" else model
                        dets, _ = r.roi_heads(feats, props, image_list.image_sizes)
                        return r.transform.postprocess(dets, image_list.image_sizes, [(480, 640)] * batch)

                def whole(arm=arm, det=det):
                    with arm_context(arm):
                        return det.get_detections(obs)

                fns[arm] = dict(heads=heads, rest=rest, detector=whole)
            for arm in arms:  # warm-up: algorithm selection, graph capture
                for fn in fns[arm].values():
                    for _ in range(3):
                        fn()
            times = {arm: {s: [] for s in fns[arm]} for arm in arms}
            for _ in range(args.windows):
                for arm in arms:
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
                        detector_speedup_vs_fp32=med["fp32"]["detector"] / med["engine"]["detector"])
            out["cases"].append(case)
            print(json.dumps(case), file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
