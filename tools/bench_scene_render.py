"""Scene renderer microbench: the 21 objects of workloads.scenes.ycbv_scene(21) at their ground-truth poses, 480x640,
rgb + normals + depth + instance map.

For one frame and for a batch of 64 such frames it times
  * scene: one mpx_raster_render_scene call (all instances of a frame in one view, shared depth test);
  * per_object: one mpx_raster_render call with one view per object (21 views per frame, each a full-frame buffer) plus
    a torch composite -- the nearest positive depth per pixel, its object's rgb / normals / depth gathered.
Both are checked to agree on every pixel whose nearest depth is unique (ties are where the composite has no rule).
Inputs are resident on the device; CUDA events around `--iters` calls (20x that for one frame) after `--warmup` calls;
medians of `--repeats` windows.  Prints one JSON line with the GPU's name, power limit and max SM clock.
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from megapose6d_b200 import _abi  # noqa: E402
from megapose6d_b200.renderer import BatchRenderer  # noqa: E402
from megapose6d_b200.scene_renderer import Panda3dSceneRenderer  # noqa: E402
from workloads.scenes import ycbv_scene  # noqa: E402


def gpu_info() -> dict:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in q.split(",")]
        return dict(name=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:  # noqa: BLE001
        return dict(name=torch.cuda.get_device_name(0), error=str(e))


def time_ms(fn, warmup: int, iters: int, repeats: int) -> float:
    for _ in range(warmup):
        fn()
    times = []
    for _ in range(repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) / iters)
    return sorted(times)[len(times) // 2]


def run(n_frames: int, warmup: int, iters: int, repeats: int, scene_r, batch_r, labels, TCO, K, h, w) -> dict:
    lib = _abi.lib()
    dev = "cuda"
    n_obj = len(labels)
    n_inst = n_frames * n_obj
    lab = scene_r.mesh_db.label_ids(labels * n_frames, dev)
    T = TCO.to(dev).repeat(n_frames, 1, 1).contiguous()
    Kf = K.to(dev).reshape(1, 3, 3).repeat(n_frames, 1, 1).contiguous()
    Ki = K.to(dev).reshape(1, 3, 3).repeat(n_inst, 1, 1).contiguous()
    offsets = torch.arange(0, n_inst + 1, n_obj, dtype=torch.int32, device=dev)
    rgb = torch.empty(n_frames, 3, h, w, device=dev)
    nrm = torch.empty(n_frames, 3, h, w, device=dev)
    dep = torch.empty(n_frames, 1, h, w, device=dev)
    iid = torch.empty(n_frames, h, w, dtype=torch.int32, device=dev)
    ws = scene_r.workspace(h, w, dev)

    def scene():
        _abi.check(lib.mpx_raster_render_scene(scene_r.mesh_db.handle, n_frames, n_inst, _abi.ptr(offsets), _abi.ptr(lab),
                                               _abi.ptr(T), None, _abi.ptr(Kf), h, w, scene_r.flags, _abi.ptr(rgb),
                                               _abi.ptr(nrm), _abi.ptr(dep), _abi.ptr(iid), _abi.ptr(ws), ws.numel(),
                                               _abi.stream_ptr()))

    lab_b = batch_r.mesh_db.label_ids(labels * n_frames, dev)
    s_rgb = torch.empty(n_inst, 3, h, w, device=dev)
    s_nrm = torch.empty(n_inst, 3, h, w, device=dev)
    s_dep = torch.empty(n_inst, 1, h, w, device=dev)
    ws_b = batch_r.workspace(h, w, dev)
    rows = torch.arange(h, device=dev)[:, None]
    cols = torch.arange(w, device=dev)[None, :]
    frames = torch.arange(n_frames, device=dev)[:, None, None]
    out = {}

    def per_object():
        _abi.check(lib.mpx_raster_render(batch_r.mesh_db.handle, _abi.ptr(lab_b), _abi.ptr(T), _abi.ptr(Ki), n_inst, h, w,
                                         batch_r.flags, _abi.ptr(s_rgb), _abi.ptr(s_nrm), _abi.ptr(s_dep), _abi.ptr(ws_b),
                                         ws_b.numel(), _abi.stream_ptr()))
        d = s_dep.view(n_frames, n_obj, h, w)
        d_eff = torch.where(d > 0, d, torch.full_like(d, float("inf")))
        best = d_eff.min(1)
        k = best.indices
        out["id"] = torch.where(torch.isfinite(best.values), k, torch.full_like(k, -1))
        out["rgb"] = s_rgb.view(n_frames, n_obj, 3, h, w)[frames, k, :, rows, cols].permute(0, 3, 1, 2)
        out["nrm"] = s_nrm.view(n_frames, n_obj, 3, h, w)[frames, k, :, rows, cols].permute(0, 3, 1, 2)
        out["dep"] = torch.where(torch.isfinite(best.values), best.values, torch.zeros_like(best.values))
        out["ties"] = ((d_eff == best.values[:, None]) & torch.isfinite(d_eff)).sum(1) > 1

    ms_scene = time_ms(scene, warmup, iters, repeats)
    ms_obj = time_ms(per_object, warmup, iters, repeats)
    # agreement where the nearest positive depth is unique (a pixel covered only at depth 0 -- beyond the far plane's
    # depth cut -- has no depth for the composite to compare)
    ok = (out["id"] >= 0) & ~out["ties"]
    agree = (iid.long() == out["id"])[ok].float().mean().item()
    same_rgb = (rgb == out["rgb"]).all(1)[ok].float().mean().item()
    same_dep = (dep[:, 0] == out["dep"])[ok].float().mean().item()
    return dict(frames=n_frames, instances=n_inst, scene_ms=ms_scene, per_object_plus_composite_ms=ms_obj,
                speedup=ms_obj / ms_scene, covered_fraction=(iid >= 0).float().mean().item(),
                agree_inst_id=agree, agree_rgb=same_rgb, agree_depth=same_dep)


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--batch", type=int, default=64)
    args = ap.parse_args(argv)
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    sc = ycbv_scene(21)
    ds, K, TCO = sc["ds"], sc["K"][0], sc["TCO_gt"]
    labels = list(sc["labels"])
    h, w = sc["images"].shape[-2:]
    scene_r = Panda3dSceneRenderer(ds)
    batch_r = BatchRenderer(object_dataset=ds)
    res = {"workload": f"ycbv_scene(21): 21 objects x 10k triangles at ground-truth poses, {h}x{w}, rgb+normals+depth",
           "gpu": gpu_info(), "sm_count": _abi.lib().mpx_sm_count(),
           # one frame takes tens of microseconds: 20x the calls per window
           "one_frame": run(1, args.warmup, 20 * args.iters, args.repeats, scene_r, batch_r, labels, TCO, K, h, w),
           f"batch_{args.batch}": run(args.batch, args.warmup, args.iters, args.repeats, scene_r, batch_r,
                                      labels, TCO, K, h, w)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
