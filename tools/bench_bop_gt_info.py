"""Time the ground-truth annotation of a BOP split on the device (bop_dataset.compute_gt_info: canvas renders +
mpx_bop_gt_info) against oracle/bop_gt_ref.py on the host, and check that both give the same outputs on one image.

The split is YCB-V-sized: the 21 procedural objects of `workloads.scenes.ycbv_scene` as models (mm), 640x480 images with
all 21 objects each (written by workloads/bop_split.py through the device scene renderer).  Reported: the whole annotate
call with and without the mask PNGs (file writes included), the annotation kernel alone (CUDA events, every gt of the
split in one launch), and the host oracle per gt on the same canvases.  Prints one JSON line with the card's name and
power limit.

    python tools/bench_bop_gt_info.py [--images 8] [--repeats 20]
"""
from __future__ import annotations

import argparse
import json
import shutil
import sys
import tempfile
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from megapose6d_b200 import bop_dataset  # noqa: E402
from megapose6d_b200.bop_eval import load_json, read_depth_png  # noqa: E402
from megapose6d_b200.meshes import TriMesh  # noqa: E402
from megapose6d_b200.object_dataset import RigidObject, RigidObjectDataset  # noqa: E402
from megapose6d_b200.renderer import BatchRenderer  # noqa: E402
from megapose6d_b200.scene_renderer import Panda3dSceneRenderer  # noqa: E402
from oracle import bop_gt_ref  # noqa: E402
from tools.bench_bop_eval import gpu_info  # noqa: E402
from workloads import bop_split  # noqa: E402
from workloads.scenes import ycbv_scene  # noqa: E402


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=20, help="timed launches of the annotation kernel")
    args = ap.parse_args()
    ds = ycbv_scene()["ds"]
    models, info = {}, {}
    for k, obj in enumerate(ds.list_objects):
        v = np.asarray(obj.mesh.vertices, np.float64) * obj.scale * 1000.0
        models[k + 1] = TriMesh(v, obj.mesh.faces)
        sub = v[:: max(1, len(v) // 2000)]
        info[k + 1] = dict(diameter=float(np.sqrt(((sub[:, None] - sub[None]) ** 2).sum(-1)).max()))
    objs = tuple(range(1, 22))
    delta = bop_dataset.GT_INFO_DELTA_DEFAULT
    res = {}
    with tempfile.TemporaryDirectory() as tmp:
        root = Path(tmp)
        cache = {}

        def render(models_, views, TCO, K, resolution):
            if "r" not in cache:
                rds = RigidObjectDataset([RigidObject(label=f"obj_{o:06d}", mesh=models_[o], mesh_units="mm")
                                          for o in sorted(models_)])
                cache["r"] = Panda3dSceneRenderer(rds)
            out = cache["r"].render_scene_tensors([[f"obj_{o:06d}" for o in v] for v in views], torch.from_numpy(TCO),
                                                  torch.from_numpy(K), resolution, render_normals=False)
            return out.depths[:, 0].cpu().numpy(), out.inst_id.cpu().numpy()

        bop_split.write_split(root, render, n_scenes=1, n_images=args.images, objects=objs, models=models, info=info)
        shutil.copytree(root / "models_eval", root / "models")
        sdir = root / "test" / "000001"
        n_gt = 21 * args.images

        for masks in (False, True):
            bop_dataset.compute_gt_info(root, "test", write_masks=masks)  # warm-up: mesh upload, module load
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            bop_dataset.compute_gt_info(root, "test", write_masks=masks)
            torch.cuda.synchronize()
            res["annotate_with_masks_s" if masks else "annotate_s"] = round(time.perf_counter() - t0, 4)

        # the annotation kernel alone, every gt of the split in one launch
        cams = load_json(sdir / "scene_camera.json", keys_to_int=True)
        gts = load_json(sdir / "scene_gt.json", keys_to_int=True)
        ims = sorted(gts)
        rend = BatchRenderer(RigidObjectDataset([RigidObject(label=f"obj_{o:06d}", mesh=models[o], mesh_units="mm")
                                                 for o in sorted(models)]))
        raws = [read_depth_png(sdir / "depth" / f"{i:06d}.png") for i in ims]
        Ks = [np.asarray(cams[i]["cam_K"], np.float64).reshape(3, 3) for i in ims]
        pairs = [(k, g) for k, i in enumerate(ims) for g in gts[i]]
        t0 = time.perf_counter()
        large = bop_dataset.render_canvas_depth(rend, [g["obj_id"] for _, g in pairs], [g["cam_R_m2c"] for _, g in pairs],
                                                [g["cam_t_m2c"] for _, g in pairs], np.stack([Ks[k] for k, _ in pairs]),
                                                480, 640)
        torch.cuda.synchronize()
        res["canvas_render_s"] = round(time.perf_counter() - t0, 4)
        test = torch.from_numpy(np.stack(raws).view(np.int16)).cuda()
        scale = torch.tensor([cams[i]["depth_scale"] for i in ims], dtype=torch.float32, device="cuda")
        K = torch.from_numpy(np.stack(Ks)).cuda()
        idx = torch.tensor([k for k, _ in pairs], dtype=torch.int32, device="cuda")
        out = bop_dataset.gt_info_from_depths(test, scale, K, large, idx, delta)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.repeats):
            bop_dataset.gt_info_from_depths(test, scale, K, large, idx, delta)
        e1.record()
        torch.cuda.synchronize()
        kernel_ms = e0.elapsed_time(e1) / args.repeats
        # the canvases are read whole; the test depth only under the silhouettes, so it is left out: a lower bound
        canvas_bytes = large.numel() * 4
        res.update(kernel_ms=round(kernel_ms, 4), kernel_us_per_gt=round(1e3 * kernel_ms / n_gt, 3),
                   kernel_canvas_GBps=round(canvas_bytes / (kernel_ms * 1e-3) / 1e9, 1))

        # the host oracle on the first image, on the same canvases: same outputs, and its time
        counts, bbox, mask, mask_visib = (t.cpu().numpy() for t in out)
        large_h = large[:21].cpu().numpy()
        t0 = time.perf_counter()
        equal = True
        for g in range(21):
            want, m, mv = bop_gt_ref.annotate(raws[0], cams[ims[0]]["depth_scale"], Ks[0], large_h[g], delta)
            equal &= bop_dataset.gt_info_entry(counts[g], bbox[g]) == want
            equal &= bool(np.array_equal(mask[g].astype(bool), m) and np.array_equal(mask_visib[g].astype(bool), mv))
        host_s = time.perf_counter() - t0
        res.update(oracle_ms_per_gt=round(1e3 * host_s / 21, 2), oracle_equal=bool(equal),
                   annotate_ms_per_gt=round(1e3 * res["annotate_s"] / n_gt, 3))
    print(json.dumps(dict(metric="bop_gt_info", images=args.images, gts=n_gt, h=480, w=640, objects=21, **res,
                          **gpu_info())))


if __name__ == "__main__":
    main()
