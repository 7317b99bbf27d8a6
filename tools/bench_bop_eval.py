"""Time the BOP evaluator on the device against the host oracle (oracle/bop_ref.py, oracle/bop_other_ref.py) on the host
cores, per error type: the bop19 ones (vsd, mssd, mspd) and the toolkit's others (ad, add, adi, cus, proj, re, te, rete).

The split is YCB-V-sized: the 21 procedural objects of `workloads.scenes.ycbv_scene` as models_eval (mm), 640x480 images
with all 21 objects each (written by workloads/bop_split.py through the device scene renderer), estimates = ground truth
perturbed by a few mm.  The host side renders with the C oracle (oracle/raster_ref.c) on all cores.  Prints one JSON line.

    python tools/bench_bop_eval.py [--images 4] [--oracle-images 1]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from megapose6d_b200 import bop_eval  # noqa: E402
from megapose6d_b200.meshes import TriMesh  # noqa: E402
from megapose6d_b200.object_dataset import RigidObject, RigidObjectDataset  # noqa: E402
from megapose6d_b200.scene_renderer import Panda3dSceneRenderer  # noqa: E402
from oracle import bop_other_ref, bop_ref, pipeline_ref  # noqa: E402
from workloads import bop_split  # noqa: E402
from workloads.scenes import ycbv_scene  # noqa: E402

OTHER_TYPES = ("ad", "add", "adi", "cus", "proj", "re", "te", "rete")


def gpu_info() -> dict:
    out = dict(gpu=torch.cuda.get_device_name(0))
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        out["power_limit"], out["max_sm_clock"] = [x.strip() for x in q.split(",")]
    except Exception:  # noqa: BLE001
        pass
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=4)
    ap.add_argument("--oracle-images", type=int, default=1, help="images the (slow) host oracle is timed on")
    args = ap.parse_args()
    ds = ycbv_scene()["ds"]
    models, info = {}, {}
    for k, obj in enumerate(ds.list_objects):
        m = obj.mesh
        v = np.asarray(m.vertices, np.float64) * obj.scale * 1000.0
        models[k + 1] = TriMesh(v, m.faces)
        sub = v[:: max(1, len(v) // 2000)]
        info[k + 1] = dict(diameter=float(np.sqrt(((sub[:, None] - sub[None]) ** 2).sum(-1)).max()))
    info[1]["symmetries_continuous"] = [dict(axis=[0, 0, 1], offset=[0, 0, 0])]  # one object with 314 symmetries
    objs = tuple(range(1, 22))
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

        gt = bop_split.write_split(root, render, n_scenes=1, n_images=args.images, objects=objs, models=models, info=info)
        r = np.random.RandomState(0)
        ests = [dict(scene_id=s, im_id=i, obj_id=o, score=1.0, R=R, t=t + r.normal(0, 3.0, 3), time=0.1)
                for (s, i), inst in gt.items() for o, R, t in inst]
        ev = bop_eval.BopEvaluator(root)
        ests_n = bop_eval.normalize_results(ests)
        sub = [e for e in ests_n if e["im_id"] < args.oracle_images]
        ms = [ev.split.models[o].with_defaults() for o in sorted(ev.split.models)]
        rm = pipeline_ref.RefMeshes([f"obj_{o:06d}" for o in sorted(ev.split.models)], [m.vertices * 1e-3 for m in ms],
                                    [m.vertex_normals for m in ms], [m.vertex_colors for m in ms], [m.faces for m in ms])
        rr = pipeline_ref.RefRenderer(rm)

        def host_render(obj_id, R, t, K, shape):
            T = np.eye(4)
            T[:3, :3], T[:3, 3] = R, np.reshape(t, 3) / 1000.0
            return rr.render([f"obj_{obj_id:06d}"], torch.from_numpy(T).float()[None], torch.from_numpy(K).float()[None],
                             None, tuple(shape), render_depth=True)["depths"][0, 0].numpy()

        split_sub = bop_eval.BopSplit(ev.split.root, ev.split.split, ev.split.models_info, ev.split.models,
                                      [t for t in ev.split.targets if t["im_id"] < args.oracle_images],
                                      ev.split.scene_camera, ev.split.scene_gt, ev.split.scene_gt_info)
        for t in ("vsd", "mssd", "mspd") + OTHER_TYPES:
            ev.errors(ests_n, types=(t,))  # warm-up: mesh upload, module load
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            df = ev.errors(ests_n, types=(t,))
            torch.cuda.synchronize()
            dev_s = time.perf_counter() - t0
            t0 = time.perf_counter()
            if t in OTHER_TYPES:
                rows = bop_other_ref.calc_other_errors(split_sub, sub, host_render, (t,), ev.symmetric_obj_ids)
            else:
                rows = bop_ref.calc_errors(split_sub, sub, host_render, types=(t,))
            host_s = time.perf_counter() - t0
            dev_per_pair = dev_s / len(df)
            host_per_pair = host_s / max(1, len(rows))
            res[t] = dict(pairs=len(df), device_s=round(dev_s, 4), oracle_pairs=len(rows), oracle_s=round(host_s, 3),
                          device_ms_per_pair=round(1e3 * dev_per_pair, 4),
                          oracle_ms_per_pair=round(1e3 * host_per_pair, 3),
                          speedup=round(host_per_pair / dev_per_pair, 1))
    print(json.dumps(dict(metric="bop_eval_per_type", images=args.images, h=480, w=640, objects=21, types=res, **gpu_info())))


if __name__ == "__main__":
    main()
