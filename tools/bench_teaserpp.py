"""Time the TEASER++ depth refiner (megapose6d_b200/teaserpp_refiner.py) on a YCB-V-sized frame.

Scene: the 21 procedural objects of `workloads.scenes.ycbv_scene` at 480x640.  "Measured" depth = the device rasteriser
at the true poses, one render per object composed by the nearest surface, with a seeded fraction of pixels replaced by
uniform depths in [0.2, 1.5] m.  Predictions = the true poses perturbed by a few degrees and millimetres, x1 and x5
hypotheses per object.  Reports CUDA-event times of warm `refine_poses` calls (render included) and of each stage run
alone on the same inputs, the device name and its power limit, as one JSON line.

    python tools/bench_teaserpp.py [--calls 5] [--corrupt 0.1]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import pandas as pd
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from megapose6d_b200 import teaserpp_refiner as tr  # noqa: E402
from megapose6d_b200.renderer import BatchRenderer  # noqa: E402
from megapose6d_b200.tensor_collection import PandasTensorCollection  # noqa: E402
from workloads.scenes import ycbv_scene  # noqa: E402


def gpu_info() -> dict:
    out = dict(gpu=torch.cuda.get_device_name(0))
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        out["power_limit"], out["max_sm_clock"] = [x.strip() for x in q.split(",")]
    except Exception:  # noqa: BLE001
        pass
    return out


def timed(fn, calls: int) -> float:
    """Mean milliseconds per call between CUDA events, after one warm call."""
    fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(calls):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / calls


def perturb(T: torch.Tensor, n_hyp: int, seed: int) -> torch.Tensor:
    rng = np.random.RandomState(seed)
    out = T.repeat_interleave(n_hyp, 0).clone()
    for i in range(len(out)):
        w = rng.randn(3)
        w = torch.from_numpy(w / np.linalg.norm(w) * np.deg2rad(rng.uniform(1, 3))).float()
        Kx = torch.tensor([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
        out[i, :3, :3] = torch.matrix_exp(Kx) @ out[i, :3, :3]
        out[i, :3, 3] += torch.from_numpy(rng.uniform(-0.005, 0.005, 3)).float()
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--corrupt", type=float, default=0.1)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark measures the H100; there is no CPU path"
    sc = ycbv_scene(21)
    ds, K, T_true, labels = sc["ds"], sc["K"].cuda(), sc["TCO_gt"].cuda(), sc["labels"]
    n_obj = len(labels)
    renderer = BatchRenderer(ds)
    refiner = tr.TeaserppRefiner(renderer.mesh_db, renderer)
    h, w = 480, 640
    d = renderer.render(labels, T_true, K.repeat(n_obj, 1, 1), None, (h, w), render_depth=True).depths[:, 0]
    depth = torch.where(d > 0, d, torch.inf).amin(0)
    depth = torch.where(torch.isinf(depth), 0.0, depth)
    g = torch.Generator(device="cuda").manual_seed(0)
    bad = torch.rand(h, w, device="cuda", generator=g) < args.corrupt
    depth = torch.where(bad, 0.2 + 1.3 * torch.rand(h, w, device="cuda", generator=g), depth)[None].contiguous()
    result = dict(metric="TeaserppRefiner.refine_poses ms per call", workload=f"ycbv_scene(21) 480x640, "
                  f"{args.corrupt:.0%} corrupted measured pixels, poses perturbed 1-3 deg / <= 5 mm", **gpu_info())
    for n_hyp in (1, 5):
        T_pred = perturb(T_true.cpu(), n_hyp, 7).cuda()
        n = len(T_pred)
        infos = pd.DataFrame(dict(label=[l for l in labels for _ in range(n_hyp)], batch_im_id=0,
                                  instance_id=np.repeat(np.arange(n_obj), n_hyp)))
        preds = PandasTensorCollection(infos, poses=T_pred)
        total = timed(lambda: refiner.refine_poses(preds, depth=depth, K=K), args.calls)
        # the stages alone on this call's inputs
        Kn = K.repeat(n, 1, 1)
        rend = renderer.render(infos.label.tolist(), T_pred, Kn, None, (h, w), render_depth=True).depths[:, 0]
        vi = torch.zeros(n, dtype=torch.int32, device="cuda")
        src, tgt, count = tr.points(rend, depth, vi, Kn)
        _, ss, st = tr.farthest_point_sampling(src, tgt, count, refiner.n_points)
        m = torch.where(count >= refiner.n_min_points, refiner.n_points, 0).to(torch.int32)
        params = tr.get_solver_params(refiner.noise_bound)
        adj = tr.consistency_graph(ss, st, m, params.noise_bound)
        clique, size, status, nodes = tr.max_clique(adj, m)
        poses = T_pred.clone().contiguous()
        stages = dict(
            render=timed(lambda: renderer.render(infos.label.tolist(), T_pred, Kn, None, (h, w), render_depth=True), args.calls),
            points=timed(lambda: tr.points(rend, depth, vi, Kn), args.calls),
            fps=timed(lambda: tr.farthest_point_sampling(src, tgt, count, refiner.n_points), args.calls),
            graph=timed(lambda: tr.consistency_graph(ss, st, m, params.noise_bound), args.calls),
            clique=timed(lambda: tr.max_clique(adj, m), args.calls),
            solve=timed(lambda: tr.solve(ss, st, m, clique, size, poses.clone(), poses.clone(), params,
                                         refiner.min_num_inliers), args.calls))
        result[f"x{n_hyp}"] = dict(predictions=n, ms_per_call=round(total, 3),
                                   stage_ms={k: round(v, 3) for k, v in stages.items()},
                                   masked_points_max=int(count.max()), clique_sizes=size.tolist(),
                                   clique_nodes_max=int(nodes.max()), budget_exhausted=int((status & 1).sum()))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
