"""A small synthetic BOP split (models, scenes, ground truth, targets) written to a directory, for the BOP evaluator.

Three models in mm: a bumpy sphere (no symmetry), a box with discrete symmetries (the three 180-degree turns) and a closed
cylinder with a continuous symmetry about z plus the 180-degree turn about x.  Each image holds several objects close
together, so they occlude one another; its test depth is the scene's depth over a back wall, quantised with depth_scale
0.1, with noise and holes.  visib_fract is the share of an instance's pixels in its single render that the scene's
instance map keeps.

The renderer is an argument: render(models, obj_ids_per_view, TCO [n_inst, 4, 4] float32 metres, K [n_views, 3, 3],
(h, w)) -> (depth [n_views, h, w] float32 metres, inst_id [n_views, h, w] int32, -1 = background), e.g. the device's
`mpx_raster_render_scene` or a CPU restatement of it.
"""
from __future__ import annotations

import json
from pathlib import Path
from typing import Callable, Dict, List, Tuple

import numpy as np

from megapose6d_b200.bop_eval import write_depth_png
from megapose6d_b200.meshes import TriMesh

DEPTH_SCALE = 0.1


def _grid_faces(n_rows: int, n_cols: int, wrap: bool) -> List[List[int]]:
    faces = []
    cols = n_cols if wrap else n_cols - 1
    for i in range(n_rows - 1):
        for j in range(cols):
            a, b = i * n_cols + j, i * n_cols + (j + 1) % n_cols
            c, d = a + n_cols, b + n_cols
            faces += [[a, c, b], [b, c, d]]
    return faces


def bumpy_sphere(radius=40.0, n_lat=24, n_lon=32) -> TriMesh:
    th = np.linspace(0.02, np.pi - 0.02, n_lat)[:, None]
    ph = np.linspace(0, 2 * np.pi, n_lon, endpoint=False)[None, :]
    r = radius * (1.0 + 0.15 * np.sin(3 * th) * np.cos(2 * ph + 0.5) + 0.05 * np.cos(5 * ph))
    v = np.stack([r * np.sin(th) * np.cos(ph), r * np.sin(th) * np.sin(ph), r * np.cos(th) * np.ones_like(ph)], -1)
    v = v.reshape(-1, 3)
    faces = _grid_faces(n_lat, n_lon, wrap=True)
    top, bot = len(v), len(v) + 1
    v = np.vstack([v, [[0, 0, radius]], [[0, 0, -radius]]])
    faces += [[top, j, (j + 1) % n_lon] for j in range(n_lon)]
    last = (n_lat - 1) * n_lon
    faces += [[bot, last + (j + 1) % n_lon, last + j] for j in range(n_lon)]
    return TriMesh(v, np.asarray(faces, np.int32))


def box(size=(70.0, 50.0, 30.0), n=6) -> TriMesh:
    """Axis-aligned box centred at the origin, each face an n x n grid (so the evaluation points cover the surface)."""
    verts, faces = [], []
    s = np.asarray(size) / 2
    g = np.linspace(-1, 1, n)
    for axis in range(3):
        for sign in (-1, 1):
            u, w = [a for a in range(3) if a != axis]
            base = len(verts)
            for a in g:
                for b in g:
                    p = np.zeros(3)
                    p[axis], p[u], p[w] = sign * s[axis], a * s[u], b * s[w]
                    verts.append(p)
            for f in _grid_faces(n, n, wrap=False):
                faces.append([base + k for k in (f if sign > 0 else f[::-1])])
    return TriMesh(np.asarray(verts), np.asarray(faces, np.int32))


def cylinder(radius=25.0, height=80.0, n_seg=36, n_rings=5) -> TriMesh:
    ph = np.linspace(0, 2 * np.pi, n_seg, endpoint=False)
    zs = np.linspace(-height / 2, height / 2, n_rings)
    v = np.array([[radius * np.cos(p), radius * np.sin(p), z] for z in zs for p in ph])
    faces = _grid_faces(n_rings, n_seg, wrap=True)
    top, bot = len(v), len(v) + 1
    v = np.vstack([v, [[0, 0, height / 2]], [[0, 0, -height / 2]]])
    last = (n_rings - 1) * n_seg
    faces += [[top, last + j, last + (j + 1) % n_seg] for j in range(n_seg)]
    faces += [[bot, (j + 1) % n_seg, j] for j in range(n_seg)]
    return TriMesh(v, np.asarray(faces, np.int32))


def _flip(axis: int) -> List[float]:
    m = -np.eye(4)
    m[axis, axis] = 1.0
    m[3, 3] = 1.0
    return m.reshape(-1).tolist()


def models_and_info() -> Tuple[Dict[int, TriMesh], Dict[int, dict]]:
    models = {1: bumpy_sphere(), 2: box(), 3: cylinder()}
    info = {}
    for o, m in models.items():
        v = m.vertices
        d = np.sqrt(((v[:, None, :] - v[None, :, :]) ** 2).sum(-1)).max()
        lo, hi = v.min(0), v.max(0)
        info[o] = dict(diameter=float(d), min_x=lo[0], min_y=lo[1], min_z=lo[2], size_x=hi[0] - lo[0],
                       size_y=hi[1] - lo[1], size_z=hi[2] - lo[2])
    info[2]["symmetries_discrete"] = [_flip(0), _flip(1), _flip(2)]
    info[3]["symmetries_continuous"] = [dict(axis=[0, 0, 1], offset=[0, 0, 0])]
    info[3]["symmetries_discrete"] = [_flip(0)]
    return models, {o: {k: (float(v) if not isinstance(v, list) else v) for k, v in i.items()} for o, i in info.items()}


def write_ply(path: Path, m: TriMesh) -> None:
    lines = ["ply", "format ascii 1.0", f"element vertex {len(m.vertices)}", "property float x", "property float y",
             "property float z", f"element face {len(m.faces)}", "property list uchar int vertex_indices", "end_header"]
    lines += [f"{x:.6f} {y:.6f} {z:.6f}" for x, y, z in m.vertices]
    lines += [f"3 {a} {b} {c}" for a, b, c in m.faces]
    Path(path).write_text("\n".join(lines) + "\n")


def random_rotation(rng) -> np.ndarray:
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def write_split(root: Path, render: Callable, n_scenes=2, n_images=2, objects=(1, 2, 3, 2), h=480, w=640, seed=0,
                split="test", model_ids=None, models=None, info=None) -> dict:
    """Writes models_eval/, <split>/<scene>/{scene_camera, scene_gt, scene_gt_info}.json + depth/*.png and
    test_targets_bop19.json under root.  objects: the obj_ids of each image (repeats = several instances).  Returns
    {(scene_id, im_id): [(obj_id, R, t_mm)]}, the ground truth as written."""
    root = Path(root)
    rng = np.random.RandomState(seed)
    if models is None:
        models, info = models_and_info()
    (root / "models_eval").mkdir(parents=True, exist_ok=True)
    for o, m in models.items():
        write_ply(root / "models_eval" / f"obj_{o:06d}.ply", m)
    (root / "models_eval" / "models_info.json").write_text(json.dumps({str(o): i for o, i in info.items()}, indent=1))
    f = 1.1 * w
    K = np.array([[f, 0, w / 2 - 0.5 + 3.25], [0, f, h / 2 - 0.5 - 2.5], [0, 0, 1]])
    targets, gt_all = [], {}
    for scene_id in range(1, n_scenes + 1):
        sdir = root / split / f"{scene_id:06d}"
        (sdir / "depth").mkdir(parents=True, exist_ok=True)
        cams, gts, infos = {}, {}, {}
        for im_id in range(n_images):
            inst = []
            for k, o in enumerate(objects):
                ang = 2 * np.pi * k / len(objects) + rng.uniform(-0.3, 0.3)
                rad = rng.uniform(15, 40)  # close together: the objects occlude one another
                t = np.array([rad * np.cos(ang), rad * np.sin(ang), rng.uniform(450, 700)])
                inst.append((o, random_rotation(rng), t))
            T = np.zeros((len(inst), 4, 4), np.float32)
            for k, (_, R, t) in enumerate(inst):
                T[k, :3, :3], T[k, :3, 3], T[k, 3, 3] = R, t / 1000.0, 1.0
            Kv = np.repeat(K[None].astype(np.float32), 1 + len(inst), 0)
            views = [[o for o, _, _ in inst]] + [[o] for o, _, _ in inst]
            Tv = np.concatenate([T, T])
            depth, iid = render(models, views, Tv, Kv, (h, w))
            depth, iid = np.asarray(depth), np.asarray(iid)
            mm = depth[0].astype(np.float64) * 1000.0
            wall = 1100.0 + 0.05 * (np.arange(w)[None, :] - w / 2)
            mm = np.where(mm > 0, mm, wall)
            mm = mm + rng.normal(0, 1.0, mm.shape)
            raw = np.round(mm / DEPTH_SCALE)
            raw[rng.uniform(size=raw.shape) < 0.02] = 0  # sensor holes
            raw[h // 2 - 20:h // 2 + 20, w // 2 - 10:w // 2 + 30] = 0
            write_depth_png(sdir / "depth" / f"{im_id:06d}.png", np.clip(raw, 0, 65535).astype(np.uint16))
            cams[str(im_id)] = dict(cam_K=K.reshape(-1).tolist(), depth_scale=DEPTH_SCALE)
            gts[str(im_id)] = [dict(obj_id=int(o), cam_R_m2c=R.reshape(-1).tolist(), cam_t_m2c=t.tolist()) for o, R, t in inst]
            infos[str(im_id)] = []
            for k in range(len(inst)):
                n_all = int((depth[1 + k] > 0).sum())
                n_vis = int((iid[0] == k).sum())
                infos[str(im_id)].append(dict(px_count_all=n_all, px_count_visib=n_vis,
                                              visib_fract=n_vis / n_all if n_all else 0.0))
            for o in sorted(set(objects)):
                targets.append(dict(scene_id=scene_id, im_id=im_id, obj_id=int(o), inst_count=int(list(objects).count(o))))
            gt_all[(scene_id, im_id)] = inst
        (sdir / "scene_camera.json").write_text(json.dumps(cams))
        (sdir / "scene_gt.json").write_text(json.dumps(gts))
        (sdir / "scene_gt_info.json").write_text(json.dumps(infos))
    (root / "test_targets_bop19.json").write_text(json.dumps(targets))
    return gt_all
