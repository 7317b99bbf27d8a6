"""BOP datasets on the host: oracle/bop_gt_ref.py against the stored outputs of the BOP toolkit's own functions, the readers
of megapose6d_b200/bop_dataset.py against the stored outputs of the reference's BOPDataset + keep_bop19, and the CLI's
argument errors.

The stored outputs are recorded with MPX_RECORD_REFERENCE=1 and $MEGAPOSE_REFERENCE naming a checkout of the reference
(tests/helpers.py: reference_outputs); the toolkit runs on C-oracle renders and on hand-made canvases, the reference's
reader on the split that `write_reader_split` writes."""
from __future__ import annotations

import importlib.util
import json
import sys
import types
from pathlib import Path

import numpy as np
import pytest
import torch

from megapose6d_b200 import bop_dataset, prediction_runner
from megapose6d_b200.bop_eval import write_depth_png
from oracle import bop_gt_ref, pipeline_ref
from tests import helpers
from workloads import bop_split

MODELS, INFO = bop_split.models_and_info()
DELTA = 15


# ------------------------------------------------------------------------------------------------------ gt info cases
def camera(h: int, w: int) -> np.ndarray:
    f = 1.1 * w
    return np.array([[f, 0, w / 2 - 0.5 + 3.25], [0, f * 1.01, h / 2 - 0.5 - 2.5], [0, 0, 1]])


def gt_poses(h: int, w: int, seed: int = 0):
    """(obj_id, R, t_mm) per gt: in view, truncated by the left and top borders (negative bbox_obj), outside the image but on
    the canvas, behind the camera, and one in front of another (occluded)."""
    r = np.random.RandomState(seed)
    K = camera(h, w)
    z = 520.0

    def at(u, v, zz):  # centre projected at pixel (u, v)
        return np.array([(u - K[0, 2]) * zz / K[0, 0], (v - K[1, 2]) * zz / K[1, 1], zz])

    rot = lambda: bop_split.random_rotation(r)  # noqa: E731
    return [(1, rot(), at(0.5 * w, 0.5 * h, z)), (2, rot(), at(0.6 * w, 0.45 * h, z - 150)),  # occluder of the first
            (3, rot(), at(-0.02 * w, 0.5 * h, z)), (2, rot(), at(0.5 * w, -0.03 * h, z)),  # truncated left / top
            (1, rot(), at(1.45 * w, 0.5 * h, z)),  # outside the image, on the canvas
            (3, rot(), np.array([0.0, 0.0, -400.0])),  # behind the camera
            (2, rot(), at(0.3 * w, 0.7 * h, z + 40))]


def scene_test_depth(window_mm: np.ndarray, h: int, w: int, seed: int = 0, scale: float = 0.1) -> np.ndarray:
    """raw uint16 test depth: the nearest rendered surface over a back wall, noise, holes (random and a block)."""
    r = np.random.RandomState(seed + 1)
    near = np.where(window_mm > 0, window_mm, np.inf).min(0)
    mm = np.where(np.isfinite(near), near, 900.0 + 0.1 * np.arange(w)[None, :]) + r.normal(0, 4.0, (h, w))
    raw = np.round(mm / scale)
    raw[r.uniform(size=(h, w)) < 0.03] = 0
    raw[h // 3:h // 3 + 4, w // 2:w // 2 + 6] = 0
    return np.clip(raw, 0, 65535).astype(np.uint16)


def boundary_case(h: int, w: int, K: np.ndarray, delta: float = DELTA, scale: float = 0.1):
    """A hand-made canvas (metres) and raw test depth whose rendered distance is delta behind the test distance, give or
    take a few float32 steps, over the whole image: visibility flips within a few float32 steps of the rendered depth.  The
    principal point pixel holds an exact difference of delta (X = Y = 0 there).  Both distance conversions agree on every
    pixel here; `conversion_case` holds a pixel where they do not."""
    raw = np.full((h, w), 5000, np.uint16)  # 500 mm
    dt = np.float32(5000) * np.float32(scale)
    ys, xs = np.mgrid[:h, :w]
    ray = np.sqrt(1 + ((xs - K[0, 2]) / K[0, 0]) ** 2 + ((ys - K[1, 2]) / K[1, 1]) ** 2)
    dg_m = ((float(dt) + delta / ray) / 1000.0).astype(np.float32)
    steps = ((xs * 7 + ys * 3) % 9 - 4).astype(np.int32)
    dg_m = (dg_m.view(np.int32) + steps).view(np.float32)
    cx, cy = int(K[0, 2]), int(K[1, 2])
    if cx == K[0, 2] and cy == K[1, 2]:
        dg_m[cy, cx] = np.float32(0.515)  # fp32(515.0 mm) - 500 mm == delta exactly
    large = np.zeros((3 * h, 3 * w), np.float32)
    large[h:2 * h, w:2 * w] = dg_m
    large[h + 2, w - 5:w + 3] = np.float32(0.6)  # a strip that leaves the image on the left
    return raw, large


CONVERSION_XC = 19  # the pixel of conversion_case: (cx + 19, cy)


def conversion_case(h: int, w: int):
    """(raw, scale, K, large_m) with one rendered pixel whose bop19 visibility is true under the distance conversion of
    scene_gt_info (misc.depth_im_to_dist_im_fast) and false under that of the masks (misc.depth_im_to_dist_im).

    Construction: the Pythagorean triple (a, b, c) = (m^2 - n^2, 2mn, m^2 + n^2) with m = 5733, n = 106 has an odd
    hypotenuse c in [2^24, 2^25), a float32 midpoint.  The test depth is d = b 2^-15 mm (raw 4 times scale d / 4, both
    exact) at the pixel 19 columns right of the principal point with fx = 19 b / a, so that X d = a 2^-15 and the exact
    distance is the midpoint c 2^-15.  The two conversions round X d differently, and the larger leg (a / b = 27) carries
    that difference into the float64 distances, which then round to neighbouring float32 values: 16053.9677734375 (fast)
    and 16053.966796875.  The rendered depth (0.5940095782279968 m, found by a search over float32 steps) puts the
    rendered distance at the fast test distance + 15 mm under both conversions: visible by exactly delta in one, by delta
    plus one float32 step in the other."""
    cx, cy = float(w // 2), float(h // 2)
    K = np.array([[0.702839260698782, 0, cx], [0, 1.0, cy], [0, 0, 1]])
    scale = float(np.float32(593.455078125 / 4))
    x, y = w // 2 + CONVERSION_XC, h // 2
    raw = np.zeros((h, w), np.uint16)
    raw[y, x] = 4
    large = np.zeros((3 * h, 3 * w), np.float32)
    large[h + y, w + x] = np.float32(0.5940095782279968)
    return raw, scale, K, large


def c_oracle_canvases(poses, h, w, K):
    """[n, 3h, 3w] float32 metre depth of each gt alone on the enlarged canvas, by the C oracle (oracle/raster_ref.c)."""
    from tests.test_bop_eval_host import ref_meshes

    rr = pipeline_ref.RefRenderer(ref_meshes(MODELS))
    Kc = K.copy()
    Kc[0, 2] += w
    Kc[1, 2] += h
    out = []
    for o, R, t in poses:
        T = np.eye(4)
        T[:3, :3], T[:3, 3] = R, t / 1000.0
        d = rr.render([f"obj_{o:06d}"], torch.from_numpy(T).float()[None], torch.from_numpy(Kc).float()[None], None,
                      (3 * h, 3 * w), render_depth=True)
        out.append(d["depths"][0, 0].numpy())
    return np.stack(out)


def toolkit_outputs(tk, raw, scale, K, large_m, delta):
    """The scripts' loop bodies with the toolkit's own misc / visibility functions (calc_gt_info.py:126-191,
    calc_gt_masks.py:105-127) on the same depth images."""
    h, w = raw.shape
    depth = raw.astype(np.float32)
    depth *= np.float32(scale)
    large = (large_m.astype(np.float32) * np.float32(1000.0)).astype(np.float32)
    depth_gt = large[h:2 * h, w:2 * w]
    dist_gt = tk.misc.depth_im_to_dist_im_fast(depth_gt, K)
    dist_im = tk.misc.depth_im_to_dist_im_fast(depth, K)
    visib = tk.visibility.estimate_visib_mask_gt(dist_im, dist_gt, delta, visib_mode="bop19")
    n_all = int(np.sum(large > 0))
    n_valid = int(np.sum(dist_im[dist_gt > 0] > 0))
    n_visib = int(visib.sum())
    bbox, bbox_visib = [-1] * 4, [-1] * 4
    if n_visib > 0:
        ys, xs = (large > 0).nonzero()
        bbox = [int(v) for v in tk.misc.calc_2d_bbox(xs - w, ys - h, (w, h))]
        ys, xs = visib.nonzero()
        bbox_visib = [int(v) for v in tk.misc.calc_2d_bbox(xs, ys, (w, h))]
    dist_im_s = tk.misc.depth_im_to_dist_im(depth, K)
    dist_gt_s = tk.misc.depth_im_to_dist_im(depth_gt, K)
    mask_visib = tk.visibility.estimate_visib_mask_gt(dist_im_s, dist_gt_s, delta, visib_mode="bop19")
    return dict(counts=np.array([n_all, n_valid, n_visib]), visib_fract=n_visib / float(n_all) if n_all > 0 else 0.0,
                bbox=np.array(bbox + bbox_visib), visib=np.packbits(visib), mask=np.packbits(dist_gt_s > 0),
                mask_visib=np.packbits(mask_visib))


def host_cases(h=48, w=64):
    """[(name, raw, scale, K, large_m)]: C-oracle renders of gt_poses over a scene depth, and the boundary canvas."""
    K = camera(h, w)
    poses = gt_poses(h, w)
    large = c_oracle_canvases(poses, h, w, K)
    raw = scene_test_depth((large[:, h:2 * h, w:2 * w] * 1000).astype(np.float32), h, w)
    cases = [(f"render{k}", raw, 0.1, K, large[k]) for k in range(len(poses))]
    Kb = K.copy()
    Kb[0, 2], Kb[1, 2] = 30.0, 20.0
    braw, blarge = boundary_case(h, w, Kb)
    cases.append(("boundary", braw, 0.1, Kb, blarge))
    cases.append(("conversions",) + conversion_case(h, w))
    return cases


def test_oracle_matches_toolkit():
    cases = host_cases()

    def compute():
        from oracle import bop_toolkit

        tk = bop_toolkit.load()
        out = {}
        for name, raw, scale, K, large in cases:
            out.update({f"{name}/{k}": v for k, v in toolkit_outputs(tk, raw, scale, K, large, DELTA).items()})
        return out

    want = helpers.reference_outputs("bop_gt_info_toolkit", compute)
    seen = set()
    for name, raw, scale, K, large in cases:
        info, mask, mask_visib = bop_gt_ref.annotate(raw, scale, K, large, DELTA)
        assert [info["px_count_all"], info["px_count_valid"], info["px_count_visib"]] == want[f"{name}/counts"].tolist(), name
        assert info["visib_fract"] == float(want[f"{name}/visib_fract"]), name
        assert info["bbox_obj"] + info["bbox_visib"] == want[f"{name}/bbox"].tolist(), name
        h, w = raw.shape
        unpack = lambda k: np.unpackbits(want[f"{name}/{k}"].numpy())[:h * w].reshape(h, w).astype(bool)  # noqa: E731
        assert np.array_equal(mask, unpack("mask")) and np.array_equal(mask_visib, unpack("mask_visib")), name
        visib = unpack("visib")
        assert int(visib.sum()) == info["px_count_visib"]
        if info["px_count_visib"] == 0:
            seen.add("invisible")
        if info["px_count_all"] == 0:
            seen.add("empty")
        if min(info["bbox_obj"][:2]) < 0:
            seen.add("truncated")
        if (visib != mask_visib).any():
            seen.add("conversions differ")
    assert seen == {"invisible", "empty", "truncated", "conversions differ"}, seen
    # the conversion case: visible by scene_gt_info's conversion, not by the masks' one, at its one pixel
    raw, scale, K, large = conversion_case(48, 64)
    info, mask, mask_visib = bop_gt_ref.annotate(raw, scale, K, large, DELTA)
    y, x = 24, 32 + CONVERSION_XC
    assert info["px_count_visib"] == 1 and info["bbox_visib"] == [x, y, 0, 0] and mask[y, x] and not mask_visib.any()
    dt = bop_gt_ref.test_depth_mm(raw, scale)
    dg = bop_gt_ref.render_mm(large)[48:96, 64:128]
    fast = np.float32(bop_gt_ref.dist_image_fast(dg, K)[y, x]) - np.float32(bop_gt_ref.dist_image_fast(dt, K)[y, x])
    slow = np.float32(bop_gt_ref.dist_image(dg, K)[y, x]) - np.float32(bop_gt_ref.dist_image(dt, K)[y, x])
    assert fast == DELTA and slow > DELTA


# ----------------------------------------------------------------------------------------------------------- readers
def write_reader_split(root: Path, h: int = 12, w: int = 16) -> None:
    """Two scenes: scene 1 with rgb PNGs and world-frame cameras (cam_R_w2c / cam_t_w2c), scene 2 with gray JPGs, no world
    frame and an invisible gt; one view without ground truth; targets naming a subset of the views."""
    from PIL import Image

    r = np.random.RandomState(5)
    targets = []
    for scene_id, (kind, n_views) in {1: ("rgb", 3), 2: ("gray", 2)}.items():
        sdir = root / "test" / f"{scene_id:06d}"
        (sdir / kind).mkdir(parents=True)
        (sdir / "depth").mkdir()
        cams, gts, infos = {}, {}, {}
        for v in range(n_views):
            im_id = 10 * v + scene_id
            if kind == "rgb":
                Image.fromarray(r.randint(0, 256, (h, w, 3)).astype(np.uint8)).save(sdir / kind / f"{im_id:06d}.png")
            else:
                Image.fromarray(r.randint(0, 256, (h, w)).astype(np.uint8)).save(sdir / kind / f"{im_id:06d}.jpg", quality=90)
            write_depth_png(sdir / "depth" / f"{im_id:06d}.png", r.randint(0, 9000, (h, w)).astype(np.uint16))
            cam = dict(cam_K=[20.0 + v, 0, w / 2 + 0.25, 0, 21.0, h / 2 - 0.5, 0, 0, 1], depth_scale=0.1 + 0.9 * (scene_id - 1))
            if kind == "rgb":
                cam.update(cam_R_w2c=bop_split.random_rotation(r).reshape(-1).tolist(),
                           cam_t_w2c=r.uniform(-300, 300, 3).tolist())
            cams[str(im_id)] = cam
            if scene_id == 1 and v == 2:
                continue  # a view without ground truth
            gts[str(im_id)], infos[str(im_id)] = [], []
            for k, o in enumerate((1, 3, 2)[:2 + v % 2]):
                gts[str(im_id)].append(dict(obj_id=o, cam_R_m2c=bop_split.random_rotation(r).reshape(-1).tolist(),
                                            cam_t_m2c=[float(x) for x in r.uniform(-50, 50, 2)] + [float(r.uniform(400, 800))]))
                invisible = scene_id == 2 and k == 1
                (sdir / "mask_visib").mkdir(exist_ok=True)  # the reference reads them: its segmentation map
                Image.fromarray((255 * (r.uniform(size=(h, w)) < (0 if invisible else 0.3))).astype(np.uint8)).save(
                    sdir / "mask_visib" / f"{im_id:06d}_{k:06d}.png")
                infos[str(im_id)].append(dict(
                    px_count_all=int(r.randint(1, 200)), px_count_valid=3, px_count_visib=0 if invisible else 7,
                    visib_fract=0.0 if invisible else float(r.uniform(0.1, 1)),
                    bbox_obj=[int(r.randint(-5, 10)), int(r.randint(-5, 8)), int(r.randint(0, 9)), int(r.randint(0, 7))],
                    bbox_visib=[-1, -1, -1, -1] if invisible else [int(r.randint(0, 10)), int(r.randint(0, 8)), 2, 3]))
            if v != 1 or scene_id == 2:
                targets += [dict(scene_id=scene_id, im_id=im_id, obj_id=g["obj_id"], inst_count=1) for g in gts[str(im_id)]]
        # scene_camera in a non-sorted key order: the frame order within a scene is the file's
        (sdir / "scene_camera.json").write_text(json.dumps(dict(reversed(list(cams.items())))))
        (sdir / "scene_gt.json").write_text(json.dumps(gts))
        (sdir / "scene_gt_info.json").write_text(json.dumps(infos))
    (root / "test_targets_bop19.json").write_text(json.dumps(targets))
    mdir = root / "models"
    mdir.mkdir()
    for o, m in MODELS.items():
        bop_split.write_ply(mdir / f"obj_{o:06d}.ply", m)
    (mdir / "models_info.json").write_text(json.dumps({str(o): i for o, i in INFO.items()}))


def _reference_readers():
    """The reference's datasets/bop_scene_dataset.py (BOPDataset, remap_bop_targets) and keep_bop19
    (datasets/datasets_cfg.py:53-62, exec'ed alone: the module imports every dataset of the package), loaded by path on
    top of the reference caller of tests/test_prediction_runner.py.  Substituted: pinocchio's Transform (numpy 4x4:
    R | t, inverse, product), megapose.config (BOP_TOOLKIT_DIR, MEMORY unused), imageio.imread (PIL)."""
    from PIL import Image

    from oracle import bop_toolkit
    from tests.test_prediction_runner import _ref_caller

    R = _ref_caller()
    bop_toolkit.load()
    io = types.ModuleType("imageio")
    io.imread = lambda p: np.asarray(Image.open(p))
    sys.modules["imageio"] = io
    sys.modules.setdefault("png", types.ModuleType("png"))
    cfg = types.ModuleType("megapose.config")
    cfg.BOP_TOOLKIT_DIR, cfg.MEMORY = bop_toolkit.TOOLKIT, None
    sys.modules["megapose.config"] = cfg

    class Transform:
        def __init__(self, *args):
            if len(args) == 1:
                self.matrix = np.asarray(args[0], np.float64)
            else:
                self.matrix = np.eye(4)
                self.matrix[:3, :3], self.matrix[:3, 3] = np.asarray(args[0], np.float64), np.asarray(args[1], np.float64)

        def inverse(self):
            m = np.eye(4)
            m[:3, :3] = self.matrix[:3, :3].T
            m[:3, 3] = -self.matrix[:3, :3].T.dot(self.matrix[:3, 3])
            return Transform(m)

        def __mul__(self, other):
            return Transform(self.matrix.dot(other.matrix))

    old = sys.modules["megapose.lib3d.transform"]
    mod = types.ModuleType("megapose.lib3d.transform")
    mod.Transform = Transform
    sys.modules[mod.__name__] = mod
    try:
        spec = importlib.util.spec_from_file_location("megapose.datasets.bop_scene_dataset",
                                                      R.ns.camera_geometry.__file__.replace("lib3d/camera_geometry.py",
                                                                                            "datasets/bop_scene_dataset.py"))
        bsd = importlib.util.module_from_spec(spec)
        sys.modules[spec.name] = bsd
        spec.loader.exec_module(bsd)
    finally:
        sys.modules["megapose.lib3d.transform"] = old
    src = Path(spec.origin).with_name("datasets_cfg.py").read_text().splitlines()
    a = next(i for i, l in enumerate(src) if l.startswith("def keep_bop19"))
    b = next(i for i, l in enumerate(src) if l.startswith("def make_scene_dataset"))
    import pandas as pd

    ns = dict(pd=pd, BOPDataset=bsd.BOPDataset, remap_bop_targets=bsd.remap_bop_targets, SceneDataset=object)
    exec(compile("\n".join(src[a:b]), str(Path(spec.origin).with_name("datasets_cfg.py")), "exec"), ns)
    return bsd, ns["keep_bop19"]


def _observation_arrays(prefix, obs, twc, two):
    out = {f"{prefix}/rgb": obs.rgb, f"{prefix}/K": np.asarray(obs.camera_data.K, np.float64),
           f"{prefix}/resolution": np.asarray(obs.camera_data.resolution), f"{prefix}/TWC": twc,
           f"{prefix}/depth": obs.depth, f"{prefix}/n_objects": len(obs.object_datas)}
    for n, o in enumerate(obs.object_datas):
        p = f"{prefix}/obj{n}"
        out.update({f"{p}/label": np.asarray(o.label), f"{p}/TWO": two(o), f"{p}/bbox_modal": np.asarray(o.bbox_modal),
                    f"{p}/bbox_amodal": np.asarray(o.bbox_amodal), f"{p}/visib_fract": o.visib_fract,
                    f"{p}/unique_id": o.unique_id})
    return out


def test_readers_match_the_reference(tmp_path):
    write_reader_split(tmp_path)

    def compute():
        bsd, keep = _reference_readers()
        ds = keep(bsd.BOPDataset(tmp_path, label_format="synt-{label}", split="test", load_depth=True))
        out = dict(frames=np.asarray(ds.frame_index[["scene_id", "view_id"]].to_numpy(), np.int64))
        for k in range(len(ds)):
            obs = ds[k]
            out.update(_observation_arrays(f"{obs.infos.scene_id}/{obs.infos.view_id}", obs, obs.camera_data.TWC.matrix,
                                           lambda o: o.TWO.matrix))
        targets = bsd.remap_bop_targets(__import__("pandas").read_json(tmp_path / "test_targets_bop19.json"))
        out["targets"] = np.asarray(targets.to_csv(index=False))
        return out

    want = helpers.reference_outputs("bop_dataset_reader", compute)
    ds = bop_dataset.keep_bop19(bop_dataset.BOPDataset(tmp_path, label_format="synt-{label}", split="test", load_depth=True))
    frames = [tuple(f) for f in ds.frame_index[["scene_id", "view_id"]].to_numpy().tolist()]
    assert sorted(frames) == sorted(tuple(f) for f in want["frames"].tolist())
    assert [f[0] for f in frames] == sorted(f[0] for f in frames)  # scenes in sorted order
    assert frames == [(1, 1), (2, 12), (2, 2)]  # views in scene_camera.json order, the view without gt dropped
    for scene_id, view_id in frames:
        obs = ds[frames.index((scene_id, view_id))]
        p = f"{scene_id}/{view_id}"
        tol = 0 if scene_id == 1 else 2  # scene 2: JPEG
        assert obs.rgb.dtype == np.uint8 and obs.rgb.shape == tuple(want[f"{p}/rgb"].shape)
        assert np.abs(obs.rgb.astype(int) - want[f"{p}/rgb"].numpy().astype(int)).max() <= tol
        assert np.array_equal(np.asarray(obs.camera_data.K, np.float64), want[f"{p}/K"].numpy())
        assert tuple(obs.camera_data.resolution) == tuple(want[f"{p}/resolution"].tolist())
        np.testing.assert_allclose(obs.camera_data.TWC, want[f"{p}/TWC"].numpy(), rtol=0, atol=1e-12)
        assert obs.depth.dtype == np.float32 and np.array_equal(obs.depth, want[f"{p}/depth"].numpy())
        assert len(obs.object_datas) == int(want[f"{p}/n_objects"])
        for n, o in enumerate(obs.object_datas):
            q = f"{p}/obj{n}"
            assert o.label == str(want[f"{q}/label"]) and o.unique_id == int(want[f"{q}/unique_id"]) == n + 1
            np.testing.assert_allclose(o.TWO, want[f"{q}/TWO"].numpy(), rtol=0, atol=1e-12)
            assert list(o.bbox_modal) == want[f"{q}/bbox_modal"].tolist()
            assert list(o.bbox_amodal) == want[f"{q}/bbox_amodal"].tolist()
            assert o.visib_fract == float(want[f"{q}/visib_fract"])
    invisible = ds[frames.index((2, 2))].object_datas[1]
    assert list(invisible.bbox_modal) == [-1, -1, -2, -2] and invisible.visib_fract == 0.0
    targets = bop_dataset.remap_bop_targets(__import__("pandas").read_json(tmp_path / "test_targets_bop19.json"))
    assert str(want["targets"]) == targets.to_csv(index=False)
    # the collated frame feeds the runner: the gt detections are bbox_visib as (x1, y1, x2, y2)
    batch = prediction_runner.SceneObservation.collate_fn([ds[0]])
    assert batch["gt_detections"].bboxes.tolist() == [list(map(float, o.bbox_modal)) for o in ds[0].object_datas]


def test_object_dataset(tmp_path):
    write_reader_split(tmp_path)
    ds = bop_dataset.BOPObjectDataset(tmp_path / "models", label_format="synt-{label}")
    assert [o.label for o in ds] == ["synt-obj_000001", "synt-obj_000002", "synt-obj_000003"]
    for o in ds:
        obj_id = int(o.label[-6:])
        assert o.mesh_path == tmp_path / "models" / f"obj_{obj_id:06d}.ply" and o.mesh_units == "mm" and o.scale == 0.001
        assert o.mesh_diameter == INFO[obj_id]["diameter"]
        assert len(o.symmetries_discrete) == len(INFO[obj_id].get("symmetries_discrete", []))
        assert len(o.symmetries_continuous) == len(INFO[obj_id].get("symmetries_continuous", []))
    assert ds[1].is_symmetric and not ds[0].is_symmetric
    np.testing.assert_array_equal(ds[1].symmetries_discrete[0], np.asarray(INFO[2]["symmetries_discrete"][0]).reshape(4, 4))


def test_reader_without_gt_info_names_the_annotate_command(tmp_path):
    write_reader_split(tmp_path)
    (tmp_path / "test" / "000001" / "scene_gt_info.json").unlink()
    with pytest.raises(FileNotFoundError, match="bop_dataset annotate"):
        bop_dataset.BOPDataset(tmp_path, split="test")
    with pytest.raises(FileNotFoundError):
        bop_dataset.BOPDataset(tmp_path / "missing", split="test")


def test_reader_refuses_gt_info_shorter_than_gt(tmp_path):
    write_reader_split(tmp_path)
    path = tmp_path / "test" / "000002" / "scene_gt_info.json"
    info = json.loads(path.read_text())
    info["2"] = info["2"][:1]
    path.write_text(json.dumps(info))
    ds = bop_dataset.BOPDataset(tmp_path, split="test")
    frames = [tuple(f) for f in ds.frame_index[["scene_id", "view_id"]].to_numpy().tolist()]
    assert len(ds[frames.index((2, 12))].object_datas) == 3
    with pytest.raises(ValueError, match="2 ground-truth instances in scene_gt.json but 1 in scene_gt_info.json"):
        ds[frames.index((2, 2))]


def test_gt_info_entry():
    e = bop_dataset.gt_info_entry([0, 0, 0], [-1] * 8)
    assert e == dict(px_count_all=0, px_count_valid=0, px_count_visib=0, visib_fract=0.0, bbox_obj=[-1] * 4,
                     bbox_visib=[-1] * 4)
    e = bop_dataset.gt_info_entry(np.array([7, 5, 3]), np.array([-2, 1, 4, 5, 0, 1, 2, 3], np.int32))
    assert e["visib_fract"] == 3 / 7.0 and e["bbox_obj"] == [-2, 1, 4, 5] and type(e["bbox_obj"][0]) is int


# --------------------------------------------------------------------------------------------------------------- CLI
@pytest.mark.parametrize("argv", [[], ["frame0", "--bop-dataset", "ds"], ["frame0", "--evaluate"],
                                  ["--bop-dataset", "ds", "--meshes-from", "m"]])
def test_runner_cli_usage_errors(argv, tmp_path, capsys):
    with pytest.raises(SystemExit) as e:
        prediction_runner.main(argv + ["--save-dir", str(tmp_path / "out")])
    assert e.value.code == 2 and "error" in capsys.readouterr().err
    assert not (tmp_path / "out").exists()


def test_annotate_cli_usage_errors(tmp_path, capsys):
    for argv in ([], ["annotate"], ["annotate", str(tmp_path), "--split", "nope"], ["annotate", str(tmp_path), "--delta", "x"]):
        with pytest.raises(SystemExit) as e:
            bop_dataset.main(argv)
        assert e.value.code == 2, argv
    assert "nope" in capsys.readouterr().err
