"""Ground-truth annotation on the device (csrc/bop_eval.cu: mpx_bop_gt_info): counts, boxes and both masks equal to
oracle/bop_gt_ref.py bit for bit on the device's own renders, refusals before any launch, `annotate` on a written split,
and `prediction_runner --bop-dataset ... --evaluate` end to end."""
from __future__ import annotations

import json
import shutil

import numpy as np
import pytest
import torch

from megapose6d_b200 import _abi, bop_dataset, prediction_runner
from megapose6d_b200.bop_eval import load_json, read_depth_png
from megapose6d_b200.object_dataset import RigidObject, RigidObjectDataset
from megapose6d_b200.renderer import BatchRenderer
from oracle import bop_gt_ref
from tests.test_bop_dataset_host import (CONVERSION_XC, DELTA, MODELS, boundary_case, camera, conversion_case,
                                         gt_poses, scene_test_depth)
from workloads import bop_split

pytestmark = pytest.mark.gpu


def _renderer():
    return BatchRenderer(RigidObjectDataset([RigidObject(label=f"obj_{o:06d}", mesh=MODELS[o], mesh_units="mm")
                                             for o in sorted(MODELS)]))


def _check(counts, bbox, mask, mask_visib, raw, scale, K, large, delta):
    info, m, mv = bop_gt_ref.annotate(raw, scale, K, large, delta)
    assert counts.tolist() == [info["px_count_all"], info["px_count_valid"], info["px_count_visib"]]
    assert bbox.tolist() == info["bbox_obj"] + info["bbox_visib"]
    assert np.array_equal(mask.astype(bool), m) and np.array_equal(mask_visib.astype(bool), mv)
    assert set(np.unique(mask)) <= {0, 1} and set(np.unique(mask_visib)) <= {0, 1}
    return info


def _plain_depth(rend, poses, K, h, w) -> np.ndarray:
    """[n, h, w] depth (metres) of each pose rendered alone at the image's own size and principal point."""
    T = np.zeros((len(poses), 4, 4), np.float32)
    for k, (_, R, t) in enumerate(poses):
        T[k, :3, :3], T[k, :3, 3], T[k, 3, 3] = R, t / 1000.0, 1.0
    out = rend.render([f"obj_{o:06d}" for o, _, _ in poses], torch.from_numpy(T).cuda(),
                      torch.from_numpy(np.stack([K] * len(poses))).float().cuda(), None, (h, w), render_depth=True)
    return out.depths[:, 0].cpu().numpy()


@pytest.mark.parametrize("h,w", [(480, 640), (103, 150)])
def test_device_equals_oracle(h, w):
    """Four images in one launch: two scenes of device renders (in view, occluded, truncated, off the image, behind the
    camera) with holes in the test depth, the hand-made canvas whose distances sit on delta, and the pixel where the
    distance conversions of scene_gt_info and of the masks fall on opposite sides of delta."""
    rend = _renderer()
    K = camera(h, w)
    Kb = K.copy()
    Kb[0, 2], Kb[1, 2] = float(w // 2), float(h // 2)
    images, gts = [], []  # (raw, scale, K); (image index, canvas)
    for k in range(2):
        poses = gt_poses(h, w, seed=k)
        large = bop_dataset.render_canvas_depth(rend, [o for o, _, _ in poses], [R for _, R, _ in poses],
                                                [t for _, _, t in poses], np.stack([K] * len(poses)), h, w).cpu().numpy()
        scale = 0.1 if k == 0 else 0.25
        images.append((scene_test_depth((large[:, h:2 * h, w:2 * w] * 1000).astype(np.float32), h, w, seed=k, scale=scale),
                       scale, K))
        gts += [(k, large[g]) for g in range(len(poses))]
        # the canvas geometry: its image window is the render at the image's own size and principal point, up to the
        # float32 rounding of the shifted projection (a silhouette pixel may fall to the other side, a depth may move in
        # its last bits); a wrong shift or window would move whole silhouettes
        plain = _plain_depth(rend, poses, K, h, w)
        win = large[:, h:2 * h, w:2 * w]
        both = (win > 0) & (plain > 0)
        assert ((win > 0) != (plain > 0)).sum() <= 0.01 * max(1, ((win > 0) | (plain > 0)).sum())
        rel = np.abs(win[both] - plain[both]) / plain[both]
        assert both.sum() > 0 and (rel > 1e-4).sum() <= 1e-3 * both.sum() and np.median(rel) < 1e-6, rel.max()
    braw, blarge = boundary_case(h, w, Kb)
    images.append((braw, 0.1, Kb))
    gts.append((2, blarge))
    b_gt = len(gts) - 1
    craw, cscale, cK, clarge = conversion_case(h, w)
    images.append((craw, cscale, cK))
    gts.append((3, clarge))
    order = [b_gt] + [g for g in range(len(gts)) if g != b_gt]  # gts of different images interleaved
    cuda = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    test = cuda(np.stack([i[0] for i in images]).view(np.int16))
    scale = cuda(np.array([i[1] for i in images], np.float32))
    Ks = cuda(np.stack([i[2] for i in images]))
    large = cuda(np.stack([gts[g][1] for g in order]))
    idx = cuda(np.array([gts[g][0] for g in order], np.int32))
    counts, bbox, mask, mask_visib = (t.cpu().numpy() for t in
                                      bop_dataset.gt_info_from_depths(test, scale, Ks, large, idx, DELTA))
    seen = set()
    for k, g in enumerate(order):
        i, canvas = gts[g]
        info = _check(counts[k], bbox[k], mask[k], mask_visib[k], images[i][0], images[i][1], images[i][2], canvas, DELTA)
        seen |= {"empty"} if info["px_count_all"] == 0 else set()
        seen |= {"invisible"} if info["px_count_all"] > 0 and info["px_count_visib"] == 0 else set()
        seen |= {"truncated"} if info["px_count_visib"] > 0 and min(info["bbox_obj"][:2]) < 0 else set()
        seen |= {"holes"} if info["px_count_valid"] < info["px_count_visib"] else set()
    assert seen == {"empty", "invisible", "truncated", "holes"}, seen
    # the conversion pixel: counted visible by scene_gt_info's conversion, absent from mask_visib
    cy, cx = h // 2, w // 2 + CONVERSION_XC
    assert counts[-1].tolist() == [1, 1, 1] and bbox[-1].tolist() == [cx, cy, 0, 0] * 2
    assert mask[-1, cy, cx] == 1 and mask_visib[-1].sum() == 0
    # the boundary pixel: distance difference exactly delta is visible; one float32 step further is not
    cy, cx = h // 2, w // 2
    assert mask_visib[0, cy, cx] == 1
    c2 = blarge.copy()
    c2[h + cy, w + cx] = np.nextafter(np.float32(0.515), np.float32(1))
    _, _, _, mv2 = bop_dataset.gt_info_from_depths(test, scale, Ks, cuda(c2[None]), cuda(np.array([2], np.int32)), DELTA)
    assert mv2[0, cy, cx].item() == 0
    # launch shape: the same gts one per call give the same result
    c1, b1, _, _ = bop_dataset.gt_info_from_depths(test, scale, Ks, large[3:4].contiguous(), idx[3:4].contiguous(), DELTA,
                                                   masks=False)
    assert c1.cpu().numpy().tolist() == [counts[3].tolist()] and b1.cpu().numpy().tolist() == [bbox[3].tolist()]


def test_out_of_range_image_index():
    h, w = 8, 10
    test = torch.zeros(1, h, w, dtype=torch.int16, device="cuda")
    large = torch.full((2, 3 * h, 3 * w), 0.5, device="cuda")
    K = torch.from_numpy(camera(h, w))[None].cuda()
    counts, bbox, mask, mv = bop_dataset.gt_info_from_depths(test, torch.ones(1, device="cuda"), K, large,
                                                             torch.tensor([1, 0], dtype=torch.int32, device="cuda"), DELTA)
    assert counts[0].tolist() == [-1, -1, -1] and bbox[0].tolist() == [-1] * 8 and int(mask[0].sum()) == 0
    assert counts[1].tolist() == [9 * h * w, 0, h * w] and bbox[1].tolist() == [-w, -h, 3 * w - 1, 3 * h - 1, 0, 0, w - 1, h - 1]


def test_refusals_before_any_launch():
    lib = _abi.lib()
    d = torch.zeros(4096, dtype=torch.float64, device="cuda")
    p = d.data_ptr()
    host = np.zeros(4096)
    hp = host.ctypes.data
    n0 = lib.mpx_launch_count()
    call = lambda **kw: lib.mpx_bop_gt_info(*[kw.get(k, v) for k, v in dict(  # noqa: E731
        n=1, h=4, w=4, test=p, n_img=1, scale=p, K=p, large=p, idx=p, delta=15.0, counts=p, bbox=p, mask=p, mv=p,
        stream=None).items()])
    assert call(n=-1) == -1 and b"n_gt" in lib.mpx_last_error()
    assert call(h=0) == -1 and call(w=-1) == -1 and call(h=20000, w=20000) == -1
    assert call(n_img=0) == -1
    for k in ("test", "scale", "K", "large", "idx", "counts", "bbox"):
        assert call(**{k: None}) == -1, k
        assert call(**{k: hp}) == -1 and b"not device memory" in lib.mpx_last_error(), k
    for k in ("mask", "mv"):
        assert call(**{k: hp}) == -1, k
    assert call(n=0, test=None) == 0
    torch.cuda.synchronize()
    assert lib.mpx_launch_count() == n0
    assert call(mask=None, mv=None) == 0  # optional masks
    torch.cuda.synchronize()
    assert lib.mpx_launch_count() == n0 + 2


# ------------------------------------------------------------------------------------------------------ split, CLI
@pytest.fixture(scope="module")
def split(tmp_path_factory):
    """workloads/bop_split.write_split on the device renderer, without scene_gt_info.json, plus models/ (PLY in mm), rgb/
    and one gt behind the camera (invisible)."""
    from PIL import Image

    from tests.test_gpu_bop_eval import device_scene_renderer

    root = tmp_path_factory.mktemp("bop_gt")
    bop_split.write_split(root, device_scene_renderer(), n_scenes=2, n_images=2, h=480, w=640, seed=4)
    shutil.copytree(root / "models_eval", root / "models")
    # a finer model that no scene shows: the pose models sample 2000 points per mesh (meshes are padded to the largest)
    fine = bop_split.bumpy_sphere(n_lat=48, n_lon=48)
    bop_split.write_ply(root / "models" / "obj_000004.ply", fine)
    info = json.loads((root / "models" / "models_info.json").read_text())
    info["4"] = dict(diameter=80.0)
    (root / "models" / "models_info.json").write_text(json.dumps(info))
    r = np.random.RandomState(0)
    for sdir in sorted((root / "test").iterdir()):
        (sdir / "scene_gt_info.json").unlink()
        (sdir / "rgb").mkdir()
        for p in sorted((sdir / "depth").iterdir()):
            Image.fromarray(r.randint(0, 256, (480, 640, 3)).astype(np.uint8)).save(sdir / "rgb" / p.name)
    gt_path = root / "test" / "000001" / "scene_gt.json"
    gt = json.loads(gt_path.read_text())
    gt["1"].append(dict(obj_id=1, cam_R_m2c=np.eye(3).reshape(-1).tolist(), cam_t_m2c=[0.0, 0.0, -400.0]))
    gt_path.write_text(json.dumps(gt))
    return root


def test_annotate_matches_oracle(split, capsys):
    bop_dataset.main(["annotate", str(split), "--split", "test"])
    assert "annotated 17 ground-truth instance(s)" in capsys.readouterr().out
    from PIL import Image

    rend = _renderer()
    for sdir in sorted((split / "test").iterdir()):
        cams = load_json(sdir / "scene_camera.json", keys_to_int=True)
        gts = load_json(sdir / "scene_gt.json", keys_to_int=True)
        infos = load_json(sdir / "scene_gt_info.json", keys_to_int=True)
        assert sorted(infos) == sorted(gts)
        for im_id, inst in gts.items():
            raw = read_depth_png(sdir / "depth" / f"{im_id:06d}.png")
            h, w = raw.shape
            K = np.asarray(cams[im_id]["cam_K"], np.float64).reshape(3, 3)
            large = bop_dataset.render_canvas_depth(rend, [g["obj_id"] for g in inst], [g["cam_R_m2c"] for g in inst],
                                                    [g["cam_t_m2c"] for g in inst], np.stack([K] * len(inst)), h, w)
            assert len(infos[im_id]) == len(inst)
            for k in range(len(inst)):
                want, m, mv = bop_gt_ref.annotate(raw, cams[im_id]["depth_scale"], K, large[k].cpu().numpy(), DELTA)
                assert infos[im_id][k] == want, (sdir.name, im_id, k)
                for sub, ref in (("mask", m), ("mask_visib", mv)):
                    png = np.asarray(Image.open(sdir / sub / f"{im_id:06d}_{k:06d}.png"))
                    assert png.dtype == np.uint8 and set(np.unique(png)) <= {0, 255}
                    assert np.array_equal(png == 255, ref), (sub, im_id, k)
    assert json.loads((split / "test" / "000001" / "scene_gt_info.json").read_text())["1"][-1]["bbox_visib"] == [-1] * 4


def test_runner_on_the_split_end_to_end(split, tmp_path, capsys):
    from megapose6d_b200 import load_model
    from tests import helpers

    if not (split / "test" / "000001" / "scene_gt_info.json").exists():
        bop_dataset.compute_gt_info(split, "test")
    ckpt = tmp_path / "ckpt"
    load_model.write_run(ckpt, "coarse-rgb-906902141", helpers.make_state_dict(helpers.COARSE_CFG, 5))
    load_model.write_run(ckpt, "refiner-rgb-653307694", helpers.make_state_dict(helpers.REFINER_CFG, 6))
    ds = bop_dataset.keep_bop19(bop_dataset.BOPDataset(split, split="test"))
    n_gt = 0
    for k in range(len(ds)):
        obs = ds[k]
        info = load_json(split / "test" / f"{obs.infos.scene_id:06d}" / "scene_gt_info.json", keys_to_int=True)
        boxes = prediction_runner.SceneObservation.collate_fn([obs])["gt_detections"].bboxes.tolist()
        want = [[x, y, x + bw, y + bh] for x, y, bw, bh in (e["bbox_visib"] for e in info[int(obs.infos.view_id)])]
        assert boxes == want
        n_gt += len(want)
    capsys.readouterr()
    prediction_runner.main(["--bop-dataset", str(split), "--model", "megapose-1.0-RGB", "--models-root", str(ckpt),
                            "--save-dir", str(tmp_path / "out"), "--evaluate"])
    lines = capsys.readouterr().out.strip().splitlines()
    scores = json.loads(lines[-1])
    assert 0.0 <= scores["bop19_average_recall"] <= 1.0 and scores["bop19_average_time_per_image"] > 0
    assert json.loads((tmp_path / "out" / "bop19_scores.json").read_text()) == scores
    rows = prediction_runner.load_bop_results(tmp_path / "out" / "bop_refiner_final.csv")
    assert len(rows) == n_gt == 17
    assert sum(1 for r in rows if (r["scene_id"], r["im_id"]) == (1, 1)) == 5  # the frame with the invisible gt ran
