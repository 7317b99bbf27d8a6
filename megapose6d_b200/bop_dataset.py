"""BOP datasets: ground-truth annotation on the device and the reference's readers.

Annotation.  `compute_gt_info` writes what the BOP toolkit's `scripts/calc_gt_info.py` and `scripts/calc_gt_masks.py`
(vendored by the reference under deps/bop_toolkit_challenge) write for a split: `scene_gt_info.json` (pixel counts,
visible fraction, bounding boxes) and the `mask/` and `mask_visib/` PNGs, which official splits ship and custom recordings
in the BOP format lack.  Each ground-truth instance is rendered alone, depth only, by the engine's rasteriser on the
scripts' enlarged canvas (3w x 3h, principal point shifted by (w, h), so that truncated objects keep their whole
silhouette); everything after the render is one launch of the kernel of csrc/bop_eval.cu (include/mpx.h:
mpx_bop_gt_info) for all instances of a chunk.

    python -m megapose6d_b200.bop_dataset annotate <dataset_dir> [--split test] [--delta 15] [--models-dir DIR] [--no-masks]

Readers.  `BOPDataset`, `remap_bop_targets` and `keep_bop19` restate the reference's datasets/bop_scene_dataset.py:55-291
and datasets/datasets_cfg.py:53-62; `BOPObjectDataset` its datasets/bop_object_datasets.py:33-61.  They feed the
frame-level `prediction_runner.PredictionRunner`.
"""
from __future__ import annotations

import argparse
import json
from pathlib import Path
from typing import Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import pandas as pd
import torch

from . import _abi
from .bop_eval import load_json, read_depth_png
from .example import CameraData, ObjectData
from .object_dataset import RigidObject, RigidObjectDataset
from .prediction_runner import ObservationInfos, SceneDataset, SceneObservation

GT_INFO_DELTA_DEFAULT = 15  # mm, the scripts' default


# ------------------------------------------------------------------------------------------------------ device kernel
def gt_info_from_depths(depth_test: torch.Tensor, depth_scale: torch.Tensor, K: torch.Tensor,
                        depth_gt_large: torch.Tensor, img_idx: torch.Tensor, delta: float, masks: bool = True):
    """mpx_bop_gt_info on device tensors: depth_test [I,h,w] int16 (raw uint16 bits), depth_scale [I] float32, K [I,3,3]
    float64, depth_gt_large [G,3h,3w] float32 metres (each gt alone on the enlarged canvas), img_idx [G] int32.
    Returns (counts [G,3] int64 = px_count_all / valid / visib, bbox [G,8] int32 = bbox_obj, bbox_visib as x, y, w, h,
    mask [G,h,w] uint8 0/1 | None, mask_visib [G,h,w] uint8 0/1 | None), on the device, without a host sync."""
    n = int(img_idx.numel())
    dev = depth_gt_large.device
    h, w = depth_test.shape[-2:]
    if n and tuple(depth_gt_large.shape[-2:]) != (3 * h, 3 * w):
        raise ValueError(f"depth_gt_large is {tuple(depth_gt_large.shape)}, the canvas of a {h}x{w} image is {3 * h}x{3 * w}")
    counts = torch.empty(n, 3, dtype=torch.int64, device=dev)
    bbox = torch.empty(n, 8, dtype=torch.int32, device=dev)
    mask = torch.empty(n, h, w, dtype=torch.uint8, device=dev) if masks else None
    mask_visib = torch.empty(n, h, w, dtype=torch.uint8, device=dev) if masks else None
    _abi.check(_abi.lib().mpx_bop_gt_info(
        n, h, w, _abi.ptr(depth_test), depth_test.shape[0], _abi.ptr(depth_scale), _abi.ptr(K), _abi.ptr(depth_gt_large),
        _abi.ptr(img_idx), float(delta), _abi.ptr(counts), _abi.ptr(bbox), _abi.ptr(mask), _abi.ptr(mask_visib),
        _abi.stream_ptr()))
    return counts, bbox, mask, mask_visib


def gt_info_entry(counts: Sequence[int], bbox: Sequence[int]) -> dict:
    """One scene_gt_info.json entry from a row of gt_info_from_depths (visib_fract in float64, 0.0 for an empty silhouette)."""
    n_all, n_valid, n_visib = (int(c) for c in counts)
    return dict(px_count_all=n_all, px_count_valid=n_valid, px_count_visib=n_visib,
                visib_fract=n_visib / float(n_all) if n_all > 0 else 0.0,
                bbox_obj=[int(v) for v in bbox[:4]], bbox_visib=[int(v) for v in bbox[4:]])


# -------------------------------------------------------------------------------------------------------- annotation
def _mesh_renderer(models_dir: Path):
    from .meshes import load_ply
    from .renderer import BatchRenderer

    info = load_json(models_dir / "models_info.json", keys_to_int=True)
    ds = RigidObjectDataset([RigidObject(label=f"obj_{o:06d}", mesh=load_ply(models_dir / f"obj_{o:06d}.ply"), mesh_units="mm")
                             for o in sorted(info)])
    return BatchRenderer(ds)


def render_canvas_depth(renderer, obj_ids: Sequence[int], R: np.ndarray, t_mm: np.ndarray, K: np.ndarray,
                        h: int, w: int) -> torch.Tensor:
    """[n, 3h, 3w] float32 depth in metres: each object alone on the enlarged canvas of an h x w image (cx + w, cy + h)."""
    n = len(obj_ids)
    dev = torch.device("cuda")
    T = np.zeros((n, 4, 4), np.float64)
    T[:, :3, :3] = np.asarray(R, np.float64).reshape(n, 3, 3)
    T[:, :3, 3] = np.asarray(t_mm, np.float64).reshape(n, 3) / 1000.0
    T[:, 3, 3] = 1.0
    Kc = np.asarray(K, np.float64).reshape(n, 3, 3).copy()
    Kc[:, 0, 2] += w
    Kc[:, 1, 2] += h
    H, W = 3 * h, 3 * w
    TCO = torch.from_numpy(T).float().to(dev)
    Kt = torch.from_numpy(Kc).float().to(dev)
    label_idx = renderer.mesh_db.label_ids([f"obj_{o:06d}" for o in obj_ids], dev)
    depth = torch.empty(n, H, W, dtype=torch.float32, device=dev)
    if n:
        ws = renderer.workspace(H, W, dev)
        _abi.check(_abi.lib().mpx_raster_render(renderer.mesh_db.handle, _abi.ptr(label_idx), _abi.ptr(TCO), _abi.ptr(Kt), n,
                                                H, W, renderer.flags, None, None, _abi.ptr(depth), _abi.ptr(ws), ws.numel(),
                                                _abi.stream_ptr()))
    return depth


def _write_mask(path: Path, m: np.ndarray) -> None:
    from PIL import Image

    Image.fromarray((m.astype(np.uint8) * 255)).save(path)


def compute_gt_info(dataset_dir: Union[str, Path], split: str = "test", models_dir: Optional[Union[str, Path]] = None,
                    delta: float = GT_INFO_DELTA_DEFAULT, write_masks: bool = True,
                    max_canvas_bytes: int = 1 << 30) -> Dict[int, Dict[int, List[dict]]]:
    """Writes <split>/<scene>/scene_gt_info.json and, with write_masks, mask/ and mask_visib/ {im_id:06d}_{gt_id:06d}.png
    (0 / 255) for every scene of the split, from scene_camera.json, scene_gt.json, the depth images and the models of
    `models_dir` (default <dataset_dir>/models, PLY in mm).  Instances are rendered and annotated in chunks whose canvases
    take at most `max_canvas_bytes` of device memory.  Returns {scene_id: {im_id: [entry per gt]}}, as written."""
    root = Path(dataset_dir)
    renderer = _mesh_renderer(Path(models_dir) if models_dir is not None else root / "models")
    out: Dict[int, Dict[int, List[dict]]] = {}
    for sdir in sorted(p for p in (root / split).iterdir() if p.is_dir() and p.name.isdigit()):
        scene_camera = load_json(sdir / "scene_camera.json", keys_to_int=True)
        scene_gt = load_json(sdir / "scene_gt.json", keys_to_int=True)
        im_ids = sorted(scene_gt)
        depths = {i: read_depth_png(sdir / "depth" / f"{i:06d}.png") for i in im_ids}
        infos: Dict[int, List[Optional[dict]]] = {i: [None] * len(scene_gt[i]) for i in im_ids}
        if write_masks:
            (sdir / "mask").mkdir(exist_ok=True)
            (sdir / "mask_visib").mkdir(exist_ok=True)
        by_size: Dict[Tuple[int, int], List[int]] = {}
        for i in im_ids:
            by_size.setdefault(depths[i].shape, []).append(i)
        for (h, w), ims in by_size.items():
            per_chunk = max(1, int(max_canvas_bytes // (9 * h * w * 4)))
            gts = [(i, g) for i in ims for g in range(len(scene_gt[i]))]
            for c0 in range(0, len(gts), per_chunk):
                chunk = gts[c0:c0 + per_chunk]
                imgs = list(dict.fromkeys(i for i, _ in chunk))
                im_k = {i: k for k, i in enumerate(imgs)}
                K = np.stack([np.asarray(scene_camera[i]["cam_K"], np.float64).reshape(3, 3) for i in imgs])
                large = render_canvas_depth(renderer, [scene_gt[i][g]["obj_id"] for i, g in chunk],
                                            [scene_gt[i][g]["cam_R_m2c"] for i, g in chunk],
                                            [scene_gt[i][g]["cam_t_m2c"] for i, g in chunk],
                                            np.stack([K[im_k[i]] for i, _ in chunk]), h, w)
                test = torch.from_numpy(np.stack([depths[i] for i in imgs]).view(np.int16)).cuda()
                scale = torch.tensor([scene_camera[i]["depth_scale"] for i in imgs], dtype=torch.float32, device="cuda")
                idx = torch.tensor([im_k[i] for i, _ in chunk], dtype=torch.int32, device="cuda")
                counts, bbox, mask, mask_visib = gt_info_from_depths(test, scale, torch.from_numpy(K).cuda(), large, idx,
                                                                     delta, masks=write_masks)
                counts, bbox = counts.cpu().numpy(), bbox.cpu().numpy()
                if write_masks:
                    mask, mask_visib = mask.cpu().numpy(), mask_visib.cpu().numpy()
                for k, (i, g) in enumerate(chunk):
                    infos[i][g] = gt_info_entry(counts[k], bbox[k])
                    if write_masks:
                        _write_mask(sdir / "mask" / f"{i:06d}_{g:06d}.png", mask[k])
                        _write_mask(sdir / "mask_visib" / f"{i:06d}_{g:06d}.png", mask_visib[k])
        (sdir / "scene_gt_info.json").write_text(json.dumps({str(i): infos[i] for i in im_ids}, indent=2))
        out[int(sdir.name)] = infos
    return out


# ------------------------------------------------------------------------------------------------------------ readers
def remap_bop_targets(targets: pd.DataFrame) -> pd.DataFrame:
    """im_id -> view_id, and label = obj_{obj_id:06d} (bop_scene_dataset.py:55-58)."""
    targets = targets.rename(columns={"im_id": "view_id"})
    targets["label"] = targets["obj_id"].apply(lambda x: f"obj_{x:06d}")
    return targets


def _load_image(path_png: Path) -> np.ndarray:
    from PIL import Image

    path = path_png
    for suffix in (".png", ".jpg", ".tif"):
        path = path_png.with_suffix(suffix)
        if path.exists():
            break
    with Image.open(path) as im:
        return np.array(im)


def _inverse(T: np.ndarray) -> np.ndarray:
    out = np.eye(4)
    out[:3, :3] = T[:3, :3].T
    out[:3, 3] = -T[:3, :3].T.dot(T[:3, 3])
    return out


def _pose(R, t_mm) -> np.ndarray:
    T = np.eye(4)
    T[:3, :3] = np.asarray(R, np.float64).reshape(3, 3)
    T[:3, 3] = np.asarray(t_mm, np.float64) * 0.001
    return T


def _xywh_to_xyxy(b) -> list:
    x, y, w, h = np.array(b).tolist()
    return [x, y, x + w, y + h]


class BOPDataset(SceneDataset):
    """A split of a dataset in the BOP format, frame by frame (datasets/bop_scene_dataset.py:109-291).

    Every frame is (scene_id, view_id) of <ds_dir>/<split>/<scene>/scene_camera.json; its observation holds the rgb image
    (`rgb/` or `gray/`, .png, .jpg or .tif; gray repeated to 3 channels), the camera (K, and TWC from cam_R_w2c / cam_t_w2c
    in mm, else the identity), depth in metres = fp32(raw) * fp32(depth_scale / 1000) when `load_depth`, and one ObjectData
    per ground-truth instance of scene_gt.json: TWO = TWC TCO, label = label_format.format(label=obj_{obj_id:06d}) (or
    str(obj_id) with `use_raw_object_id`), visib_fract, unique_id = n + 1, bbox_modal / bbox_amodal = bbox_visib / bbox_obj
    of scene_gt_info.json as (x1, y1, x2, y2).  Invisible instances are kept, with bbox_visib [-1, -1, -1, -1].  A split
    with ground truth needs scene_gt_info.json (`python -m megapose6d_b200.bop_dataset annotate` writes it).

    Differences from the reference: scenes are indexed in sorted order (the reference follows `iterdir()`, so only the
    frame order can differ); no per-view annotation or index cache is written into the dataset; the `mask_visib/`
    segmentation is not read, as `SceneObservation` carries none."""

    def __init__(self, ds_dir: Union[str, Path], label_format: str = "{label}", split: str = "train",
                 load_depth: bool = False, use_raw_object_id: bool = False):
        self.ds_dir = Path(ds_dir)
        if not self.ds_dir.exists():
            raise FileNotFoundError(f"dataset {self.ds_dir} does not exist")
        self.split = split
        self.base_dir = self.ds_dir / split
        self.label_format = label_format
        self.use_raw_object_id = use_raw_object_id
        self.annotations: Dict[str, dict] = {}
        scene_ids, view_ids = [], []
        for sdir in sorted(p for p in self.base_dir.iterdir() if p.is_dir()):
            ann = {}
            for f in ("scene_camera", "scene_gt_info", "scene_gt"):
                if (sdir / f"{f}.json").exists():
                    ann[f] = json.loads((sdir / f"{f}.json").read_text())
            if "scene_gt" in ann and "scene_gt_info" not in ann:
                raise FileNotFoundError(f"{sdir} has scene_gt.json but no scene_gt_info.json: write it with "
                                        f"`python -m megapose6d_b200.bop_dataset annotate {self.ds_dir} --split {split}`")
            self.annotations[sdir.name] = ann
            for view_id in ann["scene_camera"]:
                scene_ids.append(int(sdir.name))
                view_ids.append(int(view_id))
        super().__init__(pd.DataFrame({"scene_id": scene_ids, "view_id": view_ids}), load_depth)

    def _load_scene_observation(self, image_infos: ObservationInfos) -> SceneObservation:
        view_id = int(image_infos.view_id)
        scene_key = f"{int(image_infos.scene_id):06d}"
        scene_dir = self.base_dir / scene_key
        ann = self.annotations[scene_key]
        cam = ann["scene_camera"][str(view_id)]
        scene_gt = ann.get("scene_gt")
        gt = gt_info = None
        if scene_gt is not None and str(view_id) in scene_gt:
            gt, gt_info = scene_gt[str(view_id)], ann["scene_gt_info"][str(view_id)]
            if len(gt_info) < len(gt):  # the reference fails here too (an IndexError)
                raise ValueError(f"{scene_dir}: view {view_id} has {len(gt)} ground-truth instances in scene_gt.json but "
                                 f"{len(gt_info)} in scene_gt_info.json")

        rgb_dir = scene_dir / "rgb" if (scene_dir / "rgb").exists() else scene_dir / "gray"
        rgb = _load_image(rgb_dir / f"{view_id:06d}.png")
        if rgb.ndim == 2:
            rgb = np.repeat(rgb[..., None], 3, axis=-1)
        rgb = rgb[..., :3]

        TCW = _pose(cam["cam_R_w2c"], cam["cam_t_w2c"]) if "cam_R_w2c" in cam else np.eye(4)
        TWC = _inverse(TCW)
        camera_data = CameraData(K=np.array(cam["cam_K"]).reshape(3, 3), resolution=rgb.shape[:2], TWC=TWC)

        object_datas = []
        for n, (g, info) in enumerate(zip(gt or [], gt_info or [])):
            name = str(g["obj_id"]) if self.use_raw_object_id else f"obj_{int(g['obj_id']):06d}"
            object_datas.append(ObjectData(label=self.label_format.format(label=name),
                                           TWO=TWC.dot(_pose(g["cam_R_m2c"], g["cam_t_m2c"])),
                                           unique_id=n + 1, bbox_modal=_xywh_to_xyxy(info["bbox_visib"]),
                                           bbox_amodal=_xywh_to_xyxy(info["bbox_obj"]), visib_fract=info["visib_fract"]))

        depth = None
        if self.load_depth:
            path = scene_dir / "depth" / f"{view_id:06d}.png"
            if not path.exists():
                path = path.with_suffix(".tif")
            depth = np.asarray(_load_image(path), np.float32) * np.float32(cam["depth_scale"] / 1000)
        return SceneObservation(rgb=rgb, depth=depth, infos=image_infos, object_datas=object_datas,
                                camera_data=camera_data)


def keep_bop19(ds: BOPDataset) -> BOPDataset:
    """Only the frames named by <ds_dir>/test_targets_bop19.json, in the dataset's order (datasets_cfg.py:53-62)."""
    assert ds.frame_index is not None and isinstance(ds, BOPDataset)
    targets = remap_bop_targets(pd.read_json(ds.ds_dir / "test_targets_bop19.json"))
    targets = targets.loc[:, ["scene_id", "view_id"]].drop_duplicates()
    index = ds.frame_index.merge(targets, on=["scene_id", "view_id"]).reset_index(drop=True)
    if len(index) != len(targets):
        raise ValueError(f"{len(targets)} target frames in test_targets_bop19.json, {len(index)} of them in the split")
    ds.frame_index = index
    return ds


class BOPObjectDataset(RigidObjectDataset):
    """The models of a BOP dataset (datasets/bop_object_datasets.py:33-61): <models_dir>/obj_{id:06d}.ply in mm, one object
    per models_info.json entry with its diameter (mm) and symmetries (discrete: 4x4 arrays; continuous: {axis, offset})."""

    def __init__(self, ds_dir: Union[str, Path], label_format: str = "{label}"):
        ds_dir = Path(ds_dir)
        infos = json.loads((ds_dir / "models_info.json").read_text())
        objects = []
        for obj_id, info in infos.items():
            obj_label = f"obj_{int(obj_id):06d}"
            objects.append(RigidObject(
                label=label_format.format(label=obj_label), mesh_path=(ds_dir / obj_label).with_suffix(".ply"),
                mesh_units="mm", mesh_diameter=info["diameter"],
                symmetries_discrete=[np.array(x).reshape(4, 4) for x in info.get("symmetries_discrete", [])],
                symmetries_continuous=[dict(offset=d["offset"], axis=d["axis"]) for d in info.get("symmetries_continuous", [])]))
        self.ds_dir = ds_dir
        super().__init__(objects)


# ---------------------------------------------------------------------------------------------------------------- CLI
def main(argv: Optional[Sequence[str]] = None) -> None:
    ap = argparse.ArgumentParser(description="BOP datasets")
    sub = ap.add_subparsers(dest="command", required=True)
    a = sub.add_parser("annotate", help="write scene_gt_info.json, mask/ and mask_visib/ of a split on the device")
    a.add_argument("dataset_dir", type=Path)
    a.add_argument("--split", default="test")
    a.add_argument("--models-dir", type=Path, default=None, help="default: <dataset_dir>/models")
    a.add_argument("--delta", type=float, default=GT_INFO_DELTA_DEFAULT, help="visibility tolerance in mm")
    a.add_argument("--no-masks", action="store_true", help="write scene_gt_info.json only")
    args = ap.parse_args(argv)
    if not (args.dataset_dir / args.split).is_dir():
        ap.error(f"{args.dataset_dir / args.split} is not a directory")
    out = compute_gt_info(args.dataset_dir, args.split, args.models_dir, args.delta, write_masks=not args.no_masks)
    n = sum(len(v) for s in out.values() for v in s.values())
    print(f"annotated {n} ground-truth instance(s) in {sum(len(s) for s in out.values())} image(s) of "
          f"{len(out)} scene(s) under {args.dataset_dir / args.split}")


if __name__ == "__main__":
    main()
