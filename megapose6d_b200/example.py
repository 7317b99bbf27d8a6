"""Caller side of the reference's example (src/megapose/scripts/run_inference_on_example.py:36-148, README.md:200-260):
read an example directory, build the object dataset and the detections, run a named model, write the poses.

Directory layout (the reference's): `image_rgb.png` (+ `image_depth.png`, uint16 millimetres), `camera_data.json`
(`{"K": 3x3, "resolution": [h, w]}`), `inputs/object_data.json` (`[{"label", "bbox_modal": [x1, y1, x2, y2]}, ...]`),
`meshes/<label>/<file>.obj|.ply` in millimetres; output `outputs/object_data.json` with `TWO = [quaternion xyzw,
translation]` per object (datasets/scene_dataset.py:67-120).  The JSON structures are restated here with numpy only (the
reference wraps them in pinocchio `Transform`s).

    python -m megapose6d_b200.example <example_dir> --model megapose-1.0-RGB-multi-hypothesis [--vis-outputs]

`--vis-outputs` then renders every estimated pose into the image (one scene, run_inference_on_example.py:151-193) and
writes visualizations/{mesh_overlay, contour_overlay, all_results}.png; `--vis-only` does only that, from an existing
outputs/object_data.json.
"""
from __future__ import annotations

import argparse
import json
from dataclasses import dataclass
from pathlib import Path
from typing import List, Optional, Tuple

import numpy as np
import pandas as pd
import torch

from .load_model import NAMED_MODELS, load_named_model
from .object_dataset import RigidObject, RigidObjectDataset
from .tensor_collection import PandasTensorCollection
from .types import DetectionsType, ObservationTensor, PoseEstimatesType


@dataclass
class CameraData:
    """datasets/scene_dataset.py:122-180.  Transforms are 4x4 float64 matrices here; on disk `[quaternion xyzw, translation]`."""
    K: Optional[np.ndarray] = None
    resolution: Optional[Tuple[int, int]] = None
    TWC: Optional[np.ndarray] = None
    camera_id: Optional[str] = None
    TWC_init: Optional[np.ndarray] = None

    @staticmethod
    def from_json(text: str) -> "CameraData":
        d = json.loads(text)
        assert isinstance(d, dict), "camera_data.json must hold one object"
        out = CameraData()
        for key in ("TWC", "TWC_init"):
            if key in d:
                quat, trans = d[key]
                setattr(out, key, transform_from_quat_trans(quat, trans))
        if "camera_id" in d:
            out.camera_id = d["camera_id"]
        if "K" in d:
            out.K = np.asarray(d["K"], dtype=np.float64)
            assert out.K.shape == (3, 3), "camera_data.json: K must be 3x3"
        if "resolution" in d:
            h, w = d["resolution"]
            assert isinstance(h, int) and isinstance(w, int), "camera_data.json: resolution must be two integers [h, w]"
            out.resolution = (h, w)
        return out

    def to_json(self) -> str:
        d: dict = {}
        for key in ("TWC", "TWC_init"):
            T = getattr(self, key)
            if T is not None:
                d[key] = transform_to_list(T)
        if self.K is not None:
            d["K"] = np.asarray(self.K).tolist()
        if self.camera_id is not None:
            d["camera_id"] = self.camera_id
        if self.resolution is not None:
            d["resolution"] = [int(self.resolution[0]), int(self.resolution[1])]
        return json.dumps(d)


@dataclass
class ObjectData:
    """datasets/scene_dataset.py:71-120: label + boxes in, label + TWO out."""
    label: str
    TWO: Optional[np.ndarray] = None  # 4x4
    unique_id: Optional[int] = None
    bbox_amodal: Optional[np.ndarray] = None  # [xmin, ymin, xmax, ymax]
    bbox_modal: Optional[np.ndarray] = None
    visib_fract: Optional[float] = None
    TWO_init: Optional[np.ndarray] = None

    @staticmethod
    def from_json(d: dict) -> "ObjectData":
        assert isinstance(d, dict) and isinstance(d["label"], str)
        out = ObjectData(label=d["label"])
        for key in ("TWO", "TWO_init"):
            if key in d:
                quat, trans = d[key]
                setattr(out, key, transform_from_quat_trans(quat, trans))
        for key in ("unique_id", "visib_fract"):
            if key in d:
                setattr(out, key, d[key])
        for key in ("bbox_amodal", "bbox_modal"):
            if key in d:
                setattr(out, key, np.asarray(d[key], dtype=np.float64))
        return out

    def to_json(self) -> dict:
        d: dict = dict(label=self.label)
        for key in ("TWO", "TWO_init"):
            T = getattr(self, key)
            if T is not None:
                d[key] = transform_to_list(T)
        for key in ("bbox_amodal", "bbox_modal"):
            if getattr(self, key) is not None:
                d[key] = np.asarray(getattr(self, key)).tolist()
        for key in ("visib_fract", "unique_id"):
            if getattr(self, key) is not None:
                d[key] = getattr(self, key)
        return d


def transform_to_list(T: np.ndarray) -> list:
    """4x4 -> [quaternion xyzw, translation] (datasets/scene_dataset.py:67-68)."""
    T = np.asarray(T, dtype=np.float64)
    return [rotmat_to_quat_xyzw(T[:3, :3]).tolist(), T[:3, 3].tolist()]


def rotmat_to_quat_xyzw(R: np.ndarray) -> np.ndarray:
    """Unit quaternion (x, y, z, w), w >= 0 branch-stable (Shepperd)."""
    R = np.asarray(R, dtype=np.float64)
    t = np.trace(R)
    if t > 0:
        s = np.sqrt(t + 1.0) * 2
        q = np.array([(R[2, 1] - R[1, 2]) / s, (R[0, 2] - R[2, 0]) / s, (R[1, 0] - R[0, 1]) / s, 0.25 * s])
    else:
        i = int(np.argmax(np.diag(R)))
        j, k = (i + 1) % 3, (i + 2) % 3
        s = np.sqrt(1.0 + R[i, i] - R[j, j] - R[k, k]) * 2
        q = np.zeros(4)
        q[i] = 0.25 * s
        q[j] = (R[j, i] + R[i, j]) / s
        q[k] = (R[k, i] + R[i, k]) / s
        q[3] = (R[k, j] - R[j, k]) / s
    return q / np.linalg.norm(q)


def transform_from_quat_trans(quat_xyzw, trans) -> np.ndarray:
    x, y, z, w = (float(v) for v in quat_xyzw)
    n = np.sqrt(x * x + y * y + z * z + w * w)
    x, y, z, w = x / n, y / n, z / n, w / n
    T = np.eye(4)
    T[:3, :3] = [[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                 [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                 [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]]
    T[:3, 3] = np.asarray(trans, dtype=np.float64)
    return T


def load_observation(example_dir: Path, load_depth: bool = False) -> Tuple[np.ndarray, Optional[np.ndarray], CameraData]:
    """run_inference_on_example.py:36-50: rgb uint8 [h,w,3], depth float32 metres [h,w] (optional), camera."""
    from PIL import Image

    example_dir = Path(example_dir)
    camera = CameraData.from_json((example_dir / "camera_data.json").read_text())
    with Image.open(example_dir / "image_rgb.png") as im:
        rgb = np.asarray(im.convert("RGB"), dtype=np.uint8)
    assert camera.K is not None and camera.resolution is not None, "camera_data.json needs K and resolution"
    assert rgb.shape[:2] == camera.resolution, f"image {rgb.shape[:2]} != camera resolution {camera.resolution}"
    depth = None
    if load_depth:
        with Image.open(example_dir / "image_depth.png") as im:
            depth = np.asarray(im, dtype=np.float32) / 1000.0
        assert depth.shape[:2] == camera.resolution
    return rgb, depth, camera


def load_observation_tensor(example_dir: Path, load_depth: bool = False) -> ObservationTensor:
    rgb, depth, camera = load_observation(example_dir, load_depth)
    return ObservationTensor.from_numpy(rgb, depth, camera.K)


def load_object_data(path: Path) -> List[ObjectData]:
    return [ObjectData.from_json(d) for d in json.loads(Path(path).read_text())]


def make_detections_from_object_data(object_data: List[ObjectData]) -> DetectionsType:
    """inference/utils.py:214-225."""
    infos = pd.DataFrame(dict(label=[d.label for d in object_data], batch_im_id=0, instance_id=np.arange(len(object_data))))
    bboxes = torch.as_tensor(np.stack([d.bbox_modal for d in object_data]))
    return PandasTensorCollection(infos=infos, bboxes=bboxes)


def load_detections(example_dir: Path) -> DetectionsType:
    return make_detections_from_object_data(load_object_data(Path(example_dir) / "inputs" / "object_data.json")).cuda()


def make_object_dataset(example_dir: Path, mesh_units: str = "mm") -> RigidObjectDataset:
    """One object per directory under meshes/, exactly one .obj or .ply in each (run_inference_on_example.py:76-91)."""
    objects = []
    for object_dir in sorted(p for p in (Path(example_dir) / "meshes").iterdir() if p.is_dir()):
        files = [f for f in sorted(object_dir.iterdir()) if f.suffix.lower() in (".obj", ".ply")]
        assert len(files) == 1, f"expected exactly one .obj / .ply in {object_dir}, found {len(files)}"
        objects.append(RigidObject(label=object_dir.name, mesh_path=files[0], mesh_units=mesh_units))
    assert objects, f"no meshes under {Path(example_dir) / 'meshes'}"
    return RigidObjectDataset(objects)


def save_predictions(example_dir: Path, pose_estimates: PoseEstimatesType) -> Path:
    labels = pose_estimates.infos["label"].tolist()
    poses = pose_estimates.poses.detach().cpu().double().numpy()
    data = [ObjectData(label=l, TWO=T).to_json() for l, T in zip(labels, poses)]
    out = Path(example_dir) / "outputs" / "object_data.json"
    out.parent.mkdir(exist_ok=True)
    out.write_text(json.dumps(data))
    return out


def run_inference(example_dir: Path, model_name: str, models_root: Optional[Path] = None) -> PoseEstimatesType:
    """run_inference_on_example.py:126-148.  `models_root` overrides $MEGAPOSE_DATA_DIR/megapose-models."""
    info = NAMED_MODELS[model_name]
    observation = load_observation_tensor(example_dir, load_depth=info["requires_depth"]).cuda()
    detections = load_detections(example_dir)
    object_dataset = make_object_dataset(example_dir)
    pose_estimator = load_named_model(model_name, object_dataset, models_root=models_root).cuda()
    output, _ = pose_estimator.run_inference_pipeline(observation, detections=detections, **info["inference_parameters"])
    save_predictions(example_dir, output)
    return output


def get_mask_from_rgb(img: np.ndarray) -> np.ndarray:
    """visualization/utils.py:47-53: a pixel belongs to the rendering when any channel is > 0."""
    return (np.asarray(img) > 0).any(axis=-1)


def make_mesh_overlay(rgb_input: np.ndarray, rgb_rendered: np.ndarray) -> np.ndarray:
    """BokehPlotter.plot_overlay (visualization/bokeh_plotter.py:106-130): the image lightened where nothing is rendered,
    the rendering lightened where it is."""
    assert rgb_input.dtype == np.uint8 and rgb_rendered.dtype == np.uint8
    mask = get_mask_from_rgb(rgb_rendered)
    overlay = np.zeros_like(rgb_input).astype(np.float32)
    overlay[~mask] = rgb_input[~mask] * 0.6 + 255 * 0.4
    overlay[mask] = rgb_rendered[mask] * 0.8 + 255 * 0.2
    return overlay.astype(np.uint8)


def _box3(mask: np.ndarray, op) -> np.ndarray:
    """3x3 box max (op = np.logical_or) or min (np.logical_and) of a boolean image, edges replicated."""
    p = np.pad(mask, 1, mode="edge")
    h, w = mask.shape
    out = p[1:h + 1, 1:w + 1].copy()
    for di in range(3):
        for dj in range(3):
            out = op(out, p[di:di + h, dj:dj + w])
    return out


def make_contour_overlay(img: np.ndarray, render: np.ndarray, color: Tuple[int, int, int] = (0, 255, 0),
                         dilate_iterations: int = 1) -> dict:
    """The silhouette of the rendering drawn on the image (what visualization/utils.py:55-83 draws): the mask's boundary
    pixels -- in the mask, with a 3x3 neighbour outside it -- dilated `dilate_iterations` times with a 3x3 box and
    painted `color`.  The boundary is computed directly, not with an edge detector."""
    mask = get_mask_from_rgb(render)
    contour = mask & ~_box3(mask, np.logical_and)
    for _ in range(dilate_iterations):
        contour = _box3(contour, np.logical_or)
    out = np.copy(img)
    out[contour] = color
    return dict(img=out, mask=mask, contour=contour)


def render_object_data(example_dir: Path, object_datas: List[ObjectData], resolution: Tuple[int, int],
                       K: np.ndarray) -> np.ndarray:
    """All estimated poses in one scene seen by the image's camera (TWC = I), white ambient light: rgb (h, w, 3) uint8."""
    from .renderer import Panda3dLightData
    from .scene_renderer import Panda3dCameraData, Panda3dObjectData, Panda3dSceneRenderer

    renderer = Panda3dSceneRenderer(make_object_dataset(example_dir))
    camera = Panda3dCameraData(K=K, resolution=resolution, TWC=np.eye(4))
    objects = [Panda3dObjectData(label=o.label, TWO=o.TWO) for o in object_datas]
    lights = [Panda3dLightData(light_type="ambient", color=(1.0, 1.0, 1.0, 1.0))]
    return renderer.render_scene(objects, [camera], lights, render_depth=False, render_binary_mask=False,
                                 render_normals=False, copy_arrays=True)[0].rgb


def make_output_visualization(example_dir: Path) -> Path:
    """run_inference_on_example.py:151-193: visualizations/{mesh_overlay, contour_overlay, all_results}.png from
    outputs/object_data.json."""
    from PIL import Image

    example_dir = Path(example_dir)
    rgb, _, camera = load_observation(example_dir, load_depth=False)
    object_datas = load_object_data(example_dir / "outputs" / "object_data.json")
    rendered = render_object_data(example_dir, object_datas, camera.resolution, camera.K)
    mesh_overlay = make_mesh_overlay(rgb, rendered)
    contour_overlay = make_contour_overlay(rgb, rendered, color=(0, 255, 0), dilate_iterations=1)["img"]
    vis_dir = example_dir / "visualizations"
    vis_dir.mkdir(exist_ok=True)
    Image.fromarray(mesh_overlay).save(vis_dir / "mesh_overlay.png")
    Image.fromarray(contour_overlay).save(vis_dir / "contour_overlay.png")
    Image.fromarray(np.concatenate([rgb, contour_overlay, mesh_overlay], axis=1)).save(vis_dir / "all_results.png")
    return vis_dir


def main(argv: Optional[List[str]] = None) -> None:
    parser = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    parser.add_argument("example_dir", type=Path)
    parser.add_argument("--model", type=str, default="megapose-1.0-RGB-multi-hypothesis", choices=sorted(NAMED_MODELS))
    parser.add_argument("--models-root", type=Path, default=None, help="directory holding <run_id>/{config.yaml,checkpoint.pth.tar}")
    parser.add_argument("--vis-outputs", action="store_true",
                        help="also render the estimated poses and write visualizations/*.png")
    parser.add_argument("--vis-only", action="store_true",
                        help="only visualise an existing outputs/object_data.json (no inference)")
    args = parser.parse_args(argv)
    if not args.vis_only:
        out = run_inference(args.example_dir, args.model, args.models_root)
        print(f"wrote {len(out)} pose(s) to {args.example_dir / 'outputs' / 'object_data.json'}")
    if args.vis_outputs or args.vis_only:
        print(f"wrote visualizations to {make_output_visualization(args.example_dir)}")


if __name__ == "__main__":
    main()
