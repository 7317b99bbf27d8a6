"""Scene renderer: several posed objects per camera on the CUDA rasteriser, with one shared depth test.

Mirror of Panda3dSceneRenderer (src/megapose/panda3d_renderer/panda3d_scene_renderer.py:139-358) and its types
(panda3d_renderer/types.py:43-125): `render_scene(object_datas, camera_datas, light_datas, ...)` returns one
CameraRenderingData(rgb, normals, depth, binary_mask) per camera as host arrays.  Every camera sees every object; all
cameras of one resolution are drawn by one mpx_raster_render_scene call.  `render_scene_tensors` is the device-side form,
which also returns the per-pixel instance map.

What the engine draws is what the batch renderer draws (include/mpx.h: mpx_raster_render_scene): white ambient light,
near / far planes 0.1 / 10 m, one sample per pixel, 8-bit colour and normal levels.  What the reference configures beyond
that is refused with NotImplementedError rather than drawn differently.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Sequence, Set, Tuple

import numpy as np
import torch

from . import _abi
from .meshes import BatchedMeshes, MeshDataBase
from .object_dataset import RigidObjectDataset

# renderer.py re-exports this module, so the flag values are restated rather than imported from it
RASTER_QUANTIZE8 = 1
RASTER_NORMALS_GL = 2
MAX_INSTANCES_PER_VIEW = 1024


@dataclass
class Panda3dObjectData:
    """types.py:43-56.  TWO: object -> world, 4x4 float64; color (r, g, b, a) replaces the object's albedo."""

    label: str
    TWO: np.ndarray = None
    color: Optional[Tuple[float, float, float, float]] = None
    material: Optional[object] = None
    remove_mesh_material: bool = False
    scale: float = 1
    positioning_function: Optional[object] = None

    def __post_init__(self):
        self.TWO = np.eye(4) if self.TWO is None else np.asarray(self.TWO, dtype=np.float64)


@dataclass
class Panda3dCameraData:
    """types.py:58-101.  K 3x3; resolution (h, w); TWC: camera -> world, 4x4 float64."""

    K: np.ndarray
    resolution: Tuple[int, int]
    TWC: np.ndarray = None
    z_near: float = 0.1
    z_far: float = 10
    node_name: str = "camera"
    positioning_function: Optional[object] = None

    def __post_init__(self):
        self.TWC = np.eye(4) if self.TWC is None else np.asarray(self.TWC, dtype=np.float64)


@dataclass
class CameraRenderingData:
    """types.py:104-125: rgb (h, w, 3) uint8; normals (h, w, 3) uint8; depth (h, w, 1) float32 metres; binary_mask (h, w)
    bool.  Fields that were not asked for are None."""

    rgb: np.ndarray
    normals: Optional[np.ndarray] = None
    depth: Optional[np.ndarray] = None
    binary_mask: Optional[np.ndarray] = None


@dataclass
class SceneRenderOutput:
    """Device-side result of render_scene_tensors: rgbs / normals [V,3,h,w] in [0,1] (8-bit levels), depths [V,1,h,w]
    metres, inst_id [V,h,w] int32 (index of the instance within its view, -1 = background)."""

    rgbs: torch.Tensor
    normals: Optional[torch.Tensor]
    depths: Optional[torch.Tensor]
    inst_id: torch.Tensor


def compose_TCO(TWC: np.ndarray, TWO: np.ndarray, scale: float = 1.0) -> np.ndarray:
    """Pose of an object in a camera's frame: inv(TWC) @ TWO @ diag(scale, scale, scale, 1), in float64, cast to float32
    once."""
    S = np.diag([float(scale)] * 3 + [1.0])
    return (np.linalg.inv(np.asarray(TWC, np.float64)) @ np.asarray(TWO, np.float64) @ S).astype(np.float32)


def to_uint8(x: torch.Tensor) -> torch.Tensor:
    """8-bit levels k / 255 back to k: round(255 x) is exact for every level."""
    return (x * 255.0).round().to(torch.uint8)


def check_scene_inputs(object_datas: Sequence[Panda3dObjectData], camera_datas: Sequence[Panda3dCameraData],
                       light_datas) -> None:
    """What the engine does not draw raises NotImplementedError (messages in the style of BatchRenderer._light_flags)."""
    lights = list(light_datas or [])
    if len(lights) != 1 or getattr(lights[0], "light_type", None) != "ambient" \
            or getattr(lights[0], "positioning_function", None) is not None \
            or tuple(float(c) for c in tuple(lights[0].color)[:3]) != (1.0, 1.0, 1.0):
        raise NotImplementedError("scenes are rendered under one white ambient light only "
                                  "(point lights and coloured light are not implemented for scenes)")
    for obj in object_datas:
        if obj.positioning_function is not None:
            raise NotImplementedError("object positioning functions are not implemented: give the pose as TWO")
        if obj.material is not None:
            raise NotImplementedError("object materials are not implemented: the mesh's own colours / texture are drawn")
        if obj.remove_mesh_material:
            raise NotImplementedError("remove_mesh_material=True is not implemented")
        if obj.color is not None and len(obj.color) > 3 and float(obj.color[3]) < 1.0:
            raise NotImplementedError("object colours with alpha < 1 (transparency) are not implemented")
    for cam in camera_datas:
        if cam.positioning_function is not None:
            raise NotImplementedError("camera positioning functions are not implemented: give the pose as TWC")
        if float(cam.z_near) != 0.1 or float(cam.z_far) != 10.0:
            raise NotImplementedError("near / far planes other than 0.1 / 10 m are not implemented")


class Panda3dSceneRenderer:
    def __init__(self, asset_dataset: Optional[RigidObjectDataset] = None, preload_labels: Set[str] = set(),
                 debug: bool = False, verbose: bool = False, mesh_db: Optional[BatchedMeshes] = None,
                 normals_gl_axes: bool = False):
        """`preload_labels`, `debug`, `verbose` are accepted for the reference's signature: every mesh of the dataset is
        uploaded once, as BatchRenderer does."""
        if mesh_db is None:
            assert asset_dataset is not None
            mesh_db = MeshDataBase.from_object_ds(asset_dataset).batched()
        self.mesh_db = mesh_db
        self.flags = RASTER_QUANTIZE8 | (RASTER_NORMALS_GL if normals_gl_axes else 0)
        self._workspace: Optional[torch.Tensor] = None

    def workspace(self, h: int, w: int, device) -> torch.Tensor:
        need = _abi.lib().mpx_raster_workspace_bytes(h, w)
        if self._workspace is None or self._workspace.numel() < need or self._workspace.device != torch.device(device):
            self._workspace = torch.empty(need, dtype=torch.uint8, device=device)
        return self._workspace

    def render_scene_tensors(self, labels_per_view: Sequence[Sequence[str]], TCO_per_instance: torch.Tensor,
                             K: torch.Tensor, resolution: Tuple[int, int], render_depth: bool = True,
                             render_normals: bool = True, colors: Optional[torch.Tensor] = None,
                             device="cuda") -> SceneRenderOutput:
        """View v draws the instances labels_per_view[v]; TCO_per_instance [n_inst,4,4] lists their poses in the views'
        camera frames, view after view; K [n_views,3,3]; colors [n_inst,3] (a negative first component: no override)."""
        n_views = len(labels_per_view)
        counts = [len(v) for v in labels_per_view]
        if any(c > MAX_INSTANCES_PER_VIEW for c in counts):
            raise ValueError(f"at most {MAX_INSTANCES_PER_VIEW} instances per view")
        n_inst = sum(counts)
        h, w = resolution
        dev = torch.device(device)
        TCO = torch.as_tensor(TCO_per_instance).detach().to(dev, torch.float32).reshape(n_inst, 4, 4).contiguous()
        K = torch.as_tensor(K).detach().to(dev, torch.float32).reshape(n_views, 3, 3).contiguous()
        offsets = torch.tensor(np.cumsum([0] + counts), dtype=torch.int32, device=dev)
        labels = [l for v in labels_per_view for l in v]
        label_idx = self.mesh_db.label_ids(labels, dev) if n_inst else torch.zeros(1, dtype=torch.int32, device=dev)
        col = None
        if colors is not None:
            col = torch.as_tensor(colors).detach().to(dev, torch.float32).reshape(n_inst, 3).contiguous()
        rgbs = torch.empty(n_views, 3, h, w, device=dev, dtype=torch.float32)
        normals = torch.empty(n_views, 3, h, w, device=dev, dtype=torch.float32) if render_normals else None
        depths = torch.empty(n_views, 1, h, w, device=dev, dtype=torch.float32) if render_depth else None
        inst_id = torch.empty(n_views, h, w, device=dev, dtype=torch.int32)
        ws = self.workspace(h, w, dev)
        _abi.check(_abi.lib().mpx_raster_render_scene(
            self.mesh_db.handle, n_views, n_inst, _abi.ptr(offsets), _abi.ptr(label_idx), _abi.ptr(TCO), _abi.ptr(col),
            _abi.ptr(K), h, w, self.flags, _abi.ptr(rgbs), _abi.ptr(normals), _abi.ptr(depths), _abi.ptr(inst_id),
            _abi.ptr(ws), ws.numel(), _abi.stream_ptr()))
        return SceneRenderOutput(rgbs=rgbs, normals=normals, depths=depths, inst_id=inst_id)

    def render_scene(self, object_datas: List[Panda3dObjectData], camera_datas: List[Panda3dCameraData],
                     light_datas: list, render_depth: bool = False, copy_arrays: bool = True,
                     render_binary_mask: bool = False, render_normals: bool = False,
                     clear: bool = True) -> List[CameraRenderingData]:
        """panda3d_scene_renderer.py:298-358.  `copy_arrays` and `clear` have no effect: the arrays returned are always
        new, and nothing stays in a scene graph between calls."""
        check_scene_inputs(object_datas, camera_datas, light_datas)
        if render_binary_mask:
            assert render_depth, "the binary mask is computed from the depth: it needs render_depth=True"
        labels = [o.label for o in object_datas]
        colors = None
        if any(o.color is not None for o in object_datas):
            colors = torch.tensor([[float(c) for c in tuple(o.color)[:3]] if o.color is not None else [-1.0, 0.0, 0.0]
                                   for o in object_datas], dtype=torch.float32)
        groups = {}
        for n, cam in enumerate(camera_datas):
            groups.setdefault(tuple(int(r) for r in cam.resolution), []).append(n)
        results: List[Optional[CameraRenderingData]] = [None] * len(camera_datas)
        for resolution, cams in groups.items():
            TCO = np.stack([compose_TCO(camera_datas[c].TWC, o.TWO, o.scale) for c in cams for o in object_datas]) \
                if object_datas else np.zeros((0, 4, 4), np.float32)
            K = np.stack([np.asarray(camera_datas[c].K, np.float64) for c in cams]).astype(np.float32)
            out = self.render_scene_tensors([labels] * len(cams), torch.from_numpy(TCO), torch.from_numpy(K), resolution,
                                            render_depth=render_depth, render_normals=render_normals,
                                            colors=None if colors is None else colors.repeat(len(cams), 1))
            rgb = to_uint8(out.rgbs).permute(0, 2, 3, 1).cpu().numpy()
            nrm = to_uint8(out.normals).permute(0, 2, 3, 1).cpu().numpy() if render_normals else None
            dep = out.depths.permute(0, 2, 3, 1).cpu().numpy() if render_depth else None
            for n, c in enumerate(cams):
                data = CameraRenderingData(rgb=rgb[n], normals=None if nrm is None else nrm[n],
                                           depth=None if dep is None else dep[n])
                if render_binary_mask:
                    # the reference assigns the mask to a variable that is not returned (panda3d_scene_renderer.py:329-335);
                    # here every camera's result carries it
                    data.binary_mask = dep[n, :, :, 0] > 0
                results[c] = data
        return results
