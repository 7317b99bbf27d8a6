"""Batch renderer: the CUDA rasteriser behind the reference's renderer seam.

Drop-in for Panda3dBatchRenderer (src/megapose/panda3d_renderer/panda3d_batch_renderer.py:153-340):
same constructor keywords (worker/process arguments are accepted and ignored -- there are no worker
processes), same `.render(labels, TCO, K, light_datas, resolution, render_depth, render_mask,
render_normals) -> BatchRenderOutput(rgbs, normals, depths)` contract, `.stop()` is a no-op.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Tuple

import torch

from . import _abi
from .meshes import BatchedMeshes, MeshDataBase
from .object_dataset import RigidObjectDataset

RASTER_QUANTIZE8 = 1
RASTER_NORMALS_GL = 2
RASTER_POINT_LIGHTS = 4
DEPTH_NORM_KINDS = {"tCR_scale_clamp_center": 0, "tCR_scale": 1, "tCR_center_clamp": 2, "none": 3, None: 3}
DEPTH_NORM_SHIFT = 8
# the four sample positions of 4x multisampling (standard pattern, sixteenths of a pixel about the pixel centre) -- what the
# reference's offscreen buffer is configured with (framebuffer-multisample 1, multisamples 4:
# panda3d_renderer/panda3d_scene_renderer.py:73-74)
MSAA4_OFFSETS = ((-2 / 16, -6 / 16), (6 / 16, -2 / 16), (-6 / 16, 2 / 16), (2 / 16, 6 / 16))


def is_scene_lights(lights) -> bool:
    """True for the light set of `make_scene_lights()` (ambient + point lights, what models with render_normals=False
    render under, models/pose_rigid.py:374-378), False for a single ambient light."""
    kinds = [getattr(light, "light_type", "ambient") for light in lights]
    return "point" in kinds


def make_scene_lights(ambient_light_color=(0.1, 0.1, 0.1, 1.0), point_lights_color=(0.4, 0.4, 0.4, 1.0)):
    """panda3d_scene_renderer.py:104-136: 1 ambient light + 6 point lights on the object's axes at 10 bounding radii."""
    lights = [Panda3dLightData("ambient", ambient_light_color)]
    for axis in ((1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1)):
        lights.append(Panda3dLightData("point", point_lights_color, positioning_function=axis))
    return lights


@dataclass
class Panda3dLightData:
    """Light description of the reference API (panda3d_renderer/types.py:108-130).  Two light sets are rendered, the two
    the reference's models use: one white ambient light (render_normals=True, all released models) and
    `make_scene_lights()` (render_normals=False)."""

    light_type: str = "ambient"
    color: Tuple[float, float, float, float] = (1.0, 1.0, 1.0, 1.0)
    positioning_function: Optional[object] = None


@dataclass
class BatchRenderOutput:
    """rgbs [N,3,h,w] in [0,1]; normals [N,3,h,w] in [0,1]; depths [N,1,h,w] metres."""

    rgbs: torch.Tensor
    normals: Optional[torch.Tensor]
    depths: Optional[torch.Tensor]


class BatchRenderer:
    def __init__(self, object_dataset: Optional[RigidObjectDataset] = None, n_workers: int = 0,
                 preload_cache: bool = False, split_objects: bool = False,
                 mesh_db: Optional[BatchedMeshes] = None, quantize8: bool = True, normals_gl_axes: bool = False,
                 msaa4: bool = False):
        if mesh_db is None:
            assert object_dataset is not None
            mesh_db = MeshDataBase.from_object_ds(object_dataset).batched()
        self.mesh_db = mesh_db
        self._object_dataset = object_dataset
        self.flags = (RASTER_QUANTIZE8 if quantize8 else 0) | (RASTER_NORMALS_GL if normals_gl_axes else 0)
        self._workspace: Optional[torch.Tensor] = None
        # 4x anti-aliasing of the colour / normal outputs of `render` (see _render_msaa4); off by default: the fused
        # network-input paths of the pipeline render one sample per pixel
        self.msaa4 = msaa4

    def stop(self) -> None:  # the reference joins its worker processes here
        pass

    def workspace(self, h: int, w: int, device) -> torch.Tensor:
        need = _abi.lib().mpx_raster_workspace_bytes(h, w)
        if self._workspace is None or self._workspace.numel() < need or self._workspace.device != torch.device(device):
            self._workspace = torch.empty(need, dtype=torch.uint8, device=device)
        return self._workspace

    def _light_flags(self, light_datas) -> int:
        """0 for white ambient light, RASTER_POINT_LIGHTS for make_scene_lights(); the whole batch uses one light set."""
        if light_datas is None or len(light_datas) == 0:
            return 0
        kinds = {is_scene_lights(lights) for lights in light_datas}
        if len(kinds) > 1:
            raise NotImplementedError("a batch must use one light set (ambient, or make_scene_lights())")
        if not kinds.pop():
            for lights in light_datas:
                for light in lights:
                    c = tuple(getattr(light, "color", (1.0, 1.0, 1.0, 1.0)))[:3]
                    if c != (1.0, 1.0, 1.0):
                        raise NotImplementedError("ambient light colours other than white are a training-time augmentation")
            return 0
        ref = make_scene_lights()
        for lights in light_datas:
            if [(l.light_type, tuple(l.color)) for l in lights] != [(l.light_type, tuple(l.color)) for l in ref]:
                raise NotImplementedError("point lights other than make_scene_lights() are not implemented")
        return RASTER_POINT_LIGHTS

    def render(self, labels: List[str], TCO: torch.Tensor, K: torch.Tensor, light_datas=None,
               resolution: Tuple[int, int] = (240, 320), render_depth: bool = False, render_mask: bool = False,
               render_normals: bool = False, label_idx: Optional[torch.Tensor] = None) -> BatchRenderOutput:
        """`label_idx` (int32 mesh indices on the device) may be given instead of `labels` by callers that already hold it."""
        if render_mask:
            raise NotImplementedError
        if self.msaa4:
            return self._render_msaa4(labels, TCO, K, light_datas, resolution, render_depth, render_normals, label_idx)
        flags = self.flags | self._light_flags(light_datas)
        n = TCO.shape[0]
        assert TCO.shape == (n, 4, 4) and K.shape == (n, 3, 3) and (label_idx is not None or len(labels) == n)
        h, w = resolution
        dev = TCO.device
        TCO = TCO.detach().float().contiguous()
        K = K.detach().float().contiguous()
        if label_idx is None:
            label_idx = self.mesh_db.label_ids(labels, dev)
        rgbs = torch.empty(n, 3, h, w, device=dev, dtype=torch.float32)
        normals = torch.empty(n, 3, h, w, device=dev, dtype=torch.float32) if render_normals else None
        depths = torch.empty(n, 1, h, w, device=dev, dtype=torch.float32) if render_depth else None
        ws = self.workspace(h, w, dev)
        _abi.check(_abi.lib().mpx_raster_render(self.mesh_db.handle, _abi.ptr(label_idx), _abi.ptr(TCO), _abi.ptr(K),
                                                n, h, w, flags, _abi.ptr(rgbs), _abi.ptr(normals),
                                                _abi.ptr(depths), _abi.ptr(ws), ws.numel(), _abi.stream_ptr()))
        return BatchRenderOutput(rgbs=rgbs, normals=normals, depths=depths)

    def _render_msaa4(self, labels, TCO, K, light_datas, resolution, render_depth, render_normals, label_idx=None) -> BatchRenderOutput:
        """4x anti-aliased render (contract in oracle/pipeline_ref.py: RefRenderer.render(msaa4=True)): the view is rendered
        once per sample position of the 4x multisample pattern -- pixel (i, j) sampled at (j + 0.5 + ox, i + 0.5 + oy), i.e.
        with the principal point moved to (cx - ox, cy - oy) -- every sample shaded and quantised to 8 bits on its own, and
        the pixel is the rounded mean of its four samples, (k0 + k1 + k2 + k3 + 2) >> 2 in 8-bit levels (GL's multisample
        resolve).  Depth is the single-sample (pixel-centre) depth."""
        self.msaa4 = False
        try:
            out = self.render(labels, TCO, K, light_datas, resolution, render_depth=render_depth, render_mask=False,
                              render_normals=render_normals, label_idx=label_idx)
            q8 = (self.flags & RASTER_QUANTIZE8) != 0
            parts_rgb, parts_nrm = [], []
            for ox, oy in MSAA4_OFFSETS:
                Ks = K.detach().float().clone()
                Ks[:, 0, 2] = Ks[:, 0, 2] - ox
                Ks[:, 1, 2] = Ks[:, 1, 2] - oy
                s = self.render(labels, TCO, Ks, light_datas, resolution, render_depth=False, render_mask=False,
                                render_normals=render_normals, label_idx=label_idx)
                parts_rgb.append(s.rgbs)
                if render_normals:
                    parts_nrm.append(s.normals)

            def resolve(parts):
                if q8:
                    k = sum((p * 255.0).round().to(torch.int32) for p in parts)
                    # a device-tensor divisor: CUDA torch turns `x / 255.0` into x * (1 / 255), not the IEEE quotient of the contract
                    return ((k + 2) >> 2).float() / torch.full((1,), 255.0, device=k.device)
                return ((parts[0] + parts[1]) + (parts[2] + parts[3])) * 0.25

            return BatchRenderOutput(rgbs=resolve(parts_rgb), normals=resolve(parts_nrm) if render_normals else None,
                                     depths=out.depths)
        finally:
            self.msaa4 = True

    def render_fused(self, label_idx: torch.Tensor, TCO: torch.Tensor, K: torch.Tensor, views_per_sample: int,
                     resolution: Tuple[int, int], x: torch.Tensor, c_pad: int, ch_offset: int, ch_per_view: int,
                     depth_norm_z: Optional[torch.Tensor] = None, extra_flags: int = 0) -> None:
        """Render straight into the network input tensor `x` (see include/mpx.h); `extra_flags`: RASTER_POINT_LIGHTS,
        depth-normalisation kind << DEPTH_NORM_SHIFT."""
        n = TCO.shape[0]
        h, w = resolution
        ws = self.workspace(h, w, TCO.device)
        _abi.check(_abi.lib().mpx_raster_render_fused(
            self.mesh_db.handle, _abi.ptr(label_idx), _abi.ptr(TCO), _abi.ptr(K), n, views_per_sample, h, w,
            self.flags | extra_flags,
            _abi.ptr(x), c_pad, ch_offset, ch_per_view, _abi.ptr(depth_norm_z), _abi.ptr(ws), ws.numel(),
            _abi.stream_ptr()))


    def render_crop_fused(self, label_idx: torch.Tensor, TCO: torch.Tensor, K_crop: torch.Tensor,
                          resolution: Tuple[int, int], images_nhwc4: torch.Tensor, im_idx: torch.Tensor,
                          boxes_crop: torch.Tensor, c_in: int, x: torch.Tensor, c_pad: int, ch_per_view: int,
                          depth_norm_z: Optional[torch.Tensor] = None, extra_flags: int = 0) -> None:
        """Single-view samples: render + observation crop in one pass, whole pixel vectors written once."""
        n = TCO.shape[0]
        h, w = resolution
        ws = self.workspace(h, w, TCO.device)
        _abi.check(_abi.lib().mpx_render_crop_fused(
            self.mesh_db.handle, _abi.ptr(label_idx), _abi.ptr(TCO), _abi.ptr(K_crop), n, h, w, self.flags | extra_flags,
            _abi.ptr(images_nhwc4), images_nhwc4.shape[0], images_nhwc4.shape[1], images_nhwc4.shape[2], _abi.ptr(im_idx),
            _abi.ptr(boxes_crop), c_in, _abi.ptr(x), c_pad, ch_per_view, _abi.ptr(depth_norm_z), _abi.ptr(ws), ws.numel(),
            _abi.stream_ptr()))


# name used by the reference's callers
Panda3dBatchRenderer = BatchRenderer

# the multi-object scene renderer (Panda3dSceneRenderer.render_scene) and its types
from .scene_renderer import (CameraRenderingData, Panda3dCameraData, Panda3dObjectData,  # noqa: E402,F401
                             Panda3dSceneRenderer)
