"""oracle/refload.py -- run the REAL reference code by file path.

TEST INFRASTRUCTURE ONLY, and only usable where a checkout of the reference (github.com/megapose6d/megapose6d) is named by
$MEGAPOSE_REFERENCE.  Purpose: record what the reference returns, as the golden fixtures in tests/golden/
(tools/make_golden.py; tests/golden/reference/ with MPX_RECORD_REFERENCE=1, see tests/helpers.py: reference_outputs),
against which the oracle and the product are checked.

`import megapose` fails here (pinocchio, omegaconf, roma, panda3d, ... are absent and the package
__init__ needs env vars, SURVEY.md 8c), so the reference files on the hot path are loaded with
importlib under their real module names after registering small stub modules for the missing
third-party packages.  What is substituted (and therefore NOT validated by this route):
  * the Panda3D renderer  -> any object with the same .render() signature (tests pass the C oracle)
  * megapose.lib3d.multiview.make_TCO_multiview -> oracle closed form (Panda3D scene graph absent)
  * roma.unitquat_to_rotmat (SO(3) grid) -> oracle restatement
  * torch.Tensor.cuda -> identity (CPU run)
Everything else (PosePredictor, PoseEstimator, lib3d, ResNet, tensor collections) is the
reference's own code, unmodified.
"""
from __future__ import annotations

import importlib.util
import logging
import os
import sys
import time
import types
from pathlib import Path

import numpy as np
import torch

# the reference's package directory, or None when no checkout is named
REF_ROOT = Path(os.environ["MEGAPOSE_REFERENCE"]).resolve() / "src" / "megapose" if os.environ.get("MEGAPOSE_REFERENCE") else None

_loaded = None


def available() -> bool:
    return REF_ROOT is not None and REF_ROOT.is_dir()


def _pkg(name: str) -> types.ModuleType:
    m = types.ModuleType(name)
    m.__path__ = []  # mark as package
    sys.modules[name] = m
    parent, _, child = name.rpartition(".")
    if parent in sys.modules:
        setattr(sys.modules[parent], child, m)
    return m


def _load(modname: str, relpath: str) -> types.ModuleType:
    spec = importlib.util.spec_from_file_location(modname, REF_ROOT / relpath)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[modname] = mod
    spec.loader.exec_module(mod)
    parent, _, child = modname.rpartition(".")
    if parent in sys.modules:
        setattr(sys.modules[parent], child, mod)
    return mod


class Panda3dBatchRendererStub:
    """Stands in for megapose.panda3d_renderer.panda3d_batch_renderer.Panda3dBatchRenderer so that
    pose_rigid.py:380 `isinstance(self.renderer, Panda3dBatchRenderer)` holds for substitutes."""

    def render(self, labels, TCO, K, light_datas, resolution, render_depth=False, render_mask=False,
               render_normals=False):
        raise NotImplementedError


def load():
    """Returns a namespace with the reference modules (loaded once)."""
    global _loaded
    if _loaded is not None:
        return _loaded
    if not available():
        raise RuntimeError(f"no reference source at {REF_ROOT}: set MEGAPOSE_REFERENCE to a checkout of the reference")
    from . import lib3d_ref

    for name in ["megapose", "megapose.lib3d", "megapose.models", "megapose.utils", "megapose.inference",
                 "megapose.datasets", "megapose.training", "megapose.panda3d_renderer"]:
        _pkg(name)

    # ---- third-party stubs
    t3d = types.ModuleType("transforms3d")
    t3d.euler = types.ModuleType("transforms3d.euler")
    sys.modules.setdefault("transforms3d", t3d)
    sys.modules.setdefault("transforms3d.euler", t3d.euler)

    # ---- megapose stubs
    m = types.ModuleType("megapose.datasets.pose_dataset")

    class PoseDataset:
        RGB_DIMS = [0, 1, 2]
        DEPTH_DIMS = [3]

    m.PoseDataset = PoseDataset
    sys.modules[m.__name__] = m

    m = types.ModuleType("megapose.datasets.scene_dataset")
    m.Resolution = tuple
    sys.modules[m.__name__] = m

    m = types.ModuleType("megapose.utils.logging")
    m.get_logger = lambda name: logging.getLogger(name)
    sys.modules[m.__name__] = m

    m = types.ModuleType("megapose.utils.distributed")
    m.get_rank = lambda: 0
    m.get_world_size = lambda: 1
    sys.modules[m.__name__] = m

    m = types.ModuleType("megapose.training.utils")

    class CudaTimer:
        def __init__(self, enabled=False):
            self.t0 = self.t1 = 0.0

        def start(self):
            self.t0 = time.time()

        def end(self):
            self.t1 = time.time()

        def stop(self):
            self.t1 = time.time()

        def elapsed(self):
            return self.t1 - self.t0

    class SimpleTimer(CudaTimer):
        def __init__(self):
            super().__init__()

    m.CudaTimer = CudaTimer
    m.SimpleTimer = SimpleTimer
    sys.modules[m.__name__] = m

    pr = sys.modules["megapose.panda3d_renderer"]

    class Panda3dLightData:
        def __init__(self, light_type="ambient", color=(1.0, 1.0, 1.0, 1.0), positioning_function=None):
            self.light_type = light_type
            self.color = color
            self.positioning_function = positioning_function

    pr.Panda3dLightData = Panda3dLightData
    m = types.ModuleType("megapose.panda3d_renderer.panda3d_batch_renderer")
    m.Panda3dBatchRenderer = Panda3dBatchRendererStub
    sys.modules[m.__name__] = m
    m = types.ModuleType("megapose.panda3d_renderer.panda3d_scene_renderer")
    m.make_scene_lights = lambda *a, **k: [Panda3dLightData("ambient", (0.1, 0.1, 0.1, 1.0))]
    sys.modules[m.__name__] = m

    m = types.ModuleType("megapose.lib3d.multiview")
    m.make_TCO_multiview = lib3d_ref.make_TCO_multiview
    sys.modules[m.__name__] = m

    m = types.ModuleType("megapose.lib3d.rigid_mesh_database")

    class MeshDataBase:  # only used as a type annotation on the hot path
        pass

    m.MeshDataBase = MeshDataBase
    sys.modules[m.__name__] = m

    m = types.ModuleType("megapose.inference.depth_refiner")

    class DepthRefiner:
        pass

    m.DepthRefiner = DepthRefiner
    sys.modules[m.__name__] = m

    m = types.ModuleType("megapose.utils.transform_utils")

    def load_SO3_grid(resolution):
        from . import so3_ref

        return so3_ref.load_SO3_grid_reference(resolution)

    m.load_SO3_grid = load_SO3_grid
    sys.modules[m.__name__] = m
    sys.modules["megapose.utils"].transform_utils = m

    # ---- real reference files
    ns = types.SimpleNamespace()
    ns.camera_geometry = _load("megapose.lib3d.camera_geometry", "lib3d/camera_geometry.py")
    ns.rotations = _load("megapose.lib3d.rotations", "lib3d/rotations.py")
    ns.transform_ops = _load("megapose.lib3d.transform_ops", "lib3d/transform_ops.py")
    ns.cosypose_ops = _load("megapose.lib3d.cosypose_ops", "lib3d/cosypose_ops.py")
    ns.cropping = _load("megapose.lib3d.cropping", "lib3d/cropping.py")
    ns.mesh_ops = _load("megapose.lib3d.mesh_ops", "lib3d/mesh_ops.py")
    ns.torchvision_resnet = _load("megapose.models.torchvision_resnet", "models/torchvision_resnet.py")
    ns.wide_resnet = _load("megapose.models.wide_resnet", "models/wide_resnet.py")
    ns.tensor_collection = _load("megapose.utils.tensor_collection", "utils/tensor_collection.py")
    ns.timer = _load("megapose.utils.timer", "utils/timer.py")
    ns.types = _load("megapose.inference.types", "inference/types.py")

    # inference/utils.py imports half the package; exec only the two functions the pipeline calls
    # (inference/utils.py:151-194)
    src = (REF_ROOT / "inference/utils.py").read_text().splitlines()
    start = next(i for i, l in enumerate(src) if l.startswith("def add_instance_id"))
    end = next(i for i, l in enumerate(src) if l.startswith("def make_cameras"))
    m = types.ModuleType("megapose.inference.utils")
    import pandas as pd
    from typing import List, Optional, Union

    m.__dict__.update(dict(pd=pd, np=np, torch=torch, List=List, Optional=Optional, Union=Union,
                           PoseEstimatesType=ns.types.PoseEstimatesType, DetectionsType=ns.types.DetectionsType))
    exec(compile("\n".join(src[start:end]), str(REF_ROOT / "inference/utils.py"), "exec"), m.__dict__)
    sys.modules[m.__name__] = m
    sys.modules["megapose.inference"].utils = m
    sys.modules["megapose.inference"].types = ns.types
    ns.inference_utils = m

    ns.pose_rigid = _load("megapose.models.pose_rigid", "models/pose_rigid.py")
    ns.pose_estimator = _load("megapose.inference.pose_estimator", "inference/pose_estimator.py")
    ns.Panda3dBatchRenderer = Panda3dBatchRendererStub
    _loaded = ns
    return ns


class cpu_cuda_patch:
    """Context manager: torch.Tensor.cuda -> identity (the reference hard-calls .cuda(), SURVEY A.6)."""

    def __enter__(self):
        self._orig = torch.Tensor.cuda
        torch.Tensor.cuda = lambda self, *a, **k: self
        return self

    def __exit__(self, *exc):
        torch.Tensor.cuda = self._orig
        return False
