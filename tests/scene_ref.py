"""ctypes binding of tests/scene_ref.c, the CPU restatement of the multi-object scene contract (test infrastructure).

The library is compiled with the flags of oracle/Makefile into tests/_build/ (git-ignored) on first use, or when the
source or the oracle it includes is newer."""
from __future__ import annotations

import ctypes
import subprocess
from pathlib import Path
from typing import Optional, Sequence

import numpy as np
import torch

_HERE = Path(__file__).resolve().parent
_SRC = _HERE / "scene_ref.c"
_ORACLE = _HERE.parent / "oracle"
_OUT = _HERE / "_build" / "libscene_ref.so"
_LIB: Optional[ctypes.CDLL] = None


def _compile(out: Path) -> Path:
    out.parent.mkdir(exist_ok=True)
    tmp = out.with_suffix(".so.tmp")
    subprocess.run(["gcc", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-Wall",
                    "-I", str(_ORACLE), "-o", str(tmp), str(_SRC), "-lm", "-lpthread"], check=True)
    tmp.replace(out)
    return out


def build(force: bool = False) -> Path:
    newest = max(_SRC.stat().st_mtime, (_ORACLE / "raster_ref.c").stat().st_mtime)
    if not force and _OUT.exists() and _OUT.stat().st_mtime >= newest:
        return _OUT
    try:
        return _compile(_OUT)
    except OSError:  # a read-only checkout: build into a temporary directory instead
        import tempfile

        return _compile(Path(tempfile.mkdtemp(prefix="scene_ref_")) / "libscene_ref.so")


def lib() -> ctypes.CDLL:
    global _LIB
    if _LIB is None:
        _LIB = ctypes.CDLL(str(build()))
        _LIB.raster_ref_render_scene.restype = ctypes.c_int
    return _LIB


def render_scene(meshes, labels_per_view: Sequence[Sequence[str]], TCO, K, resolution, flags: int = 1,
                 colors=None, label_idx: Optional[Sequence[int]] = None) -> dict:
    """meshes: oracle.pipeline_ref.RefMeshes.  labels_per_view: the instances of each view (or `label_idx`, their mesh
    indices concatenated, e.g. to pass an out-of-range label); TCO [n_inst,4,4]; K [n_views,3,3]; colors [n_inst,3] or
    None.  Returns rgbs / normals [V,3,h,w], depths [V,1,h,w] float32 and inst_id [V,h,w] int32 (torch, CPU)."""
    h, w = resolution
    n_views = len(labels_per_view)
    counts = [len(v) for v in labels_per_view]
    offsets = np.ascontiguousarray(np.cumsum([0] + counts), np.int32)
    if label_idx is None:
        label_idx = [meshes.label_to_id[l] for v in labels_per_view for l in v]
    idx = np.ascontiguousarray(label_idx, np.int32)
    n_inst = int(offsets[-1])
    T = np.ascontiguousarray(torch.as_tensor(TCO).detach().cpu().float().numpy().reshape(n_inst, 16))
    Kn = np.ascontiguousarray(torch.as_tensor(K).detach().cpu().float().numpy().reshape(n_views, 9))
    col = None if colors is None else np.ascontiguousarray(torch.as_tensor(colors).float().numpy().reshape(n_inst, 3))
    rgb = np.zeros((n_views, 3, h, w), np.float32)
    nrm = np.zeros((n_views, 3, h, w), np.float32)
    dep = np.zeros((n_views, 1, h, w), np.float32)
    iid = np.zeros((n_views, h, w), np.int32)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p) if a is not None else None  # noqa: E731
    m = meshes
    rc = lib().raster_ref_render_scene(
        ctypes.c_int(len(m.labels)), p(m.verts), p(m.normals), p(m.colors), p(m.vert_offsets), p(m.faces),
        p(m.face_offsets), p(getattr(m, "uv", None)), p(getattr(m, "tex", None)), p(getattr(m, "tex_offsets", None)),
        p(getattr(m, "tex_dims", None)), p(getattr(m, "tex_modulate", None)), ctypes.c_int(n_views), p(offsets), p(idx),
        p(T), p(col), p(Kn), ctypes.c_int(h), ctypes.c_int(w), ctypes.c_uint(flags), p(rgb), p(nrm), p(dep), p(iid))
    if rc != 0:
        raise RuntimeError(f"raster_ref_render_scene failed ({rc})")
    return dict(rgbs=torch.from_numpy(rgb), normals=torch.from_numpy(nrm), depths=torch.from_numpy(dep),
                inst_id=torch.from_numpy(iid))
