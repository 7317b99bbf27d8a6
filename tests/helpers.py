"""Shared builders for the tests: the synthetic workloads (re-exported from workloads/), oracle objects, reference
adapters, the stored outputs of the reference and the checker of the reference's pipeline fixtures."""
from __future__ import annotations

import hashlib
import os
from pathlib import Path

import numpy as np
import torch

from megapose6d_b200 import procedural
from oracle import pipeline_ref, resnet_ref  # noqa: F401
from workloads.scenes import (FULLSIZE, bench_scene, detection_for_pose, make_scene, pipeline_scenario,  # noqa: F401
                              rgbd_scene, ycbv_scene)
from workloads.weights import (COARSE_CFG, REFINER_CFG, REFINER_RGBD_CFG, calibration_batch, make_state_dict,  # noqa: F401
                               n_inputs)

_calibration_batch = calibration_batch
REFERENCE_GOLDEN = Path(__file__).resolve().parent / "golden" / "reference"


def reference_outputs(name: str, compute) -> dict:
    """What the reference computed for a test: {key: tensor} stored as tests/golden/reference/<name>.npz.

    `compute()` runs the reference itself (oracle/refload.py) and returns {key: tensor or array}; it is only called to
    (re)record the file, with MPX_RECORD_REFERENCE=1 on a machine that has the reference source tree.  Large outputs are
    stored as `sample_of` / `digest_of` them so that every file stays small."""
    path = REFERENCE_GOLDEN / f"{name}.npz"
    if os.environ.get("MPX_RECORD_REFERENCE") == "1":
        arrays = {k: (v.detach().cpu().numpy() if torch.is_tensor(v) else np.asarray(v)) for k, v in compute().items()}
        arrays = {k: (a.astype(str) if a.dtype == object else a) for k, a in arrays.items()}
        path.parent.mkdir(parents=True, exist_ok=True)
        np.savez_compressed(path, **arrays)
    with np.load(path) as z:  # numbers as tensors, strings as numpy arrays
        return {k: torch.from_numpy(z[k].copy()) if z[k].dtype.kind in "biuf" else z[k] for k in z.files}


class reproducible_fp32:
    """Context manager: torch's CPU convolutions, linear maps, batch norms and average pools compute in float64 and round
    the result to float32.  Their fp32 summation order depends on the host CPU's instruction set; rounded float64 results do
    not, so stored outputs of the reference can be compared at fp32 tolerances on another machine."""

    OPS = ("conv2d", "linear", "batch_norm", "adaptive_avg_pool2d")

    def __enter__(self):
        import torch.nn.functional as F

        self._orig = {name: getattr(F, name) for name in self.OPS}

        def wrap(fn):
            def run(*args, **kwargs):
                dt = next((a.dtype for a in args if torch.is_tensor(a) and a.is_floating_point()), None)
                if dt != torch.float32:
                    return fn(*args, **kwargs)
                up = [a.double() if torch.is_tensor(a) and a.dtype == torch.float32 else a for a in args]
                kw = {k: (v.double() if torch.is_tensor(v) and v.dtype == torch.float32 else v) for k, v in kwargs.items()}
                return fn(*up, **kw).float()
            return run

        for name, fn in self._orig.items():
            setattr(F, name, wrap(fn))
        return self

    def __exit__(self, *exc):
        import torch.nn.functional as F

        for name, fn in self._orig.items():
            setattr(F, name, fn)
        return False


def sample_of(t: torch.Tensor, n: int = 4096) -> torch.Tensor:
    """A fixed, seeded sample of n elements of t (all of them when t is smaller)."""
    flat = t.detach().reshape(-1).cpu()
    if flat.numel() <= n:
        return flat.clone()
    idx = torch.randperm(flat.numel(), generator=torch.Generator().manual_seed(0))[:n]
    return flat[idx]


def digest_of(t: torch.Tensor) -> np.ndarray:
    """SHA-256 of the tensor's dtype, shape and bytes: torch.equal against a stored tensor without storing it."""
    a = t.detach().cpu().contiguous().numpy()
    h = hashlib.sha256(f"{a.dtype}{a.shape}".encode())
    h.update(a.tobytes())
    return np.frombuffer(h.digest(), dtype=np.uint8).copy()


def ref_meshes_from_dataset(ds) -> pipeline_ref.RefMeshes:
    labels, v, n, c, f, uv, tex, mod = [], [], [], [], [], [], [], []
    for obj in ds.list_objects:
        m = obj.mesh.with_defaults()
        labels.append(obj.label)
        v.append(np.asarray(m.vertices, np.float64) * obj.scale)
        n.append(m.vertex_normals)
        c.append(np.clip(m.vertex_colors, 0, 1))
        f.append(m.faces)
        uv.append(m.uv)
        tex.append(m.texture)
        mod.append(1 if m.texture_modulate else 0)
    return pipeline_ref.RefMeshes(labels, v, n, c, f, uv, tex, mod)


def check_pipeline_against_golden(golden, coarse_poses, coarse_logits, kept_hypotheses, exact_network: bool,
                                  final_labels=None, final_hypotheses=None, final_poses=None):
    """`golden`: tests/golden/pipeline.npz (outputs of the reference's own PoseEstimator.run_inference_pipeline).
    coarse_poses [2*72,4,4] / coarse_logits [2*72] in the reference's row order (detection-major, grid order);
    kept_hypotheses: per detection, the set of hypothesis ids that survived the coarse filter.

    Tolerances: the initial poses are fp32 geometry -> rtol 2e-5 / atol 2e-6 (the oracle reproduces the reference to
    1e-5 / 1e-6, the CUDA path the oracle to the same).  Logits: an fp32 network (`exact_network`) must reproduce them to
    rtol 1e-4 / atol 1e-5 and give the same final result; the bf16 CUDA network is checked through what the logits are
    used for -- the same survivors wherever the reference's ranking margin is well above the observed noise."""
    want_poses = torch.from_numpy(golden["coarse_poses"])
    assert torch.allclose(coarse_poses.float().cpu(), want_poses, rtol=2e-5, atol=2e-6)
    want = torch.from_numpy(golden["coarse_logit"]).float()
    got = torch.as_tensor(np.array(torch.as_tensor(coarse_logits).cpu() if torch.is_tensor(coarse_logits) else coarse_logits, dtype=np.float32))
    err = (got - want).abs()
    if exact_network:
        assert torch.allclose(got, want, rtol=1e-4, atol=1e-5), f"coarse logits: max err {err.max():.3g}"
        tol = 1e-4
    else:
        tol = 4.0 * err.median().item() + 0.05
    n_det, m = golden["kept_hypotheses"].shape[0], want.numel() // golden["kept_hypotheses"].shape[0]
    k = golden["kept_hypotheses"].shape[1]
    checked = 0
    for det in range(n_det):
        ranked = torch.sort(want[det * m:(det + 1) * m], descending=True).values
        if (ranked[k - 1] - ranked[k]).item() > 2 * tol:
            assert set(int(h) for h in kept_hypotheses[det]) == set(int(h) for h in golden["kept_hypotheses"][det]), det
            checked += 1
    if exact_network:
        assert checked == n_det, "the scenario was chosen with clear margins"
        order_w, order_g = np.argsort(golden["final_label"]), np.argsort(np.asarray(final_labels))
        assert [int(h) for h in np.asarray(final_hypotheses)[order_g]] == [int(h) for h in golden["final_hypothesis"][order_w]]
        assert torch.allclose(final_poses.float().cpu()[order_g], torch.from_numpy(golden["final_poses"])[order_w],
                              rtol=1e-4, atol=1e-5)
    return dict(max_logit_err=err.max().item(), survivors_checked=checked)


def collection_arrays(prefix: str, c) -> dict:
    """The index, infos columns and tensors of a (Pandas)TensorCollection as {prefix/...: array} for reference_outputs."""
    d = {f"{prefix}/index": c.infos.index.to_numpy()}
    for col in c.infos.columns:
        d[f"{prefix}/col/{col}"] = c.infos[col].to_numpy()
    for k, v in c.tensors.items():
        d[f"{prefix}/t/{k}"] = v
    return d


class StoredCollection:
    """A collection rebuilt from collection_arrays: `infos` (DataFrame) and `tensors`, in the stored order."""

    def __init__(self, stored: dict, prefix: str):
        import pandas as pd

        def arr(v):
            return v.numpy() if torch.is_tensor(v) else v

        cols = {k[len(prefix) + 5:]: arr(v) for k, v in stored.items() if k.startswith(prefix + "/col/")}
        self.infos = pd.DataFrame({k: (v.astype(object) if v.dtype.kind == "U" else v) for k, v in cols.items()},
                                  index=pd.Index(arr(stored[prefix + "/index"])))
        if len(self.infos.columns) == 0:
            self.infos = pd.DataFrame(index=pd.Index(arr(stored[prefix + "/index"])))
        self.tensors = {k[len(prefix) + 3:]: v for k, v in stored.items() if k.startswith(prefix + "/t/")}

    def __len__(self):
        return len(self.infos)

    def __getattr__(self, name):
        if name != "tensors" and name in self.tensors:
            return self.tensors[name]
        raise AttributeError(name)


def json_array(value) -> np.ndarray:
    """A JSON-serialisable value as a string array for reference_outputs (read back with json.loads(str(a)))."""
    import json

    return np.asarray(json.dumps(value))
