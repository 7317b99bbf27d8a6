"""The device rasteriser on the cases of tests/raster_cases.py: bit-exact against oracle/raster_ref.c and within the
derived bounds of the float64 statement (oracle/raster_f64.py) on every unambiguous pixel, under every kernel-selection
mode, with the kernel that ran recorded; the scene renderer on the queue-overflow and tie cases; and the untiled grid
kept inside its workspace after mpx_set_sm_limit lowers the SM count below the mesh database's."""
import contextlib
import ctypes
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import pytest
import torch

from megapose6d_b200 import _abi
from oracle import raster_f64
from tests import raster_cases as rc

pytestmark = pytest.mark.gpu
DEV = "cuda"
CASES = rc.dyadic_cases() + rc.random_cases()
KERNEL = {"scatter": "raster_cover_kernel", "tiled": "raster_tiled_kernel", "untiled": "raster_kernel"}


@contextlib.contextmanager
def sm_limit(n):
    lib = _abi.lib()
    _abi.check(lib.mpx_set_sm_limit(n))
    try:
        yield
    finally:
        _abi.check(lib.mpx_set_sm_limit(0))
        _abi.check(lib.mpx_raster_set_mode(7))


class MeshDb:
    """mpx_meshdb of a case's meshes."""

    def __init__(self, meshes):
        v = np.ascontiguousarray(np.concatenate([m["verts"] for m in meshes]), np.float32)
        n = np.ascontiguousarray(np.concatenate([m["normals"] for m in meshes]), np.float32)
        c = np.ascontiguousarray(np.concatenate([m["colors"] for m in meshes]), np.float32)
        f = np.ascontiguousarray(np.concatenate([m["faces"] for m in meshes]), np.int32)
        vo = np.asarray(np.cumsum([0] + [len(m["verts"]) for m in meshes]), np.int64)
        fo = np.asarray(np.cumsum([0] + [len(m["faces"]) for m in meshes]), np.int64)
        self.handle = ctypes.c_void_p()
        _abi.check(_abi.lib().mpx_meshdb_create(len(meshes), v.ctypes.data, n.ctypes.data, c.ctypes.data, vo.ctypes.data,
                                                f.ctypes.data, fo.ctypes.data, ctypes.byref(self.handle)))

    def close(self):
        _abi.lib().mpx_meshdb_destroy(self.handle)


def _views(case, n):
    sel = np.arange(n) % len(case.labels)
    return (torch.from_numpy(case.labels[sel]).to(DEV), torch.from_numpy(case.TCO[sel]).to(DEV).contiguous(),
            torch.from_numpy(case.K[sel]).to(DEV).contiguous())


class Batch:
    """Inputs, outputs and workspace of one mpx_raster_render call of n views of `case` (views repeated cyclically),
    allocated and uploaded before any launch, so that a profiled launch holds nothing but the library's own work."""

    def __init__(self, case, n, ws=None, ws_bytes=None):
        self.n, self.h, self.w = n, case.h, case.w
        self.lab, self.T, self.K = _views(case, n)
        self.rgb = torch.empty(n, 3, case.h, case.w, device=DEV)
        self.nrm = torch.empty(n, 3, case.h, case.w, device=DEV)
        self.dep = torch.empty(n, 1, case.h, case.w, device=DEV)
        if ws is None:
            ws = torch.empty(_abi.lib().mpx_raster_workspace_bytes(case.h, case.w), dtype=torch.uint8, device=DEV)
            ws_bytes = ws.numel()
        self.ws, self.ws_bytes = ws, ws_bytes

    def poison(self):
        """NaN in every output: a pixel the launch does not write cannot equal the oracle."""
        for t in (self.rgb, self.nrm, self.dep):
            t.fill_(float("nan"))
        torch.cuda.synchronize()

    def launch(self, db):
        _abi.check(_abi.lib().mpx_raster_render(db.handle, _abi.ptr(self.lab), _abi.ptr(self.T), _abi.ptr(self.K), self.n,
                                                self.h, self.w, 1, _abi.ptr(self.rgb), _abi.ptr(self.nrm),
                                                _abi.ptr(self.dep), _abi.ptr(self.ws), self.ws_bytes, _abi.stream_ptr()))
        return self.rgb, self.nrm, self.dep


def render(db, case, n):
    return Batch(case, n).launch(db)


def _capture(fn):
    """Runs `fn` under torch.profiler between two one-element torch kernels and returns its result, the names of the
    device kernels recorded in between and whether both markers were recorded (the capture holds the window's device
    activity: a capture that lost it is taken again rather than read as 'no kernel ran')."""
    from torch.profiler import ProfilerActivity, profile

    mark = torch.zeros(1, device=DEV)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        mark.add_(1)
        out = fn()
        mark.add_(1)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    marks = [k for k, x in enumerate(names) if "raster" not in x and "lementwise" in x]
    return out, [x for x in names if "raster" in x], len(marks) >= 2


def launch_counted(db, batch, launches):
    """Launches `batch` into fresh NaN outputs and checks its launch count (mpx_launch_count); returns the outputs."""
    lib = _abi.lib()
    batch.poison()
    before = lib.mpx_launch_count()
    got = batch.launch(db)
    torch.cuda.synchronize()
    assert lib.mpx_launch_count() - before == launches
    return got


def profiled_runs():
    """Every (case, mode, batch) of test_device_equals_oracle_and_float64 launched under torch.profiler, after one warm-up
    launch: {"case/mode/batch": rasteriser kernel names, or None when no capture in five held the device activity}."""
    lib = _abi.lib()
    names = {}
    for case in CASES:
        with sm_limit(case.sm_limit):
            db = MeshDb(case.meshes)
            try:
                for mode, n in _runs(case):
                    _abi.check(lib.mpx_raster_set_mode(mode))
                    batch = Batch(case, n)
                    batch.launch(db)
                    torch.cuda.synchronize()
                    ran = None
                    for attempt in range(5):
                        time.sleep(0.2 * attempt)
                        _, found, complete = _capture(lambda: batch.launch(db))
                        if complete:
                            ran = found
                            break
                    names[f"{case.name}/{mode}/{n}"] = ran
                    del batch
            finally:
                db.close()
    return names


@pytest.fixture(scope="module")
def kernel_names():
    """The kernels each run launched, recorded in a process of its own: late in a long process (the whole GPU suite)
    torch.profiler can stop recording device activity altogether, while a fresh process records it."""
    root = Path(__file__).resolve().parent.parent
    code = (f"import json, sys; sys.path.insert(0, {str(root)!r}); from tests import test_gpu_raster_f64 as t; "
            "print('KERNELS=' + json.dumps(t.profiled_runs()))")
    res = subprocess.run([sys.executable, "-s", "-c", code], cwd=root, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-4000:]
    return json.loads([x for x in res.stdout.splitlines() if x.startswith("KERNELS=")][-1][len("KERNELS="):])


def render_scene(db, case, labels_per_view, TCO, ws=None, ws_bytes=None):
    """One view per entry of `labels_per_view` (list of (mesh label, pose index) lists), all under the case's K[0]."""
    n = len(labels_per_view)
    off = torch.tensor(np.cumsum([0] + [len(v) for v in labels_per_view]), dtype=torch.int32, device=DEV)
    lab = torch.tensor([l for v in labels_per_view for l, _ in v], dtype=torch.int32, device=DEV)
    T = torch.from_numpy(np.stack([TCO[i] for v in labels_per_view for _, i in v])).to(DEV).contiguous()
    K = torch.from_numpy(np.stack([case.K[0]] * n)).to(DEV).contiguous()
    h, w = case.h, case.w
    rgb = torch.empty(n, 3, h, w, device=DEV)
    nrm = torch.empty(n, 3, h, w, device=DEV)
    dep = torch.empty(n, 1, h, w, device=DEV)
    ids = torch.empty(n, h, w, dtype=torch.int32, device=DEV)
    if ws is None:
        ws = torch.empty(_abi.lib().mpx_raster_workspace_bytes(h, w), dtype=torch.uint8, device=DEV)
        ws_bytes = ws.numel()
    _abi.check(_abi.lib().mpx_raster_render_scene(db.handle, n, int(off[-1]), _abi.ptr(off), _abi.ptr(lab), _abi.ptr(T), None,
                                                  _abi.ptr(K), h, w, 1, _abi.ptr(rgb), _abi.ptr(nrm), _abi.ptr(dep),
                                                  _abi.ptr(ids), _abi.ptr(ws), ws_bytes, _abi.stream_ptr()))
    return rgb, nrm, dep, ids


def _refs(case):
    """Per unique view: raster_ref.c outputs on the device, and the float64 render."""
    out = []
    for v in range(len(case.labels)):
        ref, f64 = rc.rendered(case, v)
        out.append((torch.from_numpy(ref["rgb"]).to(DEV), torch.from_numpy(ref["nrm"]).to(DEV),
                    torch.from_numpy(ref["depth"]).to(DEV)[None], ref, f64))
    return out


def _check(case, refs, got, what):
    rgb, nrm, dep = got
    nu = len(refs)
    for k in range(rgb.shape[0]):
        r = refs[k % nu]
        for name, a, b in (("rgb", rgb[k], r[0]), ("normals", nrm[k], r[1]), ("depth", dep[k], r[2])):
            assert torch.equal(a, b), f"{what} view {k} {name}: {(a != b).sum().item()} values differ from raster_ref.c"
    for k in range(min(nu, rgb.shape[0])):
        res = raster_f64.check_outputs(refs[k][4], rgb[k].cpu().numpy(), nrm[k].cpu().numpy(), dep[k, 0].cpu().numpy())
        assert all(n == 0 for n, _ in res.values()), (what, k, res)


# every mode at least once per case: 7 at each batch (scatter, tiled or untiled by size), 3 at the smallest (scatter with the
# reduction), 2 at the largest (untiled, reduction), 0 at the smallest (untiled, read-then-atomic)
def _runs(case):
    b = case.batches
    return [(7, n) for n in b] + [(3, b[0]), (2, b[-1]), (0, b[0])]


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_device_equals_oracle_and_float64(case, kernel_names):
    lib = _abi.lib()
    refs = _refs(case)
    with sm_limit(case.sm_limit):
        db = MeshDb(case.meshes)
        try:
            sm = lib.mpx_sm_count()
            for mode, n in _runs(case):
                _abi.check(lib.mpx_raster_set_mode(mode))
                d = rc.dispatch(case.h, case.w, n, sm, 2 * sm, mode)
                kern = KERNEL[d["kernel"]]
                launches = 2 if d["kernel"] == "scatter" else 1
                got = launch_counted(db, Batch(case, n), launches)
                ran = kernel_names[f"{case.name}/{mode}/{n}"]
                assert ran is not None, "torch.profiler recorded no device activity in five captures"
                assert sum(kern in x for x in ran) == 1 and len(ran) == launches, (mode, n, d, ran)
                _check(case, refs, got, f"{case.name} mode {mode} batch {n}")
        finally:
            db.close()


@pytest.mark.parametrize("make", [rc.queue_case, rc.fan_grid_case], ids=["queue_overflow", "fan_grid_ties"])
def test_scene_renderer_on_queue_and_tie_cases(make):
    """One instance per view renders what mpx_raster_render renders; two instances at the same pose tie on every
    fragment, and the lower instance wins everywhere."""
    case = make()
    with sm_limit(case.sm_limit):
        db = MeshDb(case.meshes)
        try:
            single = render(db, case, 1)
            one = render_scene(db, case, [[(0, 0)]], case.TCO)
            two = render_scene(db, case, [[(0, 0), (0, 0)]], case.TCO)
            for a, b in zip(single, one[:3]):
                assert torch.equal(a, b)
            for a, b in zip(one, two):
                assert torch.equal(a, b)
            ids = two[3]
            assert ((ids == 0) == (one[2][:, 0] > 0)).all() and (ids >= 0).sum() > 100 and not (ids == 1).any()
        finally:
            db.close()


def test_untiled_grid_stays_inside_the_workspace_after_sm_limit():
    """A mesh database created at the full SM count, then mpx_set_sm_limit(16): the untiled kernel renders 4 views into a
    workspace of exactly mpx_raster_workspace_bytes (32 visibility buffers).  The workspace sits in an allocation whose
    tail could hold every buffer the database has slots for; the tail stays untouched and the pixels equal the oracle.
    The scene renderer, chunked by the current SM count, does the same with 40 views."""
    lib = _abi.lib()
    case = rc.fan_grid_case()
    h, w = case.h, case.w
    _abi.check(lib.mpx_set_sm_limit(0))
    full_slots = 2 * lib.mpx_sm_count()
    assert full_slots > 32
    db = MeshDb(case.meshes)
    try:
        with sm_limit(16):
            _abi.check(lib.mpx_raster_set_mode(2))
            need = lib.mpx_raster_workspace_bytes(h, w)
            assert need == 32 * h * w * 8
            tail = max(full_slots - 32, 0) * h * w * 8 + 4096
            buf = torch.full((need + tail,), 0xA5, dtype=torch.uint8, device=DEV)
            ws = buf[:need]
            # mode 2 turns the scatter and tiled kernels off: the one launch is the untiled kernel
            assert rc.dispatch(h, w, 4, 16, full_slots, mode=2)["kernel"] == "untiled"
            got = launch_counted(db, Batch(case, 4, ws, need), 1)
            assert (buf[need:] == 0xA5).all(), "the untiled kernel wrote past its workspace"
            refs = _refs(case)
            _check(case, refs, got, "sm limit 16, untiled")
            scene = render_scene(db, case, [[(0, 0)]] * 40, case.TCO, ws, need)
            torch.cuda.synchronize()
            assert (buf[need:] == 0xA5).all(), "the scene renderer wrote past its workspace"
            _check(case, refs, scene[:3], "sm limit 16, scene")
    finally:
        db.close()
