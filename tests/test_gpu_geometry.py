"""The hypothesis-geometry kernels (csrc/geom.cu) through the C ABI against the float64 restatement oracle/geometry_ref.py.

* Dyadic cases (tests/geometry_cases.py): every fp32 intermediate is exact, so each kernel must equal float64 bit for bit
  (torch.equal), whatever FMA contraction nvcc chose.  This pins each formula: every +1, /2, max/min and clamp.
* Random cases at the same edges: |kernel - float64| <= the running error bound of geometry_ref.Bounded, per element.
  That bound is derived operation by operation from the unit roundoff u = 2^-24 (a +- b: ea + eb + u |result|;
  a * b: |a| eb + |b| ea + u |result|; a / b: (ea + |a / b| eb) / (|b| - eb) + u |result|; sqrt: ea / (2 sqrt a) + u |result|,
  plus the second-order terms), so a 3-term dot product gets the classic gamma_3 sum of |products| and the divisions
  of the projection carry it on; it holds with or without FMA contraction.  Min / max select, so a box coordinate's
  bound is the largest bound of the points it selects from.  The largest error seen, in units of the bound, is printed.
* multiview_kernel computes in float64: within 1 fp32 ulp of fp32(float64 restatement).
* Top-K: exact indices, NaN after -inf, ties to the lower index.
"""
import numpy as np
import pandas as pd
import pytest
import torch

from megapose6d_b200 import _abi, lib3d
from megapose6d_b200.pose_estimator import PoseEstimator
from oracle import geometry_ref as G
from oracle import lib3d_ref as L
from tests import geometry_cases as C

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _d(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a)).to(DEV, dtype).contiguous()


def _launches():
    return _abi.lib().mpx_launch_count()


def crop_kernel(c):
    n = len(c["label_idx"])
    # every operand is bound to a name until the results are read: a temporary's block could be handed to the next one
    pts, lab, TCO, K, tCR = _d(c["points"]), _d(c["label_idx"], torch.int32), _d(c["TCO"]), _d(c["K"]), _d(c["tCR"])
    out = [torch.full((n, 4), 7.0, device=DEV), torch.full((n, 4), 7.0, device=DEV), torch.full((n, 3, 3), 7.0, device=DEV)]
    (im_h, im_w), (out_h, out_w) = c["im_size"], c["out_size"]
    _abi.check(_abi.lib().mpx_crop_geometry(_abi.ptr(pts), pts.shape[1], _abi.ptr(lab), _abi.ptr(TCO), _abi.ptr(K),
                                            _abi.ptr(tCR), n, float(c["lamb"]), im_h, im_w, out_h, out_w,
                                            *(_abi.ptr(o) for o in out), _abi.stream_ptr()))
    return dict(zip(("boxes_rend", "boxes_crop", "K_crop"), (o.cpu().double().numpy() for o in out)))


def pose_init_kernel(p):
    n = len(p["label_idx"])
    TCO = torch.full((n, 4, 4), 7.0, device=DEV)
    pts, lab, bb, K, R = _d(p["points"]), _d(p["label_idx"], torch.int32), _d(p["bboxes"]), _d(p["K"]), _d(p["R"])
    _abi.check(_abi.lib().mpx_pose_init_autodepth(_abi.ptr(pts), pts.shape[1], _abi.ptr(lab), _abi.ptr(bb), _abi.ptr(K),
                                                  _abi.ptr(R), n, _abi.ptr(TCO), _abi.stream_ptr()))
    return TCO.cpu().double().numpy()


def pose_update_kernel(u):
    return lib3d.update_pose(_d(u["TCO"]), _d(u["K_crop"]), _d(u["pose9"]), _d(u["tCR"])).cpu().double().numpy()


def normalize_kernel(T):
    return lib3d.normalize_T(_d(T)).cpu().double().numpy()


def _exact(got, want, what):
    got, want = torch.as_tensor(np.asarray(got, np.float64)), torch.as_tensor(np.asarray(want, np.float64))
    assert torch.equal(torch.isnan(got), torch.isnan(want)), what
    ok = torch.isnan(want) | (got == want)
    assert ok.all(), f"{what}: {(~ok).sum().item()} elements differ, max |d| = {(got - want)[~ok].abs().max().item()}"


def _within(got, v, e, what):
    got = np.asarray(got, np.float64)
    err = np.abs(got - v)
    assert np.isfinite(got).all() and (err <= e).all(), f"{what}: max err / bound = {np.max(err / np.maximum(e, 1e-300))}"
    ratio = float(np.max(np.where(e > 0, err / np.where(e > 0, e, 1), 0.0)))
    print(f"{what}: largest error = {ratio:.3f} of the bound (largest bound {e.max():.3g})")


# ---------------------------------------------------------------------------------------------------------------------
# crop geometry
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", C.DYADIC_SHAPES, ids=lambda s: f"{s[0][0]}x{s[0][1]}-{s[1][0]}x{s[1][1]}-l{s[2]}")
def test_crop_geometry_dyadic_bit_exact(shape):
    """Portrait and landscape images and outputs, lamb 1 / 1.5, every point count of N_PTS with the box-defining point in
    the last warp or a second stride, two labels with padded tables: boxes_rend, boxes_crop and K_crop equal float64."""
    for n_pts in C.N_PTS:
        c = C.dyadic_crop_case(1000 + n_pts, n_pts, shape)
        got = crop_kernel(c)
        want = G.crop_geometry(c["points"], c["label_idx"], c["TCO"], c["K"], c["tCR"], c["lamb"], c["im_size"],
                               c["out_size"])
        for k in want:
            _exact(got[k], want[k], f"{k} n_pts={n_pts}")


@pytest.mark.parametrize("shape", C.RANDOM_SHAPES, ids=lambda s: f"{s[0][0]}x{s[0][1]}-{s[1][0]}x{s[1][1]}-l{s[2]}")
def test_crop_geometry_random_within_bound(shape):
    """Random poses, three labels of unequal (padded) sizes, points and tCR on / just under / just over z = 0.1 and far
    behind it."""
    for n_pts in C.N_PTS:
        c = C.random_crop_case(n_pts, n_pts, shape, z_edges=True)
        got = crop_kernel(c)
        bounds = G.crop_geometry_bounds(c["points"], c["label_idx"], c["TCO"], c["K"], c["tCR"], c["lamb"], c["im_size"],
                                        c["out_size"])
        for k, (v, e) in bounds.items():
            _within(got[k], v, e, f"crop_geometry {k}")


def test_crop_geometry_non_finite_matches_reference():
    """A NaN in the rotation (the rendering centre is NaN too), in the translation, an inf rotation entry, a NaN tCR:
    NaN boxes and NaN K_crop entries (the zeros and the 1 kept) exactly where the reference's functions put them; the
    other hypotheses as without them."""
    c = C.random_crop_case(8, 200, C.RANDOM_SHAPES[0])
    clean = crop_kernel(c)
    c["TCO"][1, 0, 0] = np.nan
    c["TCO"][2, 1, 3] = np.nan
    c["TCO"][3, 2, 2] = np.inf
    c["tCR"][4, 2] = np.nan
    got = crop_kernel(c)
    want = G.crop_geometry(c["points"], c["label_idx"], c["TCO"], c["K"], c["tCR"], c["lamb"], c["im_size"], c["out_size"])
    for k in want:
        assert np.array_equal(np.isnan(got[k]), np.isnan(want[k])), k
        assert np.array_equal(got[k][5:], clean[k][5:]) and np.array_equal(got[k][0], clean[k][0]), k
    assert np.isnan(got["boxes_crop"][1:5]).all() and (got["K_crop"][1:5, 2] == [0, 0, 1]).all()


# ---------------------------------------------------------------------------------------------------------------------
# pose init
# ---------------------------------------------------------------------------------------------------------------------
def test_pose_init_dyadic_bit_exact():
    """bb_dx = 2^k incl. 1 (a zero-width box), and x2 = x1 - 1 (bb_dx = 0: z = inf, or NaN for one point, as in the
    reference); every point count."""
    for n_pts in C.N_PTS:
        p = C.dyadic_pose_init_case(n_pts, n_pts)
        _exact(pose_init_kernel(p), G.pose_init(**p), f"pose_init n_pts={n_pts}")
        p["bboxes"][1, 2] = p["bboxes"][1, 0] - 1
        _exact(pose_init_kernel(p), G.pose_init(**p), f"pose_init x2 = x1 - 1, n_pts={n_pts}")


def test_pose_init_random_within_bound():
    for n_pts in C.N_PTS:
        p = C.random_pose_init_case(n_pts, n_pts)
        got = pose_init_kernel(p)
        v, e = G.bounds_as_T(G.pose_init(**p, dtype="bounded"), len(p["label_idx"]))
        _within(got[:, :3, 3], v[:, :3, 3], e[:, :3, 3], "pose_init t")
        assert np.array_equal(got[:, :3, :3], p["R"]) and np.array_equal(got[:, 3], np.tile([0, 0, 0, 1.0], (16, 1)))


def test_pose_init_non_finite_matches_reference():
    p = C.random_pose_init_case(9, 257)
    p["R"][2, 1, 1] = np.nan
    p["bboxes"][3, 0] = np.nan
    p["R"][4, 0, 2] = np.inf
    got, want = pose_init_kernel(p), G.pose_init(**p)
    assert np.array_equal(np.isnan(got), np.isnan(want)) and np.isnan(got[[2, 3], :3, 3]).all()


# ---------------------------------------------------------------------------------------------------------------------
# pose update, normalize_T
# ---------------------------------------------------------------------------------------------------------------------
def test_pose_update_and_normalize_dyadic_bit_exact():
    """Signed-axis ortho6d inputs with power-of-two norms; a non-identity bottom row, which the update keeps (the
    reference clones TCO) and normalize_T replaces with (0, 0, 0, 1)."""
    u = C.dyadic_pose_update_case(11)
    _exact(pose_update_kernel(u), G.pose_update(**u), "pose_update")
    T = C.dyadic_normalize_case(12)
    _exact(normalize_kernel(T), G.normalize_T(T), "normalize_T")


def test_pose_update_and_normalize_random_within_bound():
    u = C.random_pose_update_case(4)
    got = pose_update_kernel(u)
    v, e = G.bounds_as_T(G.pose_update(**u, dtype="bounded"), 300)
    _within(got[:, :3], v[:, :3], e[:, :3], "pose_update")
    assert np.array_equal(got[:, 3], u["TCO"][:, 3])
    T = C.random_normalize_case(5)
    got = normalize_kernel(T)
    v, e = G.bounds_as_T(G.normalize_T(T, dtype="bounded"), 300)
    _within(got[:, :3], v[:, :3], e[:, :3], "normalize_T")
    assert np.array_equal(got[:, 3], np.tile([0, 0, 0, 1.0], (300, 1)))


# ---------------------------------------------------------------------------------------------------------------------
# multi-view cameras
# ---------------------------------------------------------------------------------------------------------------------
def _offsets(n_extra):
    base = np.concatenate([L.VIEW_OFFSETS["sphere_26views"], np.random.RandomState(0).randint(-2, 3, (6, 3))])
    return base[:n_extra].astype(np.float32)


@pytest.mark.parametrize("n_extra", [0, 1, 26, 32])
def test_multiview_within_one_ulp(n_extra):
    """Within 1 fp32 ulp of fp32(float64), plus 1e-14 absolute for entries that are 0 up to float64 rounding; a NaN
    pose gives NaN exactly where the restatement has it.  The rotations are signed permutations, orthonormal in fp32:
    the kernel inverts camera 0's world pose by transposition where the closed form inverts it in general, and for a
    rotation that is orthonormal only to fp32 rounding the two differ by that defect (a few ulp; test_gpu_kernels'
    test_multiview_and_pose_update covers random rotations at 2e-6)."""
    rs = np.random.RandomState(21)
    TCO = np.tile(np.eye(4), (65, 1, 1))
    TCO[:, :3, :3] = C.signed_permutations(rs, 65)
    TCO[:, :3, 3] = np.stack([rs.uniform(-0.1, 0.1, 65), rs.uniform(-0.1, 0.1, 65), rs.uniform(0.3, 1.2, 65)], 1)
    TCO = TCO.astype(np.float32)
    tCR = (TCO[:, :3, 3] + rs.uniform(-0.01, 0.01, (65, 3))).astype(np.float32)
    TCO[64, 0, 0] = np.nan
    offs = _offsets(n_extra)
    out = torch.full((65, 1 + n_extra, 4, 4), 7.0, device=DEV)
    TCO_d, tCR_d = _d(TCO), _d(tCR)
    _abi.check(_abi.lib().mpx_multiview_cameras(_abi.ptr(TCO_d), _abi.ptr(tCR_d), 65,
                                                offs.ctypes.data if n_extra else None, n_extra, _abi.ptr(out),
                                                _abi.stream_ptr()))
    got = out.cpu().numpy()
    want = G.multiview(TCO, tCR, offs.astype(np.float64)).astype(np.float32)
    assert np.array_equal(np.isnan(got), np.isnan(want))
    fin = ~np.isnan(want)
    d = np.abs(got[fin].astype(np.float64) - want[fin])
    assert (d <= np.spacing(np.abs(want[fin])).astype(np.float64) + 1e-14).all(), d.max()
    assert np.array_equal(got[:, 0], TCO, equal_nan=True)
    print(f"multiview n_extra={n_extra}: {(d > 0).sum()} of {d.size} elements off by 1 ulp")


# ---------------------------------------------------------------------------------------------------------------------
# top-K
# ---------------------------------------------------------------------------------------------------------------------
def _topk(logits, k):
    g, m = logits.shape
    idx = torch.full((g, k), -1, dtype=torch.int32, device=DEV)
    x = _d(logits)
    _abi.check(_abi.lib().mpx_topk_per_group(_abi.ptr(x), g, m, k, _abi.ptr(idx), _abi.stream_ptr()))
    return idx.cpu().long().numpy()


def _special_logits(rs, g, m):
    """Tie-heavy logits with NaN and +-inf, and rows: all equal, ties at i and i + 256 (one thread's stride), NaN
    before -inf, all NaN."""
    x = rs.randint(-4, 5, (g, m)).astype(np.float32)
    x[rs.rand(g, m) < 0.1] = np.nan
    x[rs.rand(g, m) < 0.05] = np.inf
    x[rs.rand(g, m) < 0.05] = -np.inf
    x[rs.rand(g, m) < 0.05] = -0.0
    x[0] = 1.5
    if m > 300:
        x[1] = -9
        x[1, [3, 3 + 256, 40]] = 8.0
    x[2] = -np.inf
    x[2, :m // 2] = np.nan
    x[3] = np.nan
    return x


@pytest.mark.parametrize("m", [1, 31, 33, 257, 576, 4608, 12000])
def test_topk_exact(m):
    rs = np.random.RandomState(m)
    x = np.concatenate([_special_logits(rs, 6, m), rs.randn(4, m).astype(np.float32)])
    for k in sorted({1, 5, 33, m}):
        if k <= m:
            assert np.array_equal(_topk(x, k), G.topk(x, k)), k


def test_topk_many_groups():
    rs = np.random.RandomState(7)
    x = rs.randint(-20, 21, (70000, 576)).astype(np.float32)
    x[rs.rand(70000, 576) < 0.01] = np.nan
    assert np.array_equal(_topk(x, 5), G.topk(x, 5))


def test_coarse_select_matches_pandas():
    """PoseEstimator._coarse_select (device top-K, then all survivors by descending logit) against
    sort_values(ascending=False).groupby().head(K) on tie-heavy logits with NaN and +-inf."""
    B, M, Kh = 7, 72, 5
    rs = np.random.RandomState(3)
    lg = _special_logits(rs, B, M).reshape(-1, 1)
    rows_c = dict(batch_im_ids=torch.zeros(B * M, dtype=torch.long, device=DEV),
                  label_idx=torch.zeros(B * M, dtype=torch.long, device=DEV),
                  group_base=(torch.arange(B, device=DEV) * M).unsqueeze(1))
    st = dict(K_rows=torch.zeros(B * M, 3, 3, device=DEV), bboxes=torch.zeros(B * M, 4, device=DEV),
              TCO=torch.zeros(B * M, 4, 4, device=DEV), out={})
    got = PoseEstimator._coarse_select(None, st, _d(lg), rows_c, B, M, Kh)["rows"].cpu().numpy()
    df = pd.DataFrame(dict(logit=lg.ravel().astype(np.float64), group=np.arange(B * M) // M))
    want = df.sort_values("logit", ascending=False, kind="stable").groupby("group").head(Kh).index.to_numpy()
    assert np.array_equal(got, want)


# ---------------------------------------------------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------------------------------------------------
def test_refusals_launch_nothing():
    lib = _abi.lib()
    f = torch.zeros(64, device=DEV)
    i = torch.zeros(4, dtype=torch.int32, device=DEV)
    pf, pi, s = _abi.ptr(f), _abi.ptr(i), _abi.stream_ptr()
    offs = np.zeros(99, np.float32)
    n0 = _launches()
    refused = [
        lib.mpx_pose_init_autodepth(pf, 0, pi, pf, pf, pf, 1, pf, s),
        lib.mpx_pose_init_autodepth(pf, 8, pi, pf, pf, None, 1, pf, s),
        lib.mpx_pose_init_autodepth(pf, 8, pi, pf, pf, pf, -1, pf, s),
        lib.mpx_crop_geometry(pf, 0, pi, pf, pf, pf, 1, 1.4, 480, 640, 240, 320, pf, pf, pf, s),
        lib.mpx_crop_geometry(pf, 8, pi, pf, pf, pf, 1, 1.4, 0, 640, 240, 320, pf, pf, pf, s),
        lib.mpx_crop_geometry(pf, 8, pi, pf, pf, pf, 1, 1.4, 480, 640, 240, -1, pf, pf, pf, s),
        lib.mpx_crop_geometry(pf, 8, None, pf, pf, pf, 1, 1.4, 480, 640, 240, 320, pf, pf, pf, s),
        lib.mpx_topk_per_group(pf, 1, 4, 5, pi, s),
        lib.mpx_topk_per_group(pf, 1, 12001, 5, pi, s),
        lib.mpx_topk_per_group(None, 1, 8, 2, pi, s),
        lib.mpx_topk_per_group(pf, 1, -1, 0, pi, s),
        lib.mpx_multiview_cameras(pf, pf, 1, offs.ctypes.data, 33, pf, s),
        lib.mpx_multiview_cameras(pf, pf, 1, offs.ctypes.data, -1, pf, s),
        lib.mpx_multiview_cameras(pf, pf, 1, None, 3, pf, s),
        lib.mpx_pose_update(pf, pf, None, pf, 1, pf, s),
        lib.mpx_pose_update(pf, pf, pf, pf, -1, pf, s),
        lib.mpx_normalize_T(None, 1, pf, s),
    ]
    assert all(rc != 0 for rc in refused), refused
    accepted = [  # n = 0 (or k = 0): nothing to do, nothing launched
        lib.mpx_pose_init_autodepth(None, 0, None, None, None, None, 0, None, s),
        lib.mpx_crop_geometry(None, 0, None, None, None, None, 0, 1.4, 480, 640, 240, 320, None, None, None, s),
        lib.mpx_topk_per_group(None, 0, 8, 2, None, s),
        lib.mpx_topk_per_group(None, 3, 8, 0, None, s),
        lib.mpx_multiview_cameras(None, None, 0, None, 0, None, s),
        lib.mpx_pose_update(None, None, None, None, 0, None, s),
        lib.mpx_normalize_T(None, 0, None, s),
    ]
    assert accepted == [0] * len(accepted)
    assert _launches() == n0


# ---------------------------------------------------------------------------------------------------------------------
# a NaN hypothesis through the crop + render path
# ---------------------------------------------------------------------------------------------------------------------
def test_nan_hypothesis_through_fused_and_split_crop_render():
    """A NaN pose gives NaN boxes_crop / K_crop (as in the reference).  roi_align's sample coordinates are then NaN; its
    index clamps keep every read inside the image (NaN fails the < -1 / > size tests, and converts to index 0).  The fused
    crop + render kernel and the split roi_align + render kernels write the same network input bit for bit, NaN
    included, and every other sample's slots are the same as in a batch without the NaN pose."""
    from megapose6d_b200.meshes import MeshDataBase
    from megapose6d_b200.renderer import BatchRenderer
    from tests import helpers

    ds, images, K = helpers.make_scene(3, seed=1, with_depth=True)
    db = MeshDataBase.from_object_ds(ds).batched().cuda()
    r = BatchRenderer(object_dataset=ds)
    n, h, w, c_pad = 5, 240, 320, 16
    act = _abi.act_dtype()
    labels = [ds[i % 3].label for i in range(n)]
    lab = r.mesh_db.label_ids(labels, DEV)
    nhwc4 = lib3d.image_to_nhwc4(images[:, :3].contiguous().cuda())
    im_idx = torch.zeros(n, dtype=torch.int32, device=DEV)
    TCO0 = torch.from_numpy(C.random_crop_case(5, 8, C.RANDOM_SHAPES[0], n=n)["TCO"]).cuda()
    TCO0[:, 2, 3] = 0.6

    def run(TCO):
        Kn = K.repeat(n, 1, 1).cuda()
        _, boxes, Kc = lib3d.crop_geometry(db.point_subset(200), db.label_ids(labels, DEV), TCO, Kn, TCO[:, :3, 3].contiguous(),
                                           (480, 640), (h, w))
        xa = torch.zeros(n, h // 2, w // 2, 4 * c_pad, device=DEV, dtype=act)
        xb = torch.full_like(xa, 7.0)
        _abi.check(_abi.lib().mpx_roi_align_fused(_abi.ptr(nhwc4), 1, 480, 640, _abi.ptr(im_idx), _abi.ptr(boxes), n, 3, h,
                                                  w, _abi.ptr(xa), c_pad, None, 0, _abi.stream_ptr()))
        r.render_fused(lab, TCO, Kc, 1, (h, w), xa, c_pad, 3, 6)
        r.render_crop_fused(lab, TCO, Kc, (h, w), nhwc4, im_idx, boxes, 3, xb, c_pad, 6)
        torch.cuda.synchronize()
        return boxes, Kc, xa.view(torch.int16), xb.view(torch.int16)

    TCO = TCO0.clone()
    TCO[2, 0, 1] = float("nan")
    boxes, Kc, xa, xb = run(TCO)
    assert torch.isnan(boxes[2]).all() and torch.isnan(Kc[2, :2]).any() and torch.isfinite(boxes[[0, 1, 3, 4]]).all()
    assert torch.equal(xa, xb)
    _, _, ya, _ = run(TCO0)
    keep = [0, 1, 3, 4]
    assert torch.equal(xa[keep], ya[keep])
