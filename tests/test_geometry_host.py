"""CPU checks of the float64 restatement of the hypothesis-geometry kernels (oracle/geometry_ref.py), of the dyadic case
builders (tests/geometry_cases.py) and of the device selections' NaN order."""
import numpy as np
import pandas as pd
import pytest
import torch

from megapose6d_b200.pose_estimator import best_per_group, order_desc_nan_last
from oracle import geometry_ref as G
from oracle import lib3d_ref as L
from tests import geometry_cases as C


def _t(a):
    return torch.as_tensor(np.asarray(a))


def _crop_lib3d_ref(c):
    """boxes_rend, boxes_crop, K_crop of the reference's functions (lib3d_ref, fp32 torch)."""
    pts = _t(c["points"])[_t(c["label_idx"]).long()]
    n = pts.shape[0]
    TCO, K, tCR = _t(c["TCO"]), _t(c["K"]), _t(c["tCR"])
    br = L.boxes_from_uv(L.project_points_robust(pts, K, TCO))
    img = torch.zeros(1, 3, *c["im_size"]).expand(n, -1, -1, -1)
    bc, _ = L.deepim_crops_robust(img, br, K, TCO, tCR, pts, c["out_size"], lamb=c["lamb"], return_crops=False)
    return br, bc, L.get_K_crop_resize(K, bc, c["out_size"])


def _rel_close(got, want, rtol):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    scale = np.maximum(np.abs(want), 1.0)
    assert np.array_equal(np.isnan(got), np.isnan(want))
    ok = np.isnan(want) | (np.abs(got - want) <= rtol * scale)
    assert ok.all(), np.abs(got - want)[~ok].max()


@pytest.mark.parametrize("n_pts", [1, 33, 257])
@pytest.mark.parametrize("shape", C.RANDOM_SHAPES[:2])
def test_restatement_matches_lib3d_ref(n_pts, shape):
    """The float64 restatement agrees with the reference's fp32 functions within fp32 rounding (a few ulp of the
    magnitudes involved: pixel coordinates ~1e3, translations ~1)."""
    c = C.random_crop_case(3, n_pts, shape, z_edges=True)
    got = G.crop_geometry(c["points"], c["label_idx"], c["TCO"], c["K"], c["tCR"], c["lamb"], c["im_size"], c["out_size"])
    br, bc, Kc = _crop_lib3d_ref(c)
    _rel_close(got["boxes_rend"], br, 1e-5)
    _rel_close(got["boxes_crop"], bc, 1e-5)
    _rel_close(got["K_crop"], Kc, 1e-5)
    p = C.random_pose_init_case(4, n_pts)
    want = L.TCO_init_from_boxes_autodepth_with_R(_t(p["bboxes"]), _t(p["points"])[_t(p["label_idx"]).long()], _t(p["K"]),
                                                  _t(p["R"]))
    _rel_close(G.pose_init(**p), want, 1e-5)
    u = C.random_pose_update_case(5, 64)
    _rel_close(G.pose_update(**u), L.update_pose(_t(u["TCO"]), _t(u["K_crop"]), _t(u["pose9"]), _t(u["tCR"])), 1e-5)
    T = C.random_normalize_case(6, 64)
    _rel_close(G.normalize_T(T), L.normalize_T(_t(T)), 1e-5)
    TCO = C.random_crop_case(7, 8, shape)["TCO"]
    tCR = TCO[:, :3, 3] + 0.003
    want = L.make_TCO_multiview(_t(TCO), _t(tCR), "TCO+front_3views", 4).numpy()
    _rel_close(G.multiview(TCO, tCR, L.VIEW_OFFSETS["TCO+front_3views"]).astype(np.float32), want, 1e-5)


def test_restatement_nan_matches_lib3d_ref():
    """A NaN in a pose: NaN boxes, NaN K_crop entries with the zeros kept, NaN translation of the initial pose -- in
    the restatement exactly where the reference's functions put them."""
    c = C.random_crop_case(8, 40, C.RANDOM_SHAPES[0])
    c["TCO"][1, 0, 0] = np.nan   # rotation: the rendering centre is NaN too
    c["TCO"][2, 1, 3] = np.nan   # translation
    c["TCO"][3, 2, 2] = np.inf
    c["tCR"][4, 2] = np.nan
    got = G.crop_geometry(c["points"], c["label_idx"], c["TCO"], c["K"], c["tCR"], c["lamb"], c["im_size"], c["out_size"])
    br, bc, Kc = _crop_lib3d_ref(c)
    for g, w in ((got["boxes_rend"], br), (got["boxes_crop"], bc), (got["K_crop"], Kc)):
        _rel_close(g, w, 1e-5)
    assert np.isnan(got["boxes_crop"][[1, 2, 3, 4]]).all() and np.isnan(got["boxes_rend"][[1, 2, 3]]).all()
    p = C.random_pose_init_case(9, 40)
    p["R"][2, 1, 1] = np.nan
    p["bboxes"][3, 0] = np.nan
    want = L.TCO_init_from_boxes_autodepth_with_R(_t(p["bboxes"]), _t(p["points"])[_t(p["label_idx"]).long()], _t(p["K"]),
                                                  _t(p["R"]))
    _rel_close(G.pose_init(**p), want, 1e-5)
    assert np.isnan(G.pose_init(**p)[[2, 3], :3, 3]).all()


def _dyadic_cases():
    for i, shape in enumerate(C.DYADIC_SHAPES):
        for n_pts in C.N_PTS:
            yield C.dyadic_crop_case(100 * i + n_pts, n_pts, shape)


def test_dyadic_operands_make_the_geometry_exact():
    """Every dyadic case evaluates to the same value in float32 as in float64: each intermediate is exact, so the result
    does not depend on rounding order or FMA contraction and the kernels must reproduce it bit for bit."""
    for c in _dyadic_cases():
        args = (c["points"], c["label_idx"], c["TCO"], c["K"], c["tCR"], c["lamb"], c["im_size"], c["out_size"])
        f32, f64 = G.crop_geometry(*args, dtype=np.float32), G.crop_geometry(*args)
        for k in f64:
            assert np.array_equal(f32[k].astype(np.float64), f64[k]), (k, c["im_size"], c["out_size"])
        # not degenerate: crop boxes of 16 px or more, scaled to the output size
        assert (f64["boxes_crop"][:, 2] - f64["boxes_crop"][:, 0] >= 16).all() and (f64["K_crop"][:, 0, 0] != c["K"][:, 0, 0]).any()
    for n_pts in C.N_PTS:
        p = C.dyadic_pose_init_case(n_pts, n_pts)
        assert np.array_equal(G.pose_init(**p, dtype=np.float32).astype(np.float64), G.pose_init(**p))
        p["bboxes"][1, 2] = p["bboxes"][1, 0] - 1  # x2 = x1 - 1: bb_dx = 0, z = inf (NaN for a single point: 0 / 0)
        f32, f64 = G.pose_init(**p, dtype=np.float32).astype(np.float64), G.pose_init(**p)
        assert np.array_equal(f32, f64, equal_nan=True) and not np.isfinite(f64[1, 2, 3])
    u = C.dyadic_pose_update_case(11)
    assert np.array_equal(G.pose_update(**u, dtype=np.float32).astype(np.float64), G.pose_update(**u))
    T = C.dyadic_normalize_case(12)
    assert np.array_equal(G.normalize_T(T, dtype=np.float32).astype(np.float64), G.normalize_T(T))
    # the update is not the identity: rotations change, translations move
    assert not np.array_equal(G.pose_update(**u)[:, :3, :3], u["TCO"][:, :3, :3])


def test_bounds_hold_for_an_fp32_evaluation():
    """The running error bound of geometry_ref.Bounded covers the plain fp32 evaluation of the same expressions (one
    of the fp32 evaluations it claims to bound), and is tight enough to mean something (within 2^10 ulp)."""
    for shape in C.RANDOM_SHAPES:
        for n_pts in (1, 129, 2000):
            c = C.random_crop_case(n_pts, n_pts, shape, z_edges=True)
            args = (c["points"], c["label_idx"], c["TCO"], c["K"], c["tCR"], c["lamb"], c["im_size"], c["out_size"])
            f32 = G.crop_geometry(*args, dtype=np.float32)
            b = G.crop_geometry_bounds(*args)
            for k, (v, e) in b.items():
                assert (np.abs(f32[k].astype(np.float64) - v) <= e).all(), k
                assert (e <= 2.0 ** -14 * np.maximum(np.abs(v), 1e3)).all(), k
    p = C.random_pose_init_case(3, 257)
    v, e = G.bounds_as_T(G.pose_init(**p, dtype="bounded"), 16)
    assert (np.abs(G.pose_init(**p, dtype=np.float32)[:, :3, 3] - v[:, :3, 3]) <= e[:, :3, 3]).all()
    u = C.random_pose_update_case(4)
    v, e = G.bounds_as_T(G.pose_update(**u, dtype="bounded"), 300)
    assert (np.abs(G.pose_update(**u, dtype=np.float32)[:, :3] - v[:, :3]) <= e[:, :3]).all()


def _pandas_head(logits, group, k):
    df = pd.DataFrame(dict(logit=np.asarray(logits, np.float64), group=np.asarray(group)))
    return df.sort_values("logit", ascending=False, kind="stable").groupby("group").head(k).index.to_numpy()


def selection_logits(seed: int, n: int) -> torch.Tensor:
    """Tie-heavy logits with NaN and +-inf."""
    rs = np.random.RandomState(seed)
    x = rs.randint(-3, 4, n).astype(np.float32)
    x[rs.rand(n) < 0.15] = np.nan
    x[rs.rand(n) < 0.05] = np.inf
    x[rs.rand(n) < 0.05] = -np.inf
    x[rs.rand(n) < 0.05] = -0.0
    return torch.as_tensor(x)


def test_device_selection_order_is_nan_last():
    """order_desc_nan_last / best_per_group (the fused pipeline's final pick) against pandas on tie-heavy logits with
    NaN, +-inf and -0; torch.sort(descending) alone would put NaN first."""
    for seed in range(20):
        x = selection_logits(seed, 97)
        want = np.argsort(-x.double().numpy(), kind="stable")
        assert np.array_equal(order_desc_nan_last(x).numpy(), want)
        group = torch.as_tensor(np.random.RandomState(seed).randint(0, 9, 97))
        group[:9] = torch.arange(9)
        assert np.array_equal(best_per_group(x, group, 9).numpy(), _pandas_head(x, group, 1))
    x = torch.tensor([float("nan"), 1.0, float("-inf"), float("nan"), float("-inf")])
    assert order_desc_nan_last(x).tolist() == [1, 2, 4, 0, 3]
    assert best_per_group(x, torch.tensor([0, 1, 0, 1, 2]), 3).tolist() == [1, 2, 4]
