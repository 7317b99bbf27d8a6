"""The CPU rasteriser contract (oracle/raster_ref.c) against the float64 statement (oracle/raster_f64.py), on the cases of
tests/raster_cases.py: every pixel of the dyadic cases, every unambiguous pixel of the random ones; the margins are
neither vacuous nor violated; and the case list reaches both sides of every threshold of the device rasteriser's dispatch
and path choice."""
import numpy as np
import pytest

from oracle import raster_f64
from tests import raster_cases as rc

H100_SMS = 132


rendered = rc.rendered


DYADIC = rc.dyadic_cases()
RANDOM = rc.random_cases()


def _views(case):
    return range(len(case.labels))


@pytest.mark.parametrize("case", DYADIC, ids=lambda c: c.name)
def test_dyadic_cases_match_float64_on_every_pixel(case):
    drawn = 0
    for v in _views(case):
        m, T, K = case.view(v)
        d = raster_f64.displacement(m["verts"], T, K)
        assert (d[np.isfinite(d)] == 0).all()
        for flags in (1, 0):
            ref, f64 = rendered(case, v, flags)
            bad = ref["tri"] != f64["tri"]
            assert not bad.any(), f"{case.name} view {v}: {bad.sum()} pixels with another winner, first {np.argwhere(bad)[:3]}"
            res = raster_f64.check_outputs(f64, ref["rgb"], ref["nrm"], ref["depth"], quantised=bool(flags & 1),
                                           mask=np.ones((case.h, case.w), bool))
            assert all(n == 0 for n, _ in res.values()), (case.name, v, flags, res)
        drawn += (f64["tri"] >= 0).sum()
    assert drawn > 0


def test_dyadic_cases_see_their_edges():
    """The near-plane patches are drawn at 0.1f and just beyond, rejected just before; the far-plane ones drawn at 10.0f
    and just before, rejected just beyond; shared edges go to the lower index; of the two coplanar duplicates the lower
    index wins; at z = 2^-10 the triangle is drawn, at the next depth below it is not."""
    for near in (True, False):
        case = rc.depth_window_case(near)
        drawn = [(rendered(case, v)[1]["tri"] >= 0).sum() for v in range(3)]
        assert drawn == ([0, 25, 25] if near else [25, 25, 0]), drawn
        assert all(drawn[v] == (rendered(case, v)[0]["tri"] >= 0).sum() for v in range(3))
    fan = DYADIC[0]
    tri = rendered(fan, 0)[1]["tri"]
    ids = set(np.unique(tri).tolist())
    assert 14 not in ids and 41 in ids and 42 not in ids  # face 13's copy (14) loses; face 40's copy (40) wins over it
    pm = rendered(DYADIC[3], 0)[1]["tri"]
    assert set(np.unique(pm).tolist()) == {-1, 0}


@pytest.mark.parametrize("case", RANDOM, ids=lambda c: c.name)
def test_random_cases_match_float64_on_unambiguous_pixels(case):
    for v in _views(case):
        ref, f64 = rendered(case, v)
        amb = f64["amb"]
        bad = (ref["tri"] != f64["tri"]) & ~amb
        assert not bad.any(), f"{case.name} view {v}: {bad.sum()} unambiguous pixels with another winner"
        res = raster_f64.check_outputs(f64, ref["rgb"], ref["nrm"], ref["depth"])
        assert all(n == 0 for n, _ in res.values()), (case.name, v, res)
        covered = (f64["tri"] >= 0) | (ref["tri"] >= 0)
        if case.name != "random_clamp" and covered.sum() > 200:
            assert amb[covered].mean() < 0.1, f"{case.name}: {amb[covered].mean():.3f} of the covered pixels ambiguous"


def test_margins_are_tight_on_a_mesh():
    """On the 10k-triangle mesh: under 5 % of the covered pixels are ambiguous, the colour bound is below one 8-bit level on
    99 % and the normal bound on 60 % of the unambiguous covered pixels (the texture's slope is 1 per unit of normal, 31 at
    its wrap), and the float channels stay within their bounds."""
    case = RANDOM[0]
    for v in _views(case):
        ref, f64 = rendered(case, v)
        cov = f64["tri"] >= 0
        ok = cov & ~f64["amb"]
        assert cov.sum() > 5000 and f64["amb"][cov].mean() < 0.05
        assert (f64["bound_rgb"].max(0)[ok] < 1 / 255).mean() > 0.99
        assert (f64["bound_nrm"].max(0)[ok] < 1 / 255).mean() > 0.6
        ref0, f640 = rendered(case, v, flags=0)
        res = raster_f64.check_outputs(f640, ref0["rgb"], ref0["nrm"], ref0["depth"], quantised=False)
        assert all(n == 0 for n, _ in res.values()), res


def test_clamp_domain():
    """Vertices projected beyond 2^20 px are moved onto the clamp.  Their triangles' coverage then differs from float64 on
    some pixels, and every such pixel lies inside the displacement-derived exclusion (the contract's domain: the float64
    statement holds for triangles whose vertices project within the clamp)."""
    case = RANDOM[-1]
    ref, f64 = rendered(case, 0)
    assert f64["clamped"].sum() >= 6
    differ = ref["tri"] != f64["tri"]
    assert differ.any() and f64["amb"][differ].all()
    clamped_tris = np.nonzero(f64["clamped"][case.meshes[0]["faces"]].any(1))[0]
    assert np.isin(ref["tri"][differ], clamped_tris).any() or np.isin(f64["tri"][differ], clamped_tris).any()


@pytest.mark.parametrize("case", DYADIC + RANDOM, ids=lambda c: c.name)
def test_displacement_bound(case):
    """|snapped - float64| <= half a sub-pixel per axis plus the fp32 error of the projection, for every projectable
    vertex inside the clamp; 0 on dyadic cases."""
    for v in _views(case):
        m, T, K = case.view(v)
        P, u, vv, ok = raster_f64.project_f64(m["verts"], T, K)
        X, Y, _, behind = raster_f64.snap_f32(m["verts"], T, K)
        d = raster_f64.displacement(m["verts"], T, K)
        live = ok & ~behind & (np.abs(u) < 2 ** 20) & (np.abs(vv) < 2 ** 20)
        A = np.abs(np.asarray(m["verts"], np.float64)) @ np.abs(np.asarray(T, np.float64)[:3, :3]).T + np.abs(T[:3, 3])
        z = P[:, 2]
        ex = 8 * raster_f64.U * (abs(K[0, 0]) * (A[:, 0] + np.abs(P[:, 0] / z) * A[:, 2]) / z + np.abs(u) + abs(K[0, 2]))
        ey = 8 * raster_f64.U * (abs(K[1, 1]) * (A[:, 1] + np.abs(P[:, 1] / z) * A[:, 2]) / z + np.abs(vv) + abs(K[1, 2]))
        bound = np.hypot(1 / 512 + ex, 1 / 512 + ey)
        assert (d[live] <= bound[live]).all()
        if case.dyadic:
            assert (d[live] == 0).all()


def _observe(cases, sm=H100_SMS):
    obs = []
    for case in cases:
        s = case.sm_limit or sm
        for n in case.batches:
            for mode in (7, 2, 3):
                obs.append((case.name, n, mode, rc.triangle_paths(case, n, s, 2 * s, mode)))
    return obs


def test_case_list_reaches_both_sides_of_every_threshold():
    obs = _observe(DYADIC + RANDOM)
    paths = set().union(*(o["paths"] for *_, o in obs))
    assert {"walk32", "walk64", "queued", "queue-full", "tiled-small", "tiled-big", "strip-span"} <= paths, paths
    assert any(o["ext_le"] for *_, o in obs) and any(o["ext_gt_x"] for *_, o in obs) and any(o["ext_gt_y"] for *_, o in obs)
    assert {1023, 1024, 1025} <= set().union(*(o["area"] for *_, o in obs))
    # exactly 2048 in one scatter CTA, 2304 in another (queue case under the 16-SM limit, one view); 4352 in each CTA of
    # the untiled kernel at 32 views
    qc = RANDOM[1]
    d = rc.triangle_paths(qc, 1, 16, 32, 7)
    assert d["dispatch"] == dict(kernel="scatter", parts=16) and {2048, 2304} <= d["queue"]
    d = rc.triangle_paths(qc, 32, 16, 32, 2)
    assert d["dispatch"]["kernel"] == "untiled" and d["dispatch"]["strips"] == 1 and d["queue"] == {4352}
    tiled = [o for *_, o in obs if o["dispatch"]["kernel"] == "tiled"]
    assert max(o["max_row"] for o in tiled) == 4094
    assert max(o["max_span"] for o in tiled) >= 3
    disp = {(name, n, mode): o["dispatch"] for name, n, mode, o in obs}
    assert disp[("random_tiled_4095x64", 17, 7)]["kernel"] == "tiled"
    assert disp[("random_untiled_4096x16", 17, 7)]["kernel"] == "untiled"
    assert disp[("random_strips_128", 17, 7)]["n_strips"] == 128 and disp[("random_strips_128", 17, 7)]["R"] == 16
    assert disp[("random_strips_129", 17, 7)]["kernel"] == "untiled"
    assert disp[("random_rows_16", 17, 7)]["R"] == 16 and disp[("random_rows_15", 17, 7)]["kernel"] == "untiled"
    assert disp[("random_1x320", 17, 7)]["kernel"] == "untiled" and disp[("random_240x1", 17, 7)]["kernel"] == "tiled"
    assert disp[("random_mesh_10k", 4, 7)] == dict(kernel="scatter", parts=33)
    assert disp[("random_37x53", 1, 7)] == dict(kernel="scatter", parts=40)
    # projectability edge and clamp
    pm = rc.proj_min_case()
    m, T, K = pm.view(0)
    _, _, _, behind = raster_f64.snap_f32(m["verts"], T, K)
    z = m["verts"][:, 2]
    assert not behind[z == np.float32(2 ** -10)].any() and behind[z == np.nextafter(np.float32(2 ** -10), np.float32(0))].all()
    cm = RANDOM[-1]
    X, Y, _, _ = raster_f64.snap_f32(cm.meshes[0]["verts"], cm.TCO[0], cm.K[0])
    assert (np.abs(X) == 2 ** 28).sum() >= 6


def test_untiled_grid_fits_workspace_after_sm_limit():
    """A mesh database created at 132 SMs holds 264 CTA slots.  After mpx_set_sm_limit(16) the workspace holds 32
    visibility buffers; the untiled grid of 4 views (16 strips each) was 64 CTAs, 32 past the workspace.  Capped at
    min(slots, 2 x SMs) it is 32.  The scene renderer's chunks follow the current SM count and always fit."""
    h, w, n = 64, 80, 4
    buffers = 2 * 16
    parent = rc.dispatch(h, w, n, 16, 2 * H100_SMS, mode=2, cap_slots=False)
    fixed = rc.dispatch(h, w, n, 16, 2 * H100_SMS, mode=2)
    assert parent["kernel"] == "untiled" and parent["grid"] == 64 > buffers
    assert fixed["grid"] == buffers and fixed["strips"] == 8
    for n in (1, 2, 3, 5, 31, 33, 300):
        assert rc.dispatch(h, w, n, 16, 2 * H100_SMS, mode=2)["grid"] <= buffers
