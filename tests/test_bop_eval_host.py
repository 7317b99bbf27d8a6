"""BOP 2019 evaluation on the host: oracle/bop_ref.py against the stored outputs of the BOP toolkit itself, the product's
host scoring against the oracle on the same error tables, and the split reader against workloads/bop_split.py."""
from __future__ import annotations

import numpy as np
import pandas as pd
import pytest
import torch

from megapose6d_b200 import bop_eval
from oracle import bop_ref, pipeline_ref
from tests import helpers, scene_ref
from workloads import bop_split


def ref_meshes(models) -> pipeline_ref.RefMeshes:
    ids = sorted(models)
    ms = [models[o].with_defaults() for o in ids]
    return pipeline_ref.RefMeshes([f"obj_{o:06d}" for o in ids], [m.vertices * 1e-3 for m in ms],
                                  [m.vertex_normals for m in ms], [m.vertex_colors for m in ms], [m.faces for m in ms])


def host_scene_renderer():
    """workloads.bop_split renderer on tests/scene_ref.c (the CPU restatement of mpx_raster_render_scene)."""
    cache = {}

    def render(models, views, TCO, K, resolution):
        if "m" not in cache:
            cache["m"] = ref_meshes(models)
        out = scene_ref.render_scene(cache["m"], [[f"obj_{o:06d}" for o in v] for v in views], torch.from_numpy(TCO),
                                     torch.from_numpy(K), resolution, flags=1)
        return out["depths"][:, 0].numpy(), out["inst_id"].numpy()

    return render


def single_renderer(models):
    """oracle render callback: the C oracle's depth (metres) of one object."""
    meshes = ref_meshes(models)
    rr = pipeline_ref.RefRenderer(meshes)

    def render(obj_id, R, t_mm, K, shape):
        T = np.eye(4)
        T[:3, :3], T[:3, 3] = R, np.reshape(t_mm, 3) / 1000.0
        out = rr.render([f"obj_{obj_id:06d}"], torch.from_numpy(T).float()[None], torch.from_numpy(K).float()[None], None,
                        tuple(shape), render_depth=True)
        return out["depths"][0, 0].numpy()

    return render


MODELS, INFO = bop_split.models_and_info()


def poses(n, seed):
    r = np.random.RandomState(seed)
    out = []
    for _ in range(n):
        R = bop_split.random_rotation(r)
        t = np.array([r.uniform(-30, 30), r.uniform(-30, 30), r.uniform(400, 700)])
        out.append((R, t.reshape(3, 1)))
    return out


# ------------------------------------------------------------------------------------------------ oracle vs the toolkit
def test_symmetries_match_toolkit():
    def compute():
        tk = helpers_toolkit()
        out = {}
        for o in (1, 2, 3):
            s = tk.misc.get_symmetry_transformations(INFO[o], 0.01)
            out[f"obj{o}"] = np.stack([np.concatenate([x["R"].reshape(9), x["t"].reshape(3)]) for x in s])
        return out

    want = helpers.reference_outputs("bop_eval_symmetries", compute)
    assert want["obj3"].shape == (628, 12) and want["obj2"].shape == (4, 12) and want["obj1"].shape == (1, 12)
    for o in (1, 2, 3):
        got = np.stack([np.concatenate([R.reshape(9), t.reshape(3)]) for R, t in bop_ref.symmetries(INFO[o])])
        np.testing.assert_array_equal(got, want[f"obj{o}"].numpy())
        np.testing.assert_allclose(bop_eval.symmetry_transformations(INFO[o]), want[f"obj{o}"].numpy(), rtol=0, atol=1e-15)


def helpers_toolkit():
    from oracle import bop_toolkit

    return bop_toolkit.load()


def _point_cases():
    cases = []
    ps = poses(8, 1)
    for o in (1, 2, 3):
        for k in range(3):
            R_g, t_g = ps[k]
            R_e = ps[k + 3][0] if k else R_g
            t_e = t_g + np.array([[2.0], [-1.0], [3.0]]) * k
            if o == 3 and k == 2:  # a symmetric flip of the gt pose: errors ~0 under MSSD / MSPD
                Rs, ts = bop_ref.symmetries(INFO[3])[400]
                R_e, t_e = R_g.dot(Rs), R_g.dot(ts) + t_g
            cases.append((o, R_e, t_e, R_g, t_g))
    return cases


K0 = np.array([[572.4, 0, 325.3], [0, 573.6, 242.0], [0, 0, 1]])


def test_point_errors_match_toolkit():
    cases = _point_cases()

    def compute():
        tk = helpers_toolkit()
        out = {k: [] for k in ("mssd", "mspd", "add", "adi")}
        for o, R_e, t_e, R_g, t_g in cases:
            pts = np.asarray(MODELS[o].vertices, np.float64)
            syms = tk.misc.get_symmetry_transformations(INFO[o], 0.01)
            out["mssd"].append(tk.pose_error.mssd(R_e, t_e, R_g, t_g, pts, syms))
            out["mspd"].append(tk.pose_error.mspd(R_e, t_e, R_g, t_g, K0, pts, syms))
            out["add"].append(tk.pose_error.add(R_e, t_e, R_g, t_g, pts))
            out["adi"].append(tk.pose_error.adi(R_e, t_e, R_g, t_g, pts))
        return {k: np.asarray(v) for k, v in out.items()}

    want = helpers.reference_outputs("bop_eval_point_errors", compute)
    for i, (o, R_e, t_e, R_g, t_g) in enumerate(cases):
        pts = np.asarray(MODELS[o].vertices, np.float64)
        syms = bop_ref.symmetries(INFO[o])
        got = dict(mssd=bop_ref.mssd(R_e, t_e, R_g, t_g, pts, syms), mspd=bop_ref.mspd(R_e, t_e, R_g, t_g, K0, pts, syms),
                   add=bop_ref.add(R_e, t_e, R_g, t_g, pts), adi=bop_ref.adi(R_e, t_e, R_g, t_g, pts))
        for k, v in got.items():
            assert v == pytest.approx(float(want[k][i]), rel=1e-12, abs=1e-9), (k, i)
    assert float(want["mssd"][-1]) < 1e-9 and float(want["mspd"][-1]) < 1e-9  # the flip is free under symmetries


def _vsd_cases():
    """(depth_test mm, depth_est mm, depth_gt mm, K, diameter): rendered cases with noise and holes, an empty union, and
    hand-made images whose principal-point column puts differences exactly on delta and on a tau."""
    h, w = 48, 64
    K = np.array([[70.0, 0, 20.0], [0, 70.0, 17.0], [0, 0, 1]])
    render = single_renderer(MODELS)
    cases = []
    ps = poses(4, 2)
    r = np.random.RandomState(3)
    for o in (1, 2):
        (R_g, t_g), (R_e, _) = ps[o], ps[o + 1]
        t_e = t_g + np.array([[4.0], [-3.0], [10.0]])
        dg = bop_ref.render_mm(render, o, R_g, t_g.reshape(3), K, (h, w))
        de = bop_ref.render_mm(render, o, R_e if o == 2 else R_g, t_e.reshape(3), K, (h, w))
        test = np.where(dg > 0, dg, 900.0) + r.normal(0, 2.0, (h, w))
        test[r.uniform(size=(h, w)) < 0.1] = 0  # holes
        test[:, : w // 4] -= 200.0  # an occluder in front of part of the object
        test = (np.round(test / 0.1) * np.float32(0.1)).astype(np.float32)
        cases.append((test, de, dg, K, INFO[o]["diameter"]))
    z = np.zeros((h, w), np.float32)
    cases.append((np.full((h, w), 500.0, np.float32), z, z, K, 100.0))  # empty union
    dg = np.zeros((h, w), np.float32)
    de = np.zeros((h, w), np.float32)
    test = np.zeros((h, w), np.float32)
    cx = 20  # X = 0 in this column, and Y = 0 in row 17: there the distance is the depth itself
    dg[:, cx] = 500.0
    test[:, cx] = 485.0  # dist_gt - dist_test == delta exactly: visible
    test[::3, cx] = 484.0  # just behind: not visible
    de[:, cx] = 490.0  # |dist_gt - dist_est| / 100 == 0.1, a tau exactly
    de[2::4, cx] = 470.0
    cases.append((test, de, dg, K, 100.0))
    return cases


def test_vsd_matches_toolkit():
    cases = _vsd_cases()

    def compute():
        tk = helpers_toolkit()

        class Stub:  # the toolkit's renderer interface, returning the case's depth images (mm)
            def __init__(self, de, dg):
                self.seq = [de, dg]

            def render_object(self, obj_id, R, t, fx, fy, cx, cy):
                return {"depth": self.seq.pop(0)}

        out = []
        for test, de, dg, K, diam in cases:
            out.append(tk.pose_error.vsd(np.eye(3), np.zeros((3, 1)), np.eye(3), np.zeros((3, 1)), test, K, 15,
                                         bop_ref.VSD_TAUS, True, diam, Stub(de, dg), 1, "step"))
        return {"vsd": np.asarray(out)}

    want = helpers.reference_outputs("bop_eval_vsd", compute)["vsd"].numpy()
    for i, (test, de, dg, K, diam) in enumerate(cases):
        got, counts = bop_ref.vsd_from_depths(test, de, dg, K, 15, bop_ref.VSD_TAUS, diam, return_counts=True)
        np.testing.assert_array_equal(np.asarray(got), want[i])
    assert (want[2] == 1.0).all()  # empty union
    assert 0 < want[0].min() and want[0].max() <= 1.0


def test_sphere_gating_and_matching_match_toolkit():
    spheres = [(20.0, np.array([0, 0, 500.0]), np.array([30.0, 0, 500.0])),
               (20.0, np.array([0, 0, 500.0]), np.array([80.0, 0, 500.0])),
               (20.0, np.array([0, 0, 0.0]), np.array([0, 0, 500.0])),
               (20.0, np.array([40.0, 0, 500.0]), np.array([0, 0, 500.0]))]
    # tied scores, invalid gts, errors on the threshold
    errs = [dict(est_id=0, score=0.5, errors={0: [0.1], 1: [0.05], 2: [0.01]}),
            dict(est_id=1, score=0.9, errors={0: [0.2], 1: [0.3], 2: [0.01]}),
            dict(est_id=2, score=0.5, errors={0: [0.3], 1: [0.02], 2: [0.2]}),
            dict(est_id=3, score=0.1, errors={0: [0.0], 1: [0.0], 2: [0.0]})]
    valid = [True, True, False]

    def compute():
        tk = helpers_toolkit()
        gate = [tk.misc.overlapping_sphere_projections(r, a, b) for r, a, b in spheres]
        ms = tk.pose_matching.match_poses(errs, [0.3], -1, valid)
        matches = [dict(scene_id=1, im_id=0, obj_id=1, gt_id=g, est_id=-1, valid=v) for g, v in enumerate(valid)]
        for m in ms:
            matches[m["gt_id"]]["est_id"] = m["est_id"]
        sc = tk.score.calc_localization_scores([1], [1], matches, -1, do_print=False)
        return dict(gate=np.asarray(gate), est=np.asarray([m["est_id"] for m in ms]),
                    gt=np.asarray([m["gt_id"] for m in ms]), recall=np.asarray(sc["recall"]))

    want = helpers.reference_outputs("bop_eval_matching", compute)
    assert [bop_ref.spheres_overlap(r, a, b) for r, a, b in spheres] == want["gate"].tolist()
    assert [bop_eval.spheres_projections_overlap(r, a, b) for r, a, b in spheres] == want["gate"].tolist()
    flat = [dict(e, errors={g: v[0] for g, v in e["errors"].items()}) for e in errs]
    ms = bop_ref.match_poses(flat, 0.3, valid)
    assert [m["est_id"] for m in ms] == want["est"].tolist() and [m["gt_id"] for m in ms] == want["gt"].tolist()
    matches = [dict(gt_id=g, est_id=-1, valid=v) for g, v in enumerate(valid)]
    for m in ms:
        matches[m["gt_id"]]["est_id"] = m["est_id"]
    assert bop_ref.localization_recall(matches) == float(want["recall"])


# ----------------------------------------------------------------------------------- the product's host side vs the oracle
@pytest.fixture(scope="module")
def split_dir(tmp_path_factory):
    root = tmp_path_factory.mktemp("bop")
    gt = bop_split.write_split(root, host_scene_renderer(), n_scenes=2, n_images=2, h=96, w=128)
    return root, gt


def estimates(gt, seed=0):
    """perturbed, duplicated (tied scores), missing and wrong-object estimates, with per-image times"""
    r = np.random.RandomState(seed)
    out = []
    for (s, i), inst in gt.items():
        for k, (o, R, t) in enumerate(inst):
            if (s + i + k) % 5 == 3:
                continue  # missing
            t_e = t + r.normal(0, 4.0, 3) * (k % 3)
            out.append(dict(scene_id=s, im_id=i, obj_id=o, score=round(r.uniform(), 1), R=R, t=t_e, time=0.25 + s))
            if k % 2 == 0:  # a duplicate with a tied score and a worse pose
                out.append(dict(scene_id=s, im_id=i, obj_id=o, score=out[-1]["score"],
                                R=bop_split.random_rotation(r), t=t_e + 30.0, time=0.25 + s))
        out.append(dict(scene_id=s, im_id=i, obj_id=3 if inst[0][0] != 3 else 1, score=0.99, R=inst[0][1], t=inst[0][2],
                        time=0.25 + s))
    return out


def test_split_reader_roundtrip(split_dir):
    root, gt = split_dir
    sp = bop_eval.load_split(root)
    assert sorted(sp.models) == [1, 2, 3] and sp.models_info[3]["symmetries_continuous"][0]["axis"] == [0, 0, 1]
    for (s, i), inst in gt.items():
        got = sp.scene_gt[s][i]
        assert [g["obj_id"] for g in got] == [o for o, _, _ in inst]
        np.testing.assert_array_equal(np.reshape(got[1]["cam_R_m2c"], (3, 3)), inst[1][1])
        assert sp.scene_camera[s][i]["depth_scale"] == 0.1
        d = sp.depth(s, i)
        assert d.dtype == np.uint16 and d.shape == (96, 128) and (d == 0).any() and d.max() > 4000
        assert all(x["px_count_all"] > 0 and 0 <= x["visib_fract"] <= 1 for x in sp.scene_gt_info[s][i])
    assert any(x["visib_fract"] < 0.95 for v in sp.scene_gt_info.values() for im in v.values() for x in im)  # occlusion
    np.testing.assert_array_equal(sp.models[2].vertices, np.round(bop_split.box().vertices, 6))


def test_host_scoring_matches_oracle(split_dir):
    root, gt = split_dir
    sp = bop_eval.load_split(root)
    ests = bop_eval.normalize_results(estimates(gt))
    render = single_renderer(sp.models)
    rows = bop_ref.calc_errors(sp, ests, render)
    want = bop_ref.evaluate(sp, ests, render)
    sel = bop_eval.select_estimates(sp, ests)
    assert [(e["scene_id"], e["im_id"], e["obj_id"], e["est_id"]) for e in sel] == \
        list(dict.fromkeys((r["scene_id"], r["im_id"], r["obj_id"], r["est_id"]) for r in rows))
    df = pd.DataFrame({k: [r[k] for r in rows] for k in ("scene_id", "im_id", "obj_id", "est_id", "gt_id", "score")})
    for k in range(len(bop_eval.VSD_TAUS)):
        df[f"vsd_{k}"] = [r["vsd"][k] for r in rows]
    df["mssd"] = [r["mssd"] for r in rows]
    df["mspd"] = [r["mspd"] for r in rows]
    got = bop_eval.score_errors(sp, df, ests)
    assert got == want
    assert 0 < want["bop19_average_recall"] < 1 and want["bop19_average_time_per_image"] == pytest.approx(1.75)


def test_selection_ties_and_inst_count():
    sp = bop_eval.BopSplit(None, "test", {}, {}, [dict(scene_id=1, im_id=0, obj_id=2, inst_count=2)])
    ests = [dict(scene_id=1, im_id=0, obj_id=2, score=s, n=n) for n, s in enumerate([0.5, 0.9, 0.5, 0.5, 0.1])]
    ests.append(dict(scene_id=1, im_id=0, obj_id=3, score=1.0, n=9))  # not a target
    sel = bop_eval.select_estimates(sp, ests)
    assert [(e["n"], e["est_id"]) for e in sel] == [(1, 1), (0, 0)]


def test_time_per_image():
    e = [dict(scene_id=1, im_id=0, time=1.0), dict(scene_id=1, im_id=0, time=1.0005), dict(scene_id=1, im_id=1, time=3.0)]
    assert bop_eval.average_time_per_image(e) == 2.0
    assert bop_eval.average_time_per_image(e + [dict(scene_id=2, im_id=0, time=-1)]) == -1.0
    with pytest.raises(ValueError):
        bop_eval.average_time_per_image(e + [dict(scene_id=1, im_id=1, time=3.5)])
