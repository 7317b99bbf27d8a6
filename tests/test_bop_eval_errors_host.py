"""The BOP toolkit's other pose errors on the host: oracle/bop_other_ref.py's proj, re, te, cus, multi-element matching and
localization scores against the stored outputs of the toolkit itself, and the product's host scoring of ad, add, adi,
cus, proj, re, te and rete against the oracle on a synthetic split."""
from __future__ import annotations

import numpy as np
import pandas as pd
import pytest

from megapose6d_b200 import bop_eval
from oracle import bop_other_ref, bop_ref
from tests import helpers
from tests.test_bop_eval_host import K0, MODELS, helpers_toolkit, host_scene_renderer, poses, single_renderer
from workloads import bop_split

NEW_TYPES = ("ad", "add", "adi", "cus", "proj", "re", "te", "rete")


def _turn(axis, ang):
    a = np.zeros(3)
    a[axis] = 1.0
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * K.dot(K)


def _pose_cases():
    """(obj_id, R_e, t_e, R_g, t_g): identical poses, 180-degree turns, rotations whose cosine falls just outside
    [-1, 1], and random pairs."""
    ps = poses(6, 7)
    R0, t0 = ps[0]
    cases = [(1, R0, t0, R0, t0)]
    for axis in range(3):  # 180 degrees about each axis, composed with a random gt rotation
        cases.append((2, R0.dot(_turn(axis, np.pi)), t0 + 1.0, R0, t0))
    cases.append((1, np.eye(3) * (1 + 4e-16), t0, np.eye(3), t0))  # cosine just above 1
    cases.append((3, np.diag([1.0, -1.0, -1.0]) * (1 + 4e-16), t0, np.eye(3), t0 + 2.0))  # just below -1
    for k in range(1, 5):
        (R_g, t_g), (R_e, _) = ps[k], ps[(k + 1) % 6]
        cases.append((1 + k % 3, R_e, t_g + np.array([[3.0], [-2.0], [15.0]]) * k, R_g, t_g))
    return cases


def _pose_compute():
    tk = helpers_toolkit()
    out = {k: [] for k in ("proj", "re", "te")}
    for o, R_e, t_e, R_g, t_g in _pose_cases():
        pts = np.asarray(MODELS[o].vertices, np.float64)
        out["proj"].append(tk.pose_error.proj(R_e, t_e, R_g, t_g, K0, pts))
        out["re"].append(tk.pose_error.re(R_e, R_g))
        out["te"].append(tk.pose_error.te(t_e, t_g))
    return {k: np.asarray(v) for k, v in out.items()}


def stored():
    """The toolkit's outputs for every case of this file (one stored file)."""
    return helpers.reference_outputs("bop_eval_more_errors", lambda: dict(
        _pose_compute(), **_cus_compute(), **_matching_compute(), **_scores_compute()))


def test_pose_errors_match_toolkit():
    cases = _pose_cases()
    want = stored()
    for i, (o, R_e, t_e, R_g, t_g) in enumerate(cases):
        pts = np.asarray(MODELS[o].vertices, np.float64)
        assert bop_other_ref.proj(R_e, t_e, R_g, t_g, K0, pts) == pytest.approx(float(want["proj"][i]), rel=1e-12, abs=1e-9)
        assert bop_other_ref.re(R_e, R_g) == pytest.approx(float(want["re"][i]), rel=0, abs=2e-6), i
        assert bop_other_ref.te(t_e, t_g) == pytest.approx(float(want["te"][i]), rel=1e-12, abs=0)
    re = want["re"].numpy()
    assert re[0] == 0.0 and (np.abs(re[1:4] - 180.0) < 1e-6).all()
    assert re[4] == 0.0 and re[5] == 180.0  # clipped cosines
    assert float(want["proj"][0]) == 0.0 and float(want["te"][0]) == 0.0


# --------------------------------------------------------------------------------------------------------------- cus
def _cus_cases():
    """(depth_est mm, depth_gt mm): C-oracle renders, disjoint silhouettes, an empty union, one inside the other."""
    h, w = 48, 64
    K = np.array([[70.0, 0, 20.0], [0, 70.0, 17.0], [0, 0, 1]])
    render = single_renderer(MODELS)
    ps = poses(4, 5)
    cases = []
    for o in (1, 2):
        (R_g, t_g), (R_e, _) = ps[o], ps[o + 1]
        dg = bop_ref.render_mm(render, o, R_g, t_g.reshape(3), K, (h, w))
        de = bop_ref.render_mm(render, o, R_e, (t_g + np.array([[6.0], [-4.0], [10.0]])).reshape(3), K, (h, w))
        cases.append((de, dg))
    a = np.zeros((h, w), np.float32)
    b = np.zeros((h, w), np.float32)
    a[5:15, 5:15], b[30:40, 40:50] = 500.0, 600.0
    cases.append((a, b))  # disjoint: error 1
    cases.append((np.zeros((h, w), np.float32), np.zeros((h, w), np.float32)))  # empty union: error 1
    c = np.zeros((h, w), np.float32)
    c[10:30, 10:40] = 700.0
    d = np.zeros((h, w), np.float32)
    d[15:22, 12:19] = 650.0
    cases.append((d, c))  # the estimate inside the gt
    cases.append((c, d))
    return cases


def _cus_compute():
    tk = helpers_toolkit()

    class Stub:  # the toolkit's renderer interface, returning the case's depth images (mm)
        def __init__(self, de, dg):
            self.seq = [de, dg]

        def render_object(self, obj_id, R, t, fx, fy, cx, cy):
            return {"depth": self.seq.pop(0)}

    K = np.array([[70.0, 0, 20.0], [0, 70.0, 17.0], [0, 0, 1]])
    return {"cus": np.asarray([tk.pose_error.cus(np.eye(3), np.zeros((3, 1)), np.eye(3), np.zeros((3, 1)), K, Stub(de, dg), 1)
                               for de, dg in _cus_cases()])}


def test_cus_matches_toolkit():
    want = stored()["cus"].numpy()
    for i, (de, dg) in enumerate(_cus_cases()):
        got, counts = bop_other_ref.cus_from_depths(de, dg, return_counts=True)
        assert got == want[i], (i, got, want[i])
    assert want[2] == 1.0 and want[3] == 1.0
    assert want[4] == want[5] == 1.0 - 49 / 600.0
    assert 0 < want[0] < 1 and 0 < want[1] < 1


# ---------------------------------------------------------------------------------------------------------- matching
# two-element (rete) errors: better in one element and worse in the other, errors on a threshold, tied scores
RETE_ERRS = [dict(est_id=0, score=0.5, errors={0: [1.0, 4.0], 1: [0.5, 4.5], 2: [0.1, 0.1], 3: [2.0, 2.0]}),
             dict(est_id=1, score=0.9, errors={0: [5.0, 1.0], 1: [4.9, 4.9], 2: [0.2, 0.2], 3: [3.0, 1.0]}),
             dict(est_id=2, score=0.5, errors={0: [2.0, 3.0], 1: [1.0, 5.0], 2: [0.0, 0.0], 3: [1.0, 3.0]}),
             dict(est_id=3, score=0.1, errors={0: [0.0, 0.0], 1: [0.0, 0.0], 2: [0.0, 0.0], 3: [4.0, 4.0]}),
             dict(est_id=4, score=0.5, errors={0: [3.0, 0.5], 1: [0.1, 0.1], 2: [0.0, 0.0], 3: [0.5, 4.99]})]
RETE_VALID = [True, True, False, True]
RETE_THS = [(5.0, 5.0), (2.0, 5.0), (5.0, 3.0)]


def _matching_compute():
    tk = helpers_toolkit()
    out = {}
    for k, th in enumerate(RETE_THS):
        ms = tk.pose_matching.match_poses(RETE_ERRS, list(th), -1, RETE_VALID)
        out[f"rete_est_{k}"] = np.asarray([m["est_id"] for m in ms])
        out[f"rete_gt_{k}"] = np.asarray([m["gt_id"] for m in ms])
    return out


def test_multi_element_matching_matches_toolkit():
    want = stored()
    rows = [dict(scene_id=1, im_id=0, obj_id=1, est_id=e["est_id"], gt_id=g, score=e["score"])
            for e in RETE_ERRS for g in e["errors"]]
    errs = np.array([v for e in RETE_ERRS for v in e["errors"].values()])
    for k, th in enumerate(RETE_THS):
        ms = bop_other_ref.match_poses_multi(RETE_ERRS, th, RETE_VALID)
        assert [m["est_id"] for m in ms] == want[f"rete_est_{k}"].tolist(), k
        assert [m["gt_id"] for m in ms] == want[f"rete_gt_{k}"].tolist(), k
        got = bop_eval.match_errors(rows, errs, th, {(1, 0): RETE_VALID})
        assert got == {(1, 0, g) for g in want[f"rete_gt_{k}"].tolist()}, k
    assert len(want["rete_gt_0"]) >= 2
    # one element: the same rule as recall()'s
    one = bop_eval.match_errors(rows, errs[:, :1], [2.0], {(1, 0): RETE_VALID})
    assert one == {(1, 0, m["gt_id"]) for m in bop_ref.match_poses(
        [dict(e, errors={g: v[0] for g, v in e["errors"].items()}) for e in RETE_ERRS], 2.0, RETE_VALID)}
    with pytest.raises(ValueError):
        bop_eval.match_errors(rows, errs, [5.0], {(1, 0): RETE_VALID})


# ---------------------------------------------------------------------------------------------------------- scores
# gts of three target images in scenes 1 and 2; scene 3 has no targets, object 4 no instances
SCORE_MATCHES = [dict(scene_id=1, im_id=0, obj_id=1, gt_id=0, est_id=0, valid=True),
                 dict(scene_id=1, im_id=0, obj_id=2, gt_id=1, est_id=-1, valid=True),
                 dict(scene_id=1, im_id=0, obj_id=2, gt_id=2, est_id=1, valid=True),
                 dict(scene_id=1, im_id=1, obj_id=3, gt_id=0, est_id=2, valid=False),
                 dict(scene_id=1, im_id=1, obj_id=1, gt_id=1, est_id=-1, valid=True),
                 dict(scene_id=2, im_id=0, obj_id=3, gt_id=0, est_id=4, valid=True),
                 dict(scene_id=2, im_id=0, obj_id=1, gt_id=1, est_id=-1, valid=False)]
SCORE_SCENES, SCORE_OBJS = [1, 2, 3], [1, 2, 3, 4]
SCORE_KEYS = ("recall", "mean_obj_recall", "mean_scene_recall", "gt_count", "targets_count", "tp_count")


def _scores_compute():
    tk = helpers_toolkit()
    sc = tk.score.calc_localization_scores(SCORE_SCENES, SCORE_OBJS, [dict(m) for m in SCORE_MATCHES], -1, do_print=False)
    out = {f"score_{k}": np.asarray(sc[k]) for k in SCORE_KEYS}
    out["score_obj_recalls"] = np.asarray([sc["obj_recalls"][o] for o in SCORE_OBJS])
    out["score_scene_recalls"] = np.asarray([sc["scene_recalls"][s] for s in SCORE_SCENES])
    return out


def _want_scores(want) -> dict:
    out = {k: want[f"score_{k}"].item() for k in SCORE_KEYS}
    out["obj_recalls"] = dict(zip(SCORE_OBJS, want["score_obj_recalls"].tolist()))
    out["scene_recalls"] = dict(zip(SCORE_SCENES, want["score_scene_recalls"].tolist()))
    return out


def test_localization_scores_match_toolkit(tmp_path):
    want = _want_scores(stored())
    assert want["obj_recalls"][4] == 0.0 and want["scene_recalls"][3] == 0.0
    assert 0 < want["mean_obj_recall"] < want["recall"]
    got = bop_other_ref.localization_scores(SCORE_SCENES, SCORE_OBJS, SCORE_MATCHES)
    assert got == dict(want, gt_count=int(want["gt_count"]), targets_count=int(want["targets_count"]),
                       tp_count=int(want["tp_count"]))
    # the product's scores from the same matches: a split whose scene 3 is a directory without targets
    for s in SCORE_SCENES:
        (tmp_path / "test" / f"{s:06d}").mkdir(parents=True)
    scene_gt, valid, matched = {}, {}, set()
    for m in SCORE_MATCHES:
        scene_gt.setdefault(m["scene_id"], {}).setdefault(m["im_id"], []).append(dict(obj_id=m["obj_id"]))
        valid.setdefault((m["scene_id"], m["im_id"]), []).append(m["valid"])
        if m["est_id"] != -1:
            matched.add((m["scene_id"], m["im_id"], m["gt_id"]))
    sp = bop_eval.BopSplit(tmp_path, "test", {o: {} for o in SCORE_OBJS}, {},
                           [dict(scene_id=1, im_id=0, obj_id=1, inst_count=1)], scene_gt=scene_gt)
    assert bop_eval.split_scene_ids(sp) == SCORE_SCENES
    assert bop_eval.localization_scores(sp, matched, valid) == got


# ----------------------------------------------------------------------------------- the product's host side vs the oracle
@pytest.fixture(scope="module")
def split_dir(tmp_path_factory):
    """two scenes of (sphere, box, box) and an empty third scene: the cylinder and scene 3 have no targets"""
    root = tmp_path_factory.mktemp("bop_more")
    gt = bop_split.write_split(root, host_scene_renderer(), n_scenes=2, n_images=2, h=96, w=128, objects=(1, 2, 2), seed=4)
    (root / "test" / "000003").mkdir()
    return root, gt


def estimates(gt, seed=0):
    """perturbed (a few within each threshold), rotated, symmetric flips, duplicated (tied scores) and missing estimates"""
    r = np.random.RandomState(seed)
    _, info = bop_split.models_and_info()
    out = []
    for (s, i), inst in gt.items():
        for k, (o, R, t) in enumerate(inst):
            if (s + i + k) % 5 == 3:
                continue
            R_e = R.dot(_turn(k % 3, np.radians(r.uniform(0, 8)))) if k else R
            t_e = t + r.normal(0, 3.0, 3) * (k % 3)
            if o == 2 and k == 2:  # a symmetric flip of the box: correct under ADI, not under ADD
                S = bop_eval.symmetry_transformations(info[2])[1]
                R_e, t_e = R.dot(S[:9].reshape(3, 3)), R.dot(S[9:]) + t
            out.append(dict(scene_id=s, im_id=i, obj_id=o, score=round(r.uniform(), 1), R=R_e, t=t_e, time=0.5))
            if k % 2 == 0:
                out.append(dict(scene_id=s, im_id=i, obj_id=o, score=out[-1]["score"], R=bop_split.random_rotation(r),
                                t=t_e + 12.0, time=0.5))
    return out


def _frame(rows, types):
    df = pd.DataFrame({k: [r[k] for r in rows] for k in ("scene_id", "im_id", "obj_id", "est_id", "gt_id", "score")})
    for t in types:
        if t == "rete":
            df["re"], df["te"] = [r["rete"][0] for r in rows], [r["rete"][1] for r in rows]
        else:
            df[t] = [r[t] for r in rows]
    return df


def test_host_scoring_matches_oracle(split_dir):
    root, gt = split_dir
    sp = bop_eval.load_split(root)
    ests = bop_eval.normalize_results(estimates(gt))
    render = single_renderer(sp.models)
    sym = bop_eval.default_symmetric_obj_ids(sp.models_info)
    assert sym == [2, 3] and bop_eval.split_scene_ids(sp) == [1, 2, 3]
    rows = bop_other_ref.calc_other_errors(sp, ests, render, NEW_TYPES, sym)
    want = bop_other_ref.evaluate_localization(sp, ests, render, NEW_TYPES, symmetric_obj_ids=sym)
    got = bop_eval.score_errors(sp, _frame(rows, NEW_TYPES), ests, types=NEW_TYPES)
    for t in NEW_TYPES:
        assert got[t] == want[t], t
        assert set(got[t]["obj_recalls"]) == {1, 2, 3} and got[t]["obj_recalls"][3] == 0.0
        assert got[t]["scene_recalls"][3] == 0.0
    assert not any(k.startswith("bop19_average_recall") for k in got)
    recalls = {t: got[t]["recall"] for t in NEW_TYPES}
    assert 0 < recalls["proj"] < 1 and 0 < recalls["rete"] <= min(recalls["re"], recalls["te"])
    assert recalls["adi"] >= recalls["ad"] >= recalls["add"] and recalls["adi"] > recalls["add"]
    # a te threshold override moves exactly te and rete
    ths = {"te": [50.0], "rete": [5.0, 50.0]}
    over = bop_eval.score_errors(sp, _frame(rows, NEW_TYPES), ests, types=NEW_TYPES, thresholds=ths)
    want_over = bop_other_ref.evaluate_localization(sp, ests, render, ("te", "rete"), thresholds=ths, symmetric_obj_ids=sym)
    assert over["te"] == want_over["te"] and over["rete"] == want_over["rete"]
    assert over["te"]["recall"] > got["te"]["recall"]
    assert all(over[t] == got[t] for t in NEW_TYPES if t not in ("te", "rete"))


def test_threshold_and_option_parsing():
    assert bop_eval.resolve_thresholds({"te": 50})["te"] == [50.0]
    assert bop_eval.resolve_thresholds()["rete"] == [5.0, 5.0]
    with pytest.raises(ValueError):
        bop_eval.resolve_thresholds({"rete": [5.0]})
    with pytest.raises(ValueError):
        bop_eval.resolve_thresholds({"vsd": [0.3]})
    import argparse

    ap = argparse.ArgumentParser()
    bop_eval.add_error_type_arguments(ap)
    args = ap.parse_args(["--error-types", "ad,rete", "--correct-th", "te=50", "--correct-th", "rete=5,10",
                          "--symmetric-obj-ids", "10,11"])
    assert bop_eval.error_type_options(args) == dict(types=["ad", "rete"], thresholds={"te": [50.0], "rete": [5.0, 10.0]},
                                                     symmetric_obj_ids=[10, 11])
    assert bop_eval.error_type_options(ap.parse_args([])) == dict(types=["vsd", "mssd", "mspd"], thresholds={},
                                                                  symmetric_obj_ids=None)
    for bad in (["--error-types", "ad,xyz"], ["--correct-th", "te"], ["--correct-th", "vsd=0.3"]):
        with pytest.raises(SystemExit):
            ap.parse_args(bad)
