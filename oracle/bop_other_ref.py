"""oracle/bop_other_ref.py -- the BOP toolkit's other pose errors and its localization scores, restated in numpy float64 on
the host (test infrastructure).

What the toolkit's scripts/eval_calc_errors.py computes for the error types ad, add, adi, cus, proj, re, te and rete
(bop_toolkit_lib/pose_error: add, adi, cus, proj, re, te, with the script's gating), and what scripts/eval_calc_scores.py
makes of them with n_top = -1 and visib_gt_min = -1 (pose_matching.match_poses for errors of several elements,
score.calc_localization_scores), written out plainly on top of oracle/bop_ref.py (transforms, projections, renders in mm,
sphere gating, valid gts).  Depth renders come from the same callback as bop_ref's.  The product's
megapose6d_b200/bop_eval.py is checked against this module, and this module against the stored outputs of the toolkit
itself (tests/golden/reference/bop_eval_more_errors.npz).
"""
from __future__ import annotations

import math
import os
from typing import Callable, Dict, List, Sequence

import numpy as np

from oracle.bop_ref import add, adi, gt_valid, project, render_mm, spheres_overlap


def proj(R_e, t_e, R_g, t_g, K, pts):
    """mean distance of the projections of the model points (px)"""
    return np.linalg.norm(project(pts, K, R_e, t_e) - project(pts, K, R_g, t_g), axis=1).mean()


def re(R_e, R_g):
    """rotation error in degrees: acos(0.5 (trace(R_e inv(R_g)) - 1)), the cosine clipped to [-1, 1]"""
    c = float(0.5 * (np.trace(R_e.dot(np.linalg.inv(R_g))) - 1.0))
    return 180.0 * math.acos(min(1.0, max(-1.0, c))) / np.pi


def te(t_e, t_g):
    """translation error, in the unit of t (mm)"""
    return np.linalg.norm(np.reshape(t_g, 3) - np.reshape(t_e, 3))


def cus_from_depths(depth_est: np.ndarray, depth_gt: np.ndarray, return_counts: bool = False):
    """complement over union of the silhouettes (depth > 0) of two renders; 1.0 for an empty union"""
    me, mg = depth_est > 0, depth_gt > 0
    n_inter, n_union = int(np.logical_and(me, mg).sum()), int(np.logical_or(me, mg).sum())
    e = 1.0 - np.int64(n_inter) / float(n_union) if n_union > 0 else 1.0
    return (e, [n_inter, n_union]) if return_counts else e


def ad(obj_id, symmetric_obj_ids, R_e, t_e, R_g, t_g, pts):
    """ADI for an object of symmetric_obj_ids, ADD otherwise"""
    return adi(R_e, t_e, R_g, t_g, pts) if obj_id in symmetric_obj_ids else add(R_e, t_e, R_g, t_g, pts)


def calc_other_errors(split, ests: Sequence[dict], render: Callable, types, symmetric_obj_ids=()) -> List[dict]:
    """calc_errors for the toolkit's other error types: ad (adi for symmetric_obj_ids, add otherwise), add, adi, cus, proj,
    re, te, rete ([re, te]), with eval_calc_errors.py's gating: ad / add / adi inf where the centres are a diameter or
    more apart, cus 1.0 where the sphere projections do not overlap, proj / re / te / rete never gated."""
    org: Dict[tuple, List[dict]] = {}
    for e in ests:
        org.setdefault((e["scene_id"], e["im_id"], e["obj_id"]), []).append(e)
    out = []
    for tgt in split.targets:
        scene_id, im_id, obj_id = tgt["scene_id"], tgt["im_id"], tgt["obj_id"]
        K = np.asarray(split.scene_camera[scene_id][im_id]["cam_K"], np.float64).reshape(3, 3)
        shape = split.depth(scene_id, im_id).shape if "cus" in types else None
        cands = org.get((scene_id, im_id, obj_id), [])
        top = sorted(enumerate(cands), key=lambda x: x[1]["score"], reverse=True)[:tgt["inst_count"]]
        diameter = split.models_info[obj_id]["diameter"]
        pts = np.asarray(split.models[obj_id].vertices, np.float64)
        for est_id, est in top:
            R_e, t_e = est["R"], np.reshape(est["t"], (3, 1))
            for gt_id, gt in enumerate(split.scene_gt[scene_id][im_id]):
                if gt["obj_id"] != obj_id:
                    continue
                R_g = np.asarray(gt["cam_R_m2c"], np.float64).reshape(3, 3)
                t_g = np.asarray(gt["cam_t_m2c"], np.float64).reshape(3, 1)
                row = dict(scene_id=scene_id, im_id=im_id, obj_id=obj_id, est_id=est_id, gt_id=gt_id, score=est["score"])
                near = np.linalg.norm(t_e - t_g) < diameter
                if "ad" in types:
                    row["ad"] = ad(obj_id, symmetric_obj_ids, R_e, t_e, R_g, t_g, pts) if near else float("inf")
                if "add" in types:
                    row["add"] = add(R_e, t_e, R_g, t_g, pts) if near else float("inf")
                if "adi" in types:
                    row["adi"] = adi(R_e, t_e, R_g, t_g, pts) if near else float("inf")
                if "cus" in types:
                    if not spheres_overlap(0.5 * diameter, t_e, t_g):
                        row["cus"] = 1.0
                    else:
                        de = render_mm(render, obj_id, R_e, t_e.reshape(3), K, shape)
                        dg = render_mm(render, obj_id, R_g, t_g.reshape(3), K, shape)
                        row["cus"] = cus_from_depths(de, dg)
                if "proj" in types:
                    row["proj"] = proj(R_e, t_e, R_g, t_g, K, pts)
                if "re" in types:
                    row["re"] = re(R_e, R_g)
                if "te" in types:
                    row["te"] = te(t_e, t_g)
                if "rete" in types:
                    row["rete"] = [re(R_e, R_g), te(t_e, t_g)]
                out.append(row)
    return out


# ------------------------------------------------------------------------------ the other error types' localization scores
LOCALIZATION_THRESHOLDS = {"ad": [0.1], "add": [0.1], "adi": [0.1], "cus": [0.5], "proj": [5.0], "re": [5.0], "te": [5.0],
                           "rete": [5.0, 5.0]}  # te in the unit of its errors (mm)
NORMALIZED_BY_DIAMETER = ("ad", "add", "adi", "mssd")


def match_poses_multi(errs: Sequence[dict], thresholds: Sequence[float], gt_valid: Sequence[bool]) -> List[dict]:
    """match_poses for errors of several elements: an estimate takes a valid, unmatched gt only when every element is
    strictly below the best so far, which starts at the thresholds.  errs: [{est_id, score, errors: {gt_id: [e, ...]}}]."""
    matched, out = [], []
    for e in sorted(errs, key=lambda e: e["score"], reverse=True):
        best_gt, best = -1, list(thresholds)
        for gt_id, err in e["errors"].items():
            if gt_valid[gt_id] and gt_id not in matched and all(err[i] < best[i] for i in range(len(thresholds))):
                best_gt, best = gt_id, err
        if best_gt >= 0:
            matched.append(best_gt)
            out.append(dict(est_id=e["est_id"], gt_id=best_gt, score=e["score"], error=best))
    return out


def localization_scores(scene_ids, obj_ids, matches: Sequence[dict]) -> dict:
    """calc_localization_scores with n_top = -1: matches = one dict per gt of the target images (scene_id, im_id, obj_id,
    est_id (-1 = unmatched), valid); a zero-target object or scene has recall 0 and counts in the means."""
    obj_tars, obj_tps = dict.fromkeys(obj_ids, 0), dict.fromkeys(obj_ids, 0)
    scene_tars, scene_tps = dict.fromkeys(scene_ids, 0), dict.fromkeys(scene_ids, 0)
    for m in matches:
        if m["valid"]:
            obj_tars[m["obj_id"]] += 1
            scene_tars[m["scene_id"]] += 1
            if m["est_id"] != -1:
                obj_tps[m["obj_id"]] += 1
                scene_tps[m["scene_id"]] += 1
    tars, tps = sum(obj_tars.values()), sum(obj_tps.values())

    def rec(tp, n):
        return 0.0 if n == 0 else tp / float(n)

    obj_recalls = {o: rec(obj_tps[o], obj_tars[o]) for o in obj_ids}
    scene_recalls = {s: float(rec(scene_tps[s], scene_tars[s])) for s in scene_ids}
    return dict(recall=float(rec(tps, tars)), obj_recalls=obj_recalls,
                mean_obj_recall=float(np.mean(list(obj_recalls.values())).squeeze()), scene_recalls=scene_recalls,
                mean_scene_recall=float(np.mean(list(scene_recalls.values())).squeeze()), gt_count=len(matches),
                targets_count=int(tars), tp_count=int(tps))


def split_scene_ids(split) -> List[int]:
    """the numbered scene directories of the split (and the scenes of its targets)"""
    ids = {t["scene_id"] for t in split.targets}
    if split.root is not None and os.path.isdir(os.path.join(split.root, split.split)):
        ids |= {int(d) for d in os.listdir(os.path.join(split.root, split.split)) if d.isdigit()}
    return sorted(ids)


def localization_score(split, rows: Sequence[dict], err_type: str, thresholds: Sequence[float]) -> dict:
    """eval_calc_scores.py for one error type of calc_errors' rows: normalise, match per (image, object), score"""
    valid = gt_valid(split)
    matches = []
    for (s, i), vmask in valid.items():
        gts = split.scene_gt[s][i]
        im = [dict(scene_id=s, im_id=i, obj_id=g["obj_id"], gt_id=k, est_id=-1, valid=vmask[k]) for k, g in enumerate(gts)]
        for obj_id in set(g["obj_id"] for g in gts):
            errs: Dict[int, dict] = {}
            for r in rows:
                if (r["scene_id"], r["im_id"], r["obj_id"]) == (s, i, obj_id):
                    e = errs.setdefault(r["est_id"], dict(est_id=r["est_id"], score=r["score"], errors={}))
                    v = r[err_type] if isinstance(r[err_type], list) else [r[err_type]]
                    if err_type in NORMALIZED_BY_DIAMETER:
                        v = [x / float(split.models_info[obj_id]["diameter"]) for x in v]
                    e["errors"][r["gt_id"]] = v
            for m in match_poses_multi(list(errs.values()), thresholds, vmask):
                im[m["gt_id"]]["est_id"] = m["est_id"]
        matches += im
    return localization_scores(split_scene_ids(split), sorted(split.models_info), matches)


def evaluate_localization(split, ests: Sequence[dict], render: Callable, types, thresholds=None,
                          symmetric_obj_ids=()) -> dict:
    """{type: localization_score} for the other error types, at LOCALIZATION_THRESHOLDS or the given ones"""
    ths = dict(LOCALIZATION_THRESHOLDS, **(thresholds or {}))
    rows = calc_other_errors(split, ests, render, tuple(types), symmetric_obj_ids)
    return {t: localization_score(split, rows, t, ths[t]) for t in types}
