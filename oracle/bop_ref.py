"""oracle/bop_ref.py -- the BOP 2019 pose-error protocol restated in numpy float64 on the host (test infrastructure).

What the toolkit's scripts/eval_bop19.py -> eval_calc_errors.py -> eval_calc_scores.py compute (bop_toolkit_lib/pose_error,
visibility, misc, pose_matching, score), with its bop19 defaults, written out plainly: one pose pair at a time, whole
images as numpy arrays.  Depth renders come from a callback `render(obj_id, R, t_mm, K, (h, w)) -> [h, w] float32 depth in
METRES` (0 = no surface), so that tests can feed it the device's renders or the C oracle's.  The product's
megapose6d_b200/bop_eval.py is checked against this module, and this module against the stored outputs of the toolkit
itself (tests/golden/reference/bop_eval_*.npz).
"""
from __future__ import annotations

import math
from typing import Callable, Dict, List, Sequence, Tuple

import numpy as np

VSD_TAUS = np.arange(0.05, 0.51, 0.05)
MSSD_THRESHOLDS = np.arange(0.05, 0.51, 0.05)
MSPD_THRESHOLDS = np.arange(5, 51, 5)


def symmetries(model_info: dict, max_sym_disc_step: float = 0.01) -> List[Tuple[np.ndarray, np.ndarray]]:
    """[(R 3x3, t 3x1)]: identity + discrete symmetries, each combined with every discretised continuous rotation."""
    disc = [(np.eye(3), np.zeros((3, 1)))]
    for s in model_info.get("symmetries_discrete", []):
        m = np.reshape(np.asarray(s, np.float64), (4, 4))
        disc.append((m[:3, :3], m[:3, 3].reshape(3, 1)))
    cont = []
    for s in model_info.get("symmetries_continuous", []):
        axis = np.array(s["axis"], np.float64)
        axis = axis / math.sqrt(np.dot(axis, axis))
        offset = np.array(s["offset"], np.float64).reshape(3, 1)
        n = int(np.ceil(np.pi / max_sym_disc_step))
        for i in range(1, n):
            ang = i * (2.0 * np.pi / n)
            ca, sa = math.cos(ang), math.sin(ang)
            R = np.diag([ca, ca, ca]) + np.outer(axis, axis) * (1.0 - ca)
            d = axis * sa
            R += np.array([[0.0, -d[2], d[1]], [d[2], 0.0, -d[0]], [-d[1], d[0], 0.0]])
            cont.append((R, -R.dot(offset) + offset))
    if not cont:
        return disc
    return [(Rc.dot(Rd), Rc.dot(td) + tc) for Rd, td in disc for Rc, tc in cont]


def transform(pts, R, t):
    return (R.dot(pts.T) + np.reshape(t, (3, 1))).T


def project(pts, K, R, t):
    P = K.dot(np.hstack((R, np.reshape(t, (3, 1)))))
    x = P.dot(np.hstack((pts, np.ones((len(pts), 1)))).T)
    x /= x[2, :]
    return x[:2, :].T


def dist_image(depth: np.ndarray, K: np.ndarray) -> np.ndarray:
    """distance from the camera centre per pixel, float64: sqrt((X d)^2 + (Y d)^2 + d^2), X = (x - cx) / fx"""
    h, w = depth.shape
    xs, ys = np.meshgrid(np.arange(w), np.arange(h))
    X = (xs - K[0, 2]) / np.float64(K[0, 0])
    Y = (ys - K[1, 2]) / np.float64(K[1, 1])
    return np.sqrt(np.multiply(X, depth) ** 2 + np.multiply(Y, depth) ** 2 + depth.astype(np.float64) ** 2)


def visib_mask(dist_test, dist_model, delta):
    diff = dist_model.astype(np.float32) - dist_test.astype(np.float32)
    return np.logical_and(np.logical_or(diff <= delta, dist_test == 0), dist_model > 0)


def vsd_from_depths(depth_test_mm: np.ndarray, depth_est_mm: np.ndarray, depth_gt_mm: np.ndarray, K, delta, taus, diameter,
                    return_counts: bool = False):
    """VSD (step cost, bop19 visibility, normalised by the diameter) from depth images in mm."""
    dt, de, dg = dist_image(depth_test_mm, K), dist_image(depth_est_mm, K), dist_image(depth_gt_mm, K)
    vg = visib_mask(dt, dg, delta)
    ve = np.logical_or(visib_mask(dt, de, delta), np.logical_and(vg, de > 0))
    inter = np.logical_and(vg, ve)
    n_union = int(np.logical_or(vg, ve).sum())
    n_inter = int(inter.sum())
    d = np.abs(dg[inter] - de[inter]) / diameter
    counts = [int((d >= tau).sum()) for tau in taus]
    if n_union == 0:
        errs = [1.0] * len(taus)
    else:
        errs = [(c + (n_union - n_inter)) / float(n_union) for c in counts]
    return (errs, [n_union, n_inter] + counts) if return_counts else errs


def render_mm(render: Callable, obj_id, R, t, K, shape) -> np.ndarray:
    """rendered depth in mm, float32: fp32(metres * 1000)"""
    return (np.asarray(render(obj_id, R, t, K, shape), np.float32) * np.float32(1000.0)).astype(np.float32)


def spheres_overlap(radius, p1, p2) -> bool:
    p1, p2 = np.reshape(p1, 3), np.reshape(p2, 3)
    if p1[2] == 0 or p2[2] == 0:
        return False
    return bool(np.linalg.norm((p1 / p1[2])[:2] - (p2 / p2[2])[:2]) < radius * (1.0 / p1[2] + 1.0 / p2[2]))


def mssd(R_e, t_e, R_g, t_g, pts, syms, return_argmin: bool = False):
    pe = transform(pts, R_e, t_e)
    es = [np.linalg.norm(pe - transform(pts, R_g.dot(Rs), R_g.dot(ts) + np.reshape(t_g, (3, 1))), axis=1).max()
          for Rs, ts in syms]
    return (min(es), int(np.argmin(es))) if return_argmin else min(es)


def mspd(R_e, t_e, R_g, t_g, K, pts, syms, return_argmin: bool = False):
    pe = project(pts, K, R_e, t_e)
    es = [np.linalg.norm(pe - project(pts, K, R_g.dot(Rs), R_g.dot(ts) + np.reshape(t_g, (3, 1))), axis=1).max()
          for Rs, ts in syms]
    return (min(es), int(np.argmin(es))) if return_argmin else min(es)


def add(R_e, t_e, R_g, t_g, pts):
    return np.linalg.norm(transform(pts, R_e, t_e) - transform(pts, R_g, t_g), axis=1).mean()


def adi(R_e, t_e, R_g, t_g, pts):
    """mean distance from each point in the gt pose to its nearest point in the estimated pose (brute force, chunked)"""
    pe, pg = transform(pts, R_e, t_e), transform(pts, R_g, t_g)
    best = np.empty(len(pg))
    for i in range(0, len(pg), 512):
        d = pg[i:i + 512, None, :] - pe[None, :, :]
        best[i:i + 512] = np.sqrt((d * d).sum(-1).min(1))
    return best.mean()


# ------------------------------------------------------------------------------------------------------------- protocol
def calc_errors(split, ests: Sequence[dict], render: Callable, types=("vsd", "mssd", "mspd"), delta=15) -> List[dict]:
    """One dict per (selected estimate, gt of its object): scene_id, im_id, obj_id, est_id, gt_id, score, and per type the
    error (vsd: list over VSD_TAUS).  `split` is a megapose6d_b200.bop_eval.BopSplit (plain data); ests as
    bop_eval.normalize_results."""
    org: Dict[tuple, List[dict]] = {}
    for e in ests:
        org.setdefault((e["scene_id"], e["im_id"], e["obj_id"]), []).append(e)
    syms = {o: symmetries(info) for o, info in split.models_info.items()}
    out = []
    for tgt in split.targets:
        scene_id, im_id, obj_id = tgt["scene_id"], tgt["im_id"], tgt["obj_id"]
        K = np.asarray(split.scene_camera[scene_id][im_id]["cam_K"], np.float64).reshape(3, 3)
        depth = None
        if "vsd" in types:
            depth = split.depth(scene_id, im_id).astype(np.float32)
            depth *= split.scene_camera[scene_id][im_id]["depth_scale"]
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
                if "vsd" in types:
                    if not spheres_overlap(0.5 * diameter, t_e, t_g):
                        row["vsd"] = [1.0] * len(VSD_TAUS)
                    else:
                        de = render_mm(render, obj_id, R_e, t_e.reshape(3), K, depth.shape)
                        dg = render_mm(render, obj_id, R_g, t_g.reshape(3), K, depth.shape)
                        row["vsd"] = vsd_from_depths(depth, de, dg, K, delta, VSD_TAUS, diameter)
                if "mssd" in types:
                    row["mssd"] = mssd(R_e, t_e, R_g, t_g, pts, syms[obj_id]) if near else float("inf")
                if "mspd" in types:
                    row["mspd"] = mspd(R_e, t_e, R_g, t_g, K, pts, syms[obj_id])
                if "add" in types:
                    row["add"] = add(R_e, t_e, R_g, t_g, pts) if near else float("inf")
                if "adi" in types:
                    row["adi"] = adi(R_e, t_e, R_g, t_g, pts) if near else float("inf")
                out.append(row)
    return out


def match_poses(errs: Sequence[dict], threshold: float, gt_valid: Sequence[bool]) -> List[dict]:
    """Greedy matching by decreasing score: each estimate takes the valid, unmatched gt of lowest error below threshold.
    errs: [{est_id, score, errors: {gt_id: error}}]."""
    matched, out = [], []
    for e in sorted(errs, key=lambda e: e["score"], reverse=True):
        best_gt, best = -1, threshold
        for gt_id, err in e["errors"].items():
            if gt_valid[gt_id] and gt_id not in matched and err < best:
                best_gt, best = gt_id, err
        if best_gt >= 0:
            matched.append(best_gt)
            out.append(dict(est_id=e["est_id"], gt_id=best_gt, score=e["score"], error=best))
    return out


def gt_valid(split) -> Dict[tuple, List[bool]]:
    tg: Dict[tuple, Dict[int, int]] = {}
    for t in split.targets:
        tg.setdefault((t["scene_id"], t["im_id"]), {})[t["obj_id"]] = t["inst_count"]
    out = {}
    for (s, i), to_add in tg.items():
        gts, info = split.scene_gt[s][i], split.scene_gt_info[s][i]
        to_add = dict(to_add)
        valid = [False] * len(gts)
        for g in sorted(range(len(gts)), key=lambda g: info[g]["visib_fract"], reverse=True):
            if to_add.get(gts[g]["obj_id"], 0) > 0:
                valid[g] = True
                to_add[gts[g]["obj_id"]] -= 1
        out[(s, i)] = valid
    return out


def localization_recall(matches: Sequence[dict]) -> float:
    """calc_localization_scores(...)['recall'] with n_top = -1: true positives over valid gt poses."""
    tars = sum(1 for m in matches if m["valid"])
    tps = sum(1 for m in matches if m["valid"] and m["est_id"] != -1)
    return tps / float(tars) if tars else 0.0


def recall(split, rows: Sequence[dict], key, threshold, normalize) -> float:
    valid = gt_valid(split)
    matches = []
    for (s, i), vmask in valid.items():
        gts = split.scene_gt[s][i]
        im = [dict(obj_id=g["obj_id"], gt_id=k, est_id=-1, valid=vmask[k]) for k, g in enumerate(gts)]
        for obj_id in set(g["obj_id"] for g in gts):
            errs: Dict[int, dict] = {}
            for r in rows:
                if (r["scene_id"], r["im_id"], r["obj_id"]) == (s, i, obj_id):
                    e = errs.setdefault(r["est_id"], dict(est_id=r["est_id"], score=r["score"], errors={}))
                    e["errors"][r["gt_id"]] = normalize(r, key(r))
            for m in match_poses(list(errs.values()), threshold, vmask):
                im[m["gt_id"]]["est_id"] = m["est_id"]
        matches += im
    return localization_recall(matches)


def evaluate(split, ests: Sequence[dict], render: Callable, delta=15) -> dict:
    rows = calc_errors(split, ests, render, delta=delta)
    out = {}
    rec_vsd = [[recall(split, rows, lambda r, k=k: r["vsd"][k], th, lambda r, e: e) for th in VSD_TAUS]
               for k in range(len(VSD_TAUS))]

    def by_diameter(r, e):
        return e / float(split.models_info[r["obj_id"]]["diameter"])

    def by_width(r, e):
        return (640.0 / float(split.depth_width(r["scene_id"], r["im_id"]))) * e

    rec_mssd = [recall(split, rows, lambda r: r["mssd"], th, by_diameter) for th in MSSD_THRESHOLDS]
    rec_mspd = [recall(split, rows, lambda r: r["mspd"], th, by_width) for th in MSPD_THRESHOLDS]
    ar = dict(vsd=float(np.mean(rec_vsd)), mssd=float(np.mean(rec_mssd)), mspd=float(np.mean(rec_mspd)))
    out.update(bop19_recalls_vsd=rec_vsd, bop19_recalls_mssd=rec_mssd, bop19_recalls_mspd=rec_mspd)
    for k, v in ar.items():
        out[f"bop19_average_recall_{k}"] = v
    out["bop19_average_recall"] = float(np.mean([ar["vsd"], ar["mssd"], ar["mspd"]]))
    times, avail = {}, True
    for e in ests:
        if e["time"] < 0:
            avail = False
            break
        times.setdefault((e["scene_id"], e["im_id"]), e["time"])
    out["bop19_average_time_per_image"] = float(np.mean(list(times.values()))) if avail and times else -1.0
    return out
