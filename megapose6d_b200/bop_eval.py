"""BOP 2019 evaluation of pose estimates: VSD, MSSD and MSPD errors on the device, matching and average recall on the host.

The protocol is that of the BOP toolkit's `scripts/eval_bop19.py` (the toolkit is vendored by the reference under
deps/bop_toolkit_challenge) with its bop19 defaults: the top `inst_count` estimates per (scene, image, object) by score
(stable sort), the `inst_count` most visible ground-truth poses valid, VSD with delta 15 mm (5 for itodd), taus 0.05..0.5
of the diameter, step cost and bop19 visibility, MSSD thresholds 0.05..0.5 x diameter, MSPD thresholds 5..50 px scaled by
640 / image width, symmetries discretised with max_sym_disc_step 0.01, models from `models_eval/`.

Depth renders come from the engine's rasteriser (`BatchRenderer.render(render_depth=True)`, near/far planes 0.1 / 10 m);
the per-pixel VSD reduction and the per-point MSSD / MSPD / ADD / ADI reductions are the kernels of csrc/bop_eval.cu
(include/mpx.h: mpx_bop_vsd, mpx_bop_point_errors).

The toolkit's other error types (scripts/eval_calc_errors.py: ad, add, adi, cus, proj, re, te, rete) are scored as its
scripts/eval_calc_scores.py does with n_top = -1 and visib_gt_min = -1: a recall per type at its own threshold
(LOCALIZATION_THRESHOLDS, overridable per type), with per-object and per-scene recalls.  CUS uses the VSD renders
(mpx_bop_cus), PROJ / RE / TE the point store (mpx_bop_pose_errors).

    python -m megapose6d_b200.bop_eval <dataset_dir> <results.csv> [--split test] [--errors-out DIR]
        [--error-types ad,add,adi,cus,proj,re,te,rete] [--correct-th te=50 ...] [--symmetric-obj-ids 10,11]
"""
from __future__ import annotations

import argparse
import json
import math
from dataclasses import dataclass, field
from pathlib import Path
from typing import Dict, Iterable, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from . import _abi

VSD_TAUS = np.arange(0.05, 0.51, 0.05)
MSSD_THRESHOLDS = np.arange(0.05, 0.51, 0.05)
MSPD_THRESHOLDS = np.arange(5, 51, 5)
VSD_DELTAS = {"itodd": 5}
VSD_DELTA_DEFAULT = 15
MAX_SYM_DISC_STEP = 0.01
KINDS = {"mssd": 0, "mspd": 1, "add": 2, "adi": 3}
BOP19_TYPES = ("vsd", "mssd", "mspd")
# The toolkit's other error types (scripts/eval_calc_errors.py) and their default correctness thresholds
# (scripts/eval_calc_scores.py): one threshold per error element.  ad / add / adi are fractions of the diameter, cus a
# fraction of the union, proj pixels, re degrees.  te is compared in the unit of its errors, mm, although the toolkit
# labels its thresholds "cm": te 5 and the second element of rete 5 mean 5 mm.
LOCALIZATION_THRESHOLDS = {"ad": [0.1], "add": [0.1], "adi": [0.1], "cus": [0.5], "proj": [5.0], "re": [5.0], "te": [5.0],
                           "rete": [5.0, 5.0]}
ERROR_TYPES = BOP19_TYPES + ("add", "adi") + tuple(t for t in LOCALIZATION_THRESHOLDS if t not in ("add", "adi"))
NORMALIZED_BY_DIAMETER = ("ad", "add", "adi")


# ------------------------------------------------------------------------------------------------------------ split reader
def load_json(path: Path, keys_to_int: bool = False):
    """JSON with object keys that are integers converted to int (the toolkit's `inout.load_json(keys_to_int=True)`)."""
    hook = (lambda d: {int(k) if k.lstrip("-").isdigit() else k: v for k, v in d.items()}) if keys_to_int else None
    with open(path) as f:
        return json.load(f, object_hook=hook)


def read_depth_png(path: Path) -> np.ndarray:
    """16-bit depth PNG -> [h, w] uint16 raw values."""
    from PIL import Image

    with Image.open(path) as im:
        return np.asarray(im).astype(np.uint16)


def write_depth_png(path: Path, raw: np.ndarray) -> None:
    from PIL import Image

    Image.fromarray(np.ascontiguousarray(raw, np.uint16)).save(path)


def symmetry_transformations(model_info: dict, max_sym_disc_step: float = MAX_SYM_DISC_STEP) -> np.ndarray:
    """[n, 12] float64 (R row-major, t): the identity and the discrete symmetries, each composed with the discretised
    continuous symmetries when the model has any (the toolkit's `misc.get_symmetry_transformations`)."""
    disc = [(np.eye(3), np.zeros(3))]
    for s in model_info.get("symmetries_discrete", []):
        m = np.asarray(s, np.float64).reshape(4, 4)
        disc.append((m[:3, :3], m[:3, 3]))
    cont = []
    for s in model_info.get("symmetries_continuous", []):
        axis = np.asarray(s["axis"], np.float64)
        axis = axis / math.sqrt(np.dot(axis, axis))
        offset = np.asarray(s["offset"], np.float64)
        n_steps = int(np.ceil(np.pi / max_sym_disc_step))
        step = 2.0 * np.pi / n_steps
        for i in range(1, n_steps):
            c, s_ = math.cos(i * step), math.sin(i * step)
            R = np.diag([c, c, c]) + np.outer(axis, axis) * (1.0 - c)
            a = axis * s_
            R = R + np.array([[0.0, -a[2], a[1]], [a[2], 0.0, -a[0]], [-a[1], a[0], 0.0]])
            cont.append((R, -R.dot(offset) + offset))
    out = []
    for Rd, td in disc:
        if cont:
            out += [(Rc.dot(Rd), Rc.dot(td) + tc) for Rc, tc in cont]
        else:
            out.append((Rd, td))
    return np.stack([np.concatenate([R.reshape(9), t.reshape(3)]) for R, t in out])


@dataclass
class BopSplit:
    """A BOP dataset split: cameras, ground truth, visibility, targets and the evaluation models (points in mm)."""

    root: Path
    split: str
    models_info: Dict[int, dict]
    models: Dict[int, "object"]  # obj_id -> meshes.TriMesh (mm)
    targets: List[dict]
    scene_camera: Dict[int, Dict[int, dict]] = field(default_factory=dict)
    scene_gt: Dict[int, Dict[int, List[dict]]] = field(default_factory=dict)
    scene_gt_info: Dict[int, Dict[int, List[dict]]] = field(default_factory=dict)
    _widths: Dict[Tuple[int, int], int] = field(default_factory=dict, repr=False)

    def depth_path(self, scene_id: int, im_id: int) -> Path:
        return self.root / self.split / f"{scene_id:06d}" / "depth" / f"{im_id:06d}.png"

    def depth(self, scene_id: int, im_id: int) -> np.ndarray:
        return read_depth_png(self.depth_path(scene_id, im_id))

    def depth_width(self, scene_id: int, im_id: int) -> int:
        key = (scene_id, im_id)
        if key not in self._widths:
            from PIL import Image

            with Image.open(self.depth_path(scene_id, im_id)) as im:
                self._widths[key] = im.size[0]
        return self._widths[key]

    def K(self, scene_id: int, im_id: int) -> np.ndarray:
        return np.asarray(self.scene_camera[scene_id][im_id]["cam_K"], np.float64).reshape(3, 3)


def split_scene_ids(split: BopSplit) -> List[int]:
    """Every scene of the split: its numbered scene directories and the scenes of its targets (the toolkit's
    `dataset_params` lists a dataset's scenes by hand)."""
    ids = {t["scene_id"] for t in split.targets}
    if split.root is not None and (Path(split.root) / split.split).is_dir():
        ids |= {int(d.name) for d in (Path(split.root) / split.split).iterdir() if d.is_dir() and d.name.isdigit()}
    return sorted(ids)


def default_symmetric_obj_ids(models_info: Dict[int, dict]) -> List[int]:
    """The objects whose models_info entry lists discrete or continuous symmetries.  The toolkit keeps a hand-written
    per-dataset table instead (`dataset_params`); the two can differ."""
    return sorted(o for o, info in models_info.items()
                  if info.get("symmetries_discrete") or info.get("symmetries_continuous"))


def load_split(dataset_dir: Union[str, Path], split: str = "test", targets_filename: str = "test_targets_bop19.json") -> BopSplit:
    from .meshes import load_ply

    root = Path(dataset_dir)
    models_dir = root / "models_eval"
    models_info = load_json(models_dir / "models_info.json", keys_to_int=True)
    models = {obj_id: load_ply(models_dir / f"obj_{obj_id:06d}.ply") for obj_id in sorted(models_info)}
    targets = load_json(root / targets_filename)
    out = BopSplit(root, split, models_info, models, targets)
    for scene_id in sorted({t["scene_id"] for t in targets}):
        d = root / split / f"{scene_id:06d}"
        out.scene_camera[scene_id] = load_json(d / "scene_camera.json", keys_to_int=True)
        out.scene_gt[scene_id] = load_json(d / "scene_gt.json", keys_to_int=True)
        out.scene_gt_info[scene_id] = load_json(d / "scene_gt_info.json", keys_to_int=True)
    return out


def normalize_results(results) -> List[dict]:
    """A bop19 CSV path or the dicts of `prediction_runner.load_bop_results` / `predictions_to_bop` -> dicts with float64
    R [3,3] and t [3] (mm)."""
    if isinstance(results, (str, Path)):
        from .prediction_runner import load_bop_results

        results = load_bop_results(Path(results))
    out = []
    for r in results:
        out.append(dict(scene_id=int(r["scene_id"]), im_id=int(r["im_id"]), obj_id=int(r["obj_id"]), score=float(r["score"]),
                        R=np.asarray(torch.as_tensor(r["R"]).double().numpy() if torch.is_tensor(r["R"]) else r["R"],
                                     np.float64).reshape(3, 3),
                        t=np.asarray(torch.as_tensor(r["t"]).double().numpy() if torch.is_tensor(r["t"]) else r["t"],
                                     np.float64).reshape(3),
                        time=float(r.get("time", -1))))
    return out


def average_time_per_image(ests: Sequence[dict]) -> float:
    """Mean of the per-image `time` (every estimate of an image must give the same time); -1 when any time is negative."""
    times: Dict[Tuple[int, int], float] = {}
    for e in ests:
        key = (e["scene_id"], e["im_id"])
        if e["time"] < 0:
            return -1.0
        if key in times:
            if abs(times[key] - e["time"]) > 0.001:
                raise ValueError(f"the running time of scene {key[0]} image {key[1]} differs between its estimates")
        else:
            times[key] = e["time"]
    return float(np.mean(list(times.values()))) if times else -1.0


# --------------------------------------------------------------------------------------------------------- device kernels
def vsd_from_depths(depth_test: torch.Tensor, depth_scale: torch.Tensor, K: torch.Tensor, depth_est: torch.Tensor,
                    depth_gt: torch.Tensor, est_idx: torch.Tensor, gt_idx: torch.Tensor, img_idx: torch.Tensor,
                    diameter: torch.Tensor, delta: float, taus: Sequence[float] = VSD_TAUS):
    """mpx_bop_vsd on device tensors: depth_test [I,h,w] int16 (raw uint16 bits), depth_scale [I] float32, K [I,3,3]
    float64, depth_est [E,h,w] / depth_gt [G,h,w] float32 metres, index tensors [P] int32, diameter [P] float64 mm.
    Returns (errors [P, n_taus] float64, counts [P, 2 + n_taus] int64), on the device, without a host sync."""
    n = int(est_idx.numel())
    dev = depth_est.device
    h, w = depth_est.shape[-2:]
    taus_h = np.ascontiguousarray(np.asarray(taus, np.float64))
    err = torch.empty(n, len(taus_h), dtype=torch.float64, device=dev)
    counts = torch.empty(n, 2 + len(taus_h), dtype=torch.int64, device=dev)
    _abi.check(_abi.lib().mpx_bop_vsd(
        n, h, w, _abi.ptr(depth_test), depth_test.shape[0], _abi.ptr(depth_scale), _abi.ptr(K), _abi.ptr(depth_est),
        depth_est.shape[0], _abi.ptr(depth_gt), depth_gt.shape[0], _abi.ptr(est_idx), _abi.ptr(gt_idx), _abi.ptr(img_idx),
        _abi.ptr(diameter), taus_h.ctypes.data, len(taus_h), float(delta), _abi.ptr(counts), _abi.ptr(err),
        _abi.stream_ptr()))
    return err, counts


def cus_from_depths(depth_est: torch.Tensor, depth_gt: torch.Tensor, est_idx: torch.Tensor, gt_idx: torch.Tensor):
    """mpx_bop_cus on device tensors: depth_est [E,h,w] / depth_gt [G,h,w] float32 metres, index tensors [P] int32.
    Returns (errors [P] float64, counts [P, 2] int64 = (intersection, union)), on the device, without a host sync."""
    n = int(est_idx.numel())
    dev = depth_est.device
    h, w = depth_est.shape[-2:]
    err = torch.empty(n, dtype=torch.float64, device=dev)
    counts = torch.empty(n, 2, dtype=torch.int64, device=dev)
    _abi.check(_abi.lib().mpx_bop_cus(n, h, w, _abi.ptr(depth_est), depth_est.shape[0], _abi.ptr(depth_gt),
                                      depth_gt.shape[0], _abi.ptr(est_idx), _abi.ptr(gt_idx), _abi.ptr(counts),
                                      _abi.ptr(err), _abi.stream_ptr()))
    return err, counts


class PointStore:
    """Model points (float64 mm) and symmetry transforms of several models, concatenated on the device."""

    def __init__(self, points: Sequence[np.ndarray], syms: Sequence[np.ndarray], device="cuda"):
        self.n_models = len(points)
        self.pts = torch.from_numpy(np.ascontiguousarray(np.concatenate(points), np.float64)).to(device)
        self.pt_off = torch.tensor(np.cumsum([0] + [len(p) for p in points]), dtype=torch.int64, device=device)
        self.syms = torch.from_numpy(np.ascontiguousarray(np.concatenate(syms), np.float64)).to(device)
        self.sym_off = torch.tensor(np.cumsum([0] + [len(s) for s in syms]), dtype=torch.int64, device=device)

    def errors(self, kind: str, model_idx: torch.Tensor, pose_est: torch.Tensor, pose_gt: torch.Tensor,
               K: Optional[torch.Tensor] = None):
        """mpx_bop_point_errors: pose_* [P, 12] float64 (R row-major, t mm), K [P, 3, 3] float64 (mspd).  Returns
        (errors [P] float64, argmin symmetry [P] int32) on the device."""
        n = int(model_idx.numel())
        dev = self.pts.device
        err = torch.empty(n, dtype=torch.float64, device=dev)
        arg = torch.empty(n, dtype=torch.int32, device=dev)
        _abi.check(_abi.lib().mpx_bop_point_errors(
            KINDS[kind], n, self.n_models, _abi.ptr(self.pts), _abi.ptr(self.pt_off), self.pts.shape[0], _abi.ptr(self.syms),
            _abi.ptr(self.sym_off), self.syms.shape[0], _abi.ptr(model_idx), _abi.ptr(pose_est), _abi.ptr(pose_gt),
            _abi.ptr(K), _abi.ptr(err), _abi.ptr(arg), _abi.stream_ptr()))
        return err, arg

    def pose_errors(self, pose_est: torch.Tensor, pose_gt: torch.Tensor, model_idx: Optional[torch.Tensor] = None,
                    K: Optional[torch.Tensor] = None, types: Iterable[str] = ("proj", "re", "te")) -> Dict[str, torch.Tensor]:
        """mpx_bop_pose_errors: pose_* [P, 12] float64 (R row-major, t mm); model_idx [P] int32 and K [P, 3, 3] float64
        for proj.  Returns {type: [P] float64} on the device for the requested types (proj px, re degrees, te mm)."""
        types = tuple(types)
        n = int(pose_est.shape[0])
        out = {t: torch.empty(n, dtype=torch.float64, device=self.pts.device) for t in ("proj", "re", "te") if t in types}
        _abi.check(_abi.lib().mpx_bop_pose_errors(
            n, self.n_models, _abi.ptr(self.pts), _abi.ptr(self.pt_off), self.pts.shape[0], _abi.ptr(model_idx),
            _abi.ptr(pose_est), _abi.ptr(pose_gt), _abi.ptr(K), _abi.ptr(out.get("proj")), _abi.ptr(out.get("re")),
            _abi.ptr(out.get("te")), _abi.stream_ptr()))
        return out


def _pose12(R: np.ndarray, t: np.ndarray) -> np.ndarray:
    return np.concatenate([np.asarray(R, np.float64).reshape(9), np.asarray(t, np.float64).reshape(3)])


def spheres_projections_overlap(radius: float, t1: np.ndarray, t2: np.ndarray) -> bool:
    """Whether the projections of two spheres of `radius` centred at t1, t2 overlap (approximately)."""
    if t1[2] == 0 or t2[2] == 0:
        return False
    d = np.linalg.norm((t1 / t1[2])[:2] - (t2 / t2[2])[:2])
    return bool(d < radius * (1.0 / t1[2] + 1.0 / t2[2]))


# ------------------------------------------------------------------------------------------------------------ host scoring
def gt_valid_masks(split: BopSplit) -> Dict[Tuple[int, int], List[bool]]:
    """visib_gt_min = -1: per target image, the inst_count most visible ground-truth poses of each target object."""
    targets: Dict[Tuple[int, int], Dict[int, int]] = {}
    for t in split.targets:
        targets.setdefault((t["scene_id"], t["im_id"]), {})[t["obj_id"]] = t["inst_count"]
    out = {}
    for (scene_id, im_id), to_add in targets.items():
        gts = split.scene_gt[scene_id][im_id]
        info = split.scene_gt_info[scene_id][im_id]
        order = sorted(range(len(gts)), key=lambda g: info[g]["visib_fract"], reverse=True)
        to_add = dict(to_add)
        valid = [False] * len(gts)
        for g in order:
            o = gts[g]["obj_id"]
            if to_add.get(o, 0) > 0:
                valid[g] = True
                to_add[o] -= 1
        out[(scene_id, im_id)] = valid
    return out


def recall(split: BopSplit, rows: Sequence[dict], errors: np.ndarray, threshold: float,
           valid: Dict[Tuple[int, int], List[bool]]) -> float:
    """Recall of one error type at one threshold.  rows[k] = {scene_id, im_id, obj_id, est_id, gt_id, score} of error k,
    in the order the estimates were selected (by decreasing score); errors[k] already normalised."""
    tars = sum(sum(v) for v in valid.values())
    if tars == 0:
        return 0.0
    by_est: Dict[Tuple[int, int, int, int], List[Tuple[int, float]]] = {}
    for r, e in zip(rows, errors):
        by_est.setdefault((r["scene_id"], r["im_id"], r["obj_id"], r["est_id"]), []).append((r["gt_id"], e))
    # estimates of one (image, object) in selection order; python's sort is stable, as the toolkit's
    groups: Dict[Tuple[int, int, int], List[Tuple[float, List[Tuple[int, float]]]]] = {}
    score = {(r["scene_id"], r["im_id"], r["obj_id"], r["est_id"]): r["score"] for r in rows}
    for key, errs in by_est.items():
        groups.setdefault(key[:3], []).append((score[key], errs))
    tps = 0
    for (scene_id, im_id, _), ests in groups.items():
        mask = valid.get((scene_id, im_id))
        if mask is None:
            continue
        matched = set()
        for _, errs in sorted(ests, key=lambda e: e[0], reverse=True):
            best_gt, best = -1, threshold
            for gt_id, e in errs:
                if mask[gt_id] and gt_id not in matched and e < best:
                    best_gt, best = gt_id, e
            if best_gt >= 0:
                matched.add(best_gt)
                tps += 1
    return tps / float(tars)


def match_errors(rows: Sequence[dict], errors: np.ndarray, thresholds: Sequence[float],
                 valid: Dict[Tuple[int, int], List[bool]]) -> set:
    """The toolkit's `pose_matching.match_poses` for errors of one or more elements (rete: [re, te]), over every (image,
    object): by decreasing score (stable), each estimate takes the valid, unmatched gt whose error is strictly below the
    best so far in EVERY element, starting from the thresholds.  errors [n_rows, n_elems] (or [n_rows]) already
    normalised.  Returns the matched (scene_id, im_id, gt_id)."""
    ths = [float(x) for x in thresholds]
    errors = np.asarray(errors, np.float64).reshape(len(rows), -1 if len(rows) else len(ths))
    if errors.shape[1] != len(ths):
        raise ValueError(f"{errors.shape[1]} error elements but {len(ths)} thresholds")
    by_est: Dict[Tuple[int, int, int, int], List[Tuple[int, np.ndarray]]] = {}
    for r, e in zip(rows, errors):
        by_est.setdefault((r["scene_id"], r["im_id"], r["obj_id"], r["est_id"]), []).append((r["gt_id"], e))
    score = {(r["scene_id"], r["im_id"], r["obj_id"], r["est_id"]): r["score"] for r in rows}
    groups: Dict[Tuple[int, int, int], List[Tuple[float, List[Tuple[int, np.ndarray]]]]] = {}
    for key, errs in by_est.items():
        groups.setdefault(key[:3], []).append((score[key], errs))
    matched = set()
    for (scene_id, im_id, _), ests in groups.items():
        mask = valid.get((scene_id, im_id))
        if mask is None:
            continue
        for _, errs in sorted(ests, key=lambda e: e[0], reverse=True):
            best_gt, best = -1, ths
            for gt_id, e in errs:
                if mask[gt_id] and (scene_id, im_id, gt_id) not in matched and all(e[j] < best[j] for j in range(len(ths))):
                    best_gt, best = gt_id, e
            if best_gt >= 0:
                matched.add((scene_id, im_id, best_gt))
    return matched


def localization_scores(split: BopSplit, matched: set, valid: Dict[Tuple[int, int], List[bool]]) -> dict:
    """The toolkit's `score.calc_localization_scores` with n_top = -1: recall over the valid gts of the target images,
    per object (every model of models_info) and per scene (every scene of the split); an object or scene without targets
    has recall 0 and counts in the means."""
    obj_ids, scene_ids = sorted(split.models_info), split_scene_ids(split)
    obj_tars, obj_tps = {o: 0 for o in obj_ids}, {o: 0 for o in obj_ids}
    scene_tars, scene_tps = {s: 0 for s in scene_ids}, {s: 0 for s in scene_ids}
    gt_count = tars = tps = 0
    for (scene_id, im_id), mask in valid.items():
        gts = split.scene_gt[scene_id][im_id]
        gt_count += len(gts)
        for gt_id, ok in enumerate(mask):
            if not ok:
                continue
            o = gts[gt_id]["obj_id"]
            tars += 1
            obj_tars[o] += 1
            scene_tars[scene_id] += 1
            if (scene_id, im_id, gt_id) in matched:
                tps += 1
                obj_tps[o] += 1
                scene_tps[scene_id] += 1

    def calc_recall(tp: int, n: int) -> float:
        return tp / float(n) if n else 0.0

    obj_recalls = {o: calc_recall(obj_tps[o], obj_tars[o]) for o in obj_ids}
    scene_recalls = {s: calc_recall(scene_tps[s], scene_tars[s]) for s in scene_ids}
    return dict(recall=calc_recall(tps, tars), obj_recalls=obj_recalls,
                mean_obj_recall=float(np.mean(list(obj_recalls.values()))), scene_recalls=scene_recalls,
                mean_scene_recall=float(np.mean(list(scene_recalls.values()))), gt_count=gt_count, targets_count=tars,
                tp_count=tps)


def resolve_thresholds(thresholds: Optional[Dict[str, Sequence[float]]] = None) -> Dict[str, List[float]]:
    """LOCALIZATION_THRESHOLDS with per-type overrides (the toolkit's --correct_th_<type>), one value per error element."""
    out = {t: list(v) for t, v in LOCALIZATION_THRESHOLDS.items()}
    for t, v in (thresholds or {}).items():
        if t not in out:
            raise ValueError(f"no correctness threshold for error type {t!r} (one of {', '.join(out)})")
        v = [float(x) for x in (v if isinstance(v, (list, tuple, np.ndarray)) else [v])]
        if len(v) != len(out[t]):
            raise ValueError(f"{t} takes {len(out[t])} threshold(s), got {v}")
        out[t] = v
    return out


def score_errors(split: BopSplit, errors_df, ests: Sequence[dict], types=("vsd", "mssd", "mspd"),
                 thresholds: Optional[Dict[str, Sequence[float]]] = None) -> dict:
    """Average recalls of an error table (BopEvaluator.errors) under the bop19 thresholds, then, for each of the other
    types asked for (LOCALIZATION_THRESHOLDS), the toolkit's score dict under `<type>`: recall, obj_recalls,
    mean_obj_recall, scene_recalls, mean_scene_recall, gt_count, targets_count, tp_count.  ad / add / adi errors are
    divided by the diameter; rete is matched on the re and te columns together.  thresholds overrides the defaults per
    type; te thresholds are in mm (the unit of the te errors), as the toolkit compares them."""
    valid = gt_valid_masks(split)
    rows = errors_df[["scene_id", "im_id", "obj_id", "est_id", "gt_id", "score"]].to_dict("records")
    out: dict = {}
    ar = {}
    if "vsd" in types:
        rec = [[recall(split, rows, errors_df[f"vsd_{k}"].to_numpy(), th, valid) for th in VSD_TAUS]
               for k in range(len(VSD_TAUS))]
        out["bop19_recalls_vsd"] = rec
        ar["vsd"] = float(np.mean(rec))
    if "mssd" in types:
        diam = np.array([float(split.models_info[o]["diameter"]) for o in errors_df["obj_id"]], np.float64)
        e = errors_df["mssd"].to_numpy(np.float64) / diam
        rec = [recall(split, rows, e, th, valid) for th in MSSD_THRESHOLDS]
        out["bop19_recalls_mssd"] = rec
        ar["mssd"] = float(np.mean(rec))
    if "mspd" in types:
        widths = np.array([float(split.depth_width(s, i)) for s, i in zip(errors_df["scene_id"], errors_df["im_id"])])
        e = (640.0 / widths) * errors_df["mspd"].to_numpy(np.float64)
        rec = [recall(split, rows, e, th, valid) for th in MSPD_THRESHOLDS]
        out["bop19_recalls_mspd"] = rec
        ar["mspd"] = float(np.mean(rec))
    for k, v in ar.items():
        out[f"bop19_average_recall_{k}"] = v
    if all(k in ar for k in ("vsd", "mssd", "mspd")):
        out["bop19_average_recall"] = float(np.mean([ar["vsd"], ar["mssd"], ar["mspd"]]))
    out["bop19_average_time_per_image"] = average_time_per_image(ests)
    ths = resolve_thresholds(thresholds)
    for t in types:
        if t not in ths:
            continue
        if t == "rete":
            e = errors_df[["re", "te"]].to_numpy(np.float64)
        else:
            e = errors_df[t].to_numpy(np.float64)
            if t in NORMALIZED_BY_DIAMETER:
                e = e / np.array([float(split.models_info[o]["diameter"]) for o in errors_df["obj_id"]], np.float64)
        out[t] = localization_scores(split, match_errors(rows, e, ths[t], valid), valid)
    return out


def select_estimates(split: BopSplit, ests: Sequence[dict]) -> List[dict]:
    """Per target, the top inst_count estimates of its (scene, image, object) by score, ties in input order; each gets
    `est_id`, its index among that (scene, image, object)'s estimates in input order."""
    by_key: Dict[Tuple[int, int, int], List[dict]] = {}
    for e in ests:
        by_key.setdefault((e["scene_id"], e["im_id"], e["obj_id"]), []).append(e)
    out = []
    for t in split.targets:
        cands = by_key.get((t["scene_id"], t["im_id"], t["obj_id"]), [])
        top = sorted(enumerate(cands), key=lambda x: x[1]["score"], reverse=True)[:t["inst_count"]]
        out += [dict(e, est_id=i) for i, e in top]
    return out


# ------------------------------------------------------------------------------------------------------------- evaluator
class BopEvaluator:
    """BOP 2019 evaluation of pose estimates on one split of a BOP dataset, on the device.

    `errors(results)` -> one row per (selected estimate, ground truth of the same object in its image);
    `evaluate(results)` -> the bop19 average recalls, the recalls per threshold and the mean time per image, and the
    toolkit's score dict of each other error type asked for (ERROR_TYPES).

    `ad` takes ADI for the objects of `symmetric_obj_ids` and ADD for the others; by default these are the objects whose
    models_info entry lists symmetries (default_symmetric_obj_ids), which may differ from the toolkit's per-dataset table."""

    def __init__(self, dataset_dir: Union[str, Path], split: str = "test", device: str = "cuda",
                 vsd_delta: Optional[float] = None, max_renders_per_chunk: int = 256,
                 symmetric_obj_ids: Optional[Iterable[int]] = None):
        self.split = load_split(dataset_dir, split)
        self.device = torch.device(device)
        name = Path(dataset_dir).resolve().name
        self.vsd_delta = vsd_delta if vsd_delta is not None else VSD_DELTAS.get(name, VSD_DELTA_DEFAULT)
        self.max_renders = max_renders_per_chunk
        self.symmetric_obj_ids = (sorted(int(o) for o in symmetric_obj_ids) if symmetric_obj_ids is not None
                                  else default_symmetric_obj_ids(self.split.models_info))
        self.obj_ids = sorted(self.split.models)
        self.model_index = {o: i for i, o in enumerate(self.obj_ids)}
        self._renderer = None
        self._points: Optional[PointStore] = None

    # --- device resources
    @property
    def renderer(self):
        if self._renderer is None:
            from .object_dataset import RigidObject, RigidObjectDataset
            from .renderer import BatchRenderer

            ds = RigidObjectDataset([RigidObject(label=f"obj_{o:06d}", mesh=self.split.models[o], mesh_units="mm")
                                     for o in self.obj_ids])
            self._renderer = BatchRenderer(ds)
        return self._renderer

    @property
    def points(self) -> PointStore:
        if self._points is None:
            pts = [np.asarray(self.split.models[o].vertices, np.float64) for o in self.obj_ids]
            syms = [symmetry_transformations(self.split.models_info[o]) for o in self.obj_ids]
            self._points = PointStore(pts, syms, self.device)
        return self._points

    def render_depth(self, obj_ids: Sequence[int], R: np.ndarray, t_mm: np.ndarray, K: np.ndarray,
                     resolution: Tuple[int, int]) -> torch.Tensor:
        """[n, h, w] float32 depth in metres on the device: the rasteriser's depth output for poses (R, t in mm)."""
        n = len(obj_ids)
        TCO = np.zeros((n, 4, 4), np.float64)
        TCO[:, :3, :3] = np.asarray(R, np.float64).reshape(n, 3, 3)
        TCO[:, :3, 3] = np.asarray(t_mm, np.float64).reshape(n, 3) / 1000.0
        TCO[:, 3, 3] = 1.0
        T = torch.from_numpy(TCO).float().to(self.device)
        Kt = torch.from_numpy(np.asarray(K, np.float64).reshape(n, 3, 3)).float().to(self.device)
        out = self.renderer.render([f"obj_{o:06d}" for o in obj_ids], T, Kt, None, resolution, render_depth=True)
        return out.depths[:, 0]

    # --- errors
    def _pairs(self, sel: Sequence[dict]) -> List[dict]:
        rows = []
        for k, e in enumerate(sel):
            for gt_id, gt in enumerate(self.split.scene_gt[e["scene_id"]][e["im_id"]]):
                if gt["obj_id"] == e["obj_id"]:
                    rows.append(dict(scene_id=e["scene_id"], im_id=e["im_id"], obj_id=e["obj_id"], est_id=e["est_id"],
                                     gt_id=gt_id, score=e["score"], _est=k,
                                     _R_gt=np.asarray(gt["cam_R_m2c"], np.float64).reshape(3, 3),
                                     _t_gt=np.asarray(gt["cam_t_m2c"], np.float64).reshape(3)))
        return rows

    def _vsd(self, sel: Sequence[dict], rows: List[dict], types: Sequence[str] = ("vsd",)) -> Dict[str, np.ndarray]:
        """The errors that need renders, vsd and / or cus, from one set of render chunks: {type: errors}.  Both are 1.0
        without rendering where the projections of the bounding spheres do not overlap."""
        out = {}
        if "vsd" in types:
            out["vsd"] = np.ones((len(rows), len(VSD_TAUS)), np.float64)
        if "cus" in types:
            out["cus"] = np.ones(len(rows), np.float64)
        todo = [k for k, r in enumerate(rows)
                if spheres_projections_overlap(0.5 * self.split.models_info[r["obj_id"]]["diameter"], sel[r["_est"]]["t"],
                                               r["_t_gt"])]
        chunk: List[int] = []
        ests, gts = set(), set()
        for k in todo:
            r = rows[k]
            e_key, g_key = r["_est"], (r["scene_id"], r["im_id"], r["gt_id"])
            if chunk and len(ests | {e_key}) + len(gts | {g_key}) > self.max_renders:
                self._vsd_chunk(sel, rows, chunk, out)
                chunk, ests, gts = [], set(), set()
            chunk.append(k)
            ests.add(e_key)
            gts.add(g_key)
        if chunk:
            self._vsd_chunk(sel, rows, chunk, out)
        return out

    def _vsd_chunk(self, sel, rows, chunk: List[int], out: Dict[str, np.ndarray]) -> None:
        by_size: Dict[Tuple[int, int], List[int]] = {}
        depths: Dict[Tuple[int, int], np.ndarray] = {}
        for k in chunk:
            key = (rows[k]["scene_id"], rows[k]["im_id"])
            if key not in depths:
                depths[key] = self.split.depth(*key)
            by_size.setdefault(depths[key].shape, []).append(k)
        for (h, w), ks in by_size.items():
            imgs = list(dict.fromkeys((rows[k]["scene_id"], rows[k]["im_id"]) for k in ks))
            est_keys = list(dict.fromkeys(rows[k]["_est"] for k in ks))
            gt_keys = list(dict.fromkeys((rows[k]["scene_id"], rows[k]["im_id"], rows[k]["gt_id"]) for k in ks))
            im_i = {key: i for i, key in enumerate(imgs)}
            est_i = {key: i for i, key in enumerate(est_keys)}
            gt_i = {key: i for i, key in enumerate(gt_keys)}
            d_est = self.render_depth([sel[e]["obj_id"] for e in est_keys], [sel[e]["R"] for e in est_keys],
                                      [sel[e]["t"] for e in est_keys],
                                      [self.split.K(sel[e]["scene_id"], sel[e]["im_id"]) for e in est_keys], (h, w))
            gt_rows = {(rows[k]["scene_id"], rows[k]["im_id"], rows[k]["gt_id"]): rows[k] for k in ks}
            d_gt = self.render_depth([gt_rows[g]["obj_id"] for g in gt_keys], [gt_rows[g]["_R_gt"] for g in gt_keys],
                                     [gt_rows[g]["_t_gt"] for g in gt_keys], [self.split.K(g[0], g[1]) for g in gt_keys],
                                     (h, w))
            idx = lambda keys: torch.tensor(keys, dtype=torch.int32, device=self.device)  # noqa: E731
            e_idx = idx([est_i[rows[k]["_est"]] for k in ks])
            g_idx = idx([gt_i[(rows[k]["scene_id"], rows[k]["im_id"], rows[k]["gt_id"])] for k in ks])
            if "vsd" in out:
                test = torch.from_numpy(np.stack([depths[key] for key in imgs]).view(np.int16)).to(self.device)
                scale = torch.tensor([self.split.scene_camera[s][i]["depth_scale"] for s, i in imgs],
                                     dtype=torch.float32, device=self.device)
                K = torch.from_numpy(np.stack([self.split.K(s, i) for s, i in imgs])).to(self.device)
                diam = torch.tensor([float(self.split.models_info[rows[k]["obj_id"]]["diameter"]) for k in ks],
                                    dtype=torch.float64, device=self.device)
                err, _ = vsd_from_depths(test, scale, K, d_est, d_gt, e_idx, g_idx,
                                         idx([im_i[(rows[k]["scene_id"], rows[k]["im_id"])] for k in ks]), diam,
                                         self.vsd_delta)
                out["vsd"][ks] = err.cpu().numpy()
            if "cus" in out:
                err, _ = cus_from_depths(d_est, d_gt, e_idx, g_idx)
                out["cus"][ks] = err.cpu().numpy()

    def _point(self, kind: str, sel, rows: List[dict], todo: Optional[List[int]] = None) -> Tuple[np.ndarray, np.ndarray]:
        """Errors of `kind` for rows `todo` (default: every row that the toolkit computes), inf elsewhere."""
        err = np.full(len(rows), np.inf)
        arg = np.full(len(rows), -1, np.int64)
        if kind == "mspd":
            todo = list(range(len(rows)))
        else:  # the toolkit gives inf without computing when the centres are a diameter or more apart
            todo = [k for k in (range(len(rows)) if todo is None else todo)
                    if np.linalg.norm(sel[rows[k]["_est"]]["t"] - rows[k]["_t_gt"])
                    < self.split.models_info[rows[k]["obj_id"]]["diameter"]]
        if not todo:
            return err, arg
        dev = self.device
        m = torch.tensor([self.model_index[rows[k]["obj_id"]] for k in todo], dtype=torch.int32, device=dev)
        pe = torch.from_numpy(np.stack([_pose12(sel[rows[k]["_est"]]["R"], sel[rows[k]["_est"]]["t"]) for k in todo])).to(dev)
        pg = torch.from_numpy(np.stack([_pose12(rows[k]["_R_gt"], rows[k]["_t_gt"]) for k in todo])).to(dev)
        K = None
        if kind == "mspd":
            K = torch.from_numpy(np.stack([self.split.K(rows[k]["scene_id"], rows[k]["im_id"]) for k in todo])).to(dev)
        e, a = self.points.errors(kind, m, pe, pg, K)
        err[todo] = e.cpu().numpy()
        arg[todo] = a.cpu().numpy()
        return err, arg

    def _ad(self, sel, rows: List[dict]) -> np.ndarray:
        """ADI for the rows of symmetric objects, ADD for the others (gated as ADD / ADI)."""
        sym = set(self.symmetric_obj_ids)
        e_adi, _ = self._point("adi", sel, rows, [k for k, r in enumerate(rows) if r["obj_id"] in sym])
        e_add, _ = self._point("add", sel, rows, [k for k, r in enumerate(rows) if r["obj_id"] not in sym])
        return np.where([r["obj_id"] in sym for r in rows], e_adi, e_add)

    def _pose(self, types: Sequence[str], sel, rows: List[dict]) -> Dict[str, np.ndarray]:
        """proj (px), re (degrees) and te (mm) of every row, never gated."""
        if not rows:
            return {t: np.zeros(0) for t in types}
        dev = self.device
        pe = torch.from_numpy(np.stack([_pose12(sel[r["_est"]]["R"], sel[r["_est"]]["t"]) for r in rows])).to(dev)
        pg = torch.from_numpy(np.stack([_pose12(r["_R_gt"], r["_t_gt"]) for r in rows])).to(dev)
        m = K = None
        if "proj" in types:
            m = torch.tensor([self.model_index[r["obj_id"]] for r in rows], dtype=torch.int32, device=dev)
            K = torch.from_numpy(np.stack([self.split.K(r["scene_id"], r["im_id"]) for r in rows])).to(dev)
        return {t: v.cpu().numpy() for t, v in self.points.pose_errors(pe, pg, m, K, types).items()}

    def errors(self, results, types: Iterable[str] = BOP19_TYPES):
        """pandas DataFrame, one row per (selected estimate, ground truth of its object in its image): scene_id, im_id,
        obj_id, est_id, gt_id, score, then per type: vsd_0 .. vsd_9 (one per tau of VSD_TAUS), mssd / mspd / add / adi /
        ad (mm), mspd / proj (px), cus, re (degrees), te (mm), and mssd_sym / mspd_sym (index of the minimising symmetry, -1
        where the error was not computed).  rete writes the re and te columns.  The toolkit's gating: ad / add / adi / mssd
        are inf where the centres are a diameter or more apart, vsd / cus 1.0 where the projections of the bounding
        spheres do not overlap; mspd, proj, re and te are always computed."""
        import pandas as pd

        types = list(dict.fromkeys(types))
        for t in types:
            if t not in ERROR_TYPES:
                raise ValueError(f"unknown error type {t!r} (one of {', '.join(ERROR_TYPES)})")
        sel = select_estimates(self.split, normalize_results(results))
        rows = self._pairs(sel)
        df = pd.DataFrame({k: [r[k] for r in rows] for k in ("scene_id", "im_id", "obj_id", "est_id", "gt_id", "score")})
        rendered = self._vsd(sel, rows, [t for t in types if t in ("vsd", "cus")]) if {"vsd", "cus"} & set(types) else {}
        pose_types = [t for t in ("proj", "re", "te") if t in types or (t != "proj" and "rete" in types)]
        posed = self._pose(pose_types, sel, rows) if pose_types else {}
        for t in types:
            if t == "vsd":
                v = rendered["vsd"]
                for k in range(v.shape[1]):
                    df[f"vsd_{k}"] = v[:, k]
            elif t == "cus":
                df["cus"] = rendered["cus"]
            elif t in KINDS:
                e, a = self._point(t, sel, rows)
                df[t] = e
                if t in ("mssd", "mspd"):
                    df[f"{t}_sym"] = a
            elif t == "ad":
                df["ad"] = self._ad(sel, rows)
            elif t == "rete":
                for c in ("re", "te"):
                    if c not in df:
                        df[c] = posed[c]
            elif t not in df:  # proj, re, te
                df[t] = posed[t]
        return df

    def evaluate(self, results, errors_out: Optional[Union[str, Path]] = None, types: Iterable[str] = BOP19_TYPES,
                 thresholds: Optional[Dict[str, Sequence[float]]] = None) -> dict:
        """score_errors of `errors(results, types)`.  The bop19 keys are those of the bop19 types asked for; each other type
        gets the toolkit's score dict under its name, at LOCALIZATION_THRESHOLDS or the `thresholds` given per type (te in
        mm).  With `ad`, `symmetric_obj_ids` records the objects it scored with ADI."""
        types = list(dict.fromkeys(types))
        ths = resolve_thresholds(thresholds)
        ests = normalize_results(results)
        df = self.errors(ests, types)
        if errors_out is not None:
            Path(errors_out).mkdir(parents=True, exist_ok=True)
            df.to_csv(Path(errors_out) / "errors.csv", index=False)
        scores = score_errors(self.split, df, ests, types, ths)
        if "ad" in types:
            scores["symmetric_obj_ids"] = list(self.symmetric_obj_ids)
        return scores


def parse_error_types(text: str) -> List[str]:
    types = [t.strip() for t in text.split(",") if t.strip()]
    for t in types:
        if t not in ERROR_TYPES:
            raise argparse.ArgumentTypeError(f"unknown error type {t!r} (one of {', '.join(ERROR_TYPES)})")
    return types


def parse_correct_th(text: str) -> Tuple[str, List[float]]:
    """`te=50` or `rete=5,10` -> (type, thresholds)."""
    t, sep, v = text.partition("=")
    if not sep or t.strip() not in LOCALIZATION_THRESHOLDS:
        raise argparse.ArgumentTypeError(f"expected <type>=<threshold>[,<threshold>] with a type among "
                                         f"{', '.join(LOCALIZATION_THRESHOLDS)}, got {text!r}")
    try:
        return t.strip(), [float(x) for x in v.split(",")]
    except ValueError as e:
        raise argparse.ArgumentTypeError(str(e)) from None


def add_error_type_arguments(ap: argparse.ArgumentParser, prefix: str = "") -> None:
    """--[prefix]error-types, --correct-th, --symmetric-obj-ids (shared with prediction_runner --evaluate)."""
    ap.add_argument(f"--{prefix}error-types", type=parse_error_types, default=None,
                    help="comma-separated error types to score instead of the bop19 ones (vsd, mssd, mspd): any of "
                         f"{', '.join(ERROR_TYPES)}; each type other than the bop19 ones gets the BOP toolkit's score dict "
                         "(recall, per-object and per-scene recalls)")
    ap.add_argument("--correct-th", type=parse_correct_th, action="append", default=[], metavar="TYPE=TH[,TH]",
                    help="correctness threshold(s) of one error type, repeatable (the toolkit's --correct_th_<type>); "
                         "defaults: " + ", ".join(f"{t}={','.join(f'{x:g}' for x in v)}"
                                                  for t, v in LOCALIZATION_THRESHOLDS.items())
                         + ". ad/add/adi are fractions of the diameter, proj px, re degrees; te is in mm, the unit of "
                           "its errors, although the toolkit labels it cm")
    ap.add_argument("--symmetric-obj-ids", default=None,
                    help="comma-separated objects that `ad` scores with ADI (default: those with symmetries in "
                         "models_info)")


def error_type_options(args: argparse.Namespace, prefix: str = "") -> dict:
    """BopEvaluator keyword arguments and evaluate() keyword arguments from add_error_type_arguments' options."""
    types = getattr(args, f"{prefix}error_types".replace("-", "_"))
    sym = args.symmetric_obj_ids
    return dict(types=list(types) if types else list(BOP19_TYPES), thresholds=dict(args.correct_th),
                symmetric_obj_ids=[int(o) for o in sym.split(",") if o.strip()] if sym is not None else None)


def main(argv: Optional[Sequence[str]] = None) -> dict:
    ap = argparse.ArgumentParser(description="BOP 2019 average recall (VSD, MSSD, MSPD) of a bop19 results CSV, and the "
                                             "BOP toolkit's other pose-error scores (--error-types)")
    ap.add_argument("dataset_dir")
    ap.add_argument("results_csv")
    ap.add_argument("--split", default="test")
    ap.add_argument("--errors-out", default=None, help="directory for the per-pair error table (errors.csv)")
    add_error_type_arguments(ap)
    args = ap.parse_args(argv)
    opt = error_type_options(args)
    ev = BopEvaluator(args.dataset_dir, args.split, symmetric_obj_ids=opt["symmetric_obj_ids"])
    scores = ev.evaluate(args.results_csv, errors_out=args.errors_out, types=opt["types"], thresholds=opt["thresholds"])
    print(json.dumps(scores))
    return scores


if __name__ == "__main__":
    main()
