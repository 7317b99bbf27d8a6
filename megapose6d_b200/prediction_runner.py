"""Frame-level caller of the pose estimator: a scene dataset sharded over the ranks, one pipeline run per frame, predictions
gathered on every rank, BOP-format export.

Mirrors the caller side of the reference (SURVEY.md 8f.3):
  * `SceneObservation`, `ObservationInfos`, `SceneDataset`            datasets/scene_dataset.py:178-420
  * `DistributedSceneSampler`                                        datasets/samplers.py:41-55
  * `PredictionRunner.{run_inference_pipeline, get_predictions}`     evaluation/prediction_runner.py:49-209
  * `gather_predictions`, `format_results`                           evaluation/runner_utils.py:56-90,
                                                                     utils/tensor_collection.py:165-186
  * `save_bop_results` / `load_bop_results` / `convert_results_to_bop`  evaluation/bop.py:101-137 and the BOP toolkit's
                                                                     `inout.save_bop_results` (bop19 CSV)

Two levels of data parallelism exist and they compose: the hypotheses of ONE frame are sharded over the ranks of the pose
estimator's process group (`parallel.HypothesisSharder`, lowest latency per frame), and FRAMES are sharded over the ranks
of the runner's group (this file; highest throughput, no collective on the data path).  With `frame_parallel=True` (the
reference's scheme) the estimator must not shard hypotheses over the same ranks — every rank then works on a different
frame — and `PredictionRunner` asserts that.

What differs from the reference, deliberately: predictions are exchanged with one `all_gather_object` per prediction key
(the reference writes `rank=<r>.pth.tar` files into a shared temporary directory between two barriers) and EVERY rank gets
the concatenated result (the reference: rank 0 only; the order — rank 0's rows, then rank 1's, ... — is the same); the
next frame's host->device copy is issued on a side stream from pinned memory while the current frame runs; the PyTorch
`DataLoader` worker processes are replaced by a one-frame look-ahead thread (decoding a PNG is ~100x cheaper than the
reference's pipeline was, but not cheaper than a 13 ms pipeline).
"""
from __future__ import annotations

import copy
import threading
import time
from collections import defaultdict
from dataclasses import dataclass
from pathlib import Path
from typing import Any, Dict, Iterator, List, Optional, Sequence

import numpy as np
import pandas as pd
import torch
import torch.distributed as dist

from . import tensor_collection as tc
from .example import CameraData, ObjectData, load_object_data, load_observation
from .tensor_collection import PandasTensorCollection
from .types import DetectionsType, InferenceConfig, ObservationTensor, PoseEstimatesType


# ----------------------------------------------------------------------------------------------- scene observations
@dataclass
class ObservationInfos:
    scene_id: Any
    view_id: Any


@dataclass
class SceneObservation:
    """One frame: image(s), camera, annotated objects (datasets/scene_dataset.py:194-205)."""
    rgb: Optional[np.ndarray] = None  # [h,w,3] uint8
    depth: Optional[np.ndarray] = None  # [h,w] float32, metres
    infos: Optional[ObservationInfos] = None
    object_datas: Optional[List[ObjectData]] = None
    camera_data: Optional[CameraData] = None

    def as_pandas_tensor_collection(self, object_labels: Optional[Sequence[str]] = None) -> PandasTensorCollection:
        """infos{label, scene_id, view_id, visib_fract} + TCO/poses [B,4,4], bboxes [B,4] (modal), K [B,3,3]
        (+ TCO_init/poses_init when the objects carry initial poses): datasets/scene_dataset.py:301-381."""
        assert self.camera_data is not None and self.object_datas is not None and self.infos is not None
        keep = None if object_labels is None else set(object_labels)
        TWC = np.eye(4) if self.camera_data.TWC is None else np.asarray(self.camera_data.TWC, dtype=np.float64)
        TCW = torch.linalg.inv(torch.as_tensor(TWC).float())
        rows, TWO, TWO_init, boxes = [], [], [], []
        for obj in self.object_datas:
            if keep is not None and obj.label not in keep:
                continue
            rows.append(dict(label=obj.label, scene_id=self.infos.scene_id, view_id=self.infos.view_id,
                             visib_fract=1 if obj.visib_fract is None else obj.visib_fract))
            TWO.append(torch.as_tensor(np.eye(4) if obj.TWO is None else obj.TWO).float())
            assert obj.bbox_modal is not None, f"object {obj.label}: bbox_modal is required"
            boxes.append(torch.as_tensor(np.asarray(obj.bbox_modal)).float())
            if obj.TWO_init is not None:
                TWO_init.append(torch.as_tensor(obj.TWO_init).float())
        assert rows, "no object left in this observation"
        TCO = TCW.unsqueeze(0) @ torch.stack(TWO)
        K = torch.as_tensor(np.asarray(self.camera_data.K)).unsqueeze(0).expand(len(rows), -1, -1)
        data = PandasTensorCollection(infos=pd.DataFrame(rows), TCO=TCO, bboxes=torch.stack(boxes), poses=TCO.clone(), K=K)
        if TWO_init:
            assert len(TWO_init) == len(rows), "either all objects or none carry TWO_init"
            TWC_init = TWC if self.camera_data.TWC_init is None else self.camera_data.TWC_init
            TCO_init = torch.linalg.inv(torch.as_tensor(np.asarray(TWC_init)).float()).unsqueeze(0) @ torch.stack(TWO_init)
            data.register_tensor("TCO_init", TCO_init)
            data.register_tensor("poses_init", TCO_init.clone())
        return data

    @staticmethod
    def collate_fn(batch: List["SceneObservation"], object_labels: Optional[Sequence[str]] = None) -> Dict[str, Any]:
        """cameras{K}, rgb [B,3,H,W] uint8, depth [B,1,H,W] | [B,0], im_infos, gt_detections (score = 1), gt_data,
        initial_data | None (datasets/scene_dataset.py:206-299)."""
        cam_rows, Ks, im_infos, rgbs, depths, gt, det, init = [], [], [], [], [], [], [], []
        for batch_im_id, obs in enumerate(batch):
            assert obs.infos is not None and obs.camera_data is not None and obs.rgb is not None
            im_infos.append(dict(scene_id=obs.infos.scene_id, view_id=obs.infos.view_id, batch_im_id=batch_im_id))
            Ks.append(np.asarray(obs.camera_data.K))
            cam_rows.append(dict(TWC=obs.camera_data.TWC, resolution=obs.camera_data.resolution))
            rgbs.append(torch.from_numpy(np.array(obs.rgb, dtype=np.uint8)).permute(2, 0, 1))
            depths.append(np.array([]) if obs.depth is None else np.expand_dims(obs.depth, 0))
            g = obs.as_pandas_tensor_collection(object_labels)
            g.infos["batch_im_id"] = batch_im_id
            gt.append(g)
            if "poses_init" in g.tensors:
                i = copy.deepcopy(g)
                i.poses = i.poses_init
                init.append(i)
            d = copy.deepcopy(g)
            d.infos["score"] = 1.0
            det.append(d)
        return dict(cameras=PandasTensorCollection(infos=pd.DataFrame(cam_rows), K=torch.as_tensor(np.stack(Ks))),
                    rgb=torch.stack(rgbs), depth=torch.as_tensor(np.stack(depths)), im_infos=im_infos,
                    gt_detections=tc.concatenate(det), gt_data=tc.concatenate(gt),
                    initial_data=tc.concatenate(init) if init else None)


class SceneDataset:
    """Map-style dataset over `frame_index` (columns scene_id, view_id): datasets/scene_dataset.py:384-420."""

    def __init__(self, frame_index: Optional[pd.DataFrame], load_depth: bool = False):
        self.frame_index = frame_index
        self.load_depth = load_depth

    def _load_scene_observation(self, image_infos: ObservationInfos) -> SceneObservation:
        raise NotImplementedError

    def __getitem__(self, idx: int) -> SceneObservation:
        assert self.frame_index is not None
        row = self.frame_index.iloc[idx]
        return self._load_scene_observation(ObservationInfos(scene_id=row.scene_id, view_id=row.view_id))

    def __len__(self) -> int:
        assert self.frame_index is not None
        return len(self.frame_index)


class ListSceneDataset(SceneDataset):
    """In-memory frames (synthetic scenes of the tests and benches)."""

    def __init__(self, observations: Sequence[SceneObservation], load_depth: bool = False):
        frame_index = pd.DataFrame(dict(scene_id=[o.infos.scene_id for o in observations],
                                        view_id=[o.infos.view_id for o in observations]))
        super().__init__(frame_index, load_depth)
        self._by_key = {(o.infos.scene_id, o.infos.view_id): o for o in observations}
        assert len(self._by_key) == len(observations), "(scene_id, view_id) must be unique"

    def _load_scene_observation(self, image_infos: ObservationInfos) -> SceneObservation:
        obs = self._by_key[(image_infos.scene_id, image_infos.view_id)]
        return obs if self.load_depth else SceneObservation(obs.rgb, None, obs.infos, obs.object_datas, obs.camera_data)


class ExampleDirSceneDataset(SceneDataset):
    """Frames stored as directories in the README example's layout (`image_rgb.png`, `image_depth.png`, `camera_data.json`,
    `inputs/object_data.json`): scene_id = position of the directory in `example_dirs`, view_id = 0."""

    def __init__(self, example_dirs: Sequence[Path], load_depth: bool = False):
        self.example_dirs = [Path(d) for d in example_dirs]
        super().__init__(pd.DataFrame(dict(scene_id=np.arange(len(self.example_dirs)), view_id=0)), load_depth)

    def _load_scene_observation(self, image_infos: ObservationInfos) -> SceneObservation:
        d = self.example_dirs[int(image_infos.scene_id)]
        rgb, depth, camera = load_observation(d, load_depth=self.load_depth)
        return SceneObservation(rgb, depth, image_infos, load_object_data(d / "inputs" / "object_data.json"), camera)


# -------------------------------------------------------------------------------------------------- frame sharding
class DistributedSceneSampler:
    """Rank r's frames: `np.array_split` of the (seed-0 shuffled) frame indices (datasets/samplers.py:41-55).  The shuffle
    spreads the scenes, whose frames differ in cost, evenly over the ranks; the global numpy state is left untouched."""

    def __init__(self, scene_ds, num_replicas: int, rank: int, shuffle: bool = True):
        assert 0 <= rank < num_replicas
        indices = np.arange(len(scene_ds))
        if shuffle:
            state = np.random.get_state()
            np.random.seed(0)
            try:
                indices = np.random.permutation(indices)
            finally:
                np.random.set_state(state)
        self.local_indices = np.array_split(indices, num_replicas)[rank].tolist()

    def __len__(self) -> int:
        return len(self.local_indices)

    def __iter__(self) -> Iterator[int]:
        return iter(self.local_indices)


def _world(group) -> tuple:
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(group), dist.get_world_size(group)
    return 0, 1


def gather_distributed(data: PandasTensorCollection, group=None) -> PandasTensorCollection:
    """Concatenation of every rank's collection in rank order, on every rank, on the CPU
    (utils/tensor_collection.py:165-186 exchanges files and returns the concatenation on rank 0 only)."""
    rank, world = _world(group)
    data = data.cpu()
    if world == 1:
        return tc.concatenate([data])
    parts: List[Optional[PandasTensorCollection]] = [None] * world
    dist.all_gather_object(parts, data, group=group)
    return tc.concatenate(parts)


def gather_predictions(all_predictions: Dict[str, PandasTensorCollection], group=None) -> Dict[str, PandasTensorCollection]:
    """evaluation/runner_utils.py:56-59.  Keys are visited in sorted order so that the ranks issue matching collectives."""
    return {k: gather_distributed(all_predictions[k], group) for k in sorted(all_predictions)}


def format_results(predictions: Dict[str, PandasTensorCollection], eval_metrics: Optional[dict] = None,
                   eval_dfs: Optional[dict] = None) -> Dict[str, Any]:
    """The dict the reference saves as results.pth.tar (evaluation/runner_utils.py:62-90)."""
    eval_metrics, eval_dfs = eval_metrics or {}, eval_dfs or {}
    summary, table, txt = {}, defaultdict(list), ""
    for method, metrics in eval_metrics.items():
        txt += f"\n{method}\n{'-' * 80}\n"
        for name, value in metrics.items():
            summary[f"{method}/{name}"] = value
            table["method"].append(method)
            table["metric"].append(name)
            table["value"].append(value)
            txt += f"{method}/{name}: {value}\n"
        txt += "-" * 80
    return dict(summary=summary, summary_txt=txt, predictions=predictions, metrics=eval_metrics,
                summary_df=pd.DataFrame(table), dfs=eval_dfs)


# ----------------------------------------------------------------------------------------------------- BOP results
BOP19_HEADER = "scene_id,im_id,obj_id,score,R,t,time"


def save_bop_results(path: Path, results: Sequence[dict]) -> None:
    """bop19 CSV: one line per estimate, R row-major and t (millimetres) space-separated, no trailing newline (the BOP
    toolkit's `inout.save_bop_results`, vendored by the reference under deps/bop_toolkit_challenge)."""
    lines = [BOP19_HEADER]
    for r in results:
        R = " ".join(str(v) for v in np.asarray(r["R"]).flatten().tolist())
        t = " ".join(str(v) for v in np.asarray(r["t"]).flatten().tolist())
        lines.append(f"{r['scene_id']},{r['im_id']},{r['obj_id']},{r['score']},{R},{t},{r.get('time', -1)}")
    Path(path).write_text("\n".join(lines))


def load_bop_results(path: Path) -> List[dict]:
    out = []
    for n, line in enumerate(Path(path).read_text().splitlines()):
        if n == 0 and BOP19_HEADER in line:
            continue
        if not line.strip():
            continue
        e = line.split(",")
        if len(e) != 7:
            raise ValueError(f"A line does not have 7 comma-sep. elements: {line}")
        out.append(dict(scene_id=int(e[0]), im_id=int(e[1]), obj_id=int(e[2]), score=float(e[3]),
                        R=np.array([float(v) for v in e[4].split()]).reshape(3, 3),
                        t=np.array([float(v) for v in e[5].split()]).reshape(3, 1), time=float(e[6])))
    return out


def predictions_to_bop(predictions: PoseEstimatesType, use_pose_score: bool = True) -> List[dict]:
    """evaluation/bop.py:101-134: translation in millimetres, obj_id = the integer after the label's last underscore."""
    poses = predictions.poses.detach().cpu()
    out = []
    for n in range(len(predictions)):
        row = predictions.infos.iloc[n]
        out.append(dict(scene_id=row.scene_id, im_id=row.view_id, obj_id=int(str(row.label).split("_")[-1]),
                        score=row.pose_score if use_pose_score else row.score,
                        t=poses[n, :3, -1] * 1e3, R=poses[n, :3, :3], time=row.time if "time" in row else -1))
    return out


def convert_results_to_bop(results_path: Path, out_csv_path: Path, method: str, use_pose_score: bool = True) -> Path:
    """results.pth.tar (`format_results`) -> bop19 CSV for prediction key `method` (evaluation/bop.py:101-137)."""
    predictions = torch.load(results_path, weights_only=False)["predictions"][method]
    Path(out_csv_path).parent.mkdir(exist_ok=True, parents=True)
    save_bop_results(out_csv_path, predictions_to_bop(predictions, use_pose_score))
    return Path(out_csv_path)


# ----------------------------------------------------------------------------------------------- prediction runner
class _LookAhead:
    """Iterates `make(i) for i in ids`, building item k+1 on a thread while the consumer works on item k."""

    def __init__(self, ids: Sequence[int], make):
        self.ids, self.make = list(ids), make

    def __iter__(self):
        box: Dict[str, Any] = {}

        def work(i):
            try:
                box["value"] = self.make(i)
            except BaseException as e:  # re-raised in the consumer
                box["error"] = e

        thread = None
        for k, i in enumerate(self.ids):
            if thread is None:
                work(i)
            else:
                thread.join()
            if "error" in box:
                raise box.pop("error")
            value = box.pop("value")
            thread = None
            if k + 1 < len(self.ids):
                thread = threading.Thread(target=work, args=(self.ids[k + 1],), daemon=True)
                thread.start()
            yield value


class PredictionRunner:
    """evaluation/prediction_runner.py:49-209.  `device="cuda"` is the product path; `device="cpu"` only moves the containers
    (host-logic tests with a stand-in estimator — the real estimator has no CPU path)."""

    def __init__(self, scene_ds: SceneDataset, inference_cfg: InferenceConfig, batch_size: int = 1, n_workers: int = 1,
                 group=None, frame_parallel: bool = True, device: str = "cuda"):
        assert batch_size == 1, "one frame per pipeline call (evaluation/evaluation.py:158)"
        self.inference_cfg = inference_cfg
        self.group = group
        self.rank, self.world_size = _world(group) if frame_parallel else (0, 1)
        self.frame_parallel = frame_parallel
        self.sampler = DistributedSceneSampler(scene_ds, num_replicas=self.world_size, rank=self.rank)
        self.scene_ds = scene_ds
        self.batch_size = batch_size
        self.n_workers = n_workers
        self.load_depth = scene_ds.load_depth
        self.device = torch.device(device)
        self.frame_times: List[dict] = []

    # -- one frame
    def run_inference_pipeline(self, pose_estimator, obs_tensor: ObservationTensor, gt_detections: DetectionsType,
                               initial_estimates: Optional[PoseEstimatesType] = None) -> Dict[str, PoseEstimatesType]:
        """Keys: 'final', 'refiner/iteration=<n>', 'refiner/final', 'coarse' (+ 'depth_refiner')."""
        cfg = self.inference_cfg
        if cfg.detection_type == "gt":
            detections, run_detector = gt_detections, False
        elif cfg.detection_type == "detector":
            detections, run_detector = None, True
        else:
            raise ValueError(f"Unknown detection type {cfg.detection_type}")
        coarse_estimates = None
        if cfg.coarse_estimation_type == "external":
            from .pose_estimator import add_instance_id

            assert initial_estimates is not None, "coarse_estimation_type='external' needs initial poses in the dataset"
            coarse_estimates = add_instance_id(initial_estimates)
            coarse_estimates.infos["instance_id"] = 0
            run_detector = False
        preds, extra_data = pose_estimator.run_inference_pipeline(
            obs_tensor, detections=detections, run_detector=run_detector, coarse_estimates=coarse_estimates,
            n_refiner_iterations=cfg.n_refiner_iterations, n_pose_hypotheses=cfg.n_pose_hypotheses,
            run_depth_refiner=cfg.run_depth_refiner, bsz_images=cfg.bsz_images, bsz_objects=cfg.bsz_objects)
        refined = extra_data["refiner"]["preds"]
        all_preds = {"final": preds, f"refiner/iteration={cfg.n_refiner_iterations}": refined, "refiner/final": refined,
                     "coarse": extra_data["coarse"]["preds"]}
        if cfg.run_depth_refiner:
            all_preds["depth_refiner"] = extra_data["depth_refiner"]["preds"]
        scene_id = np.unique(gt_detections.infos["scene_id"]).item()
        view_id = np.unique(gt_detections.infos["view_id"]).item()
        for v in all_preds.values():
            v.infos["scene_id"] = scene_id
            v.infos["view_id"] = view_id
            if "mask" in v.tensors:
                v.delete_tensor("mask")
        return all_preds

    # -- host side of a frame: decode, collate, pin
    def _load(self, idx: int) -> Dict[str, Any]:
        data = SceneObservation.collate_fn([self.scene_ds[idx]])
        if self.device.type == "cuda":
            data["rgb"] = data["rgb"].pin_memory()
            if data["depth"].numel():
                data["depth"] = data["depth"].float().pin_memory()
        return data

    def _to_device(self, data: Dict[str, Any]) -> Dict[str, Any]:
        """Observation and detections on the device.  On CUDA the copies run on `self._copy_stream`; the event recorded
        after them is waited on by the compute stream before the frame is used."""
        depth = data["depth"] if data["depth"].numel() else None
        if self.device.type != "cuda":
            obs = ObservationTensor.from_torch_batched(data["rgb"], depth, data["cameras"].K)
            return dict(obs=obs, det=data["gt_detections"], init=data["initial_data"], ready=None)
        with torch.cuda.stream(self._copy_stream):
            rgb = data["rgb"].to(self.device, non_blocking=True)
            depth_d = None if depth is None else depth.to(self.device, non_blocking=True)
            obs = ObservationTensor.from_torch_batched(rgb, depth_d, data["cameras"].K.to(self.device))
            det = data["gt_detections"].to(self.device)
            init = None if data["initial_data"] is None else data["initial_data"].to(self.device)
            ready = torch.cuda.Event()
            ready.record(self._copy_stream)
        return dict(obs=obs, det=det, init=init, ready=ready)

    # -- all frames of this rank
    def get_predictions(self, pose_estimator) -> Dict[str, PoseEstimatesType]:
        """Runs this rank's frames (the first one twice: warm-up, as evaluation/prediction_runner.py:185-190) and returns the
        per-key concatenation of the per-frame predictions; every row carries `time` = seconds of its frame's pipeline."""
        sharder = getattr(pose_estimator, "sharder", None)
        if self.frame_parallel and self.world_size > 1 and sharder is not None and getattr(sharder, "world", 1) > 1:
            raise AssertionError("frame_parallel=True: build the estimator without a hypothesis `sharder` "
                                 "(the PoseEstimator default); every rank runs different frames")
        cuda = self.device.type == "cuda"
        if cuda:
            self._copy_stream = torch.cuda.Stream(self.device)
        predictions_list: Dict[str, List[PoseEstimatesType]] = defaultdict(list)
        self.frame_times = []
        staged = None
        frames = iter(_LookAhead(list(self.sampler), self._load))
        nxt = next(frames, None)
        if nxt is not None:
            staged = self._to_device(nxt)
        n = 0
        while staged is not None:
            cur, host = staged, nxt
            nxt = next(frames, None)
            if cuda:
                torch.cuda.current_stream(self.device).wait_event(cur["ready"])
            if n == 0:
                self.run_inference_pipeline(pose_estimator, cur["obs"], cur["det"], initial_estimates=cur["init"])
            # the next frame's copies overlap this frame's pipeline
            staged = self._to_device(nxt) if nxt is not None else None
            if cuda:
                torch.cuda.synchronize(self.device)
            t0 = time.perf_counter()
            all_preds = self.run_inference_pipeline(pose_estimator, cur["obs"], cur["det"], initial_estimates=cur["init"])
            if cuda:
                torch.cuda.synchronize(self.device)
            elapsed = time.perf_counter() - t0
            self.frame_times.append(dict(scene_id=host["im_infos"][0]["scene_id"], view_id=host["im_infos"][0]["view_id"],
                                         time=elapsed, n_detections=len(cur["det"])))
            for k, v in all_preds.items():
                v.infos["time"] = elapsed
                predictions_list[k].append(v)
            n += 1
        return {k: tc.concatenate(v) for k, v in predictions_list.items()}


def run_predictions(scene_ds: SceneDataset, pose_estimator, inference_cfg: InferenceConfig, save_dir: Optional[Path] = None,
                    group=None, device: str = "cuda") -> Dict[str, Any]:
    """The inference half of evaluation/evaluation.py:71-231 (`run_eval` with `skip_evaluation`): shard the frames, predict,
    gather, and on rank 0 save `results.pth.tar` / `predictions.pth.tar` (+ the BOP CSV of 'refiner/final') under `save_dir`."""
    runner = PredictionRunner(scene_ds, inference_cfg, group=group, device=device)
    with torch.no_grad():
        all_preds = runner.get_predictions(pose_estimator)
    # ranks without frames still take part in the collectives, with the same keys
    keys = ["final", f"refiner/iteration={inference_cfg.n_refiner_iterations}", "refiner/final", "coarse"]
    if inference_cfg.run_depth_refiner:
        keys.append("depth_refiner")
    for k in keys:
        all_preds.setdefault(k, PandasTensorCollection(infos=pd.DataFrame()))
    all_preds = gather_predictions(all_preds, group)
    results = format_results(all_preds)
    out = dict(results=results, pred_keys=list(all_preds.keys()), frame_times=runner.frame_times, save_dir=None)
    if save_dir is not None and runner.rank == 0:
        save_dir = Path(save_dir)
        save_dir.mkdir(exist_ok=True, parents=True)
        torch.save(results, save_dir / "results.pth.tar")
        torch.save(results["predictions"], save_dir / "predictions.pth.tar")
        if len(all_preds["refiner/final"]) > 0:
            convert_results_to_bop(save_dir / "results.pth.tar", save_dir / "bop_refiner_final.csv", "refiner/final")
        out["save_dir"] = save_dir
        out["results_path"] = save_dir / "results.pth.tar"
    return out


def main(argv: Optional[List[str]] = None) -> None:
    """python -m megapose6d_b200.prediction_runner <frame_dir> [<frame_dir> ...] --model <name> --save-dir <dir>
    Frames in the README example's layout; the meshes are read from `--meshes-from` (default: the first frame directory).
    python -m megapose6d_b200.prediction_runner --bop-dataset <dir> [--split test] [--label-format "{label}"] [--evaluate]
    --model <name> --save-dir <dir>
    The bop19 target frames of a BOP split (bop_dataset.keep_bop19(BOPDataset(...))) with the meshes of <dir>/models and the
    ground truth as detections; `--evaluate` scores the 'refiner/final' CSV with bop_eval.BopEvaluator on rank 0
    (`--eval-error-types`, `--correct-th`, `--symmetric-obj-ids` as bop_eval's CLI), prints the scores as one JSON line and saves them as <save-dir>/bop19_scores.json.
    Under torchrun the frames are sharded over the ranks (one process per GPU) and rank 0 writes the results."""
    import argparse
    import json
    import os

    from .example import make_object_dataset
    from .load_model import NAMED_MODELS, load_named_model

    parser = argparse.ArgumentParser(description="Pose predictions for a list of frames or a BOP split, BOP-format output")
    parser.add_argument("frame_dirs", type=Path, nargs="*")
    parser.add_argument("--bop-dataset", type=Path, default=None, help="a dataset in the BOP format (instead of frame dirs)")
    parser.add_argument("--split", default="test", help="split of --bop-dataset")
    parser.add_argument("--label-format", default="{label}", help="object labels of --bop-dataset (the reference's "
                        "label_format, e.g. 'ycbv-{label}')")
    parser.add_argument("--evaluate", action="store_true", help="BOP 2019 scores of the predictions on --bop-dataset")
    from .bop_eval import add_error_type_arguments

    add_error_type_arguments(parser, prefix="eval-")  # --eval-error-types, --correct-th, --symmetric-obj-ids
    parser.add_argument("--model", type=str, default="megapose-1.0-RGB-multi-hypothesis", choices=sorted(NAMED_MODELS))
    parser.add_argument("--models-root", type=Path, default=None)
    parser.add_argument("--meshes-from", type=Path, default=None)
    parser.add_argument("--save-dir", type=Path, required=True)
    parser.add_argument("--depth-refiner", choices=["icp", "teaserpp"], default=None,
                        help="refine the final poses against the frames' depth (evaluation/evaluation.py:132-139)")
    parser.add_argument("--detector", type=str, default=None, metavar="RUN_ID",
                        help="detect objects with this Mask R-CNN run (under --models-root) instead of using the ground "
                        "truth as detections (detection_type='detector')")
    parser.add_argument("--detector-engine", action="store_true",
                        help="run the detector's ResNet-50 FPN backbone and RPN head on the engine's convolutions")
    parser.add_argument("--detector-device-paste", action="store_true",
                        help="as --detector-engine, and turn the detector's mask logits into image-sized masks on the device")
    parser.add_argument("--detector-engine-roi-heads", action="store_true",
                        help="as --detector-device-paste, and run the detector's RoI box and mask branches on the engine")
    args = parser.parse_args(argv)
    if args.detector_engine_roi_heads:
        args.detector_device_paste = True
    if args.detector_device_paste:
        args.detector_engine = True
    if args.detector_engine and args.detector is None:
        parser.error("--detector-engine needs --detector")
    if bool(args.frame_dirs) == (args.bop_dataset is not None):
        parser.error("give either frame directories or --bop-dataset")
    if args.evaluate and args.bop_dataset is None:
        parser.error("--evaluate needs --bop-dataset")
    if args.bop_dataset is not None and args.meshes_from is not None:
        parser.error("--meshes-from applies to frame directories; --bop-dataset reads <dir>/models")
    if "RANK" in os.environ and not dist.is_initialized():
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
        dist.init_process_group("nccl")
    info = NAMED_MODELS[args.model]
    if args.depth_refiner is not None and not info["requires_depth"]:
        parser.error(f"--depth-refiner needs a model that loads depth; {args.model} does not")
    params = info["inference_parameters"]
    cfg = InferenceConfig(detection_type="gt" if args.detector is None else "detector", n_refiner_iterations=params["n_refiner_iterations"],
                          n_pose_hypotheses=params["n_pose_hypotheses"], run_depth_refiner=args.depth_refiner is not None,
                          depth_refiner=args.depth_refiner, bsz_images=576, bsz_objects=16)
    if args.bop_dataset is not None:
        from .bop_dataset import BOPDataset, BOPObjectDataset, keep_bop19

        object_dataset = BOPObjectDataset(args.bop_dataset / "models", label_format=args.label_format)
        scene_ds = keep_bop19(BOPDataset(args.bop_dataset, label_format=args.label_format, split=args.split,
                                         load_depth=info["requires_depth"]))
    else:
        object_dataset = make_object_dataset(args.meshes_from or args.frame_dirs[0])
        scene_ds = ExampleDirSceneDataset(args.frame_dirs, load_depth=info["requires_depth"])
    pose_estimator = load_named_model(args.model, object_dataset, models_root=args.models_root).cuda()
    if args.depth_refiner is not None:
        from .icp_refiner import ICPRefiner
        from .teaserpp_refiner import TeaserppRefiner

        cls = ICPRefiner if args.depth_refiner == "icp" else TeaserppRefiner
        pose_estimator.depth_refiner = cls(pose_estimator.refiner_model.mesh_db, pose_estimator.refiner_model.renderer)
    if args.detector is not None:
        from .detector import load_detector

        pose_estimator.detector_model = load_detector(args.detector, models_root=args.models_root,
                                                      engine=args.detector_engine, device_paste=args.detector_device_paste,
                                                      engine_roi_heads=args.detector_engine_roi_heads)
    out = run_predictions(scene_ds, pose_estimator, cfg, save_dir=args.save_dir)
    if out["save_dir"] is not None:
        n = len(out["results"]["predictions"]["final"])
        print(f"wrote {n} pose(s) of {len(scene_ds)} frame(s) to {out['save_dir']}")
        if args.evaluate:
            from .bop_eval import BopEvaluator, error_type_options

            csv = out["save_dir"] / "bop_refiner_final.csv"
            opt = error_type_options(args, prefix="eval-")
            scores = BopEvaluator(args.bop_dataset, args.split, symmetric_obj_ids=opt["symmetric_obj_ids"]).evaluate(
                csv if csv.exists() else [], types=opt["types"], thresholds=opt["thresholds"])
            (out["save_dir"] / "bop19_scores.json").write_text(json.dumps(scores))
            print(json.dumps(scores))
    if dist.is_initialized():
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
