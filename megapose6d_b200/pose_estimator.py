"""Pipeline orchestrator: detections -> coarse scoring of the SO(3) grid -> top-K -> refiner -> scoring.

Drop-in for the reference's PoseEstimator (src/megapose/inference/pose_estimator.py:52-667): same
constructor, attributes, methods (`run_inference_pipeline`, `forward_coarse_model`, `forward_refiner`,
`forward_scoring_model`, `filter_pose_estimates`, `forward_detection_model`, `run_depth_refiner`) and
the same structure of the returned collections and `extra_data` dictionaries.

Differences underneath: the B*M hypothesis table is built vectorised and scored in a few large fused
launches instead of ceil(B*M / bsz_images) Python iterations; the frame is never replicated per
hypothesis; pandas bookkeeping happens once per stage, after the GPU work; optionally the rows of each
stage are sharded over the ranks of a torch.distributed group (see parallel.py).
"""
from __future__ import annotations

import time
from collections import defaultdict
from typing import Any, Optional, Tuple

import numpy as np
import pandas as pd
import torch

from . import lib3d, tensor_collection as tc
from .parallel import HypothesisSharder
from .so3 import load_SO3_grid
from .tensor_collection import PandasTensorCollection
from .types import DetectionsType, ObservationTensor, PoseEstimatesType, assert_detections_valid


def order_desc_nan_last(x: torch.Tensor) -> torch.Tensor:
    """Indices that sort the 1-D `x` by descending value with NaN last and ties in index order, as the reference's
    `sort_values(ascending=False)` orders its rows (and `filter_pose_estimates` on the host).  torch.sort alone puts NaN
    first: NaN is sorted as -inf here, then moved behind the real -inf entries by a second stable sort."""
    nan = torch.isnan(x)
    order = torch.sort(torch.where(nan, torch.full_like(x, float("-inf")), x), descending=True, stable=True).indices
    return order[torch.sort(nan[order].to(torch.int32), stable=True).indices]


def best_per_group(logits: torch.Tensor, group: torch.Tensor, n_groups: int) -> torch.Tensor:
    """Rows of `sort_values(logit, ascending=False).groupby(group).head(1)`, in that order: each group's best row (NaN
    last, ties to the lower row), groups ordered by the position of their best row.  Every group must own a row."""
    order = order_desc_nan_last(logits)
    pos = torch.arange(logits.numel(), device=logits.device)
    first = torch.full((n_groups,), logits.numel(), device=logits.device, dtype=torch.long)
    first.scatter_reduce_(0, group[order], pos, "amin")
    return order[torch.sort(first).values]


def add_instance_id(inputs):
    """inference/utils.py:151-171: unique id per (batch_im_id, label) occurrence."""
    if "instance_id" in inputs.infos:
        return inputs
    df = inputs.infos
    df["instance_id"] = df.groupby(["batch_im_id", "label"]).cumcount().values
    inputs.infos = df
    return inputs


def filter_detections(detections: DetectionsType, labels=None, one_instance_per_class: bool = False) -> DetectionsType:
    """inference/utils.py:174-194."""
    if labels is not None:
        df = detections.infos
        df = df[df.label.isin(labels)]
        detections = detections[df.index.tolist()]
    if one_instance_per_class:
        df = detections.infos
        df = df.sort_values("score", ascending=False).groupby(["batch_im_id", "label"]).head(1)
        detections = detections[df.index.tolist()]
    return detections


class PendingInference:
    """Handle of PoseEstimator.submit_inference_pipeline: the frame's device work is enqueued, `.result()` waits for it."""

    def __init__(self, finish, inputs, out):
        self._finish, self._inputs, self._out = finish, inputs, out  # the inputs stay referenced until the device is done

    @property
    def done(self) -> bool:
        return self._finish is None

    def result(self):
        if self._finish is not None:
            self._out = self._finish()
            self._finish = self._inputs = None
        return self._out


class PoseEstimator(torch.nn.Module):
    """Performs inference for pose estimation."""

    def __init__(self, refiner_model: Optional[torch.nn.Module] = None, coarse_model: Optional[torch.nn.Module] = None,
                 detector_model: Optional[torch.nn.Module] = None, depth_refiner: Optional[Any] = None,
                 bsz_objects: int = 8, bsz_images: int = 256, SO3_grid_size: int = 576,
                 sharder: Optional[HypothesisSharder] = None) -> None:
        super().__init__()
        self.coarse_model = coarse_model
        self.refiner_model = refiner_model
        self.detector_model = detector_model
        self.depth_refiner = depth_refiner
        self.bsz_objects = bsz_objects
        self.bsz_images = bsz_images
        self.sharder = sharder if sharder is not None else HypothesisSharder(enabled=False)
        if SO3_grid_size is not None:
            self.load_SO3_grid(SO3_grid_size)
        if self.refiner_model is not None:
            self.cfg = getattr(self.refiner_model, "cfg", None)
            self.mesh_db = self.refiner_model.mesh_db
        elif self.coarse_model is not None:
            self.cfg = getattr(self.coarse_model, "cfg", None)
            self.mesh_db = self.coarse_model.mesh_db
        else:
            raise ValueError("At least one of refiner_model or coarse_model must be specified.")
        self.eval()
        self.fused_pipeline = True  # run_inference_pipeline enqueues all stages without intermediate host syncs
        self.keep_all_outputs = False
        self.keep_all_coarse_outputs = False
        self.refiner_outputs = None
        self.coarse_outputs = None
        self.debug_dict: dict = dict()

    def load_SO3_grid(self, grid_size: int) -> None:
        self._SO3_grid = load_SO3_grid(grid_size).cuda()
        self.__dict__.pop("_rows_cache", None)

    # ------------------------------------------------------------------------------------------
    @torch.no_grad()
    def forward_refiner(self, observation: ObservationTensor, data_TCO_input: PoseEstimatesType, n_iterations: int = 5,
                        keep_all_outputs: bool = False, cuda_timer: bool = False, **refiner_kwargs) -> Tuple[dict, dict]:
        """pose_estimator.py:102-215 -> (preds{'iteration=n': collection}, extra_data)."""
        start_time = time.time()
        assert self.refiner_model is not None
        model = self.refiner_model
        B = data_TCO_input.poses.shape[0]
        device = observation.images.device
        infos_in = data_TCO_input.infos
        labels = infos_in["label"].tolist()
        batch_im_ids = torch.as_tensor(infos_in["batch_im_id"].to_numpy(), device=device)
        K_all = observation.K[batch_im_ids]
        TCO_all = data_TCO_input.poses.to(device)

        s0, s1 = self.sharder.span(B)
        chunk = max(1, model.max_batch // max(1, model.n_rendered_views))
        model_time = 0.0
        all_outputs = []
        fields = ["poses", "poses_input", "K_crop", "K", "boxes_rend", "boxes_crop"]
        local = {n: {f: [] for f in fields} for n in range(1, n_iterations + 1)}
        for s in range(s0, s1, chunk):  # GPU work is enqueued first ...
            e = min(s1, s + chunk)
            t0 = time.time()
            outputs_ = model(images=observation.images, K=K_all[s:e], TCO=TCO_all[s:e], n_iterations=n_iterations,
                             labels=labels[s:e], batch_im_ids=batch_im_ids[s:e], cuda_timer=cuda_timer,
                             **refiner_kwargs)
            model_time += time.time() - t0
            if keep_all_outputs:
                all_outputs.append(outputs_)
            for n in range(1, n_iterations + 1):
                it = outputs_[f"iteration={n}"]
                for f, v in zip(fields, (it.TCO_output, it.TCO_input, it.K_crop, it.K, it.boxes_rend, it.boxes_crop)):
                    local[n][f].append(v)
        # ... and the DataFrame bookkeeping runs on the host while the device computes
        df = infos_in.copy()
        df["refiner_batch_idx"] = np.arange(B) // max(1, self.bsz_objects)
        df["refiner_instance_idx"] = np.arange(B) % max(1, self.bsz_objects)
        preds = dict()
        tails = dict(poses=(4, 4), poses_input=(4, 4), K_crop=(3, 3), K=(3, 3), boxes_rend=(4,), boxes_crop=(4,))
        for n in range(1, n_iterations + 1):
            tensors = dict()
            for f in fields:
                loc = torch.cat(local[n][f]) if local[n][f] else torch.empty((0,) + tails[f], device=device)
                tensors[f] = self.sharder.gather_rows(loc, B)
            preds[f"iteration={n}"] = PandasTensorCollection(df, **tensors)
        extra_data = {"n_iterations": n_iterations, "outputs": all_outputs, "model_time": model_time,
                      "time": time.time() - start_time}
        return preds, extra_data

    # ------------------------------------------------------------------------------------------
    def _score(self, observation: ObservationTensor, labels, batch_im_ids: torch.Tensor, TCO: torch.Tensor,
               cuda_timer: bool, return_debug_data: bool, label_idx: Optional[torch.Tensor] = None):
        """Enqueue the coarse model over all rows (sharded); returns (logits [n,1] on device, out dict)."""
        n = TCO.shape[0]
        K = observation.K[batch_im_ids]
        s0, s1 = self.sharder.span(n)
        out_ = self.coarse_model.forward_coarse(images=observation.images, K=K[s0:s1], labels=labels[s0:s1],
                                                TCO_input=TCO[s0:s1], cuda_timer=cuda_timer,
                                                return_debug_data=return_debug_data, batch_im_ids=batch_im_ids[s0:s1],
                                                label_idx=None if label_idx is None else label_idx[s0:s1])
        return self.sharder.gather_rows(out_["logits"], n), out_

    @torch.no_grad()
    def forward_scoring_model(self, observation: ObservationTensor, data_TCO: PoseEstimatesType, cuda_timer: bool = False,
                              return_debug_data: bool = False) -> Tuple[PoseEstimatesType, dict]:
        """pose_estimator.py:218-322: adds pose_logit / pose_score to data_TCO.infos (in place)."""
        start_time = time.time()
        assert self.coarse_model is not None
        device = observation.images.device
        df = data_TCO.infos
        batch_im_ids = torch.as_tensor(np.array(df["batch_im_id"].to_numpy(), copy=True), device=device)
        logits, out_ = self._score(observation, df["label"].tolist(), batch_im_ids, data_TCO.poses.to(device), cuda_timer,
                                   return_debug_data)
        scores = torch.sigmoid(logits)
        debug_data = dict()
        if return_debug_data:
            debug_data = {"images_crop": out_["images_crop"], "renders": out_["renders"]}
        both = torch.cat((logits.reshape(-1, 1), scores.reshape(-1, 1)), dim=1).cpu().numpy()  # one D2H read
        df["pose_logit"] = both[:, 0]
        df["pose_score"] = both[:, 1]
        elapsed = time.time() - start_time
        render_time, model_time = out_["render_time"], out_["model_time"]
        extra_data = {"render_time": render_time, "model_time": model_time, "time": elapsed, "logits": logits,
                      "scores": scores, "debug": debug_data,
                      "n_batches": int(np.ceil(len(df) / max(1, self.bsz_images))),
                      "timing_str": f"time: {elapsed:.2f}, model_time: {model_time:.2f}, render_time: {render_time:.2f}"}
        data_TCO.infos = df
        return data_TCO, extra_data

    # ------------------------------------------------------------------------------------------
    @torch.no_grad()
    def forward_coarse_model(self, observation: ObservationTensor, detections: DetectionsType, cuda_timer: bool = False,
                             return_debug_data: bool = False) -> Tuple[PoseEstimatesType, dict]:
        """pose_estimator.py:325-483: every detection x every rotation of the SO(3) grid."""
        start_time = time.time()
        assert_detections_valid(detections)
        coarse_model = self.coarse_model
        device = observation.images.device
        SO3_grid = self._SO3_grid
        B, M = len(detections), SO3_grid.shape[0]
        df = detections.infos
        # device-side row tables straight from the B detections (row = detection * M + hypothesis) ...
        det_labels = df["label"].tolist()
        bim = torch.as_tensor(np.array(df["batch_im_id"].to_numpy(), copy=True), device=device)
        batch_im_ids = bim.repeat_interleave(M)
        bbox_ids = torch.arange(B, device=device).repeat_interleave(M)
        m_idx = torch.arange(M, device=device).repeat(B)
        K = observation.K[batch_im_ids]
        bboxes = detections.bboxes.to(device)[bbox_ids]
        label_idx = coarse_model.mesh_db.label_ids(det_labels, device).repeat_interleave(M)
        labels = [l for l in det_labels for _ in range(M)]
        TCO = lib3d.TCO_init_from_boxes_autodepth_with_R(bboxes.float(), coarse_model.mesh_db.points, label_idx, K,
                                                         SO3_grid[m_idx])
        logits, out_ = self._score(observation, labels, batch_im_ids, TCO, cuda_timer, return_debug_data, label_idx)
        scores = torch.sigmoid(logits)
        both = torch.cat((logits.reshape(-1, 1), scores.reshape(-1, 1)), dim=1)
        # ... the B*M-row DataFrame is built on the host while the device scores the hypotheses
        df_hypotheses = df.loc[df.index.repeat(M)].copy()
        df_hypotheses["hypothesis_id"] = np.tile(np.arange(M), B)
        df_hypotheses["bbox_id"] = np.repeat(df.index.values, M)
        both = both.cpu().numpy()  # the stage's only synchronisation
        df_hypotheses["coarse_logit"] = both[:, 0]
        df_hypotheses["coarse_score"] = both[:, 1]
        logits = logits.reshape([B, M])
        scores = scores.reshape([B, M])
        debug_data = dict()
        if return_debug_data:
            H, W = out_["images_crop"].shape[2:]
            debug_data = {"images_crop": out_["images_crop"].reshape([B, M, -1, H, W]),
                          "renders": out_["renders"].reshape([B, M, -1, H, W])}
        elapsed = time.time() - start_time
        render_time, model_time = out_["render_time"], out_["model_time"]
        extra_data = {"render_time": render_time, "model_time": model_time, "time": elapsed, "logits": logits,
                      "scores": scores, "TCO": TCO.reshape([B, M, 4, 4]), "debug": debug_data,
                      "n_batches": int(np.ceil(B * M / max(1, self.bsz_images))),
                      "timing_str": f"time: {elapsed:.2f}, model_time: {model_time:.2f}, render_time: {render_time:.2f}"}
        data_TCO = PandasTensorCollection(df_hypotheses, poses=TCO, bboxes=bboxes)
        return data_TCO, extra_data

    # ------------------------------------------------------------------------------------------
    @torch.no_grad()
    def forward_detection_model(self, observation: ObservationTensor, *args: Any, **kwargs: Any) -> DetectionsType:
        return self.detector_model.get_detections(observation, *args, **kwargs)

    def run_depth_refiner(self, observation: ObservationTensor, predictions: PoseEstimatesType):
        assert self.depth_refiner is not None, "You must specify a depth refiner"
        return self.depth_refiner.refine_poses(predictions, depth=observation.depth, K=observation.K)

    # ------------------------------------------------------------------------------------------
    @torch.no_grad()
    def run_inference_pipeline(self, observation: ObservationTensor, detections: Optional[DetectionsType] = None,
                               run_detector: Optional[bool] = None, n_refiner_iterations: int = 5,
                               n_pose_hypotheses: int = 1, keep_all_refiner_outputs: bool = False,
                               detection_filter_kwargs: Optional[dict] = None, run_depth_refiner: bool = False,
                               bsz_images: Optional[int] = None, bsz_objects: Optional[int] = None,
                               cuda_timer: bool = False,
                               coarse_estimates: Optional[PoseEstimatesType] = None) -> Tuple[PoseEstimatesType, dict]:
        """pose_estimator.py:511-641."""
        timing_str = ""
        t_start = time.time()
        if bsz_images is not None:
            self.bsz_images = bsz_images
        if bsz_objects is not None:
            self.bsz_objects = bsz_objects
        if coarse_estimates is None and detections is None and run_detector:  # pose_estimator.py:566-572
            t0 = time.time()
            detections = self.forward_detection_model(observation).cuda()
            timing_str += f"detection={time.time() - t0:.2f}, "
        if (self.fused_pipeline and coarse_estimates is None and detections is not None and not run_depth_refiner
                and not cuda_timer and not keep_all_refiner_outputs and self.refiner_model is not None
                and self.coarse_model is not None and len(detections) > 0 and n_refiner_iterations >= 1):
            out = self._run_pipeline_fused(observation, detections, n_refiner_iterations, n_pose_hypotheses,
                                           detection_filter_kwargs, t_start)
            if out is not None:
                return out
        if coarse_estimates is None:
            assert detections is not None or run_detector, "You must either pass in `detections` or set run_detector=True"
            assert detections is not None
            detections = add_instance_id(detections)
            if detection_filter_kwargs is not None:
                detections = filter_detections(detections, **detection_filter_kwargs)
            data_TCO_coarse, coarse_extra_data = self.forward_coarse_model(observation=observation, detections=detections,
                                                                          cuda_timer=cuda_timer)
            timing_str += f"coarse={coarse_extra_data['time']:.2f}, "
            data_TCO_filtered = self.filter_pose_estimates(data_TCO_coarse, top_K=n_pose_hypotheses,
                                                           filter_field="coarse_logit")
        else:
            data_TCO_coarse = coarse_estimates
            coarse_extra_data = None
            data_TCO_filtered = coarse_estimates

        preds, refiner_extra_data = self.forward_refiner(observation, data_TCO_filtered, n_iterations=n_refiner_iterations,
                                                         keep_all_outputs=keep_all_refiner_outputs, cuda_timer=cuda_timer)
        data_TCO_refined = preds[f"iteration={n_refiner_iterations}"]
        timing_str += f"refiner={refiner_extra_data['time']:.2f}, "
        data_TCO_scored, scoring_extra_data = self.forward_scoring_model(observation, data_TCO_refined, cuda_timer=cuda_timer)
        timing_str += f"scoring={scoring_extra_data['time']:.2f}, "
        data_TCO_final_scored = self.filter_pose_estimates(data_TCO_scored, top_K=1, filter_field="pose_logit")
        if run_depth_refiner:
            t0 = time.time()
            data_TCO_depth_refiner, _ = self.run_depth_refiner(observation, data_TCO_final_scored)
            data_TCO_final = data_TCO_depth_refiner
            timing_str += f"depth refiner={time.time() - t0:.2f}"
        else:
            data_TCO_depth_refiner = None
            data_TCO_final = data_TCO_final_scored
        elapsed = time.time() - t_start
        timing_str = f"total={elapsed:.2f}, {timing_str}"
        extra_data: dict = dict()
        extra_data["coarse"] = {"preds": data_TCO_coarse, "data": coarse_extra_data}
        extra_data["coarse_filter"] = {"preds": data_TCO_filtered}
        extra_data["refiner_all_hypotheses"] = {"preds": preds, "data": refiner_extra_data}
        extra_data["scoring"] = {"preds": data_TCO_scored, "data": scoring_extra_data}
        extra_data["refiner"] = {"preds": data_TCO_final_scored, "data": refiner_extra_data}
        extra_data["timing_str"] = timing_str
        extra_data["time"] = elapsed
        if run_depth_refiner:
            extra_data["depth_refiner"] = {"preds": data_TCO_depth_refiner}
        return data_TCO_final, extra_data

    def set_tail_priority(self, mode=True) -> None:
        """Stream priorities inside a frame, for two frames in flight (frame_pipeline.py).  Everything after the coarse stage
        (refiner iterations, scoring, selection: a few hundred dependent few-CTA launches) runs on its own stream;
          True / "high": that stream and the graphs captured on it have high priority -- its launches are scheduled ahead of
                         the other frame's queued thread blocks (shortest frame latency);
          "low":         the coarse stage's graph is captured at high priority and the tail keeps the default one -- the
                         tail only takes SMs the other frame's coarse stage leaves idle;
          False / None:  one stream, default priorities.
        Call before the first frame (graphs record the priority of the stream they were captured on)."""
        dev = torch.device("cuda", torch.cuda.current_device())
        mode = {True: "high", False: None}.get(mode, mode)
        assert mode in ("high", "low", None)
        self._tail_stream = self._head_capture_stream = cap = None
        if mode == "high":
            self._tail_stream = torch.cuda.Stream(device=dev, priority=-1)  # torch: -1 = high, 0 = default
            cap = torch.cuda.Stream(device=dev, priority=-1)
        elif mode == "low":
            self._tail_stream = torch.cuda.Stream(device=dev, priority=0)
            self._head_capture_stream = torch.cuda.Stream(device=dev, priority=-1)
        for m in (self.coarse_model, self.refiner_model):
            if m is not None:
                m.graph_capture_stream = cap

    @torch.no_grad()
    def submit_inference_pipeline(self, observation: ObservationTensor, detections: DetectionsType,
                                  n_refiner_iterations: int = 5, n_pose_hypotheses: int = 1,
                                  detection_filter_kwargs: Optional[dict] = None) -> "PendingInference":
        """run_inference_pipeline in two halves: this call enqueues the whole pipeline on the current stream and returns
        without waiting for the device; `.result()` of the returned handle waits and builds what run_inference_pipeline
        returns.  Frames of one estimator execute one after the other on the device (its graphs and workspaces are
        single-buffered, the stream orders them); a second frame may be enqueued before the first one's `.result()` has been
        taken so that the device never waits for the host, not more.  FramePipeline (frame_pipeline.py) alternates frames
        over two estimators on two streams: the latency-bound refiner iterations of one frame overlap the coarse stage of
        the next."""
        pending_now = [p for p in self.__dict__.get("_in_flight", []) if not p.done]
        if len(pending_now) >= 2:
            raise RuntimeError("this estimator already has two frames enqueued: call .result() of the older handle first")
        t_start = time.time()
        kwargs = dict(n_refiner_iterations=n_refiner_iterations, n_pose_hypotheses=n_pose_hypotheses,
                      detection_filter_kwargs=detection_filter_kwargs)
        fused_ok = (self.fused_pipeline and self.refiner_model is not None and self.coarse_model is not None
                    and len(detections) > 0 and n_refiner_iterations >= 1)
        finish = self._run_pipeline_fused(observation, detections, n_refiner_iterations, n_pose_hypotheses,
                                          detection_filter_kwargs, t_start, defer=True) if fused_ok else None
        if finish is None:  # configurations the fused path does not take: computed here, the handle is already complete
            out = self.run_inference_pipeline(observation, detections=detections, **kwargs)
            pending = PendingInference(None, (observation, detections), out)
        else:
            pending = PendingInference(finish, (observation, detections), None)
        self._in_flight = pending_now + [pending]
        return pending

    # ------------------------------------------------------------------------------------------
    def _pipeline_rows(self, df: pd.DataFrame, device) -> dict:
        """Index tensors of the coarse stage (row = detection * M + hypothesis): functions of the detections' image ids
        and labels only, cached so that a stream of frames with the same detections does not rebuild them."""
        M = self._SO3_grid.shape[0]
        labels = tuple(df["label"].tolist())
        key = (tuple(df["batch_im_id"].tolist()), labels, M, str(device))
        cache = self.__dict__.setdefault("_rows_cache", {})
        ent = cache.get(key)
        if ent is None:
            if len(cache) >= 8:
                cache.clear()
            B = len(df)
            bim = torch.as_tensor(np.array(df["batch_im_id"].to_numpy(), copy=True), device=device)
            det_label_idx = self.coarse_model.mesh_db.label_ids(list(labels), device)
            ent = cache[key] = dict(
                batch_im_ids=bim.repeat_interleave(M), bbox_ids=torch.arange(B, device=device).repeat_interleave(M),
                label_idx=det_label_idx.repeat_interleave(M), R=self._SO3_grid.repeat(B, 1, 1).contiguous(),
                group_base=(torch.arange(B, device=device) * M).unsqueeze(1),
                labels_rows=[l for l in labels for _ in range(M)])
        return ent

    def _coarse_local(self, images: torch.Tensor, K_obs: torch.Tensor, bboxes_det: torch.Tensor, rows_c: dict, s0: int,
                      s1: int) -> dict:
        """Device work of the coarse stage up to this rank's logits, on tensors only: per-row intrinsics / boxes, pose
        initialisation of all B*M rows, the coarse model over rows [s0, s1).  No host synchronisation, no collective, no
        pointer-dependent input besides K_obs / bboxes_det: capturable as a CUDA graph."""
        coarse_model = self.coarse_model
        batch_im_ids, label_idx = rows_c["batch_im_ids"], rows_c["label_idx"]
        K_rows = K_obs[batch_im_ids]
        bboxes = bboxes_det[rows_c["bbox_ids"]]
        TCO = lib3d.TCO_init_from_boxes_autodepth_with_R(bboxes, coarse_model.mesh_db.points, label_idx, K_rows, rows_c["R"])
        timing = defaultdict(float)
        if s1 > s0:
            logits_local = coarse_model._iterate(images, rows_c["im_idx32"][s0:s1].contiguous(),
                                                 K_rows[s0:s1].float().contiguous(),
                                                 rows_c["label_idx32"][s0:s1].contiguous(),
                                                 TCO[s0:s1].float().contiguous(), 1, timing)[0]["out"]
        else:
            logits_local = torch.empty(0, 1, device=TCO.device)
        return dict(K_rows=K_rows, bboxes=bboxes, TCO=TCO, logits_local=logits_local,
                    out=dict(render_time=timing["render"], model_time=timing["model"]))

    def _coarse_select(self, st: dict, logits: torch.Tensor, rows_c: dict, B: int, M: int, Kh: int) -> dict:
        """Scores and the top-K rows per detection, ordered like `sort_values(descending).groupby().head(K)` (NaN last,
        ties to the lower row), on the device; `logits` are the gathered logits of all B*M rows."""
        batch_im_ids, label_idx = rows_c["batch_im_ids"], rows_c["label_idx"]
        K_rows, bboxes, TCO = st["K_rows"], st["bboxes"], st["TCO"]
        scores = torch.sigmoid(logits)
        flat = logits.flatten()
        top = lib3d.topk_per_group(logits.reshape(B, M), Kh).long()                       # [B, Kh]
        rows = (top + rows_c["group_base"]).flatten()
        rows = rows[order_desc_nan_last(flat[rows])]
        packed_c = torch.cat((flat.double(), scores.flatten().double(), rows.double()))
        return dict(K_rows=K_rows, bboxes=bboxes, TCO=TCO, logits=logits, scores=scores, rows=rows, packed_c=packed_c,
                    TCO_sel=TCO[rows], bim_sel=batch_im_ids[rows], lab_sel=label_idx[rows], K_sel=K_rows[rows],
                    bboxes_sel=bboxes[rows], out=st["out"])

    def _coarse_stage(self, images, K_obs, bboxes_det, rows_c, B, M, Kh, s0, s1, whole: bool) -> dict:
        st = self._coarse_local(images, K_obs, bboxes_det, rows_c, s0, s1)
        if whole:  # this process owns every row: selection inside the same (graph-capturable) region
            return self._coarse_select(st, st["logits_local"], rows_c, B, M, Kh)
        return st

    def _coarse_stage_graphed(self, observation: ObservationTensor, bboxes_det: torch.Tensor, rows_c: dict, B: int, M: int,
                              Kh: int) -> dict:
        """The coarse stage, with its device work up to the (local) logits -- and, when this process owns all rows, the
        selection too -- replayed as one CUDA graph: the ~25 small launches in front of the first large kernel otherwise
        leave the GPU idle for ~0.5 ms per step.  First sight of a configuration runs eagerly, the second captures, later
        ones replay.  With several ranks the logits are all-gathered (outside the graph) before the selection."""
        cm = self.coarse_model
        images = observation.images
        n = B * M
        K_obs = observation.K.float()
        if "im_idx32" not in rows_c:
            rows_c["im_idx32"] = rows_c["batch_im_ids"].to(torch.int32).contiguous()
            rows_c["label_idx32"] = rows_c["label_idx"].to(torch.int32).contiguous()
        s0, s1 = self.sharder.span(n)
        whole = not self.sharder.enabled
        if s1 - s0 > cm.max_batch:  # several launches per rank: the chunked reference-style path
            return self._coarse_stage_chunked(observation, bboxes_det, rows_c, B, M, Kh)
        cm._nhwc4(images, refresh=True)

        def finish(st: dict, static: bool) -> dict:
            if not whole:
                # the throughput-bound part of the frame ends here: the next frame in flight (FramePipeline.serialize_heads) may
                # start its coarse stage while this one's logits are gathered over the ranks and the survivors selected
                ev = torch.cuda.Event()
                ev.record(torch.cuda.current_stream(images.device))
                self.__dict__["_head_done"] = ev
                st = self._coarse_select(st, self.sharder.gather_rows(st["logits_local"], n), rows_c, B, M, Kh)
            return dict(st, static=static)

        graphable = cm.use_cuda_graphs and (s1 - s0) <= cm.graph_max_batch and not (cm.keep_images or cm.debug)
        if not graphable:
            return finish(self._coarse_stage(images, K_obs, bboxes_det, rows_c, B, M, Kh, s0, s1, whole), False)
        cm._input_buffer(s1 - s0, *cm.render_size)  # may retire older buffers and the graphs over them (bumps the epoch)
        key = (id(rows_c), Kh, s0, s1, whole, tuple(images.shape), cm._nhwc4(images).data_ptr(), tuple(K_obs.shape),
               cm.graph_epoch)
        graphs = self.__dict__.setdefault("_coarse_graphs", {})
        entry = graphs.get(key)
        if entry is None:
            if len(graphs) >= 8:
                graphs.clear()
            graphs[key] = dict(graph=None, K=K_obs.clone(), bboxes=bboxes_det.clone(), rows_c=rows_c)
            return finish(self._coarse_stage(images, K_obs, bboxes_det, rows_c, B, M, Kh, s0, s1, whole), False)
        prev = self.__dict__.get("_coarse_copies_done")
        if prev is not None:
            torch.cuda.current_stream(images.device).wait_event(prev)  # the previous step's copies out of the static buffers
        entry["K"].copy_(K_obs)
        entry["bboxes"].copy_(bboxes_det)
        if entry["graph"] is None:
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            try:
                with torch.cuda.graph(graph, stream=self.__dict__.get("_head_capture_stream")):
                    out = self._coarse_stage(images, entry["K"], entry["bboxes"], rows_c, B, M, Kh, s0, s1, whole)
            except Exception:  # noqa: BLE001 -- capture not possible here: stay eager
                torch.cuda.synchronize()
                graphs.pop(key, None)
                cm.use_cuda_graphs = False
                return finish(self._coarse_stage(images, K_obs, bboxes_det, rows_c, B, M, Kh, s0, s1, whole), False)
            entry["graph"], entry["out"] = graph, out
        entry["graph"].replay()
        return finish(dict(entry["out"]), True)

    def _coarse_stage_chunked(self, observation: ObservationTensor, bboxes_det: torch.Tensor, rows_c: dict, B: int, M: int,
                              Kh: int) -> dict:
        """The coarse stage when a rank's share of the rows needs several launches (`PosePredictor.max_batch`)."""
        coarse_model = self.coarse_model
        batch_im_ids, label_idx = rows_c["batch_im_ids"], rows_c["label_idx"]
        K_rows = observation.K[batch_im_ids]
        bboxes = bboxes_det[rows_c["bbox_ids"]]
        TCO = lib3d.TCO_init_from_boxes_autodepth_with_R(bboxes, coarse_model.mesh_db.points, label_idx, K_rows, rows_c["R"])
        logits, out_c = self._score(observation, rows_c["labels_rows"], batch_im_ids, TCO, False, False, label_idx)
        st = dict(K_rows=K_rows, bboxes=bboxes, TCO=TCO, out=out_c)
        return dict(self._coarse_select(st, logits, rows_c, B, M, Kh), static=False)

    def _pinned(self, name: str, n: int) -> torch.Tensor:
        """Pinned staging buffer of one frame's read-back.  A fresh tensor per frame (torch's caching host allocator hands the
        block back once the copy into it has completed and the frame has let go of it), so that a frame enqueued while an
        older one is still being read on the host never shares its buffer."""
        return torch.empty(max(n, 1), dtype=torch.float64, pin_memory=True)[:n]

    @torch.no_grad()
    def _run_pipeline_fused(self, observation: ObservationTensor, detections: DetectionsType, n_refiner_iterations: int,
                            n_pose_hypotheses: int, detection_filter_kwargs: Optional[dict], t_start: float,
                            defer: bool = False):
        """The same pipeline with every stage enqueued back to back.  The top-K selection between the stages and the
        final best-hypothesis selection run on the device (mpx_topk_per_group + stable sorts), so the host never waits
        for logits before it can launch the next stage.  The coarse logits come back on a side stream as soon as the
        coarse stage is done; all DataFrame bookkeeping of the reference's outputs is done while the refiner and the
        scoring pass run; after the last synchronisation only two columns are filled in.
        Returns None (caller falls back to the staged path) when two detections share a (batch_im_id, label,
        instance_id) key, because then the reference's groupby merges their hypotheses.
        `defer`: return, right after the last launch, the function that waits for the device and builds the outputs
        (submit_inference_pipeline) instead of calling it."""
        coarse_model, refiner = self.coarse_model, self.refiner_model
        device = observation.images.device
        detections = add_instance_id(detections)
        if detection_filter_kwargs is not None:
            detections = filter_detections(detections, **detection_filter_kwargs)
        assert_detections_valid(detections)
        df = detections.infos
        B, M = len(df), self._SO3_grid.shape[0]
        if B == 0 or df.duplicated(["batch_im_id", "label", "instance_id"]).any():
            return None
        Kh = min(n_pose_hypotheses, M)
        n_sel = B * Kh
        t0 = time.time()
        main = torch.cuda.current_stream(device)
        side = self.__dict__.get("_copy_stream")
        if side is None:
            side = self.__dict__["_copy_stream"] = torch.cuda.Stream(device=device)
        self.__dict__.pop("_head_done", None)  # (an event of an earlier frame that nobody collected)
        gate = self.__dict__.pop("_head_gate", None)
        if gate is not None:  # FramePipeline: this frame's coarse stage starts when the previous frame's (another estimator's,
            main.wait_event(gate)  # another stream's) has finished -- two throughput-bound heads never share the device
        # ---- coarse: B*M rows, row = detection * M + hypothesis
        rows_c = self._pipeline_rows(df, device)
        batch_im_ids, label_idx = rows_c["batch_im_ids"], rows_c["label_idx"]
        bboxes_det = detections.bboxes.to(device).float()
        st = self._coarse_stage_graphed(observation, bboxes_det, rows_c, B, M, Kh)
        K_rows, bboxes, TCO, logits, scores, rows, packed_c = (st[k] for k in ("K_rows", "bboxes", "TCO", "logits", "scores",
                                                                               "rows", "packed_c"))
        out_c = st["out"]
        pin_c = self._pinned("coarse", packed_c.numel())
        ev_c = torch.cuda.Event()
        ev_c.record(main)
        self.__dict__.setdefault("_head_done", ev_c)  # the throughput-bound part of this frame is enqueued up to here (with
        # several ranks: up to the all-gather of the coarse logits, recorded in _coarse_stage_graphed)
        with torch.cuda.stream(side):
            side.wait_event(ev_c)
            pin_c.copy_(packed_c, non_blocking=True)
            ev_c_done = torch.cuda.Event()
            ev_c_done.record(side)
            if st["static"]:
                # the stage's outputs live in the replayed graph's static buffers: what is handed to the caller is copied
                # out here, off the critical path (the next replay waits for these copies)
                K_rows, bboxes, TCO, logits, scores = (t.clone() for t in (K_rows, bboxes, TCO, logits, scores))
                sel_user = {k: st[k].clone() for k in ("TCO_sel", "K_sel", "bboxes_sel")}
                ev_copies = torch.cuda.Event()
                ev_copies.record(side)
                self.__dict__["_coarse_copies_done"] = ev_copies
                for t in (K_rows, bboxes, TCO, logits, scores, *sel_user.values()):
                    t.record_stream(main)
            else:
                sel_user = {k: st[k] for k in ("TCO_sel", "K_sel", "bboxes_sel")}
        packed_c.record_stream(side)
        # ---- refiner on the selected rows (sharded), then scoring, all enqueued without a host round trip
        head, tail = main, self.__dict__.get("_tail_stream")
        if tail is not None:  # set_tail_priority: the latency-bound rest of the frame on a high-priority stream
            tail.wait_stream(head)
            torch.cuda.set_stream(tail)
            main = tail
        head_vars = dict(observation=observation, refiner=refiner, device=device, df=df, B=B, M=M, Kh=Kh, n_sel=n_sel, t0=t0,
                         t_start=t_start, main=main, side=side, st=st, rows=rows, out_c=out_c, pin_c=pin_c,
                         ev_c_done=ev_c_done, K_rows=K_rows, bboxes=bboxes, TCO=TCO, logits=logits, scores=scores,
                         sel_user=sel_user, n_refiner_iterations=n_refiner_iterations)
        try:
            return self._run_pipeline_tail(head_vars, defer)
        finally:
            if tail is not None:
                torch.cuda.set_stream(head)
                head.wait_stream(tail)

    def _run_pipeline_tail(self, head_vars: dict, defer: bool):
        (observation, refiner, device, df, B, M, Kh, n_sel, t0, t_start, main, side, st, rows, out_c, pin_c, ev_c_done,
         K_rows, bboxes, TCO, logits, scores, sel_user, n_refiner_iterations) = (head_vars[k] for k in (
             "observation", "refiner", "device", "df", "B", "M", "Kh", "n_sel", "t0", "t_start", "main", "side", "st", "rows",
             "out_c", "pin_c", "ev_c_done", "K_rows", "bboxes", "TCO", "logits", "scores", "sel_user", "n_refiner_iterations"))
        TCO_sel, bim_sel, lab_sel, K_sel = st["TCO_sel"], st["bim_sel"], st["lab_sel"], st["K_sel"]
        s0, s1 = self.sharder.span(n_sel)
        iters = refiner.refine_tensors(observation.images, bim_sel[s0:s1], K_sel[s0:s1], lab_sel[s0:s1], TCO_sel[s0:s1],
                                       n_refiner_iterations)
        fields = dict(poses="TCO_output", poses_input="TCO_input", K_crop="K_crop", boxes_rend="boxes_rend",
                      boxes_crop="boxes_crop")
        tails = dict(poses=(4, 4), poses_input=(4, 4), K_crop=(3, 3), boxes_rend=(4,), boxes_crop=(4,))
        refined = []
        if self.sharder.world > 1:
            # one all_gather for every field of every iteration: rows -> [n_loc, n_iter * 49] floats
            widths = {f: int(np.prod(tails[f])) for f in fields}
            n_loc = s1 - s0
            if iters:
                local = torch.cat([iters[n][src].reshape(n_loc, -1).float() for n in range(n_refiner_iterations)
                                   for src in fields.values()], dim=1)
            else:
                local = torch.empty(0, n_refiner_iterations * sum(widths.values()), device=device)
            full = self.sharder.gather_rows(local, n_sel)
            col = 0
            for n in range(n_refiner_iterations):
                tensors = dict()
                for f in fields:
                    tensors[f] = full[:, col:col + widths[f]].reshape((n_sel,) + tails[f])
                    col += widths[f]
                tensors["K"] = sel_user["K_sel"]
                refined.append(tensors)
        else:
            for n in range(n_refiner_iterations):
                tensors = {f: iters[n][src] for f, src in fields.items()}
                tensors["K"] = sel_user["K_sel"]
                refined.append(tensors)
        TCO_ref = refined[-1]["poses"] if n_refiner_iterations > 0 else TCO_sel
        t_ref = time.time()
        pose_logits, out_s = self._score(observation, [""] * n_sel, bim_sel, TCO_ref, False, False, lab_sel)
        pose_scores = torch.sigmoid(pose_logits)
        # ---- best hypothesis per detection, ordered like sort_values(pose_logit, descending).groupby().head(1)
        pl = pose_logits.flatten()
        grp = torch.div(rows, M, rounding_mode="floor")
        keep = best_per_group(pl, grp, B)                                      # [B] rows of the scored collection
        if st["static"]:
            main.wait_event(self.__dict__["_coarse_copies_done"])  # the side-stream clones (K_sel ...) are read from here on
        final_tensors = {k: v[keep] for k, v in refined[-1].items()} if n_refiner_iterations > 0 else None
        packed_f = torch.cat((pl.double(), pose_scores.flatten().double(), keep.double()))
        pin_f = self._pinned("final", packed_f.numel())
        pin_f.copy_(packed_f, non_blocking=True)
        ev_f_done = torch.cuda.Event()
        ev_f_done.record(main)

        def finish():
            # ---- host bookkeeping while the device works
            df_hyp = df.loc[df.index.repeat(M)].copy()
            df_hyp.index = pd.RangeIndex(B * M)
            df_hyp["hypothesis_id"] = np.tile(np.arange(M), B)
            df_hyp["bbox_id"] = np.repeat(df.index.values, M)
            ev_c_done.synchronize()                                                # coarse stage done (refiner still running)
            coarse_np = pin_c.numpy()
            nBM = B * M
            df_hyp["coarse_logit"] = coarse_np[:nBM].astype(np.float32)
            df_hyp["coarse_score"] = coarse_np[nBM:2 * nBM].astype(np.float32)
            rows_np = coarse_np[2 * nBM:].astype(np.int64)
            data_TCO_coarse = PandasTensorCollection._wrap(df_hyp, dict(poses=TCO, bboxes=bboxes))
            t_coarse = time.time() - t0
            coarse_extra = {"render_time": out_c["render_time"], "model_time": out_c["model_time"], "time": t_coarse,
                            "logits": logits.reshape(B, M), "scores": scores.reshape(B, M), "TCO": TCO.reshape(B, M, 4, 4),
                            "debug": dict(), "n_batches": int(np.ceil(B * M / max(1, self.bsz_images))),
                            "timing_str": f"time: {t_coarse:.2f}, model_time: {out_c['model_time']:.2f}, "
                                          f"render_time: {out_c['render_time']:.2f}"}
            df_sel = df_hyp.iloc[rows_np].copy()
            df_sel.index = pd.RangeIndex(n_sel)
            data_TCO_filtered = PandasTensorCollection._wrap(df_sel, dict(poses=sel_user["TCO_sel"], bboxes=sel_user["bboxes_sel"]))
            df_ref = df_sel.copy()
            df_ref["refiner_batch_idx"] = np.arange(n_sel) // max(1, self.bsz_objects)
            df_ref["refiner_instance_idx"] = np.arange(n_sel) % max(1, self.bsz_objects)
            preds = {f"iteration={n + 1}": PandasTensorCollection._wrap(df_ref.copy(), refined[n])
                     for n in range(n_refiner_iterations)}
            refiner_extra = {"n_iterations": n_refiner_iterations, "outputs": [], "model_time": max(0.0, t_ref - t0 - t_coarse),
                             "time": max(0.0, t_ref - t0)}
            data_TCO_scored = preds[f"iteration={n_refiner_iterations}"]
            infos_scored = data_TCO_scored.infos
            ev_f_done.synchronize()                                                # everything done
            final_np = pin_f.numpy()
            infos_scored["pose_logit"] = final_np[:n_sel].astype(np.float32)
            infos_scored["pose_score"] = final_np[n_sel:2 * n_sel].astype(np.float32)
            keep_np = final_np[2 * n_sel:].astype(np.int64)
            df_final = infos_scored.iloc[keep_np].copy()
            df_final.index = pd.RangeIndex(len(keep_np))
            final = PandasTensorCollection._wrap(df_final, final_tensors)
            scoring_extra = {"render_time": out_s["render_time"], "model_time": out_s["model_time"], "time": time.time() - t_ref,
                             "logits": pose_logits, "scores": pose_scores, "debug": dict(),
                             "n_batches": int(np.ceil(n_sel / max(1, self.bsz_images))), "timing_str": ""}
            elapsed = time.time() - t_start
            extra_data: dict = dict()
            extra_data["coarse"] = {"preds": data_TCO_coarse, "data": coarse_extra}
            extra_data["coarse_filter"] = {"preds": data_TCO_filtered}
            extra_data["refiner_all_hypotheses"] = {"preds": preds, "data": refiner_extra}
            extra_data["scoring"] = {"preds": data_TCO_scored, "data": scoring_extra}
            extra_data["refiner"] = {"preds": final, "data": refiner_extra}
            extra_data["timing_str"] = (f"total={elapsed:.2f}, coarse={t_coarse:.2f}, refiner={refiner_extra['time']:.2f}, "
                                        f"scoring={scoring_extra['time']:.2f}, ")
            extra_data["time"] = elapsed
            return final, extra_data

        return finish if defer else finish()

    def filter_pose_estimates(self, data_TCO: PoseEstimatesType, top_K: int, filter_field: str,
                              ascending: bool = False) -> PoseEstimatesType:
        """pose_estimator.py:643-667: top-K rows per (batch_im_id, label, instance_id)."""
        # same selection and row order as `df.sort_values(field).groupby(cols).head(top_K)` of the reference, computed on
        # numpy arrays (sorting a 10^4-row DataFrame costs milliseconds, this costs microseconds)
        df = data_TCO.infos
        n = len(df)
        if n == 0:
            return data_TCO[[]]
        vals = df[filter_field].to_numpy(dtype=np.float64)
        order = np.argsort(vals if ascending else -vals, kind="stable")
        keys = (df["batch_im_id"].to_numpy(), df["label"].to_numpy(), df["instance_id"].to_numpy())
        codes = np.zeros(n, dtype=np.int64)
        for k in keys:
            _, inv = np.unique(k, return_inverse=True)
            codes = codes * (int(inv.max()) + 1) + inv
        sorted_codes = codes[order]
        # rank of each row inside its group, in sorted order
        by_group = np.argsort(sorted_codes, kind="stable")
        grp_sorted = sorted_codes[by_group]
        starts = np.r_[0, np.flatnonzero(np.diff(grp_sorted)) + 1]
        rank = np.empty(n, dtype=np.int64)
        rank[by_group] = np.arange(n) - np.repeat(starts, np.diff(np.r_[starts, n]))
        keep = order[rank < top_K]
        return data_TCO[keep.tolist()]
