"""Depth refinement with TEASER++ on the device: the reference's `TeaserppRefiner` (inference/teaserpp_refiner.py:164-287).

Same constructor and `refine_poses(predictions, masks, depth, K) -> (predictions_refined, extra_data)` contract as the
reference.  Per prediction: a depth render at the depth image's resolution (the call `ICPRefiner` makes), the masks of
`refiner_utils.compute_masks` (the `masks` argument is ignored, as in the reference), the point clouds of
`meshcat_utils.get_pointcloud` (rendered = source, measured = target, correspondence i = masked pixel i), farthest-point
sampling to `n_points`, then TEASER++ with known correspondences and no scale: consistency graph, maximum clique,
GNC-TLS rotation, adaptive-voting translation.  The pose is replaced by T @ pose when at least `min_num_inliers` samples
land within `noise_bound` of their target; only then is `poses_input` set to the incoming pose (teaserpp_refiner.py:276-284).

Every stage is one CUDA launch for all predictions of the call (csrc/teaser.cu, include/mpx.h "depth refinement
(TEASER++)"); the host waits for the device only after the last stage, to fill `extra_data` (a fixed number of small
read-backs and one more point-cloud launch for the raw clouds of the last prediction that reached the solver, whatever
the number of predictions).  Parity with teaserpp_python and pytorch3d is
NOT pinned (neither is installable here): the arithmetic is the contract written down in DESIGN §4 and restated by
oracle/teaser_ref.py.  Without farthest-point sampling the subset is drawn on the device by sorting uniform keys, not
with numpy's random stream.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional, Tuple

import numpy as np
import torch

from . import _abi
from .icp_refiner import DepthRefiner
from .meshes import BatchedMeshes
from .renderer import BatchRenderer, Panda3dLightData

MAX_POINTS = 1024               # MPX_TEASER_MAX_POINTS: adjacency rows of 16 64-bit words
CLIQUE_NODE_BUDGET = 20000      # MPX_TEASER_CLIQUE_NODE_BUDGET: search nodes of the max clique per prediction
MASK_TYPES = {"simple": 0, "threshold": 1}


@dataclass
class SolverParams:
    """The fields of teaserpp_python.RobustRegistrationSolver.Params that get_solver_params sets."""
    cbar2: float = 1.0
    noise_bound: float = 0.01
    estimate_scaling: bool = False
    rotation_estimation_algorithm: str = "GNC_TLS"
    rotation_gnc_factor: float = 1.4
    rotation_max_iterations: int = 100
    rotation_cost_threshold: float = 1e-12


def get_solver_params(noise_bound: float = 0.01) -> SolverParams:
    """teaserpp_refiner.py:38-50."""
    return SolverParams(cbar2=1, noise_bound=noise_bound, estimate_scaling=False, rotation_estimation_algorithm="GNC_TLS",
                        rotation_gnc_factor=1.4, rotation_max_iterations=100, rotation_cost_threshold=1e-12)


@dataclass
class Solution:
    """What teaserpp_python's getSolution() returns, for the scale-free problem."""
    rotation: np.ndarray
    translation: np.ndarray
    scale: float = 1.0
    valid: bool = False


# ---- the stages (each one launch for all predictions) ----------------------------------------------------------------
def _i32(t: torch.Tensor) -> torch.Tensor:
    return t.to(torch.int32).contiguous()


def points(depth_rendered: torch.Tensor, depth_measured: torch.Tensor, view_idx: torch.Tensor, K: torch.Tensor,
           mask_type: str = "simple", depth_delta_thresh: float = 0.1, raw: bool = False):
    """[N, H, W] rendered, [B, H, W] measured (metres), [N] view index, [N, 3, 3] K -> (src [N, H*W, 3], tgt, count [N]
    int32[, raw_src [N, H, W, 3], raw_tgt]); rows past count[n] are left as they were allocated (empty)."""
    if mask_type not in MASK_TYPES:
        raise ValueError(f"Unknown mask type {mask_type}")
    n, h, w = depth_rendered.shape
    dev = depth_rendered.device
    rend = depth_rendered.float().contiguous()
    meas = depth_measured.float().reshape(-1, h, w).contiguous()
    Kf = K.float().reshape(n, 9).contiguous()
    vi = _i32(view_idx)
    src = torch.empty(n, h * w, 3, device=dev)
    tgt = torch.empty(n, h * w, 3, device=dev)
    count = torch.zeros(n, dtype=torch.int32, device=dev)
    raw_src = torch.empty(n, h, w, 3, device=dev) if raw else None
    raw_tgt = torch.empty(n, h, w, 3, device=dev) if raw else None
    _abi.check(_abi.lib().mpx_teaser_points(n, h, w, _abi.ptr(rend), _abi.ptr(meas), meas.shape[0], _abi.ptr(vi),
                                            _abi.ptr(Kf), MASK_TYPES[mask_type], float(depth_delta_thresh), _abi.ptr(src),
                                            _abi.ptr(tgt), _abi.ptr(count), _abi.ptr(raw_src), _abi.ptr(raw_tgt),
                                            _abi.stream_ptr()))
    return (src, tgt, count, raw_src, raw_tgt) if raw else (src, tgt, count)


def farthest_point_sampling(src: torch.Tensor, tgt: torch.Tensor, count: torch.Tensor, k: int):
    """(idx [N, k] int32, samples of src [N, k, 3], samples of tgt) for the first count[n] points of src[n] / tgt[n]."""
    n, cap, _ = src.shape
    dev = src.device
    idx = torch.empty(n, k, dtype=torch.int32, device=dev)
    ss = torch.empty(n, k, 3, device=dev)
    st = torch.empty(n, k, 3, device=dev)
    lib = _abi.lib()
    nbytes = lib.mpx_teaser_fps_workspace_bytes(n, cap)
    ws = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=dev)
    _abi.check(lib.mpx_teaser_fps(n, cap, _abi.ptr(src.contiguous()), _abi.ptr(tgt.contiguous()), _abi.ptr(_i32(count)), k,
                                  _abi.ptr(idx), _abi.ptr(ss), _abi.ptr(st), _abi.ptr(ws), ws.numel(), _abi.stream_ptr()))
    return idx, ss, st


def random_sampling(src: torch.Tensor, tgt: torch.Tensor, count: torch.Tensor, k: int):
    """A uniform subset of min(k, count[n]) of the first count[n] points, without replacement (the k smallest of uniform
    keys): (idx [N, k] int64, samples of src, samples of tgt); entries past min(k, count[n]) are unused."""
    n, cap, _ = src.shape
    keys = torch.rand(n, cap, device=src.device)
    keys = torch.where(torch.arange(cap, device=src.device)[None, :] < count[:, None].long(), keys, float("inf"))
    idx = torch.topk(keys, min(k, cap), dim=1, largest=False, sorted=True).indices  # the finite keys first
    if idx.shape[1] < k:
        idx = torch.cat((idx, idx[:, :1].expand(n, k - idx.shape[1])), dim=1)
    g = idx[..., None].expand(n, k, 3)
    return idx, torch.gather(src, 1, g).contiguous(), torch.gather(tgt, 1, g).contiguous()


def consistency_graph(samp_src: torch.Tensor, samp_tgt: torch.Tensor, m: torch.Tensor, noise_bound: float,
                      cbar2: float = 1.0) -> torch.Tensor:
    """[N, k, 16] uint64 adjacency bitsets (as int64) of the first m[n] samples."""
    n, k, _ = samp_src.shape
    adj = torch.empty(n, k, 16, dtype=torch.int64, device=samp_src.device)
    bound = 2.0 * noise_bound * np.sqrt(cbar2)
    _abi.check(_abi.lib().mpx_teaser_graph(n, k, _abi.ptr(samp_src.contiguous()), _abi.ptr(samp_tgt.contiguous()),
                                           _abi.ptr(_i32(m)), float(bound), _abi.ptr(adj), _abi.stream_ptr()))
    return adj


def max_clique(adj: torch.Tensor, m: torch.Tensor, node_budget: int = 0):
    """(clique [N, k] int32 ascending then -1, size [N] int32, status [N] int32 (bit 0: node budget exhausted),
    nodes [N] int64) of each graph; node_budget <= 0 means CLIQUE_NODE_BUDGET."""
    n, k, _ = adj.shape
    dev = adj.device
    clique = torch.empty(n, k, dtype=torch.int32, device=dev)
    size = torch.empty(n, dtype=torch.int32, device=dev)
    status = torch.empty(n, dtype=torch.int32, device=dev)
    nodes = torch.empty(n, dtype=torch.int64, device=dev)
    lib = _abi.lib()
    nbytes = lib.mpx_teaser_clique_workspace_bytes(n, k)
    ws = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=dev)
    _abi.check(lib.mpx_teaser_max_clique(n, k, _abi.ptr(adj.contiguous()), _abi.ptr(_i32(m)), int(node_budget),
                                         _abi.ptr(clique), _abi.ptr(size), _abi.ptr(status), _abi.ptr(nodes), _abi.ptr(ws),
                                         ws.numel(), _abi.stream_ptr()))
    return clique, size, status, nodes


def solve(samp_src, samp_tgt, m, clique, clique_size, poses: torch.Tensor, poses_input: torch.Tensor,
          params: SolverParams, min_num_inliers: int):
    """GNC-TLS rotation, TLS translation, inlier count; updates poses / poses_input [N, 4, 4] float32 in place where
    accepted.  Returns (T [N, 4, 4] float64, num_inliers [N] int32, flags [N] int32: bit 0 valid, bit 1 accepted)."""
    n, k, _ = samp_src.shape
    dev = samp_src.device
    for t in (poses, poses_input):
        if t.dtype != torch.float32 or not t.is_contiguous():
            raise _abi.MpxError("poses must be contiguous float32")
    T = torch.empty(n, 4, 4, dtype=torch.float64, device=dev)
    n_in = torch.empty(n, dtype=torch.int32, device=dev)
    flags = torch.empty(n, dtype=torch.int32, device=dev)
    _abi.check(_abi.lib().mpx_teaser_solve(n, k, _abi.ptr(samp_src.contiguous()), _abi.ptr(samp_tgt.contiguous()),
                                           _abi.ptr(_i32(m)), _abi.ptr(clique), _abi.ptr(clique_size),
                                           float(params.noise_bound), float(params.rotation_gnc_factor),
                                           int(params.rotation_max_iterations), float(params.rotation_cost_threshold),
                                           int(min_num_inliers), _abi.ptr(poses), _abi.ptr(poses_input), _abi.ptr(T),
                                           _abi.ptr(n_in), _abi.ptr(flags), _abi.stream_ptr()))
    return T, n_in, flags


def _refine(depth_rendered, depth_measured, view_idx, K, poses, poses_input, mask_type, depth_delta_thresh, n_min_points,
            n_points, params: SolverParams, min_num_inliers, use_farthest_point_sampling, want_last: bool = True) -> dict:
    """All stages for N predictions; poses / poses_input updated in place.  Returns the reference's `out` dict for the
    last prediction that reached the solver ({} when none did)."""
    if not 1 <= n_points <= MAX_POINTS:
        raise ValueError(f"n_points={n_points} must be in 1..{MAX_POINTS}")
    if params.estimate_scaling:
        raise NotImplementedError("only the scale-free problem (estimate_scaling=False) is implemented")
    src, tgt, count = points(depth_rendered, depth_measured, view_idx, K, mask_type, depth_delta_thresh)
    reached = count >= n_min_points
    if use_farthest_point_sampling:
        _, ss, st = farthest_point_sampling(src, tgt, count, n_points)
        m = torch.where(reached, n_points, 0)
    else:
        _, ss, st = random_sampling(src, tgt, count, n_points)
        m = torch.where(reached, torch.clamp(count, max=n_points), 0)
    adj = consistency_graph(ss, st, m, params.noise_bound, params.cbar2)
    clique, size, status, _ = max_clique(adj, m)
    T, n_in, flags = solve(ss, st, m, clique, size, poses, poses_input, params, min_num_inliers)
    reached_h = reached.cpu().numpy()                       # the first wait for the device
    if not want_last or not reached_h.any():
        return {}
    last = int(np.flatnonzero(reached_h)[-1])
    status_h, count_h = status.cpu().numpy(), int(count[last])
    h, w = depth_rendered.shape[-2:]
    _, _, _, raw_src, raw_tgt = points(depth_rendered[last:last + 1], depth_measured, view_idx[last:last + 1],
                                       K[last:last + 1], mask_type, depth_delta_thresh, raw=True)
    Th = T[last].cpu().numpy()
    valid = bool(int(flags[last]) & 1)
    out = dict(solution=Solution(rotation=Th[:3, :3].copy(), translation=Th[:3, 3].copy(), scale=1.0, valid=valid),
               pc_src_raw=raw_src[0], pc_tgt_raw=raw_tgt[0], pc_src=ss[last, :int(m[last])],
               pc_tgt=st[last, :int(m[last])], pc_src_mask=src[last, :count_h], pc_tgt_mask=tgt[last, :count_h],
               T=Th, T_tgt_src=Th, num_inliers=int(n_in[last]))
    if (status_h & 1).any():
        out["clique_node_budget"] = CLIQUE_NODE_BUDGET
        out["clique_budget_exhausted"] = np.flatnonzero(status_h & 1).tolist()
    return out


def compute_teaserpp_refinement(depth_src: torch.Tensor, depth_tgt: torch.Tensor, cam_K: torch.Tensor,
                                mask: torch.Tensor, solver_params: Optional[SolverParams] = None,
                                max_num_points: int = 1000, use_farthest_point_sampling: bool = True,
                                **solver_params_kwargs) -> dict:
    """teaserpp_refiner.py:53-161 for one prediction on device tensors: [H, W] source (rendered) and target (measured)
    depth, [3, 3] K, [H, W] bool mask (pixels where either depth is not > 0 are dropped as well).  Returns the
    reference's dict ('T_tgt_src' aligns the source cloud onto the target)."""
    params = solver_params if solver_params is not None else get_solver_params(**solver_params_kwargs)
    dev = depth_src.device
    rend = torch.where(mask.bool(), depth_src.float(), 0.0)[None]
    poses = torch.eye(4, device=dev)[None].contiguous()
    return _refine(rend, depth_tgt.float()[None], torch.zeros(1, dtype=torch.int32, device=dev), cam_K.reshape(1, 3, 3),
                   poses, poses.clone(), "simple", 0.1, 1, max_num_points, params, 0, use_farthest_point_sampling)


class TeaserppRefiner(DepthRefiner):
    def __init__(self, mesh_db: BatchedMeshes, renderer: BatchRenderer, mask_type: str = "simple",
                 depth_delta_thresh: float = 0.1, n_min_points: int = 100, n_points: int = 1000,
                 noise_bound: float = 0.01, min_num_inliers: int = 50, use_farthest_point_sampling: bool = True) -> None:
        if mask_type not in MASK_TYPES:
            raise ValueError(f"Unknown mask type {mask_type}")
        if not 1 <= n_points <= MAX_POINTS:
            raise ValueError(f"n_points={n_points} must be in 1..{MAX_POINTS}")
        self.mesh_db = mesh_db
        self.renderer = renderer
        self.mask_type = mask_type
        self.depth_delta_thresh = depth_delta_thresh
        self.n_min_points = n_min_points
        self.n_points = n_points
        self.noise_bound = noise_bound
        self.min_num_inliers = min_num_inliers
        self.use_farthest_point_sampling = use_farthest_point_sampling
        self.light_datas = [Panda3dLightData("ambient")]

    @torch.no_grad()
    def refine_poses(self, predictions, masks: Optional[torch.Tensor] = None, depth: Optional[torch.Tensor] = None,
                     K: Optional[torch.Tensor] = None) -> Tuple[object, dict]:
        """teaserpp_refiner.py:188-287."""
        assert depth is not None and K is not None
        predictions_refined = predictions.clone()
        if "poses_input" not in predictions_refined.tensors:
            predictions_refined.register_tensor("poses_input", predictions.poses.clone())
        N = len(predictions)
        if N == 0:
            return predictions_refined, {}
        h, w = depth.shape[-2:]
        df = predictions.infos
        labels = df.label.tolist()
        batch_im_ids = torch.as_tensor(df.batch_im_id.to_numpy().copy(), device=K.device)
        K_ = K[batch_im_ids].float()
        out = self.renderer.render(labels, TCO=predictions.poses, K=K_, light_datas=[self.light_datas] * N,
                                   resolution=(h, w), render_depth=True)
        rendered = out.depths.reshape(N, h, w)
        poses = predictions_refined.poses.float().contiguous()
        poses_input = predictions_refined.poses_input.float().contiguous()
        extra = _refine(rendered, depth.reshape(-1, h, w), batch_im_ids, K_, poses, poses_input, self.mask_type,
                        self.depth_delta_thresh, self.n_min_points, self.n_points, get_solver_params(self.noise_bound),
                        self.min_num_inliers, self.use_farthest_point_sampling)
        predictions_refined.poses.copy_(poses)
        predictions_refined.poses_input.copy_(poses_input)
        return predictions_refined, extra
