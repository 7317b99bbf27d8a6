"""TEASER++ depth refinement on the device (csrc/teaser.cu through megapose6d_b200/teaserpp_refiner.py) against the numpy
oracle (oracle/teaser_ref.py): masks, point clouds and compaction bit for bit, farthest-point indices, adjacency words,
maximum cliques (planted, networkx, node budget), the solve given the device's clique, the refiner's gates and end-to-end
behaviour, and a launch count that does not depend on the number of predictions."""
import numpy as np
import pandas as pd
import pytest
import networkx as nx
import torch

from megapose6d_b200 import _abi, load_model, procedural
from megapose6d_b200 import teaserpp_refiner as tr
from megapose6d_b200.tensor_collection import PandasTensorCollection
from oracle import pipeline_ref
from oracle import teaser_ref as T
from tests import helpers

pytestmark = pytest.mark.gpu


def _depth_pair(h, w, seed):
    rng = np.random.RandomState(seed)
    rend = rng.uniform(0.3, 1.5, (h, w)).astype(np.float32)
    meas = (rend + rng.normal(0, 0.08, (h, w))).astype(np.float32)
    rend[rng.rand(h, w) < 0.2] = 0
    meas[rng.rand(h, w) < 0.1] = 0
    meas[rng.rand(h, w) < 0.05] = np.nan
    rend[: h // 4] = 0                      # a band without render
    return rend, meas


@pytest.mark.parametrize("h,w", [(480, 640), (103, 150)])
@pytest.mark.parametrize("mask_type", ["simple", "threshold"])
def test_points_and_compaction_bit_exact(h, w, mask_type):
    r0, m0 = _depth_pair(h, w, h)
    full = np.full((h, w), 0.8, np.float32)
    rend = np.stack([r0, np.zeros((h, w), np.float32), full])        # normal, empty, full masks
    meas = np.stack([m0, full])
    vidx = np.array([0, 1, 1])
    K = np.array([[[600.5, 0, w / 2 + 0.3], [0, 599.7, h / 2 - 0.6], [0, 0, 1]]] * 3, np.float32)
    src, tgt, count, raw_s, raw_t = tr.points(torch.from_numpy(rend).cuda(), torch.from_numpy(meas).cuda(),
                                              torch.from_numpy(vidx).cuda(), torch.from_numpy(K).cuda(), mask_type, 0.1,
                                              raw=True)
    for n in range(3):
        s_ref, t_ref = T.masked_clouds(rend[n], meas[vidx[n]], K[n], mask_type, 0.1)
        c = int(count[n])
        assert c == len(s_ref)
        assert src[n, :c].cpu().numpy().tobytes() == s_ref.tobytes()
        assert tgt[n, :c].cpu().numpy().tobytes() == t_ref.tobytes()
        assert raw_s[n].cpu().numpy().tobytes() == T.get_pointcloud(rend[n], K[n]).tobytes()
    assert int(count[1]) == 0 and int(count[2]) == h * w


def test_fps_indices_equal_oracle():
    rng = np.random.RandomState(0)
    sizes = [100, 999, 1000, 1001, 50000, 307200]
    cap = max(sizes)
    src = np.zeros((len(sizes), cap, 3), np.float32)
    for i, n in enumerate(sizes):
        p = rng.uniform(-0.2, 0.2, (n, 3)).astype(np.float32)
        if n <= 1001:
            p = np.round(p * 40) / 40                     # a grid: duplicated points and tied distances
        src[i, :n] = p
    count = torch.tensor(sizes, dtype=torch.int32).cuda()
    s = torch.from_numpy(src).cuda()
    idx, ss, st = tr.farthest_point_sampling(s, s * 2, count, 1000)
    for i, n in enumerate(sizes):
        ref = T.farthest_point_sampling(src[i, :n], 1000)
        np.testing.assert_array_equal(idx[i].cpu().numpy(), ref, err_msg=f"N={n}")
        assert ss[i].cpu().numpy().tobytes() == src[i, ref].tobytes()
        assert st[i].cpu().numpy().tobytes() == (2 * src[i, ref]).tobytes()


def test_graph_words_equal_oracle():
    rng = np.random.RandomState(1)
    k = 1000
    ss = rng.uniform(-0.1, 0.1, (2, k, 3)).astype(np.float32)
    st = (ss + rng.normal(0, 0.01, ss.shape)).astype(np.float32)
    # pairs built to sit on the 0.02 m bound: a target 2 cm longer along x
    st[1, :200] = ss[1, :200]
    st[1, 1:200:2, 0] = ss[1, 0:199:2, 0] + np.float32(0.02) + (ss[1, 1:200:2, 0] - ss[1, 0:199:2, 0])
    m = torch.tensor([k, 777], dtype=torch.int32).cuda()
    adj = tr.consistency_graph(torch.from_numpy(ss).cuda(), torch.from_numpy(st).cuda(), m, 0.01)
    for n, mm in enumerate([k, 777]):
        ref = T.pack_adjacency(T.consistency_graph(ss[n, :mm], st[n, :mm], 0.01), k)
        assert np.array_equal(adj[n].cpu().numpy().view(np.uint64), ref)


def _dev_adj(graphs, k):
    return torch.from_numpy(np.stack([T.pack_adjacency(a, k).view(np.int64) for a in graphs])).cuda()


def test_max_clique_planted():
    cases = [(0.3, 30), (0.9, 300), (0.99, 900)]
    graphs, planted = zip(*[T.planted_clique_graph(1000, p, s, 7 + i) for i, (p, s) in enumerate(cases)])
    m = torch.full((3,), 1000, dtype=torch.int32).cuda()
    clique, size, status, nodes = tr.max_clique(_dev_adj(graphs, 1000), m)
    print("nodes", nodes.tolist(), "status", status.tolist())
    for i in range(3):
        c = clique[i, :int(size[i])].cpu().tolist()
        assert int(status[i]) == 0 and c == planted[i]


def test_max_clique_small_graphs_and_budget():
    graphs = [T.random_graph(8 + 2 * s, [0.2, 0.5, 0.8, 0.95][s % 4], 100 + s) for s in range(27)]
    k = 64
    m = torch.tensor([len(a) for a in graphs], dtype=torch.int32).cuda()
    clique, size, status, nodes = tr.max_clique(_dev_adj(graphs, k), m)
    for i, a in enumerate(graphs):
        c = clique[i, :int(size[i])].cpu().tolist()
        _, ref = nx.max_weight_clique(nx.from_numpy_array(a.astype(int)), weight=None)
        ref_c, ref_nodes, _ = T.max_clique(a)
        assert len(c) == ref and T.is_clique(a, c) and c == sorted(c) and int(status[i]) == 0
        assert int(nodes[i]) == ref_nodes and c == ref_c          # the same search as the oracle's
    a, _ = T.planted_clique_graph(300, 0.8, 14, 3)
    clique, size, status, nodes = tr.max_clique(_dev_adj([a], 300), torch.tensor([300], dtype=torch.int32).cuda(),
                                                node_budget=3)
    c = clique[0, :int(size[0])].cpu().tolist()
    assert int(status[0]) == 1 and int(nodes[0]) == 3 and T.is_clique(a, c) and len(c) >= 2


def test_solve_equals_oracle_and_gates():
    rng = np.random.RandomState(5)
    k = 400
    R = T.weighted_kabsch(rng.randn(5, 3), rng.randn(5, 3), np.ones(5))
    ss = rng.uniform(-0.08, 0.08, (3, k, 3)).astype(np.float32)
    st = (ss @ R.T.astype(np.float32) + np.float32([0.01, -0.02, 0.005])).astype(np.float32)
    st += rng.normal(0, 0.002, st.shape).astype(np.float32)
    bad = rng.rand(3, k) < 0.3
    st[bad] = rng.uniform(-0.1, 0.1, (bad.sum(), 3)).astype(np.float32)
    m = torch.tensor([k, k, 1], dtype=torch.int32).cuda()          # the third: a one-vertex clique (invalid)
    S, Tt = torch.from_numpy(ss).cuda(), torch.from_numpy(st).cuda()
    clique, size, status, _ = tr.max_clique(tr.consistency_graph(S, Tt, m, 0.01), m)
    poses = torch.from_numpy(procedural.random_poses(3, 9)).float().cuda().contiguous()
    pin = torch.zeros_like(poses)
    p0 = poses.clone()
    min_inl = torch.tensor([50, 10 ** 6, 50])
    T_all, n_in, flags = [], [], []
    for n in range(3):  # per-prediction thresholds: one call each
        t, ni, f = tr.solve(S[n:n + 1], Tt[n:n + 1], m[n:n + 1], clique[n:n + 1], size[n:n + 1], poses[n:n + 1],
                            pin[n:n + 1], tr.get_solver_params(0.01), int(min_inl[n]))
        T_all.append(t[0]); n_in.append(int(ni[0])); flags.append(int(f[0]))
    for n in range(2):
        c = clique[n, :int(size[n])].cpu().tolist()
        valid, Rr, tt, ni = T.solve(ss[n], st[n], c, 0.01)
        assert valid and flags[n] & 1
        np.testing.assert_allclose(T_all[n][:3, :3].cpu().numpy(), Rr, atol=1e-9)
        np.testing.assert_allclose(T_all[n][:3, 3].cpu().numpy(), tt, atol=1e-9)
        assert n_in[n] == ni
    assert flags[0] == 3 and torch.equal(pin[0], p0[0])
    Tn = np.eye(4); Tn[:3, :3], Tn[:3, 3] = T.solve(ss[0], st[0], clique[0, :int(size[0])].cpu().tolist(), 0.01)[1:3]
    np.testing.assert_allclose(poses[0].cpu().numpy(), (Tn @ p0[0].cpu().double().numpy()).astype(np.float32), atol=1e-6)
    assert flags[1] == 1 and torch.equal(poses[1], p0[1]) and torch.equal(pin[1], torch.zeros_like(pin[1]))  # not reached
    assert flags[2] == 0 and torch.equal(poses[2], p0[2])                                                   # invalid


def _pose_err(a, b):
    dR = a[:3, :3].double().T @ b[:3, :3].double()
    ang = torch.rad2deg(torch.acos(((dR.trace() - 1) / 2).clamp(-1, 1)))
    return ang.item(), (a[:3, 3] - b[:3, 3]).norm().item() * 1000.0


def _add_mm(ds, label, a, b):
    """Mean distance of the model's vertices under poses a and b, in mm."""
    obj = next(o for o in ds.list_objects if o.label == label)
    v = torch.from_numpy(obj.mesh.vertices * obj.scale).double()
    pa = v @ a[:3, :3].double().T + a[:3, 3].double()
    pb = v @ b[:3, :3].double().T + b[:3, 3].double()
    return (pa - pb).norm(dim=1).mean().item() * 1000.0


def _scene(tmp_path, n_obj=3):
    ds, _, K = helpers.make_scene(2, seed=12)
    load_model.write_run(tmp_path, "coarse-rgb-906902141", helpers.make_state_dict(helpers.COARSE_CFG, 5))
    load_model.write_run(tmp_path, "refiner-rgb-653307694", helpers.make_state_dict(helpers.REFINER_CFG, 6))
    est = load_model.load_named_model("megapose-1.0-RGB-multi-hypothesis-icp", ds, models_root=tmp_path)
    labels = [ds[i % 2].label for i in range(n_obj)]
    T_true = torch.from_numpy(procedural.random_poses(n_obj, 23, z_range=(0.35, 0.6), xy_range=0.05)).float()
    Kn = K.repeat(n_obj, 1, 1)
    rm = helpers.ref_meshes_from_dataset(ds)
    depth = pipeline_ref.RefRenderer(rm).render(labels, T_true, Kn, None, (480, 640), render_depth=True)["depths"][:, 0]
    rng = np.random.RandomState(3)
    T_pred = T_true.clone()
    for i in range(n_obj):
        w = torch.from_numpy(rng.randn(3)).float()
        w = w / w.norm() * np.deg2rad(2.0)
        Kx = torch.tensor([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
        T_pred[i, :3, :3] = torch.matrix_exp(Kx) @ T_true[i, :3, :3]
        T_pred[i, :3, 3] += torch.from_numpy(rng.uniform(-0.005, 0.005, 3)).float()
    return est, labels, T_true, T_pred, K, depth, ds


def test_refiner_end_to_end(tmp_path):
    est, labels, T_true, T_pred, K, depth, ds = _scene(tmp_path)
    ref = tr.TeaserppRefiner(est.depth_refiner.mesh_db, est.depth_refiner.renderer)
    infos = pd.DataFrame(dict(label=labels, batch_im_id=[0, 1, 2], instance_id=[0, 0, 0]))
    preds = PandasTensorCollection(infos, poses=T_pred.cuda())
    Kc = K.repeat(3, 1, 1).cuda()
    rng = np.random.RandomState(8)
    for corrupt in (0.0, 0.3):
        d = depth.clone()
        bad = torch.from_numpy(rng.rand(*d.shape) < corrupt)
        d[bad] = torch.from_numpy(rng.uniform(0.2, 1.5, int(bad.sum()))).float()
        refined, extra = ref.refine_poses(preds, depth=d.cuda(), K=Kc)
        assert extra["num_inliers"] >= 50 and extra["solution"].valid and extra["pc_src"].shape == (1000, 3)
        assert extra["pc_src_raw"].shape == (480, 640, 3)
        for i in range(3):
            r0, t0 = _pose_err(T_pred[i], T_true[i])
            r1, t1 = _pose_err(refined.poses[i].cpu(), T_true[i])
            a0, a1 = _add_mm(ds, labels[i], T_pred[i], T_true[i]), _add_mm(ds, labels[i], refined.poses[i].cpu(), T_true[i])
            print(f"corrupt {corrupt} object {i}: {r0:.3f} deg / {t0:.2f} mm / ADD {a0:.2f} mm -> "
                  f"{r1:.3f} deg / {t1:.2f} mm / ADD {a1:.2f} mm")
            # pixel-aligned correspondences (rendered and measured point on the same ray) constrain depth, not the
            # in-image motion: the translation error shrinks, the rotation is not held to improve
            assert t1 < t0
        assert torch.equal(refined.poses_input.cpu(), T_pred)
    # the oracle on the same inputs (first object): same acceptance and pose
    rend = ref.renderer.render(labels[:1], T_pred[:1].cuda(), Kc[:1], None, (480, 640), render_depth=True).depths[0, 0]
    acc, pose, info = T.refine_one(rend.cpu().numpy(), depth[0].numpy(), K[0].numpy(), T_pred[0].numpy())
    refined, _ = ref.refine_poses(preds, depth=depth.cuda(), K=Kc)
    assert acc
    np.testing.assert_allclose(refined.poses[0].cpu().numpy(), pose, atol=1e-5)
    # two images via batch_im_id == one at a time
    both, _ = ref.refine_poses(PandasTensorCollection(pd.DataFrame(dict(label=labels[:2], batch_im_id=[0, 1],
                                                                        instance_id=[0, 0])), poses=T_pred[:2].cuda()),
                               depth=depth[:2].cuda(), K=Kc[:2])
    for i in range(2):
        one, _ = ref.refine_poses(PandasTensorCollection(pd.DataFrame(dict(label=labels[i:i + 1], batch_im_id=[0],
                                                                           instance_id=[0])), poses=T_pred[i:i + 1].cuda()),
                                  depth=depth[i:i + 1].cuda(), K=Kc[i:i + 1])
        assert torch.equal(one.poses[0], both.poses[i])
    # n_min_points gate: nothing reached the solver, nothing changes
    empty, extra = ref.refine_poses(preds, depth=torch.zeros_like(depth).cuda(), K=Kc)
    assert extra == {} and torch.equal(empty.poses.cpu(), T_pred) and torch.equal(empty.poses_input.cpu(), T_pred)
    # min_num_inliers out of reach: solved, not accepted, poses_input registered as a copy of poses
    ref_hi = tr.TeaserppRefiner(None, est.depth_refiner.renderer, min_num_inliers=10 ** 6)
    kept, extra = ref_hi.refine_poses(preds, depth=depth.cuda(), K=Kc)
    assert extra["num_inliers"] < 10 ** 6 and torch.equal(kept.poses.cpu(), T_pred)


def test_launch_count_does_not_depend_on_predictions(tmp_path):
    est, labels, T_true, T_pred, K, depth, _ = _scene(tmp_path, n_obj=21)
    ref = tr.TeaserppRefiner(None, est.depth_refiner.renderer)
    counts = []
    for n in (1, 21):
        preds = PandasTensorCollection(pd.DataFrame(dict(label=labels[:n], batch_im_id=list(range(n)),
                                                         instance_id=[0] * n)), poses=T_pred[:n].cuda())
        Kn = K.repeat(n, 1, 1).cuda()
        ref.refine_poses(preds, depth=depth[:n].cuda(), K=Kn)   # warm
        c0 = _abi.lib().mpx_launch_count()
        ref.refine_poses(preds, depth=depth[:n].cuda(), K=Kn)
        c1 = _abi.lib().mpx_launch_count()
        ref.renderer.render(labels[:n], TCO=T_pred[:n].cuda(), K=Kn, light_datas=[ref.light_datas] * n,
                            resolution=(480, 640), render_depth=True)
        counts.append((c1 - c0) - (_abi.lib().mpx_launch_count() - c1))   # the refinement's own launches
    assert counts[0] == counts[1], counts


def test_refusals():
    lib = _abi.lib()
    host = torch.zeros(16)
    assert lib.mpx_teaser_graph(1, 1025, None, None, None, 0.02, None, None) != 0
    assert lib.mpx_teaser_graph(1, 8, host.data_ptr(), host.data_ptr(), host.data_ptr(), 0.02, host.data_ptr(), None) != 0
    assert b"not device memory" in lib.mpx_last_error()
    assert lib.mpx_teaser_points(1, 0, 5, None, None, 1, None, None, 0, 0.1, None, None, None, None, None, None) != 0


def test_graph_pairs_exactly_on_the_bound():
    """Dyadic coordinates: the float64 norm differences are exact, so pairs sit exactly on the bound (an edge) or one
    ulp-scale step beyond it (no edge)."""
    nb = 2.0 ** -7                                   # bound 2 nb = 2^-6 = 0.015625, exact
    k = 6
    ss = np.zeros((1, k, 3), np.float32)
    st = np.zeros((1, k, 3), np.float32)
    ss[0, 1] = [0.25, 0, 0]; st[0, 1] = [0.25 + 2.0 ** -6, 0, 0]             # |diff| == bound with 0
    ss[0, 2] = [0, 0.5, 0]; st[0, 2] = [0, 0.5 - 2.0 ** -6, 0]               # == bound with 0, shorter
    ss[0, 3] = [0, 0, 0.125]; st[0, 3] = [0, 0, 0.125 + 2.0 ** -6 + 2.0 ** -20]  # just beyond with 0
    ss[0, 4] = [0.25, 0, 0.5]; st[0, 4] = [0.25 + 2.0 ** -6, 0, 0.5 + 2.0 ** -6]  # == bound with 1 (along z)
    ss[0, 5] = [1.0, 0, 0]; st[0, 5] = [1.0, 0, 0]
    a = T.consistency_graph(ss[0], st[0], nb)
    assert a[0, 1] and a[0, 2] and not a[0, 3] and a[1, 4]
    adj = tr.consistency_graph(torch.from_numpy(ss).cuda(), torch.from_numpy(st).cuda(),
                               torch.tensor([k], dtype=torch.int32).cuda(), nb)
    assert np.array_equal(adj[0].cpu().numpy().view(np.uint64), T.pack_adjacency(a, k))


def test_random_sampling_subset():
    cap, k = 5000, 1000
    counts = [150, 999, 1000, 1001, 4000]
    src = torch.randn(len(counts), cap, 3).cuda()
    tgt = src * 3
    c = torch.tensor(counts, dtype=torch.int32).cuda()
    idx, ss, st = tr.random_sampling(src, tgt, c, k)
    for n, cn in enumerate(counts):
        m = min(k, cn)
        i = idx[n, :m].cpu()
        assert len(set(i.tolist())) == m and int(i.max()) < cn and int(i.min()) >= 0
        assert torch.equal(ss[n, :m].cpu(), src[n, i].cpu()) and torch.equal(st[n, :m].cpu(), tgt[n, i].cpu())


def test_compute_teaserpp_refinement_equals_oracle():
    h, w = 60, 80
    rng = np.random.RandomState(6)
    K = np.array([[300, 0, 40], [0, 300, 30], [0, 0, 1]], np.float32)
    yy, xx = np.mgrid[:h, :w]
    src = (0.5 + 0.001 * xx + 0.0005 * yy + 0.01 * np.sin(xx / 7.0) * np.cos(yy / 5.0)).astype(np.float32)
    tgt = (src + 0.003 + rng.normal(0, 0.001, (h, w))).astype(np.float32)
    bad = rng.rand(h, w) < 0.2
    tgt[bad] = rng.uniform(0.3, 0.9, int(bad.sum()))
    mask = np.ones((h, w), bool)
    mask[:5] = False
    out = tr.compute_teaserpp_refinement(torch.from_numpy(src).cuda(), torch.from_numpy(tgt).cuda(),
                                         torch.from_numpy(K).cuda(), torch.from_numpy(mask).cuda(), max_num_points=300)
    _, _, info = T.refine_one(np.where(mask, src, 0).astype(np.float32), tgt, K, np.eye(4, dtype=np.float32),
                              n_min_points=1, n_points=300, min_num_inliers=0)
    assert out["solution"].valid and info["valid"]
    np.testing.assert_allclose(out["T_tgt_src"], info["T"], atol=1e-9)
    assert out["num_inliers"] == info["num_inliers"]
    assert out["pc_src"].shape == (300, 3) and out["pc_src_mask"].shape == (int(mask.sum()), 3)


def test_pose_estimator_pipeline_with_teaserpp(tmp_path):
    from megapose6d_b200.pose_estimator import PoseEstimator
    from megapose6d_b200.types import ObservationTensor

    est, labels, T_true, T_pred, K, depth, ds = _scene(tmp_path, n_obj=2)
    refiner = tr.TeaserppRefiner(est.refiner_model.mesh_db, est.refiner_model.renderer)
    pe = PoseEstimator(refiner_model=est.refiner_model, coarse_model=est.coarse_model, depth_refiner=refiner,
                       SO3_grid_size=72)
    rgb = torch.from_numpy(np.random.RandomState(4).randint(0, 256, (1, 3, 480, 640), dtype=np.uint8))
    d = torch.where(depth[1] > 0, depth[1], depth[0])[None]      # both objects in one frame (they do not overlap much)
    obs = ObservationTensor.from_torch_batched(rgb, d, K).cuda()
    bboxes = torch.stack([helpers.detection_for_pose(K[0], T_true[i], torch.from_numpy(
        next(o for o in ds.list_objects if o.label == labels[i]).mesh.vertices).float()) for i in range(2)])
    det = PandasTensorCollection(pd.DataFrame(dict(label=labels, batch_im_id=0, instance_id=np.arange(2))),
                                 bboxes=bboxes.cuda())
    final, extra = pe.run_inference_pipeline(obs, detections=det, n_refiner_iterations=1, n_pose_hypotheses=1,
                                             run_depth_refiner=True)
    dr = extra["depth_refiner"]["preds"]
    assert len(dr) == 2 and "poses_input" in dr.tensors and torch.equal(final.poses, dr.poses)
    incoming = extra["refiner"]["preds"].poses
    for i in range(2):
        assert torch.equal(dr.poses[i], incoming[i]) or torch.equal(dr.poses_input[i], incoming[i])


@pytest.mark.parametrize("which", ["teaserpp", "icp"])
def test_prediction_runner_depth_refiner_cli(tmp_path, which):
    import json
    from PIL import Image
    from megapose6d_b200 import prediction_runner

    box = procedural.textured_sphere(seed=3).with_defaults()
    frame = tmp_path / "frame"
    (frame / "meshes" / "obj_000001").mkdir(parents=True)   # BOP CSV: obj_id = the integer after the label's "_"
    lines = ["v %.6f %.6f %.6f" % tuple(v * 1000.0) for v in box.vertices]
    lines += ["vn %.6f %.6f %.6f" % tuple(n) for n in box.vertex_normals]
    lines += ["f " + " ".join(f"{i + 1}//{i + 1}" for i in f) for f in box.faces]
    (frame / "meshes" / "obj_000001" / "obj_000001.obj").write_text("\n".join(lines) + "\n")
    (frame / "inputs").mkdir()
    Kc = procedural.example_camera()
    (frame / "camera_data.json").write_text(json.dumps({"K": Kc.tolist(), "resolution": [480, 640]}))
    (frame / "inputs" / "object_data.json").write_text(json.dumps([{"label": "obj_000001", "bbox_modal": [250, 170, 390, 300]}]))
    Image.fromarray(np.random.RandomState(2).randint(0, 255, (480, 640, 3), dtype=np.uint8)).save(frame / "image_rgb.png")
    Image.fromarray(np.full((480, 640), 600, np.uint16)).save(frame / "image_depth.png")
    models = tmp_path / "models"
    load_model.write_run(models, "coarse-rgb-906902141", helpers.make_state_dict(helpers.COARSE_CFG, 1))
    load_model.write_run(models, "refiner-rgb-653307694", helpers.make_state_dict(helpers.REFINER_CFG, 2))
    out = tmp_path / "out"
    prediction_runner.main([str(frame), "--model", "megapose-1.0-RGB-multi-hypothesis-icp", "--models-root", str(models),
                            "--save-dir", str(out), "--depth-refiner", which])
    rows = (out / "bop_refiner_final.csv").read_text().strip().splitlines()
    assert rows[0].startswith("scene_id,im_id,obj_id") and len(rows) == 2
    preds = torch.load(out / "predictions.pth.tar", weights_only=False)
    assert "depth_refiner" in preds
    with pytest.raises(SystemExit):
        prediction_runner.main([str(frame), "--model", "megapose-1.0-RGB", "--models-root", str(models),
                                "--save-dir", str(out), "--depth-refiner", which])
