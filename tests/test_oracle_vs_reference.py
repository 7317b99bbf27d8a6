"""The oracle restatements must reproduce the REAL reference code.

What the reference returned for these inputs is stored under tests/golden/reference/ (helpers.reference_outputs: the
reference itself, loaded by path through oracle/refload.py, runs only to re-record them), so the comparisons run
everywhere.
"""
import numpy as np
import pandas as pd
import pytest
import torch

from oracle import lib3d_ref as L
from oracle import pipeline_ref, refload, resnet_ref, so3_ref
from tests import helpers

def _rand_pose(n, seed):
    from megapose6d_b200.procedural import random_poses

    return torch.from_numpy(random_poses(n, seed)).float()


def test_lib3d_functions_match():
    g = torch.Generator().manual_seed(0)
    n = 7
    TCO = _rand_pose(n, 1)
    K = torch.from_numpy(helpers.procedural.example_camera()).float().unsqueeze(0).repeat(n, 1, 1)
    pts = torch.randn(n, 300, 3, generator=g) * 0.05
    uv = L.project_points_robust(pts, K, TCO)
    boxes = L.boxes_from_uv(uv)
    p9 = torch.randn(n, 9, generator=g)
    Tn = TCO + 0.01 * torch.randn(n, 4, 4, generator=g)
    tCR = TCO[:, :3, 3] + 0.01
    dR = L.compute_rotation_matrix_from_ortho6d(p9[:, :6])
    Kc = L.get_K_crop_resize(K, boxes, (240, 320))
    bb = torch.tensor([[384.0, 234, 522, 455]]).repeat(n, 1) + torch.arange(n).view(-1, 1)
    R = L.compute_rotation_matrix_from_ortho6d(torch.randn(n, 6, generator=g))

    def reference():
        ref = refload.load()
        return dict(
            uv=ref.camera_geometry.project_points_robust(pts, K, TCO), boxes=ref.camera_geometry.boxes_from_uv(uv),
            K_crop=ref.camera_geometry.get_K_crop_resize(K.clone(), boxes, (480, 640), (240, 320)),
            ortho6d=ref.rotations.compute_rotation_matrix_from_ortho6d(p9[:, :6]),
            normalize_T=ref.transform_ops.normalize_T(Tn), invert=ref.transform_ops.invert_transform_matrices(TCO),
            update=ref.cosypose_ops.pose_update_with_reference_point(TCO, Kc, p9[:, 6:], dR, tCR),
            init=ref.cosypose_ops.TCO_init_from_boxes_autodepth_with_R(bb, pts, K, R))

    want = helpers.reference_outputs("lib3d_functions", reference)
    assert torch.equal(uv, want["uv"])
    assert torch.equal(boxes, want["boxes"])
    assert torch.equal(L.get_K_crop_resize(K, boxes, (240, 320)), want["K_crop"])
    assert torch.equal(L.compute_rotation_matrix_from_ortho6d(p9[:, :6]), want["ortho6d"])
    assert torch.equal(L.normalize_T(Tn), want["normalize_T"])
    assert torch.equal(L.invert_transform_matrices(TCO), want["invert"])
    assert torch.equal(L.pose_update_with_reference_point(TCO, Kc, p9[:, 6:], dR, tCR), want["update"])
    assert torch.equal(L.TCO_init_from_boxes_autodepth_with_R(bb, pts, K, R), want["init"])


def test_crops_match():
    ds, images, K = helpers.make_scene(1, seed=3, with_depth=True)
    n = 3
    TCO = _rand_pose(n, 5)
    Kn = K.repeat(n, 1, 1)
    pts = torch.from_numpy(ds[0].mesh.vertices[:2000]).float().unsqueeze(0).repeat(n, 1, 1)
    uv = L.project_points_robust(pts, Kn, TCO)
    obs = L.boxes_from_uv(uv)
    imgs = images.repeat(n, 1, 1, 1)
    b1, c1 = L.deepim_crops_robust(imgs, obs, Kn, TCO, TCO[:, :3, 3], pts, (240, 320))

    def reference():
        b2, c2 = refload.load().cropping.deepim_crops_robust(images=imgs, obs_boxes=obs, K=Kn, TCO_pred=TCO,
                                                             tCR_in=TCO[:, :3, 3], O_vertices=pts, output_size=(240, 320),
                                                             lamb=1.4)
        return dict(boxes=b2, crops_digest=helpers.digest_of(c2))

    want = helpers.reference_outputs("crops", reference)
    assert torch.equal(b1, want["boxes"]) and torch.equal(torch.from_numpy(helpers.digest_of(c1)), want["crops_digest"])


def test_sample_and_pad():
    pts = torch.arange(5002 * 3, dtype=torch.float32).view(1, 5002, 3)
    ids = L.sample_point_ids(5002, 2000)
    want = helpers.reference_outputs(
        "sample_points", lambda: dict(points=refload.load().mesh_ops.sample_points(pts, 2000, deterministic=True)))
    assert torch.equal(pts[:, ids], want["points"])


def test_so3_asset_matches_reference_file():
    from megapose6d_b200.so3 import load_SO3_grid

    # so3_ref parses the reference's own data/data_<n>.qua where the reference tree exists
    want = helpers.reference_outputs(
        "so3_grids", lambda: {str(n): helpers.digest_of(so3_ref.load_SO3_grid_reference(n)) for n in (72, 576, 4608)})
    for n in (72, 576, 4608):
        assert torch.equal(torch.from_numpy(helpers.digest_of(load_SO3_grid(n))), want[str(n)])


def test_resnet_restatement_matches_reference_module():
    for name, cfg in (("coarse", helpers.COARSE_CFG), ("refiner", helpers.REFINER_CFG)):
        sd = helpers.make_state_dict(cfg, seed=1)
        c = helpers.n_inputs(cfg)
        x = torch.rand(2, c, 64, 96, generator=torch.Generator().manual_seed(2))
        head = resnet_ref.head_name(sd)

        def reference():
            net = refload.load().torchvision_resnet.resnet34(num_classes=512, n_input_channels=c)
            net.load_state_dict({k[len("backbone."):]: v for k, v in sd.items() if k.startswith("backbone.")})
            net.eval()
            with torch.no_grad(), helpers.reproducible_fp32():
                return dict(out=torch.nn.functional.linear(net(x), sd[head + ".weight"], sd[head + ".bias"]),
                            head_weight=sd[head + ".weight"], head_bias=sd[head + ".bias"])

        want = helpers.reference_outputs(f"resnet34_{name}", reference)
        # the head make_state_dict calibrated (fp32 CPU arithmetic) when the reference ran
        sd = dict(sd, **{head + ".weight": want["head_weight"], head + ".bias": want["head_bias"]})
        with torch.no_grad(), helpers.reproducible_fp32():
            got = resnet_ref.forward(sd, x)
        assert torch.allclose(got, want["out"], rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("backbone_str,cls", [("resnet34", "WideResNet34"), ("resnet18", "WideResNet18")])
def test_wide_resnet_restatement_matches_reference_module(backbone_str, cls):
    """models/wide_resnet.py:59-126 (pre-activation blocks, bare 1x1 downsample, no fc) + the spatial mean of
    PosePredictor.net_forward (models/pose_rigid.py:323-328) + head."""
    sd = resnet_ref.init_state_dict_wide(9, "views_logits_head", 2, seed=5, backbone_str=backbone_str)
    x = torch.rand(2, 9, 64, 96, generator=torch.Generator().manual_seed(2))

    def reference():
        net = getattr(refload.load().wide_resnet, cls)(n_inputs=9)
        net.load_state_dict({k[len("backbone."):]: v for k, v in sd.items() if k.startswith("backbone.")})
        net.eval()
        with torch.no_grad():
            return dict(out=torch.nn.functional.linear(net(x).flatten(2).mean(dim=-1), sd["views_logits_head.weight"],
                                                       sd["views_logits_head.bias"]))

    want = helpers.reference_outputs(f"wide_{backbone_str}", reference)["out"]
    with torch.no_grad():
        got = resnet_ref.forward_wide(sd, x)
        emu = resnet_ref.forward_wide_act16_emulated(sd, x)
        bound = resnet_ref.act16_forward_error_bound(sd, x)
    assert torch.allclose(got, want, rtol=1e-5, atol=1e-5)
    assert ((emu - want).abs() <= bound).all()
    from workloads import weights
    sd_w = weights.init_state_dict_wide(9, "views_logits_head", 2, seed=5, backbone_str=backbone_str)
    assert all(torch.equal(sd[k], sd_w[k]) for k in sd)  # the workload generator and the oracle agree on the layout


class _MeshDbAdapter:
    """mesh_db.select(labels).{points, sample_points} as the reference's PosePredictor expects."""

    def __init__(self, meshes, ref):
        self.m, self.ref = meshes, ref

    def select(self, labels):
        pts = self.m.select_points(labels)
        ref = self.ref

        class _Sel:
            points = pts

            @staticmethod
            def sample_points(n, deterministic=False):
                return ref.mesh_ops.sample_points(pts, n, deterministic=deterministic)

        return _Sel()


def _reference_predictor(ref, cfg, sd, meshes, render_size=(240, 320), n_threads=None):
    class Renderer(ref.Panda3dBatchRenderer):
        def __init__(self, inner):
            self.inner = inner

        def render(self, labels, TCO, K, light_datas, resolution, render_depth=False, render_mask=False,
                   render_normals=False):
            d = self.inner.render(labels, TCO, K, None, resolution, render_depth, render_mask, render_normals)
            return type("Out", (), d)

    c = helpers.n_inputs(cfg)
    backbone = ref.torchvision_resnet.resnet34(num_classes=512, n_input_channels=c)
    backbone.n_features = 512
    model = ref.pose_rigid.PosePredictor(
        backbone=backbone, renderer=Renderer(pipeline_ref.RefRenderer(meshes, **({} if n_threads is None else dict(n_threads=n_threads)))),
        mesh_db=_MeshDbAdapter(meshes, ref), render_size=tuple(render_size), n_rendered_views=cfg["n_rendered_views"], multiview_type=cfg["multiview_type"],
        render_normals=True, render_depth=cfg["render_depth"], input_depth=cfg["input_depth"],
        predict_rendered_views_logits=cfg["predict_rendered_views_logits"], remove_TCO_rendering=False,
        predict_pose_update=cfg["predict_pose_update"], depth_normalization_type=cfg["depth_normalization_type"])
    model.load_state_dict(sd)
    return model.eval()


@pytest.mark.parametrize("cfg_name", ["coarse", "refiner", "refiner_rgbd"])
def test_pose_predictor_matches_reference(cfg_name):
    cfg = dict(coarse=helpers.COARSE_CFG, refiner=helpers.REFINER_CFG, refiner_rgbd=helpers.REFINER_RGBD_CFG)[cfg_name]
    ds, images, K = helpers.make_scene(2, seed=4, with_depth=cfg["input_depth"])
    meshes = helpers.ref_meshes_from_dataset(ds)
    sd = helpers.make_state_dict(cfg, seed=3)
    labels = [ds[0].label, ds[1].label]
    TCO = _rand_pose(2, 8)
    imgs, Kn = images.repeat(2, 1, 1, 1), K.repeat(2, 1, 1)
    S = helpers.sample_of  # renders and crops are compared on a fixed sample of their values (stored files stay small)
    head = resnet_ref.head_name(sd)

    def reference():
        model = _reference_predictor(refload.load(), cfg, sd, meshes)
        with torch.no_grad(), helpers.reproducible_fp32():
            if cfg["predict_pose_update"]:
                out = model(images=imgs, K=Kn, labels=labels, TCO=TCO, n_iterations=2)
                d = {}
                for it in ("iteration=1", "iteration=2"):
                    w = out[it]
                    d.update({f"{it}/TCO_output": w.TCO_output, f"{it}/K_crop": w.K_crop, f"{it}/KV_crop": w.KV_crop,
                              f"{it}/renders": S(w.renders), f"{it}/images_crop": S(w.images_crop),
                              f"{it}/network_output": w.network_outputs["pose"]})
                return dict(d, head_weight=sd[head + ".weight"], head_bias=sd[head + ".bias"])
            out = model.forward_coarse(images=imgs, K=Kn, labels=labels, TCO_input=TCO, return_debug_data=True)
            return dict(renders=S(out["renders"]), images_crop=S(out["images_crop"]), logits=out["logits"],
                        head_weight=sd[head + ".weight"], head_bias=sd[head + ".bias"])

    want = helpers.reference_outputs(f"pose_predictor_{cfg_name}", reference)
    # make_state_dict calibrates the head with fp32 CPU arithmetic (its last bits depend on the CPU): use the head the
    # reference ran with
    sd = dict(sd, **{head + ".weight": want["head_weight"], head + ".bias": want["head_bias"]})
    oracle = pipeline_ref.RefPosePredictor(sd, cfg, meshes, pipeline_ref.RefRenderer(meshes))
    with torch.no_grad(), helpers.reproducible_fp32():  # both sides: the refiner's chained iterations amplify CPU-dependent sums
        if cfg["predict_pose_update"]:
            got = oracle.forward(imgs, Kn, labels, TCO, n_iterations=2)
            for it in ("iteration=1", "iteration=2"):
                g = got[it]
                w = {k.split("/")[1]: v for k, v in want.items() if k.startswith(it + "/")}
                assert torch.allclose(g["TCO_output"], w["TCO_output"], rtol=1e-5, atol=1e-6)
                assert torch.equal(g["K_crop"], w["K_crop"]) or torch.allclose(g["K_crop"], w["K_crop"], rtol=1e-6, atol=1e-4)
                assert torch.allclose(g["KV_crop"], w["KV_crop"], rtol=1e-6, atol=1e-4)
                assert torch.allclose(S(g["renders"]), w["renders"], atol=1e-6)
                assert torch.allclose(S(g["images_crop"]), w["images_crop"], atol=1e-6)
                assert torch.allclose(g["network_output"], w["network_output"], rtol=1e-4, atol=1e-5)
        else:
            got = oracle.forward_coarse(imgs, Kn, labels, TCO)
            assert torch.allclose(S(got["renders"]), want["renders"], atol=1e-6)
            assert torch.allclose(S(got["images_crop"]), want["images_crop"], atol=1e-6)
            assert torch.allclose(got["logits"], want["logits"], rtol=1e-4, atol=1e-5)


def test_pose_estimator_pipeline_matches_reference():
    """The reference's own PoseEstimator.run_inference_pipeline vs the oracle pipeline (72-rotation grid)."""
    ds, images, K = helpers.make_scene(2, seed=6)
    meshes = helpers.ref_meshes_from_dataset(ds)
    sd_c, sd_r = helpers.make_state_dict(helpers.COARSE_CFG, 5), helpers.make_state_dict(helpers.REFINER_CFG, 6)
    head_c, head_r = resnet_ref.head_name(sd_c), resnet_ref.head_name(sd_r)
    labels = [o.label for o in ds.list_objects]
    TCO_gt = _rand_pose(2, 11)
    TCO_gt[:, 2, 3] = torch.tensor([0.55, 0.7])
    bboxes = torch.stack([helpers.detection_for_pose(K[0], TCO_gt[i], torch.from_numpy(ds[i].mesh.vertices).float())
                          for i in range(2)])
    det_df = pd.DataFrame(dict(label=labels, batch_im_id=0, instance_id=np.arange(2)))

    def reference():
        ref = refload.load()
        coarse = _reference_predictor(ref, helpers.COARSE_CFG, sd_c, meshes)
        refiner = _reference_predictor(ref, helpers.REFINER_CFG, sd_r, meshes)
        coarse.cfg = refiner.cfg = None
        with refload.cpu_cuda_patch(), helpers.reproducible_fp32():
            est = ref.pose_estimator.PoseEstimator(refiner_model=refiner, coarse_model=coarse, bsz_objects=2, bsz_images=64,
                                                   SO3_grid_size=72)
            detections = ref.tensor_collection.PandasTensorCollection(det_df.copy(), bboxes=bboxes)
            obs = ref.types.ObservationTensor(images, K)
            final, extra = est.run_inference_pipeline(obs, detections=detections, n_refiner_iterations=2, n_pose_hypotheses=2)
        coarse_preds = extra["coarse"]["preds"]
        return dict(coarse_logit=coarse_preds.infos["coarse_logit"].values, coarse_poses=coarse_preds.poses,
                    final_hypothesis_id=final.infos["hypothesis_id"].values, final_label=final.infos["label"].values,
                    final_poses=final.poses, coarse_head_weight=sd_c[head_c + ".weight"],
                    coarse_head_bias=sd_c[head_c + ".bias"], refiner_head_weight=sd_r[head_r + ".weight"],
                    refiner_head_bias=sd_r[head_r + ".bias"])

    want = helpers.reference_outputs("pose_estimator_pipeline", reference)
    # the heads make_state_dict calibrated (fp32 CPU arithmetic) when the reference ran
    sd_c = dict(sd_c, **{head_c + ".weight": want["coarse_head_weight"], head_c + ".bias": want["coarse_head_bias"]})
    sd_r = dict(sd_r, **{head_r + ".weight": want["refiner_head_weight"], head_r + ".bias": want["refiner_head_bias"]})
    oc = pipeline_ref.RefPosePredictor(sd_c, helpers.COARSE_CFG, meshes, pipeline_ref.RefRenderer(meshes))
    orf = pipeline_ref.RefPosePredictor(sd_r, helpers.REFINER_CFG, meshes, pipeline_ref.RefRenderer(meshes))
    oest = pipeline_ref.RefPoseEstimator(oc, orf, bsz_images=64, bsz_objects=2, SO3_grid_size=72)
    with helpers.reproducible_fp32():
        got = oest.run_inference_pipeline(images, K, det_df.copy(), bboxes, n_refiner_iterations=2, n_pose_hypotheses=2)
    assert np.allclose(got["coarse_df"]["coarse_logit"].values, want["coarse_logit"].numpy(), rtol=1e-4, atol=1e-5)
    assert torch.allclose(got["coarse_poses"], want["coarse_poses"], rtol=1e-5, atol=1e-6)
    assert sorted(got["final_df"]["hypothesis_id"].tolist()) == sorted(want["final_hypothesis_id"].tolist())
    order_w = np.argsort(want["final_label"])
    order_g = np.argsort(got["final_df"]["label"].values)
    assert torch.allclose(got["final_poses"][order_g], want["final_poses"][order_w], rtol=1e-4, atol=1e-5)
