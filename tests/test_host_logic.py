"""CPU tests of the host-side mirror: containers, configs, checkpoints, meshes, weight repacking, C ABI exports."""
import ctypes
import re
from pathlib import Path

import numpy as np
import pandas as pd
import pytest
import torch
import torch.nn.functional as F

from megapose6d_b200 import _abi, backbone, load_model, meshes, procedural
from megapose6d_b200 import tensor_collection as tc
from megapose6d_b200.pose_estimator import add_instance_id, filter_detections
from megapose6d_b200.types import ObservationTensor, assert_detections_valid
from oracle import resnet_ref
from tests import helpers

ROOT = Path(__file__).resolve().parents[1]


def test_abi_library_loads_and_exports_every_declared_symbol():
    header = (ROOT / "include" / "mpx.h").read_text()
    declared = set(re.findall(r"\b(mpx_[A-Za-z0-9_]+)\s*\(", header))
    assert len(declared) >= 25
    lib = ctypes.CDLL(str(_abi.lib_path()))
    missing = [name for name in sorted(declared) if not hasattr(lib, name)]
    assert not missing, f"symbols declared in include/mpx.h but not exported: {missing}"
    assert set(_abi.EXPORTS) == declared
    assert _abi.lib().mpx_abi_version() == _abi.ABI_VERSION == 5
    assert _abi.lib().mpx_act_dtype() in (0, 1)


def test_product_does_not_import_the_oracle():
    for path in (ROOT / "megapose6d_b200").rglob("*.py"):
        text = path.read_text()
        assert "import oracle" not in text and "from oracle" not in text, path


def test_tensor_collection_semantics():
    df = pd.DataFrame(dict(label=["a", "b", "c"], batch_im_id=[0, 0, 1]), index=[5, 6, 7])
    c = tc.PandasTensorCollection(df, poses=torch.arange(3 * 16).float().view(3, 4, 4))
    assert list(c.infos.index) == [0, 1, 2] and len(c) == 3
    sub = c[[2, 0]]
    assert sub.infos["label"].tolist() == ["c", "a"] and torch.equal(sub.poses[0], c.poses[2])
    sub2 = c[torch.tensor([1])]
    assert sub2.infos["label"].tolist() == ["b"]
    cat = tc.concatenate([sub, sub2])
    assert len(cat) == 3 and cat.poses.shape == (3, 4, 4)
    c.poses = c.poses * 2
    assert "poses" in c.tensors and c.poses[0, 0, 1] == 2
    with pytest.raises(AttributeError):
        _ = c.nope
    assert len(tc.concatenate([])) == 0


def test_detections_helpers():
    df = pd.DataFrame(dict(label=["a", "a", "b"], batch_im_id=[0, 0, 0], score=[0.3, 0.9, 0.5]))
    det = tc.PandasTensorCollection(df, bboxes=torch.zeros(3, 4))
    det = add_instance_id(det)
    assert det.infos["instance_id"].tolist() == [0, 1, 0]
    assert_detections_valid(det)
    one = filter_detections(det, one_instance_per_class=True)
    assert sorted(one.infos["score"].tolist()) == [0.5, 0.9]
    assert len(filter_detections(det, labels=["b"])) == 1


def test_observation_tensor():
    rgb = np.random.RandomState(0).randint(0, 255, (4, 6, 3)).astype(np.uint8)
    obs = ObservationTensor.from_numpy(rgb, depth=np.ones((4, 6), np.float32), K=np.eye(3))
    assert obs.images.shape == (1, 4, 4, 6) and obs.is_valid() and obs.depth.shape == (1, 4, 6)
    assert not ObservationTensor(obs.images * 300, obs.K).is_valid()


def test_config_compat_rules(tmp_path):
    (tmp_path / "config.yaml").write_text("input_strategy: input=obs+one_render\nbackbone_str: vanilla_resnet34\n")
    cfg = load_model.check_update_config(load_model.load_cfg(tmp_path / "config.yaml"))
    assert cfg.is_coarse_compat and cfg.predict_rendered_views_logits and not cfg.predict_pose_update and cfg.n_rendered_views == 1
    (tmp_path / "c2.yaml").write_text("multiview_type: front_3views\nn_views: 4\nrender_normals: true\ndepth_augmentation: false\n"
                                      "depth_normalization_type: tCR_scale_clamp_center\n")
    cfg = load_model.check_update_config(load_model.load_cfg(tmp_path / "c2.yaml"))
    assert cfg.multiview_type == "TCO+front_3views" and cfg.n_rendered_views == 4 and "n_views" not in cfg
    assert cfg.depth_normalization_type == "tCR_scale_clamp_center" and load_model.n_input_channels(cfg) == 27
    # pickled-object YAML written by old runs is read as a mapping
    (tmp_path / "c3.yaml").write_text("!!python/object:megapose.training.training_config.TrainingConfig\nbackbone_str: vanilla_resnet34\n"
                                      "n_rendered_views: 1\n")
    assert load_model.load_cfg(tmp_path / "c3.yaml").n_rendered_views == 1
    sd = load_model.change_keys_of_older_models({"backbone.backbone.conv1.weight": 1, "backbone.head.0.bias": 2, "pose_fc.bias": 3})
    assert set(sd) == {"backbone.conv1.weight", "views_logits_head.bias", "pose_fc.bias"}


def test_checkpoint_roundtrip_in_reference_format(tmp_path):
    sd = helpers.make_state_dict(helpers.COARSE_CFG, 1)
    run = load_model.write_run(tmp_path, "coarse-rgb-906902141", sd)
    ck = torch.load(run / "checkpoint.pth.tar", weights_only=False)
    assert set(ck) == {"state_dict", "epoch"} and torch.equal(ck["state_dict"]["backbone.conv1.weight"], sd["backbone.conv1.weight"])
    assert set(load_model.NAMED_MODELS) == {"megapose-1.0-RGB", "megapose-1.0-RGBD", "megapose-1.0-RGB-multi-hypothesis",
                                            "megapose-1.0-RGB-multi-hypothesis-icp"}


def test_stem_space_to_depth_and_bn_folding_are_exact():
    """The repacked stem (4x4/s1 over the space-to-depth input) equals conv7x7/s2 + BN in fp64-folded fp32."""
    sd = helpers.make_state_dict(helpers.COARSE_CFG, 4)
    w, b = backbone._fold(sd, "backbone.conv1", "backbone.bn1")
    x = torch.rand(2, 9, 32, 48, dtype=torch.float64)
    want = F.batch_norm(F.conv2d(x, sd["backbone.conv1.weight"].double(), stride=2, padding=3),
                        sd["backbone.bn1.running_mean"].double(), sd["backbone.bn1.running_var"].double(),
                        sd["backbone.bn1.weight"].double(), sd["backbone.bn1.bias"].double(), training=False, eps=1e-5)
    c_pad = 16
    xp = torch.zeros(2, c_pad, 32, 48, dtype=torch.float64)
    xp[:, :9] = x
    s2d = xp.view(2, c_pad, 16, 2, 24, 2).permute(0, 3, 5, 1, 2, 4).reshape(2, 4 * c_pad, 16, 24)  # (dy, dx, c) channels
    w2 = backbone._stem_s2d(w, c_pad).view(64, 4, 4, 4 * c_pad).permute(0, 3, 1, 2)
    got = F.conv2d(F.pad(s2d, (2, 1, 2, 1)), w2, bias=b)
    assert torch.allclose(got, want, rtol=1e-10, atol=1e-10)
    wp = backbone._pack(w)
    assert wp.shape == (64, 49 * 9) and torch.equal(wp[:, :9], w[:, :, 0, 0])
    Wh, bh = resnet_ref.folded_head(sd)
    feat = torch.randn(3, 512, dtype=torch.float64)
    fc = F.linear(F.linear(feat, sd["backbone.fc.weight"].double(), sd["backbone.fc.bias"].double()),
                  sd["views_logits_head.weight"].double(), sd["views_logits_head.bias"].double())
    assert torch.allclose(F.linear(feat, Wh, bh), fc, atol=1e-10)


def test_mesh_readers_and_database(tmp_path):
    m = procedural.bumpy_sphere(n_seg=24, n_lat=13)
    # ascii PLY with colours
    lines = ["ply", "format ascii 1.0", f"element vertex {len(m.vertices)}", "property float x", "property float y",
             "property float z", "property uchar red", "property uchar green", "property uchar blue",
             f"element face {len(m.faces)}", "property list uchar int vertex_indices", "end_header"]
    for v, c in zip(m.vertices, m.vertex_colors):
        lines.append(f"{v[0]:.9g} {v[1]:.9g} {v[2]:.9g} {int(round(c[0]*255))} {int(round(c[1]*255))} {int(round(c[2]*255))}")
    for f in m.faces:
        lines.append(f"3 {f[0]} {f[1]} {f[2]}")
    (tmp_path / "a.ply").write_text("\n".join(lines) + "\n")
    a = meshes.load_mesh(tmp_path / "a.ply")
    assert np.allclose(a.vertices, m.vertices, atol=1e-7) and np.array_equal(a.faces, m.faces)
    assert np.allclose(a.vertex_colors, m.vertex_colors, atol=1 / 255)
    # binary little-endian PLY
    import struct
    hdr = "\n".join(["ply", "format binary_little_endian 1.0", f"element vertex {len(m.vertices)}", "property float x",
                     "property float y", "property float z", f"element face {len(m.faces)}",
                     "property list uchar int vertex_indices", "end_header"]) + "\n"
    body = b"".join(struct.pack("<fff", *v) for v in m.vertices) + b"".join(struct.pack("<Biii", 3, *f) for f in m.faces)
    (tmp_path / "b.ply").write_bytes(hdr.encode() + body)
    b = meshes.load_mesh(tmp_path / "b.ply")
    assert np.allclose(b.vertices, m.vertices, atol=1e-6) and np.array_equal(b.faces, m.faces)
    # OBJ with a quad face -> two triangles
    (tmp_path / "c.obj").write_text("v 0 0 0\nv 1 0 0\nv 1 1 0\nv 0 1 0\nf 1 2 3 4\n")
    c = meshes.load_mesh(tmp_path / "c.obj")
    assert c.faces.tolist() == [[0, 1, 2], [0, 2, 3]]
    n = meshes.compute_vertex_normals(c.vertices, c.faces)
    assert np.allclose(n, [[0, 0, 1]] * 4)
    # database: padding and deterministic subsets follow the reference's RandomState(0) rules
    ds = procedural.make_object_dataset(2, n_seg=60, n_lat=41)
    ds.list_objects[1].mesh = procedural.bumpy_sphere(n_seg=50, n_lat=45)
    db = meshes.MeshDataBase.from_object_ds(ds).batched()
    assert db.points.shape == (2, 60 * 40 + 2, 3) and db.points.dtype == torch.float32
    sel = db.select([ds[1].label, ds[0].label])
    assert torch.equal(sel.points[1], db.points[0])
    assert torch.equal(sel.sample_points(2000, deterministic=True), db.point_subset(2000)[[1, 0]])


def test_procedural_mesh_counts():
    m = procedural.bumpy_sphere()
    assert m.faces.shape == (10000, 3) and m.vertices.shape == (5002, 3)
    assert m.faces.min() == 0 and m.faces.max() == 5001
    assert np.allclose(np.linalg.norm(m.vertex_normals, axis=1), 1, atol=1e-6)
    # outward orientation: normals point away from the centre
    assert (np.einsum("ij,ij->i", m.vertex_normals, m.vertices) > 0).mean() > 0.99


def test_so3_grid_rotations_agree_with_an_independent_quaternion_library():
    """load_SO3_grid turns the (x, y, z, w) quaternions of data_<N>.qua into matrices with roma.unitquat_to_rotmat
    (utils/transform_utils.py:27-50); roma is not installable here, so the restated formula (product: so3.py, oracle:
    lib3d_ref.unitquat_to_rotmat) is held against scipy's scalar-last Rotation.from_quat, an independent implementation of
    the same convention."""
    import numpy as np
    import torch
    from scipy.spatial.transform import Rotation

    from megapose6d_b200 import so3
    from oracle import lib3d_ref

    for n in (72, 576):
        q = np.load(so3._DATA / f"so3_grid_{n}.npy").astype(np.float64)
        assert q.shape == (n, 4) and np.allclose(np.linalg.norm(q, axis=1), 1.0, atol=1e-5)
        want = Rotation.from_quat(q).as_matrix()  # (x, y, z, w)
        got = so3.load_SO3_grid(n).double().numpy()
        ora = lib3d_ref.unitquat_to_rotmat(torch.tensor(q)).numpy()
        assert np.abs(got - want).max() < 1e-5 and np.abs(ora - want).max() < 1e-5  # fp32 grid, file quaternions unit to 1e-6
        assert np.allclose(got @ got.transpose(0, 2, 1), np.eye(3), atol=1e-5) and np.allclose(np.linalg.det(got), 1.0, atol=1e-5)
