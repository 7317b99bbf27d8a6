"""The multi-object scene contract on the CPU (tests/scene_ref.c) and the host side of the scene renderer: pose
composition, refusals, and the example's overlay helpers."""
import numpy as np
import pytest
import torch

from megapose6d_b200 import example, procedural
from megapose6d_b200.object_dataset import RigidObject, RigidObjectDataset
from megapose6d_b200.renderer import Panda3dLightData, make_scene_lights
from megapose6d_b200.scene_renderer import (CameraRenderingData, Panda3dCameraData, Panda3dObjectData,
                                            Panda3dSceneRenderer, compose_TCO)
from oracle import pipeline_ref
from tests import helpers, scene_ref


def _ds():
    return RigidObjectDataset([RigidObject("box", mesh=procedural.textured_box(seed=1)),
                               RigidObject("ball", mesh=procedural.bumpy_sphere(n_seg=40, n_lat=21)),
                               RigidObject("tinted_box", mesh=procedural.textured_box(size=(0.06, 0.09, 0.04), seed=2,
                                                                                      with_vertex_colors=True))])


K1 = torch.tensor([[500.0, 0, 80], [0, 500, 60], [0, 0, 1]])


def _poses(n, seed, **kw):
    return torch.from_numpy(procedural.random_poses(n, seed, **kw)).float()


@pytest.mark.parametrize("flags", [0, 1, 2, 3])
def test_one_instance_scene_equals_single_render(flags):
    ds = _ds()
    rm = helpers.ref_meshes_from_dataset(ds)
    n = 6
    labels = [ds[i % 3].label for i in range(n)]
    TCO = _poses(n, 4, z_range=(0.15, 0.5), xy_range=0.03)
    TCO[3, 2, 3] = 0.07   # straddles the near plane
    TCO[4, 2, 3] = 0.01   # the eye inside the mesh
    K = K1.repeat(n, 1, 1)
    r = pipeline_ref.RefRenderer(rm, quantize8=bool(flags & 1), normals_gl_axes=bool(flags & 2))
    want = r.render(labels, TCO, K, None, (120, 160), render_depth=True, render_normals=True)
    got = scene_ref.render_scene(rm, [[l] for l in labels], TCO, K, (120, 160), flags=flags)
    for key in ("rgbs", "normals", "depths"):
        assert torch.equal(got[key], want[key]), key
    ids = got["inst_id"]
    assert set(ids.unique().tolist()) <= {-1, 0}
    assert ((got["depths"][:, 0] > 0) <= (ids == 0)).all()
    assert (ids == 0).sum() > 1000


def test_two_instances_composite_nearest_and_ties_to_instance_0():
    ds = _ds()
    rm = helpers.ref_meshes_from_dataset(ds)
    TCO = _poses(2, 8, z_range=(0.3, 0.3), xy_range=0.0)
    TCO[0, :3, 3] = torch.tensor([-0.04, 0.0, 0.3])
    TCO[1, :3, 3] = torch.tensor([0.03, 0.005, 0.6])  # well behind instance 0: no depth ties
    labels = ["tinted_box", "ball"]
    K = torch.tensor([[[250.0, 0, 80], [0, 250, 60], [0, 0, 1]]])
    single = [scene_ref.render_scene(rm, [[l]], T[None], K, (120, 160)) for l, T in zip(labels, TCO)]
    got = scene_ref.render_scene(rm, [labels], TCO, K, (120, 160))
    d = torch.stack([s["depths"][0, 0] for s in single])
    cov = torch.stack([s["inst_id"][0] >= 0 for s in single])
    d_eff = torch.where(cov & (d > 0), d, torch.full_like(d, float("inf")))
    win = torch.where(cov.any(0), d_eff.argmin(0), torch.full_like(d[0], -1, dtype=torch.long))
    assert torch.equal(got["inst_id"][0].long(), win)
    assert (win == 0).sum() > 2000 and (win == 1).sum() > 200  # both visible
    assert (cov.all(0) & (win == 0)).sum() > 50  # and instance 0 hides part of instance 1
    for key in ("rgbs", "normals", "depths"):
        for k in (0, 1):
            m = win == k
            assert torch.equal(got[key][0][:, m], single[k][key][0][:, m]), (key, k)
        assert got[key][0][:, win < 0].abs().sum() == 0

    # the same instance twice: every pixel goes to instance 0, with the one-instance pixels
    twice = scene_ref.render_scene(rm, [["tinted_box", "tinted_box"]], TCO[[0, 0]], K, (120, 160))
    assert torch.equal(twice["inst_id"], single[0]["inst_id"])
    for key in ("rgbs", "normals", "depths"):
        assert torch.equal(twice[key], single[0][key])


def test_oracle_invalid_instances_views_and_colour_override():
    ds = _ds()
    rm = helpers.ref_meshes_from_dataset(ds)
    TCO = _poses(4, 3, z_range=(0.3, 0.5), xy_range=0.02)
    TCO[1, 0, 0] = float("nan")
    K = K1.repeat(3, 1, 1)
    K[2, 0, 0] = float("nan")
    labels = [["box", "ball", "tinted_box"], [], ["ball"]]
    colors = torch.tensor([[-1.0, 0, 0], [0.2, 0.4, 0.6], [0.25, 0.5, 1.0], [0.1, 0.1, 0.1]])
    got = scene_ref.render_scene(rm, labels, TCO, K, (120, 160), colors=colors)
    assert got["rgbs"][1:].abs().sum() == 0 and (got["inst_id"][1:] == -1).all()
    assert set(got["inst_id"][0].unique().tolist()) <= {-1, 0, 2}  # the NaN pose draws nothing
    m2 = got["inst_id"][0] == 2
    assert m2.sum() > 100
    assert torch.equal(got["rgbs"][0][:, m2], torch.tensor([64 / 255, 128 / 255, 1.0]).float()[:, None].expand(3, int(m2.sum())))
    # an out-of-range label contributes nothing either
    bad = scene_ref.render_scene(rm, [["box", "ball"]], TCO[[0, 2]], K[:1], (120, 160), label_idx=[0, 7])
    one = scene_ref.render_scene(rm, [["box"]], TCO[:1], K[:1], (120, 160))
    assert torch.equal(bad["inst_id"], one["inst_id"]) and torch.equal(bad["rgbs"], one["rgbs"])
    with pytest.raises(RuntimeError):
        scene_ref.render_scene(rm, [["box"]], TCO[:1], K[:1], (120, 160), flags=4)


def test_pose_composition_matches_numpy():
    rs = np.random.RandomState(0)
    for _ in range(20):
        TWC = example.transform_from_quat_trans(rs.randn(4), rs.randn(3))
        TWO = example.transform_from_quat_trans(rs.randn(4), rs.randn(3))
        s = float(rs.uniform(0.001, 2.0))
        want = (np.linalg.inv(TWC) @ TWO @ np.diag([s, s, s, 1.0])).astype(np.float32)
        got = compose_TCO(TWC, TWO, s)
        assert got.dtype == np.float32 and np.array_equal(got, want)


def test_scene_renderer_refusals():
    ds = _ds()
    r = Panda3dSceneRenderer(ds)
    cam = Panda3dCameraData(K=K1.double().numpy(), resolution=(120, 160))
    obj = Panda3dObjectData("box", TWO=np.eye(4))
    white = [Panda3dLightData("ambient", (1.0, 1.0, 1.0, 1.0))]
    cases = [
        ([obj], [cam], make_scene_lights()),
        ([obj], [cam], [Panda3dLightData("ambient", (0.5, 0.5, 0.5, 1.0))]),
        ([obj], [cam], white + white),
        ([obj], [cam], [Panda3dLightData("point", (1.0, 1.0, 1.0, 1.0))]),
        ([Panda3dObjectData("box", positioning_function=lambda *a: None)], [cam], white),
        ([Panda3dObjectData("box", material=object())], [cam], white),
        ([Panda3dObjectData("box", remove_mesh_material=True)], [cam], white),
        ([Panda3dObjectData("box", color=(1.0, 0.0, 0.0, 0.5))], [cam], white),
        ([obj], [Panda3dCameraData(K=cam.K, resolution=(120, 160), z_near=0.01)], white),
        ([obj], [Panda3dCameraData(K=cam.K, resolution=(120, 160), z_far=100)], white),
        ([obj], [Panda3dCameraData(K=cam.K, resolution=(120, 160), positioning_function=lambda *a: None)], white),
    ]
    for objs, cams, lights in cases:
        with pytest.raises(NotImplementedError):
            r.render_scene(objs, cams, lights)
    with pytest.raises(AssertionError):
        r.render_scene([obj], [cam], white, render_depth=False, render_binary_mask=True)
    assert CameraRenderingData(rgb=np.zeros((2, 2, 3), np.uint8)).binary_mask is None


def test_mesh_and_contour_overlays_on_hand_made_masks():
    h, w = 9, 12
    img = np.full((h, w, 3), 100, np.uint8)
    img[0, 0] = (10, 20, 30)
    render = np.zeros((h, w, 3), np.uint8)
    render[2:7, 3:9] = (200, 0, 0)
    render[4, 5] = (0, 0, 1)  # any channel > 0 is in the mask
    mask = example.get_mask_from_rgb(render)
    assert mask.sum() == 30 and mask[4, 5]
    ov = example.make_mesh_overlay(img, render)
    assert ov.dtype == np.uint8 and ov.shape == img.shape
    assert tuple(ov[0, 0]) == (int(10 * 0.6 + 102), int(20 * 0.6 + 102), int(30 * 0.6 + 102))
    assert tuple(ov[1, 1]) == (int(100 * 0.6 + 102),) * 3
    assert tuple(ov[2, 3]) == (int(200 * 0.8 + 51), 51, 51) and tuple(ov[4, 5]) == (51, 51, int(0.8 + 51))

    no_dilate = example.make_contour_overlay(img, render, dilate_iterations=0)
    ring = np.zeros((h, w), bool)
    ring[2:7, 3:9] = True
    ring[3:6, 4:8] = False
    assert np.array_equal(no_dilate["contour"], ring)
    assert (no_dilate["img"][ring] == (0, 255, 0)).all() and (no_dilate["img"][~ring] == img[~ring]).all()
    one = example.make_contour_overlay(img, render, color=(1, 2, 3), dilate_iterations=1)
    band = np.zeros((h, w), bool)
    band[1:8, 2:10] = True
    band[4, 5:7] = False  # the ring dilated by one pixel leaves only the centre of the 3x4 hole
    assert np.array_equal(one["contour"], band)
    assert (one["img"][band] == (1, 2, 3)).all()
    # a mask touching the image border: the border itself is not an edge
    full = np.ones((h, w, 3), np.uint8)
    assert not example.make_contour_overlay(img, full, dilate_iterations=0)["contour"].any()
