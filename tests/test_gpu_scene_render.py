"""The multi-object scene renderer (mpx_raster_render_scene, Panda3dSceneRenderer) on the GPU: bit-exact against the
single-object rasteriser for one-instance scenes and against the CPU scene contract (tests/scene_ref.c) for every
scene; refusals; the reference-style host API; the example's --vis-outputs."""
import numpy as np
import pytest
import torch

from megapose6d_b200 import _abi, procedural
from megapose6d_b200.meshes import TriMesh
from megapose6d_b200.object_dataset import RigidObject, RigidObjectDataset
from megapose6d_b200.renderer import BatchRenderer, Panda3dLightData
from megapose6d_b200.scene_renderer import Panda3dCameraData, Panda3dObjectData, Panda3dSceneRenderer
from tests import helpers, scene_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _poses(n, seed, **kw):
    return torch.from_numpy(procedural.random_poses(n, seed, **kw)).float()


def _box_mesh():
    """12 triangles: every one takes the CTA-wide path of the coverage kernel at these distances."""
    v = np.array([[x, y, z] for x in (-.05, .05) for y in (-.04, .04) for z in (-.03, .03)], dtype=np.float64)
    f = np.array([[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1], [2, 3, 7], [2, 7, 6], [0, 2, 6],
                  [0, 6, 4], [1, 5, 7], [1, 7, 3]], dtype=np.int32)
    return TriMesh(v, f, None, np.random.RandomState(0).rand(8, 3).round(2))


@pytest.fixture(scope="module")
def mixed():
    """Textured boxes, a textured box modulated by vertex colours, an untextured sphere and an untextured plain box."""
    ds = RigidObjectDataset([RigidObject("box", mesh=procedural.textured_box(seed=1)),
                             RigidObject("ball", mesh=procedural.bumpy_sphere(n_seg=40, n_lat=21)),
                             RigidObject("tinted_box", mesh=procedural.textured_box(size=(0.06, 0.09, 0.04), seed=2,
                                                                                    with_vertex_colors=True)),
                             RigidObject("plain_box", mesh=_box_mesh())])
    return ds, helpers.ref_meshes_from_dataset(ds), Panda3dSceneRenderer(ds)


@pytest.fixture(scope="module")
def ycbv():
    """The 21 objects and ground-truth poses of workloads.scenes.ycbv_scene(21) (10k triangles each), at 480x640."""
    ds, _, K = helpers.make_scene(21, seed=31)
    TCO = _poses(21, 32, z_range=(0.5, 1.0), xy_range=0.15)
    return ds, helpers.ref_meshes_from_dataset(ds), Panda3dSceneRenderer(ds), K[0], TCO


def _scene_both(r, rm, labels_per_view, TCO, K, res, colors=None):
    out = r.render_scene_tensors(labels_per_view, TCO.cuda(), K.cuda(), res, colors=None if colors is None else colors.cuda())
    ref = scene_ref.render_scene(rm, labels_per_view, TCO, K, res, flags=r.flags, colors=colors)
    return out, ref


def _assert_same_scene(out, ref, what=""):
    for name, got, want in (("rgb", out.rgbs, ref["rgbs"]), ("normals", out.normals, ref["normals"]),
                            ("depth", out.depths, ref["depths"]), ("inst_id", out.inst_id, ref["inst_id"])):
        got = got.cpu()
        assert torch.equal(got, want), f"{what}{name}: {(got != want).sum().item()} differing values"


@pytest.mark.parametrize("flags", [1, 0, 3, 2])
def test_one_instance_scenes_equal_raster_render(mixed, flags):
    """One instance per view: mpx_raster_render_scene renders exactly what mpx_raster_render renders."""
    ds, rm, r = mixed
    n = 10
    labels = [ds[i % 4].label for i in range(n)]
    TCO = _poses(n, 41, z_range=(0.15, 0.6), xy_range=0.03)
    TCO[2, 2, 3] = 0.06   # straddles the near plane
    TCO[5, 2, 3] = 0.01   # the eye inside the mesh
    TCO[7, 2, 3] = 0.1    # screen-filling triangles
    K = torch.tensor([[600.0, 0, 160], [0, 600, 120], [0, 0, 1]]).repeat(n, 1, 1)
    br = BatchRenderer(object_dataset=ds, quantize8=bool(flags & 1), normals_gl_axes=bool(flags & 2))
    single = br.render(labels, TCO.cuda(), K.cuda(), None, (240, 320), render_depth=True, render_normals=True)
    r.flags = flags
    try:
        out = r.render_scene_tensors([[l] for l in labels], TCO.cuda(), K.cuda(), (240, 320))
    finally:
        r.flags = 1
    assert torch.equal(out.rgbs, single.rgbs) and torch.equal(out.normals, single.normals)
    assert torch.equal(out.depths, single.depths)
    ids = out.inst_id
    assert set(ids.unique().tolist()) == {-1, 0} and ((out.depths[:, 0] > 0) <= (ids == 0)).all()


def test_ycbv_21_objects_vs_oracle(ycbv):
    """21 objects of 10k triangles in one 480x640 frame, interpenetrating and occluding."""
    ds, rm, r, K, TCO = ycbv
    labels = [ds[i].label for i in range(21)]
    out, ref = _scene_both(r, rm, [labels], TCO, K[None], (480, 640))
    _assert_same_scene(out, ref)
    ids = out.inst_id[0]
    assert len(ids.unique()) >= 15  # most objects are visible


def test_interpenetrating_and_repeated_instances_vs_oracle(mixed, ycbv):
    """3 to 12 instances per view, the same label several times, textured / untextured / box meshes, poses that put
    objects through each other; 480x640 and 103x150."""
    ds, rm, r = mixed
    rs = np.random.RandomState(5)
    counts = [3, 5, 8, 12, 4]
    labels = [[ds[int(rs.randint(4))].label for _ in range(c)] for c in counts]
    labels[1] = ["plain_box"] * 5
    n_inst = sum(counts)
    TCO = _poses(n_inst, 17, z_range=(0.25, 0.45), xy_range=0.04)  # close together: they intersect
    for res, f in (((480, 640), 900.0), ((103, 150), 210.0)):
        h, w = res
        K = torch.tensor([[f, 0, w / 2 - 0.3], [0, f, h / 2 + 0.2], [0, 0, 1]]).repeat(len(counts), 1, 1)
        out, ref = _scene_both(r, rm, labels, TCO, K, res)
        _assert_same_scene(out, ref, f"{res}: ")
        for v, c in enumerate(counts):
            assert len(out.inst_id[v].unique()) >= min(c, 3)


def test_invalid_instances_nan_K_and_empty_views(mixed):
    ds, rm, r = mixed
    labels = [["box", "ball", "tinted_box"], [], ["ball", "plain_box"], ["box"]]
    TCO = _poses(6, 23, z_range=(0.3, 0.5), xy_range=0.02)
    TCO[1, 1, 2] = float("nan")   # the ball of view 0 draws nothing
    K = torch.tensor([[500.0, 0, 80], [0, 500, 60], [0, 0, 1]]).repeat(4, 1, 1)
    K[3, 1, 2] = float("inf")      # view 3 is black
    out, ref = _scene_both(r, rm, labels, TCO, K, (120, 160))
    _assert_same_scene(out, ref)
    assert 1 not in out.inst_id[0].unique().tolist() and (out.inst_id[0] >= 0).sum() > 100
    for v in (1, 3):
        assert (out.inst_id[v] == -1).all() and out.rgbs[v].abs().sum() == 0 and out.depths[v].abs().sum() == 0


def test_more_views_than_one_chunk(mixed):
    """Views are processed in chunks of 2 x SMs, each with its own pass over the workspace."""
    ds, rm, r = mixed
    n = 2 * _abi.lib().mpx_sm_count() + 7
    rs = np.random.RandomState(3)
    labels = [[ds[int(rs.randint(4))].label for _ in range(1 + v % 3)] for v in range(n)]
    n_inst = sum(len(l) for l in labels)
    TCO = _poses(n_inst, 29, z_range=(0.25, 0.6), xy_range=0.03)
    K = torch.tensor([[300.0, 0, 40], [0, 300, 32], [0, 0, 1]]).repeat(n, 1, 1)
    out, ref = _scene_both(r, rm, labels, TCO, K, (64, 80))
    _assert_same_scene(out, ref)
    assert (out.inst_id[-5:] >= 0).any()


def test_composite_of_objects_separated_in_depth(ycbv):
    """Objects at distinct depths: each pixel is the single-object render of the nearest object covering it."""
    ds, rm, r, K, _ = ycbv
    n = 6
    labels = [ds[i].label for i in range(n)]
    TCO = _poses(n, 37, z_range=(0.5, 0.5), xy_range=0.05)
    TCO[:, 2, 3] = torch.tensor([0.45, 0.6, 0.75, 0.9, 1.05, 1.2])  # 15 cm apart: more than any object's depth
    out = r.render_scene_tensors([labels], TCO.cuda(), K[None].cuda(), (480, 640))
    single = BatchRenderer(object_dataset=ds).render(labels, TCO.cuda(), K[None].repeat(n, 1, 1).cuda(), None, (480, 640),
                                                     render_depth=True, render_normals=True)
    d = single.depths[:, 0]
    d_eff = torch.where(d > 0, d, torch.full_like(d, float("inf")))
    win = torch.where((d > 0).any(0), d_eff.argmin(0), torch.full_like(d[0], -1, dtype=torch.long))
    covered = win >= 0
    assert torch.equal(out.inst_id[0][covered].long(), win[covered])
    rows, cols = torch.arange(480, device=DEV)[:, None], torch.arange(640, device=DEV)[None, :]
    for got, want in ((out.rgbs, single.rgbs), (out.normals, single.normals)):
        pick = want[win.clamp(min=0), :, rows, cols].permute(2, 0, 1)  # [3,h,w]: the winner's pixel
        assert torch.equal(got[0][:, covered], pick[:, covered])
    assert torch.equal(out.depths[0, 0][covered], d.gather(0, win.clamp(min=0)[None])[0][covered])
    assert len(win.unique()) >= 5


def test_colour_override_and_ties(mixed):
    ds, rm, r = mixed
    TCO = _poses(3, 13, z_range=(0.3, 0.4), xy_range=0.03)
    K = torch.tensor([[[500.0, 0, 80], [0, 500, 60], [0, 0, 1]]])
    colors = torch.tensor([[0.25, 0.5, 1.0], [-1.0, 0.0, 0.0], [0.1, 0.9, 0.3]])
    out, ref = _scene_both(r, rm, [["box", "ball", "tinted_box"]], TCO, K, (120, 160), colors=colors)
    _assert_same_scene(out, ref)
    m0 = out.inst_id[0] == 0
    assert m0.sum() > 50
    assert torch.equal(out.rgbs[0][:, m0], torch.tensor([64 / 255, 128 / 255, 1.0], device=DEV)[:, None].expand(3, int(m0.sum())))
    # two instances at the same pose: instance 0 everywhere, with the one-instance pixels
    one = r.render_scene_tensors([["tinted_box"]], TCO[:1].cuda(), K.cuda(), (120, 160))
    two = r.render_scene_tensors([["tinted_box", "tinted_box"]], TCO[[0, 0]].cuda(), K.cuda(), (120, 160))
    assert torch.equal(two.inst_id, one.inst_id) and (one.inst_id >= 0).sum() > 100
    for a, b in ((two.rgbs, one.rgbs), (two.normals, one.normals), (two.depths, one.depths)):
        assert torch.equal(a, b)


def test_refusals_launch_nothing(mixed):
    ds, rm, r = mixed
    lib = _abi.lib()
    h, w = 64, 80
    need = lib.mpx_raster_workspace_bytes(h, w)
    ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    n_inst = 1025
    off = torch.tensor([0, n_inst], dtype=torch.int32, device=DEV)
    lab = torch.zeros(n_inst, dtype=torch.int32, device=DEV)
    T = _poses(n_inst, 1).cuda()
    K = torch.tensor([[[300.0, 0, 40], [0, 300, 32], [0, 0, 1]]], device=DEV)
    rgb = torch.empty(1, 3, h, w, device=DEV)
    handle = r.mesh_db.handle
    torch.cuda.synchronize()
    before = lib.mpx_launch_count()

    def call(n_views, n, flags, ws_bytes):
        return lib.mpx_raster_render_scene(handle, n_views, n, _abi.ptr(off), _abi.ptr(lab), _abi.ptr(T), None,
                                           _abi.ptr(K), h, w, flags, _abi.ptr(rgb), None, None, None, _abi.ptr(ws),
                                           ws_bytes, _abi.stream_ptr())

    assert call(1, 2, 1 | 4, need) != 0 and b"point lights" in lib.mpx_last_error()
    assert call(1, n_inst, 1, need) != 0 and b"instances" in lib.mpx_last_error()
    assert call(1, 2, 1, need - 1) != 0 and b"workspace" in lib.mpx_last_error()
    assert call(-1, 2, 1, need) != 0
    assert lib.mpx_launch_count() == before
    off[1] = 2
    assert call(1, 2, 1, need) == 0 and lib.mpx_launch_count() == before + 2
    with pytest.raises(ValueError):
        r.render_scene_tensors([["box"] * 1025], T.cuda(), K, (h, w))


def test_render_scene_host_api_two_resolutions(mixed):
    """Panda3dSceneRenderer.render_scene: one CameraRenderingData per camera, in the reference's host types."""
    ds, rm, r = mixed
    TWC = np.eye(4)
    TWC[:3, 3] = [0.01, -0.02, -0.05]
    objects = [Panda3dObjectData("box", TWO=procedural.random_poses(1, 3, z_range=(0.3, 0.3))[0].astype(np.float64)),
               Panda3dObjectData("ball", TWO=procedural.random_poses(1, 4, z_range=(0.35, 0.35))[0].astype(np.float64),
                                 color=(0.2, 0.4, 0.6, 1.0)),
               Panda3dObjectData("tinted_box", TWO=procedural.random_poses(1, 5, z_range=(0.4, 0.4))[0].astype(np.float64),
                                 scale=1.5)]
    cams = [Panda3dCameraData(K=np.array([[500.0, 0, 80], [0, 500, 60], [0, 0, 1]]), resolution=(120, 160)),
            Panda3dCameraData(K=np.array([[700.0, 0, 112.5], [0, 700, 75.5], [0, 0, 1]]), resolution=(151, 225), TWC=TWC),
            Panda3dCameraData(K=np.array([[450.0, 0, 81], [0, 450, 59], [0, 0, 1]]), resolution=(120, 160), TWC=TWC)]
    lights = [Panda3dLightData("ambient", (1.0, 1.0, 1.0, 1.0))]
    outs = r.render_scene(objects, cams, lights, render_depth=True, render_binary_mask=True, render_normals=True)
    assert len(outs) == 3
    for cam, o in zip(cams, outs):
        h, w = cam.resolution
        assert o.rgb.shape == (h, w, 3) and o.rgb.dtype == np.uint8
        assert o.normals.shape == (h, w, 3) and o.normals.dtype == np.uint8
        assert o.depth.shape == (h, w, 1) and o.depth.dtype == np.float32
        assert o.binary_mask.shape == (h, w) and o.binary_mask.dtype == np.bool_
        assert np.array_equal(o.binary_mask, o.depth[..., 0] > 0) and o.binary_mask.sum() > 100
        # the oracle on the same composed poses
        TCO = torch.from_numpy(np.stack([np.linalg.inv(cam.TWC) @ ob.TWO @ np.diag([ob.scale] * 3 + [1.0])
                                         for ob in objects]).astype(np.float32))
        colors = torch.tensor([[-1.0, 0, 0], [0.2, 0.4, 0.6], [-1.0, 0, 0]])
        ref = scene_ref.render_scene(rm, [[ob.label for ob in objects]], TCO, torch.from_numpy(cam.K).float()[None],
                                     (h, w), flags=1, colors=colors)
        assert np.array_equal(o.rgb, (ref["rgbs"][0] * 255).round().to(torch.uint8).permute(1, 2, 0).numpy())
        assert np.array_equal(o.normals, (ref["normals"][0] * 255).round().to(torch.uint8).permute(1, 2, 0).numpy())
        assert np.array_equal(o.depth, ref["depths"][0].permute(1, 2, 0).numpy())
    plain = r.render_scene(objects, cams[:1], lights)[0]
    assert plain.depth is None and plain.normals is None and plain.binary_mask is None
    assert np.array_equal(plain.rgb, outs[0].rgb)


def test_example_vis_outputs(tmp_path):
    """`example.py --vis-outputs` writes the three visualisations; the mesh overlay is the overlay formula applied to the
    scene render of the estimated poses."""
    from PIL import Image

    from megapose6d_b200 import example, load_model
    from tests.test_example import _make_example_dir

    rgb = (np.random.RandomState(2).rand(480, 640, 3) * 255).astype(np.uint8)
    _make_example_dir(tmp_path, rgb, dense=True)
    models = tmp_path / "models"
    load_model.write_run(models, "coarse-rgb-906902141", helpers.make_state_dict(helpers.COARSE_CFG, 1))
    load_model.write_run(models, "refiner-rgb-653307694", helpers.make_state_dict(helpers.REFINER_CFG, 2))
    example.main([str(tmp_path), "--model", "megapose-1.0-RGB", "--models-root", str(models), "--vis-outputs"])
    vis = tmp_path / "visualizations"
    ims = {}
    for name, size in (("mesh_overlay", (640, 480)), ("contour_overlay", (640, 480)), ("all_results", (3 * 640, 480))):
        with Image.open(vis / f"{name}.png") as im:
            assert im.size == size and im.mode == "RGB"
            ims[name] = np.asarray(im)
    objs = example.load_object_data(tmp_path / "outputs" / "object_data.json")
    _, _, cam = example.load_observation(tmp_path)
    rendered = example.render_object_data(tmp_path, objs, cam.resolution, cam.K)
    assert example.get_mask_from_rgb(rendered).sum() > 100
    assert np.array_equal(ims["mesh_overlay"], example.make_mesh_overlay(rgb, rendered))
    assert np.array_equal(ims["contour_overlay"], example.make_contour_overlay(rgb, rendered)["img"])
    assert np.array_equal(ims["all_results"], np.concatenate([rgb, ims["contour_overlay"], ims["mesh_overlay"]], axis=1))
    # --vis-only re-renders from the saved poses without running the estimator
    (vis / "mesh_overlay.png").unlink()
    example.main([str(tmp_path), "--vis-only"])
    with Image.open(vis / "mesh_overlay.png") as im:
        assert np.array_equal(np.asarray(im), ims["mesh_overlay"])
