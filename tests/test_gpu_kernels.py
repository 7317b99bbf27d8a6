"""GPU parity tests of the individual kernels (called through the C ABI) against the CPU oracle."""
import numpy as np
import pytest
import torch

from megapose6d_b200 import _abi, lib3d, procedural
from megapose6d_b200.meshes import MeshDataBase, TriMesh
from megapose6d_b200.object_dataset import RigidObject, RigidObjectDataset
from megapose6d_b200.renderer import BatchRenderer
from oracle import lib3d_ref as L
from oracle import pipeline_ref
from tests import helpers

pytestmark = pytest.mark.gpu
DEV = "cuda"
ACT = _abi.act_dtype() if torch.cuda.is_available() else torch.float16  # the library's 16-bit type


def _poses(n, seed, **kw):
    return torch.from_numpy(procedural.random_poses(n, seed, **kw)).float()


@pytest.fixture(scope="module")
def scene():
    ds, images, K = helpers.make_scene(3, seed=1, with_depth=True)
    db = MeshDataBase.from_object_ds(ds).batched().cuda()
    return ds, images, K, db, helpers.ref_meshes_from_dataset(ds)


def test_pose_init_and_normalize(scene):
    ds, images, K, db, rm = scene
    n = 64
    g = torch.Generator().manual_seed(0)
    labels = [ds[i % 3].label for i in range(n)]
    R = L.compute_rotation_matrix_from_ortho6d(torch.randn(n, 6, generator=g))
    bb = torch.tensor([[384.0, 234, 522, 455]]).repeat(n, 1) + 3 * torch.randn(n, 4, generator=g)
    Kn = K.repeat(n, 1, 1)
    want = L.TCO_init_from_boxes_autodepth_with_R(bb, rm.select_points(labels), Kn, R)
    got = lib3d.TCO_init_from_boxes_autodepth_with_R(bb.cuda(), db.points, db.label_ids(labels, DEV), Kn.cuda(), R.cuda())
    assert torch.allclose(got.cpu(), want, rtol=1e-5, atol=1e-6)
    noisy = want + 0.01 * torch.randn(n, 4, 4, generator=g)
    assert torch.allclose(lib3d.normalize_T(noisy.cuda()).cpu(), L.normalize_T(noisy), rtol=1e-5, atol=1e-6)
    assert lib3d.normalize_T(torch.empty(0, 4, 4, device=DEV)).shape == (0, 4, 4)


def test_crop_geometry(scene):
    ds, images, K, db, rm = scene
    n = 48
    labels = [ds[i % 3].label for i in range(n)]
    TCO = _poses(n, 3)
    TCO[5, 2, 3] = 0.05  # partly behind the z_min clamp
    Kn = K.repeat(n, 1, 1)
    tCR = TCO[:, :3, 3] + 0.003
    for npts in (2000, 200):
        pts = rm.sample_points(labels, npts)
        uv = L.project_points_robust(pts, Kn, TCO)
        br = L.boxes_from_uv(uv)
        bc, _ = L.deepim_crops_robust(torch.zeros(1, 3, 480, 640).expand(n, -1, -1, -1), br, Kn, TCO, tCR, pts, (240, 320), return_crops=False)
        Kc = L.get_K_crop_resize(Kn, bc, (240, 320))
        g_br, g_bc, g_Kc = lib3d.crop_geometry(db.point_subset(npts), db.label_ids(labels, DEV), TCO.cuda(), Kn.cuda(),
                                                tCR.cuda(), (480, 640), (240, 320))
        assert torch.allclose(g_br.cpu(), br, rtol=1e-5, atol=2e-3)
        assert torch.allclose(g_bc.cpu(), bc, rtol=1e-5, atol=4e-3)
        assert torch.allclose(g_Kc.cpu(), Kc, rtol=2e-5, atol=2e-3)


def test_multiview_and_pose_update():
    n = 33
    TCO = _poses(n, 7)
    tCR = TCO[:, :3, 3] + torch.tensor([0.002, -0.001, 0.004])
    want = L.make_TCO_multiview(TCO, tCR, "TCO+front_3views", 4)
    got = lib3d.make_TCO_multiview(TCO.cuda(), tCR.cuda(), "TCO+front_3views", 4).cpu()
    assert got.shape == (n, 4, 4, 4)
    assert torch.allclose(got, want, rtol=1e-5, atol=2e-6)
    # non-finite pose -> identity fallback (multiview.py:44-46) must not crash
    bad = TCO.clone()
    bad[0, 0, 0] = float("nan")
    lib3d.make_TCO_multiview(bad.cuda(), tCR.cuda(), "TCO+front_3views", 4)
    torch.cuda.synchronize()
    g = torch.Generator().manual_seed(1)
    out9 = torch.randn(n, 9, generator=g)
    out9[:, 8] = 1.0 + 0.05 * out9[:, 8]
    Kc = torch.tensor([[900.0, 0, 160], [0, 900, 120], [0, 0, 1]]).repeat(n, 1, 1)
    assert torch.allclose(lib3d.update_pose(TCO.cuda(), Kc.cuda(), out9.cuda(), tCR.cuda()).cpu(),
                          L.update_pose(TCO, Kc, out9, tCR), rtol=1e-5, atol=1e-6)


def test_topk():
    g = torch.Generator().manual_seed(3)
    logits = torch.randn(5, 576, generator=g)
    logits[2, 10] = logits[2, 400] = 9.0  # tie -> lower index first
    idx = lib3d.topk_per_group(logits.cuda(), 5).cpu()
    want = torch.argsort(logits, dim=1, descending=True, stable=True)[:, :5]
    assert torch.equal(idx.long(), want)
    assert idx[2, 0] == 10 and idx[2, 1] == 400


def test_roi_align_matches_torchvision(scene):
    ds, images, K, db, rm = scene
    boxes = torch.tensor([[100.0, 80, 420, 320], [-40, -30, 200, 150], [500, 380, 700, 530], [300, 200, 300.5, 200.2],
                          [0, 0, 640, 480], [610.3, 440.7, 655.1, 490.2],
                          # minification: bins of 2.8 / 3.3 px and one mixed case take the uncollapsed path
                          [-100, -100, 800, 700], [10, -200, 630, 700], [-0.4, 0.3, 820.2, 615.9]])
    n = boxes.shape[0]
    nhwc4 = lib3d.image_to_nhwc4(images.cuda())
    for c in (3, 4):
        img = images[:, :c]
        boxes5 = torch.cat((torch.zeros(n, 1), boxes), dim=1)
        want = L.crop_images(img, boxes5, (240, 320))
        got = lib3d.crop_images(nhwc4, boxes.cuda(), torch.zeros(n, dtype=torch.int32, device=DEV), c, (240, 320)).cpu()
        assert torch.allclose(got[:, :3], want[:, :3], rtol=1e-5, atol=2e-5), (c, (got - want).abs().max())  # fma contraction moves sample coordinates by an ulp
        if c == 4:  # per-pixel random depth (steep gradients) and the 0.99 validity threshold on isolated pixels
            assert ((got[:, 3] - want[:, 3]).abs() > 2e-4).float().mean() < 1e-3
    # scalar restatement on a small case (independent of torchvision)
    small = images[0, :3, :40, :48].contiguous()
    got = lib3d.crop_images(lib3d.image_to_nhwc4(small.unsqueeze(0).cuda()), torch.tensor([[-3.0, 2.5, 30.2, 41.0]], device=DEV),
                            None, 3, (6, 8)).cpu()[0]
    want = torch.from_numpy(L.roi_align_scalar(small.numpy(), [-3.0, 2.5, 30.2, 41.0], 6, 8))
    assert torch.allclose(got, want, rtol=1e-5, atol=2e-6)


def _render_both(ds, rm, labels, TCO, K, res, depth=True):
    r = BatchRenderer(object_dataset=ds)
    out = r.render(labels, TCO.cuda(), K.cuda(), None, res, render_depth=depth, render_normals=True)
    ref = pipeline_ref.RefRenderer(rm).render(labels, TCO, K, None, res, render_depth=depth, render_normals=True)
    return out, ref


@pytest.fixture(params=[7, 2, 0], ids=["scatter", "strips", "strips_read_then_atomic"])
def raster_mode(request):
    """Small batches have two implementations (include/mpx.h mpx_raster_set_mode): triangles scattered over many CTAs
    + resolve kernel (default), or one CTA per (view, row strip).  Both must match the oracle bit for bit."""
    from megapose6d_b200 import _abi
    _abi.lib().mpx_raster_set_mode(request.param)
    yield request.param
    _abi.lib().mpx_raster_set_mode(7)


@pytest.fixture(params=[7, 3], ids=["tiled", "untiled"])
def big_batch_mode(request):
    """Batches that fill the GPU: the tiled kernel (triangles binned into screen strips, z-test in shared memory; default)
    or one CTA per view with a global visibility buffer.  Same pixels, bit for bit."""
    from megapose6d_b200 import _abi
    _abi.lib().mpx_raster_set_mode(request.param)
    yield request.param
    _abi.lib().mpx_raster_set_mode(7)


def _assert_same_render(out, ref, what=""):
    for name, got, want in (("rgb", out.rgbs, ref["rgbs"]), ("normals", out.normals, ref["normals"]),
                            ("depth", out.depths, ref["depths"])):
        got = got.cpu()
        mism = (got != want).flatten(1).any(dim=0).sum().item() if got.numel() else 0
        assert torch.equal(got, want), f"{what}{name}: {mism} differing pixel positions, max |d|={(got - want).abs().max()}"


def test_raster_big_batch_bit_exact_vs_oracle(scene, big_batch_mode):
    """40 views of 10k-triangle meshes at 240x320: ten strips per view, several CTAs per view (strip groups), triangles
    that straddle strips, a view at the near plane, one mostly outside the frustum, one with an invalid pose."""
    ds, images, K, db, rm = scene
    n = 40
    labels = [ds[i % 3].label for i in range(n)]
    TCO = _poses(n, 121, z_range=(0.25, 0.9))
    TCO[3, 2, 3] = 0.12
    TCO[4, 0, 3] = 0.35
    TCO[7, 1, 1] = float("nan")
    TCO[9, 2, 3] = 0.06   # straddles the near plane: clipped per sample, screen-filling triangles
    TCO[11, 2, 3] = 0.02  # the eye inside the mesh: vertices behind the eye plane (dropped), clamped projections
    Kc = torch.tensor([[1500.0, 0, 160], [0, 1500, 120], [0, 0, 1]]).repeat(n, 1, 1)
    Kc[5] = torch.tensor([[300.0, 0, 150.3], [0, 310, 118.9], [0, 0, 1]])
    out, ref = _render_both(ds, rm, labels, TCO, Kc, (240, 320))
    _assert_same_render(out, ref)
    assert (out.depths > 0).float().mean() > 0.05 and out.rgbs[7].abs().sum() == 0


def test_raster_big_batch_low_poly_and_odd_size(big_batch_mode):
    """Boxes of 12 triangles (every triangle is 'large': the CTA-wide path of each kernel) next to a sphere, at a
    resolution that does not divide into equal strips; more views than CTA slots so that the persistent loop runs."""
    ds = RigidObjectDataset([RigidObject("box", mesh=procedural.textured_box(seed=1)),
                             RigidObject("ball", mesh=procedural.bumpy_sphere(n_seg=40, n_lat=21))])
    rm = helpers.ref_meshes_from_dataset(ds)
    n = 2 * _abi.lib().mpx_sm_count() + 5
    labels = [ds[i % 2].label for i in range(n)]
    TCO = _poses(n, 9, z_range=(0.2, 0.6))
    Kc = torch.tensor([[420.0, 0, 75], [0, 420, 50], [0, 0, 1]]).repeat(n, 1, 1)
    out, ref = _render_both(ds, rm, labels, TCO, Kc, (103, 150))
    _assert_same_render(out, ref)


def test_raster_bit_exact_vs_oracle(scene, raster_mode):
    ds, images, K, db, rm = scene
    n = 12
    labels = [ds[i % 3].label for i in range(n)]
    TCO = _poses(n, 21, z_range=(0.25, 0.9))
    TCO[3, 2, 3] = 0.12   # very close: large triangles, samples clipped at the near plane
    TCO[4, 0, 3] = 0.35   # mostly outside the frustum
    TCO[6, 2, 3] = 0.05   # straddles the near plane
    TCO[8, 2, 3] = 0.015  # the eye inside the mesh
    Kc = torch.tensor([[1500.0, 0, 160], [0, 1500, 120], [0, 0, 1]]).repeat(n, 1, 1)
    Kc[5] = torch.tensor([[300.0, 0, 150.3], [0, 310, 118.9], [0, 0, 1]])
    out, ref = _render_both(ds, rm, labels, TCO, Kc, (240, 320))
    for name, got, want in (("rgb", out.rgbs, ref["rgbs"]), ("normals", out.normals, ref["normals"]),
                            ("depth", out.depths, ref["depths"])):
        got = got.cpu()
        mism = (got != want).flatten(1).any(dim=0).sum().item() if got.numel() else 0
        assert torch.equal(got, want), f"{name}: {mism} differing pixel positions, max |d|={(got - want).abs().max()}"
    assert (out.depths > 0).float().mean() > 0.05  # the views are not empty


def test_raster_invalid_pose_and_big_triangles(raster_mode):
    # a 12-triangle box: every triangle takes the CTA-wide path; plus a non-finite pose -> black view
    v = np.array([[x, y, z] for x in (-.05, .05) for y in (-.04, .04) for z in (-.03, .03)], dtype=np.float64)
    f = np.array([[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1], [2, 3, 7], [2, 7, 6], [0, 2, 6], [0, 6, 4],
                  [1, 5, 7], [1, 7, 3]], dtype=np.int32)
    col = np.random.RandomState(0).rand(8, 3).round(2)
    ds = RigidObjectDataset([RigidObject("box", mesh=TriMesh(v, f, None, col))])
    rm = helpers.ref_meshes_from_dataset(ds)
    TCO = _poses(4, 2, z_range=(0.3, 0.5))
    TCO[2, 1, 1] = float("inf")
    Kc = torch.tensor([[600.0, 0, 160], [0, 600, 120], [0, 0, 1]]).repeat(4, 1, 1)
    out, ref = _render_both(ds, rm, ["box"] * 4, TCO, Kc, (240, 320))
    assert torch.equal(out.rgbs.cpu(), ref["rgbs"]) and torch.equal(out.depths.cpu(), ref["depths"])
    assert torch.equal(out.normals.cpu(), ref["normals"])
    assert out.rgbs[2].abs().sum() == 0 and out.depths[2].abs().sum() == 0
    assert (out.depths[0] > 0).float().mean() > 0.02


def test_raster_empty_batch():
    ds = procedural.make_object_dataset(1)
    r = BatchRenderer(object_dataset=ds)
    out = r.render([], torch.empty(0, 4, 4, device=DEV), torch.empty(0, 3, 3, device=DEV), None, (240, 320), render_normals=True)
    assert out.rgbs.shape == (0, 3, 240, 320)


def test_raster_many_views_persistent_loop(scene):
    """More views than resident CTAs: one view per CTA, persistent loop over the rest (no row strips)."""
    ds, images, K, db, rm = scene
    n = 2 * _abi.lib().mpx_sm_count() * 2 + 37
    labels = [ds[i % 3].label for i in range(n)]
    TCO = _poses(n, 77, z_range=(0.3, 0.9))
    Kc = torch.tensor([[400.0, 0, 40], [0, 400, 32], [0, 0, 1]]).repeat(n, 1, 1)
    out, ref = _render_both(ds, rm, labels, TCO, Kc, (64, 80))
    assert torch.equal(out.rgbs.cpu(), ref["rgbs"]) and torch.equal(out.normals.cpu(), ref["normals"])
    assert torch.equal(out.depths.cpu(), ref["depths"])


def test_fused_crop_render_matches_separate_kernels(scene, raster_mode):
    """mpx_render_crop_fused writes the same 16-bit network input as roi_align_fused + raster_render_fused."""
    from megapose6d_b200 import _abi

    ds, images, K, db, rm = scene
    r = BatchRenderer(object_dataset=ds)
    n, h, w, c_pad = 5, 240, 320, 16
    labels = [ds[i % 3].label for i in range(n)]
    lab = r.mesh_db.label_ids(labels, DEV)
    TCO = _poses(n, 5, z_range=(0.4, 0.8)).cuda()
    Kc = torch.tensor([[1200.0, 0, 160], [0, 1200, 120], [0, 0, 1]]).repeat(n, 1, 1).cuda()
    boxes = torch.tensor([[100.0, 80, 420, 320], [-40, -30, 200, 150], [500, 380, 700, 530], [0, 0, 640, 480],
                          [250, 150, 390, 255]]).cuda()
    im_idx = torch.zeros(n, dtype=torch.int32, device=DEV)
    nhwc4 = lib3d.image_to_nhwc4(images[:, :3].contiguous().cuda())
    xa = torch.zeros(n, h // 2, w // 2, 4 * c_pad, device=DEV, dtype=ACT)
    xb = torch.full_like(xa, 7.0)  # the fused kernel must overwrite every channel, pad included
    _abi.check(_abi.lib().mpx_roi_align_fused(_abi.ptr(nhwc4), 1, 480, 640, _abi.ptr(im_idx), _abi.ptr(boxes), n, 3, h, w,
                                              _abi.ptr(xa), c_pad, None, 0, _abi.stream_ptr()))
    r.render_fused(lab, TCO, Kc, 1, (h, w), xa, c_pad, 3, 6)
    r.render_crop_fused(lab, TCO, Kc, (h, w), nhwc4, im_idx, boxes, 3, xb, c_pad, 6)
    torch.cuda.synchronize()
    assert torch.equal(xa, xb)


def _textured_ds():
    return RigidObjectDataset([RigidObject("box", mesh=procedural.textured_box(seed=1)),
                               RigidObject("ball", mesh=procedural.bumpy_sphere(n_seg=40, n_lat=21)),
                               RigidObject("tinted_box", mesh=procedural.textured_box(size=(0.06, 0.09, 0.04), seed=2,
                                                                                      with_vertex_colors=True))])


def test_textured_meshes_bit_exact_vs_oracle(raster_mode):
    """Diffuse textures (repeat wrap, bilinear, optional modulation by vertex colours) next to an untextured mesh in the
    same store: rgb / normals / depth equal the oracle's bit for bit, through both small-batch paths."""
    ds = _textured_ds()
    rm = helpers.ref_meshes_from_dataset(ds)
    n = 9
    labels = [ds[i % 3].label for i in range(n)]
    TCO = _poses(n, 33, z_range=(0.2, 0.5))
    Kc = torch.tensor([[700.0, 0, 160], [0, 700, 120], [0, 0, 1]]).repeat(n, 1, 1)
    out, ref = _render_both(ds, rm, labels, TCO, Kc, (240, 320))
    for name, got, want in (("rgb", out.rgbs, ref["rgbs"]), ("normals", out.normals, ref["normals"]),
                            ("depth", out.depths, ref["depths"])):
        assert torch.equal(got.cpu(), want), f"{name}: max |d| = {(got.cpu() - want).abs().max()}"
    box = out.rgbs[0][:, out.depths[0, 0] > 0]
    assert box.shape[1] > 2000 and box.std() > 0.1  # the checkerboard is visible


def test_textured_meshes_many_views_and_fused_input():
    """The one-kernel path (more views than CTA slots) with textures, and the fused network-input form."""
    ds = _textured_ds()
    rm = helpers.ref_meshes_from_dataset(ds)
    n = 2 * _abi.lib().mpx_sm_count() + 19
    labels = [ds[i % 3].label for i in range(n)]
    TCO = _poses(n, 34, z_range=(0.25, 0.6))
    Kc = torch.tensor([[300.0, 0, 40], [0, 300, 32], [0, 0, 1]]).repeat(n, 1, 1)
    out, ref = _render_both(ds, rm, labels, TCO, Kc, (64, 80))
    assert torch.equal(out.rgbs.cpu(), ref["rgbs"]) and torch.equal(out.normals.cpu(), ref["normals"])
    assert torch.equal(out.depths.cpu(), ref["depths"])
    # fused 16-bit network input: channels 3..8 of each pixel vector are the contract planes rounded to the 16-bit type
    r = BatchRenderer(object_dataset=ds)
    m, h, w, c_pad = 5, 64, 80, 16
    x = torch.zeros(m, h // 2, w // 2, 4 * c_pad, device=DEV, dtype=ACT)
    lab = r.mesh_db.label_ids(labels[:m], DEV)
    r.render_fused(lab, TCO[:m].cuda().contiguous(), Kc[:m].cuda().contiguous(), 1, (h, w), x, c_pad, 3, 6, None)
    xs = x.view(m, h // 2, w // 2, 2, 2, c_pad).permute(0, 5, 1, 3, 2, 4).reshape(m, c_pad, h, w).float().cpu()
    want = torch.cat((ref["rgbs"][:m], ref["normals"][:m]), dim=1).to(ACT).float()
    assert torch.equal(xs[:, 3:9], want)
