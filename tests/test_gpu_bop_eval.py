"""BOP 2019 evaluation on the device (csrc/bop_eval.cu): VSD bit-identical to oracle/bop_ref.py on the same depth images,
MSSD / MSPD / ADD / ADI within float64 tolerances, refusals before any launch, and the evaluator end to end."""
from __future__ import annotations

import json

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

from megapose6d_b200 import _abi, bop_eval
from megapose6d_b200.object_dataset import RigidObject, RigidObjectDataset
from megapose6d_b200.scene_renderer import Panda3dSceneRenderer
from oracle import bop_ref
from workloads import bop_split

pytestmark = pytest.mark.gpu
TAUS = bop_ref.VSD_TAUS


def _vsd_images(h, w, n_img, n_est, n_gt, seed):
    """float32 metre renders with an object-like blob each, raw uint16 test depths with holes, and K per image whose
    principal point sits on a pixel, where the distance is the depth itself: delta and tau boundaries are placed there."""
    r = np.random.RandomState(seed)
    ys, xs = np.mgrid[:h, :w]
    K = np.zeros((n_img, 3, 3))
    for i in range(n_img):
        cx, cy = w // 2 + i % 3, h // 2 - i % 2
        K[i] = [[1.1 * w, 0, cx], [0, 1.1 * w, cy], [0, 0, 1]]

    def blobs(n):
        out = np.zeros((n, h, w), np.float32)
        for k in range(n):
            cx, cy, rad = r.uniform(0.3, 0.7) * w, r.uniform(0.3, 0.7) * h, r.uniform(0.15, 0.3) * min(h, w)
            m = (xs - cx) ** 2 + (ys - cy) ** 2 < rad ** 2
            out[k][m] = (r.uniform(0.5, 0.6) + 0.0002 * (xs[m] - cx) + 0.0001 * (ys[m] - cy)).astype(np.float32)
        return out

    est, gt = blobs(n_est), blobs(n_gt)
    test = np.zeros((n_img, h, w), np.uint16)
    for i in range(n_img):
        base = np.where(gt[i % n_gt] > 0, gt[i % n_gt] * 1000, 900.0) + r.normal(0, 3.0, (h, w))
        base[:, : w // 5] -= 150.0
        raw = np.round(base / 0.1)
        raw[r.uniform(size=(h, w)) < 0.05] = 0
        test[i] = raw.astype(np.uint16)
        cx, cy = int(K[i, 0, 2]), int(K[i, 1, 2])
        g = i % n_gt
        gt[g, cy, cx] = np.float32(0.5)  # 500 mm
        test[i, cy, cx] = 4850  # 485.0 mm: dist_gt - dist_test == delta exactly
    for e in range(n_est):  # on the principal point of image 0: |dist_gt - dist_est| / 100 == 0.1 exactly
        est[e, int(K[0, 1, 2]), int(K[0, 0, 2])] = np.float32(0.49)
    return test, est, gt, K


def _oracle_vsd(test, est, gt, K, scale, e, g, i, diam, delta=15):
    dt = test[i].astype(np.float32) * np.float32(scale[i])
    de = (est[e] * np.float32(1000.0)).astype(np.float32)
    dg = (gt[g] * np.float32(1000.0)).astype(np.float32)
    return bop_ref.vsd_from_depths(dt, de, dg, K[i], delta, TAUS, diam, return_counts=True)


@pytest.mark.parametrize("h,w,n_pairs", [(480, 640, 40), (103, 150, 70000)])
def test_vsd_bit_identical(h, w, n_pairs):
    n_img, n_est, n_gt = 3, 7, 5
    test, est, gt, K = _vsd_images(h, w, n_img, n_est, n_gt, seed=h)
    scale = np.array([0.1, 0.1, 0.1], np.float32)
    r = np.random.RandomState(1)
    e_idx = r.randint(0, n_est, n_pairs).astype(np.int32)
    g_idx = r.randint(0, n_gt, n_pairs).astype(np.int32)
    i_idx = r.randint(0, n_img, n_pairs).astype(np.int32)
    diam = r.uniform(80, 200, n_pairs)
    diam[:3] = 100.0
    e_idx[0], g_idx[0], i_idx[0] = 0, 0, 0
    est_z = np.concatenate([est, np.zeros((1, h, w), np.float32)])  # an empty render: union 0 with an empty gt
    gt_z = np.concatenate([gt, np.zeros((1, h, w), np.float32)])
    e_idx[1], g_idx[1] = n_est, n_gt
    cuda = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    err, counts = bop_eval.vsd_from_depths(cuda(test.view(np.int16)), cuda(scale), cuda(K), cuda(est_z), cuda(gt_z),
                                           cuda(e_idx), cuda(g_idx), cuda(i_idx), cuda(diam), 15.0, TAUS)
    err, counts = err.cpu(), counts.cpu()
    check = list(range(min(n_pairs, 40))) + list(range(40, n_pairs, 997)) + [n_pairs - 1]
    for p in check:
        want, c = _oracle_vsd(test, est_z, gt_z, K, scale, e_idx[p], g_idx[p], i_idx[p], diam[p])
        assert counts[p].tolist() == c, p
        assert torch.equal(err[p], torch.tensor(want, dtype=torch.float64)), (p, err[p], want)
    assert counts[1, 0] == 0 and (err[1] == 1.0).all()
    assert (counts[:, 0] > counts[:, 1]).any() and (counts[:, 2] > 0).any()


def _random_pose(r, z=600.0):
    return bop_split.random_rotation(r), np.array([r.uniform(-20, 20), r.uniform(-20, 20), z + r.uniform(-50, 50)])


@pytest.mark.parametrize("n_pts", [1, 31, 4097, 20000])
def test_point_errors(n_pts):
    r = np.random.RandomState(n_pts)
    pts = r.normal(0, 30.0, (n_pts, 3))
    infos = [dict(), dict(symmetries_discrete=[[1, 0, 0, 0, 0, -1, 0, 0, 0, 0, -1, 5.0, 0, 0, 0, 1]]),
             dict(symmetries_continuous=[dict(axis=[0, 0, 1], offset=[0, 0, 0])]),
             dict(symmetries_continuous=[dict(axis=[0, 0, 1], offset=[1.0, 0, 0])],
                  symmetries_discrete=[[1, 0, 0, 0, 0, -1, 0, 0, 0, 0, -1, 0, 0, 0, 0, 1]])]
    syms = [bop_eval.symmetry_transformations(i) for i in infos]
    assert [len(s) for s in syms] == [1, 2, 314, 628]
    store = bop_eval.PointStore([pts] * 4, syms)
    cases = []
    for m in range(4):
        for k in range(2):
            R_g, t_g = _random_pose(r)
            if k == 0:
                s = syms[m][len(syms[m]) // 2]
                R_s, t_s = s[:9].reshape(3, 3), s[9:]
                R_e, t_e = R_g.dot(R_s), R_g.dot(t_s) + t_g + r.normal(0, 0.5, 3)  # near a symmetric flip
            else:
                R_e, t_e = _random_pose(r)
            cases.append((m, R_e, t_e, R_g, t_g))
    K = np.array([[600.0, 0, 320.5], [0, 601.0, 240.25], [0, 0, 1]])
    mi = torch.tensor([c[0] for c in cases], dtype=torch.int32, device="cuda")
    pe = torch.from_numpy(np.stack([bop_eval._pose12(c[1], c[2]) for c in cases])).cuda()
    pg = torch.from_numpy(np.stack([bop_eval._pose12(c[3], c[4]) for c in cases])).cuda()
    Kt = torch.from_numpy(np.stack([K] * len(cases))).cuda()
    out = {k: store.errors(k, mi, pe, pg, Kt if k == "mspd" else None) for k in ("mssd", "mspd", "add", "adi")}
    for p, (m, R_e, t_e, R_g, t_g) in enumerate(cases):
        S = [(s[:9].reshape(3, 3), s[9:].reshape(3, 1)) for s in syms[m]]
        for kind in ("mssd", "mspd"):
            f = bop_ref.mssd if kind == "mssd" else bop_ref.mspd
            args = (R_e, t_e, R_g, t_g, pts, S) if kind == "mssd" else (R_e, t_e, R_g, t_g, K, pts, S)
            want, arg = f(*args, return_argmin=True)
            got = out[kind][0][p].item()
            assert got == pytest.approx(want, rel=1e-12, abs=1e-9), (kind, p)
            if kind == "mssd":
                pe_ = bop_ref.transform(pts, R_e, t_e)
                es = np.array([np.linalg.norm(pe_ - bop_ref.transform(pts, R_g.dot(Rs), R_g.dot(ts) + t_g.reshape(3, 1)),
                                              axis=1).max() for Rs, ts in S])
            else:
                pe_ = bop_ref.project(pts, K, R_e, t_e)
                es = np.array([np.linalg.norm(pe_ - bop_ref.project(pts, K, R_g.dot(Rs), R_g.dot(ts) + t_g.reshape(3, 1)),
                                              axis=1).max() for Rs, ts in S])
            close = np.abs(es - want) <= np.maximum(1e-12 * want, 1e-9)
            if close.sum() == 1:
                assert out[kind][1][p].item() == arg, (kind, p)
        assert out["add"][0][p].item() == pytest.approx(bop_ref.add(R_e, t_e, R_g, t_g, pts), rel=1e-12, abs=1e-9)
        pe_, pg_ = bop_ref.transform(pts, R_e, t_e), bop_ref.transform(pts, R_g, t_g)
        adi = cKDTree(pe_).query(pg_, k=1)[0].mean()
        assert out["adi"][0][p].item() == pytest.approx(adi, rel=1e-12, abs=1e-9)


def test_refusals_before_any_launch():
    lib = _abi.lib()
    d = torch.zeros(64, dtype=torch.float64, device="cuda")
    p = d.data_ptr()
    taus = np.asarray(TAUS)
    tp = taus.ctypes.data
    n0 = lib.mpx_launch_count()
    vsd = lambda **kw: lib.mpx_bop_vsd(*[kw.get(k, v) for k, v in dict(  # noqa: E731
        n=1, h=4, w=4, test=p, n_img=1, scale=p, K=p, est=p, n_est=1, gt=p, n_gt=1, ei=p, gi=p, ii=p, diam=p, taus=tp,
        n_taus=10, delta=15.0, counts=p, err=p, stream=None).items()])
    assert vsd(n=-1) == -1
    assert vsd(n_taus=0) == -1 and vsd(n_taus=17) == -1
    assert vsd(h=0) == -1 and vsd(w=-3) == -1 and vsd(h=65536, w=65536) == -1
    assert vsd(n_img=0) == -1 and vsd(n_est=0) == -1
    for k in ("test", "scale", "K", "est", "gt", "ei", "gi", "ii", "diam", "counts", "err", "taus"):
        assert vsd(**{k: None}) == -1, k
    pt = lambda **kw: lib.mpx_bop_point_errors(*[kw.get(k, v) for k, v in dict(  # noqa: E731
        kind=0, n=1, n_models=1, pts=p, pt_off=p, n_pts=1, syms=p, sym_off=p, n_syms=1, mi=p, pe=p, pg=p, K=p, err=p,
        arg=p, stream=None).items()])
    assert pt(kind=4) == -1 and pt(kind=-1) == -1
    assert pt(n=-1) == -1 and pt(n_models=0) == -1
    for k in ("pts", "pt_off", "mi", "pe", "pg", "err", "syms", "sym_off"):
        assert pt(**{k: None}) == -1, k
    assert pt(kind=1, K=None) == -1
    assert pt(kind=9) == -1 and b"unknown error kind" in lib.mpx_last_error()
    torch.cuda.synchronize()
    assert lib.mpx_launch_count() == n0


# ------------------------------------------------------------------------------------------------------------ end to end
def device_scene_renderer():
    cache = {}

    def render(models, views, TCO, K, resolution):
        if "r" not in cache:
            ds = RigidObjectDataset([RigidObject(label=f"obj_{o:06d}", mesh=models[o], mesh_units="mm") for o in sorted(models)])
            cache["r"] = Panda3dSceneRenderer(ds)
        out = cache["r"].render_scene_tensors([[f"obj_{o:06d}" for o in v] for v in views], torch.from_numpy(TCO),
                                              torch.from_numpy(K), resolution, render_normals=False)
        return out.depths[:, 0].cpu().numpy(), out.inst_id.cpu().numpy()

    return render


@pytest.fixture(scope="module")
def split(tmp_path_factory):
    root = tmp_path_factory.mktemp("bop_gpu")
    gt = bop_split.write_split(root, device_scene_renderer(), n_scenes=2, n_images=3, h=480, w=640, seed=3)
    return root, gt


def _ests(gt, kind, seed=0):
    r = np.random.RandomState(seed)
    out = []
    for (s, i), inst in gt.items():
        for k, (o, R, t) in enumerate(inst):
            if kind == "gt":
                out.append(dict(scene_id=s, im_id=i, obj_id=o, score=1.0, R=R, t=t, time=0.5))
            elif kind == "flip":
                info = bop_split.models_and_info()[1][o]
                S = bop_eval.symmetry_transformations(info)
                sym = S[len(S) // 2 + 1] if len(S) > 1 else S[0]
                R_s, t_s = sym[:9].reshape(3, 3), sym[9:]
                out.append(dict(scene_id=s, im_id=i, obj_id=o, score=1.0, R=R.dot(R_s), t=R.dot(t_s) + t, time=0.5))
            else:
                if (s + i + k) % 5 == 3:
                    continue
                t_e = t + r.normal(0, 5.0, 3) * (k % 3)
                out.append(dict(scene_id=s, im_id=i, obj_id=o, score=round(r.uniform(), 1), R=R, t=t_e, time=0.5 + s))
                if k % 2 == 0:
                    out.append(dict(scene_id=s, im_id=i, obj_id=o, score=out[-1]["score"], R=bop_split.random_rotation(r),
                                    t=t_e + 25.0, time=0.5 + s))
        if kind == "mixed":
            out.append(dict(scene_id=s, im_id=i, obj_id=1 if inst[0][0] != 1 else 3, score=0.99, R=inst[0][1], t=inst[0][2],
                            time=0.5 + s))
    return out


def test_ground_truth_scores_one(split):
    root, gt = split
    ev = bop_eval.BopEvaluator(root)
    sc = ev.evaluate(_ests(gt, "gt"))
    for k in ("bop19_average_recall", "bop19_average_recall_vsd", "bop19_average_recall_mssd", "bop19_average_recall_mspd"):
        assert sc[k] == 1.0, (k, sc[k])
    assert sc["bop19_average_time_per_image"] == 0.5


def test_symmetric_flips(split):
    root, gt = split
    ev = bop_eval.BopEvaluator(root)
    df = ev.errors(_ests(gt, "flip"), types=("mssd", "mspd"))
    own = df[[gt[(s, i)][g][0] == o for s, i, g, o in zip(df.scene_id, df.im_id, df.gt_id, df.obj_id)]]
    ok = own.groupby(["scene_id", "im_id", "obj_id", "est_id"])["mssd"].min()
    assert (ok < 1e-6).all()
    assert (own.groupby(["scene_id", "im_id", "obj_id", "est_id"])["mspd"].min() < 1e-6).all()
    sc = ev.evaluate(_ests(gt, "flip"))
    assert sc["bop19_average_recall_mssd"] == 1.0 and sc["bop19_average_recall_mspd"] == 1.0


def test_evaluate_matches_oracle_and_cli(split, capsys, tmp_path):
    root, gt = split
    ev = bop_eval.BopEvaluator(root, max_renders_per_chunk=7)  # several render chunks
    ests = bop_eval.normalize_results(_ests(gt, "mixed"))

    def render(obj_id, R, t, K, shape):
        return ev.render_depth([obj_id], R[None], np.reshape(t, (1, 3)), K[None], tuple(shape))[0].cpu().numpy()

    want = bop_ref.evaluate(ev.split, ests, render)
    got = ev.evaluate(ests)
    assert got == want
    assert 0 < got["bop19_average_recall"] < 1
    rows = bop_ref.calc_errors(ev.split, ests, render)
    df = ev.errors(ests)
    assert len(df) == len(rows)
    np.testing.assert_array_equal(df[[f"vsd_{k}" for k in range(10)]].to_numpy(), np.array([r["vsd"] for r in rows]))
    np.testing.assert_allclose(df["mssd"].to_numpy(), [r["mssd"] for r in rows], rtol=1e-12, atol=1e-9)
    np.testing.assert_allclose(df["mspd"].to_numpy(), [r["mspd"] for r in rows], rtol=1e-12, atol=1e-9)
    from megapose6d_b200.prediction_runner import save_bop_results

    csv = tmp_path / "res_synth-test.csv"
    save_bop_results(csv, ests)
    capsys.readouterr()
    bop_eval.main([str(root), str(csv), "--errors-out", str(tmp_path / "err")])
    line = capsys.readouterr().out.strip().splitlines()[-1]
    assert json.loads(line) == json.loads(json.dumps(bop_eval.BopEvaluator(root).evaluate(csv)))
    assert json.loads(line)["bop19_average_recall"] == pytest.approx(want["bop19_average_recall"], abs=0)
    assert (tmp_path / "err" / "errors.csv").exists()
