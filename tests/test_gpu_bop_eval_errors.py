"""The BOP toolkit's other pose errors on the device (csrc/bop_eval.cu: mpx_bop_cus, mpx_bop_pose_errors): CUS counts and
errors bit-identical to oracle/bop_other_ref.py, PROJ / RE / TE within float64 tolerances, refusals before any launch, and the
evaluator's ad / add / adi / cus / proj / re / te / rete scores end to end against the oracle."""
from __future__ import annotations

import json

import numpy as np
import pytest
import torch

from megapose6d_b200 import _abi, bop_eval
from oracle import bop_other_ref, bop_ref
from tests.test_gpu_bop_eval import _ests, _random_pose, _vsd_images, split  # noqa: F401  (split: module fixture)
from workloads import bop_split

pytestmark = pytest.mark.gpu
NEW_TYPES = ("ad", "add", "adi", "cus", "proj", "re", "te", "rete")


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _silhouettes(h, w):
    """hand-made renders (metres): disjoint, one inside the other, empty, full image"""
    out = np.zeros((5, h, w), np.float32)
    out[0, 2:10, 3:12] = 0.5
    out[1, h - 9:h - 2, w - 12:w - 4] = 0.6
    out[2, 4:8, 5:9] = 0.7  # inside render 0
    out[4] = 0.8
    return out


@pytest.mark.parametrize("h,w,n_pairs", [(480, 640, 60), (23, 37, 70000)])
def test_cus_bit_identical(h, w, n_pairs):
    _, est, gt, _ = _vsd_images(h, w, 3, 7, 7, seed=w)
    est = np.concatenate([est, _silhouettes(h, w)])
    gt = np.concatenate([gt, _silhouettes(h, w)])
    r = np.random.RandomState(n_pairs)
    e_idx = r.randint(0, len(est), n_pairs).astype(np.int32)
    g_idx = r.randint(0, len(gt), n_pairs).astype(np.int32)
    hand = [(7, 8), (7, 9), (9, 7), (10, 10), (11, 11), (10, 11), (11, 7), (0, 7)]  # disjoint, inside, empty union, full
    for k, (e, g) in enumerate(hand):
        e_idx[k], g_idx[k] = e, g
    e_idx[len(hand)], g_idx[len(hand) + 1] = len(est), -1  # out of range: NaN
    err, counts = bop_eval.cus_from_depths(cuda(est), cuda(gt), cuda(e_idx), cuda(g_idx))
    err, counts = err.cpu(), counts.cpu()
    check = list(range(min(n_pairs, 60))) + list(range(60, n_pairs, 997)) + [n_pairs - 1]
    for p in check:
        if p in (len(hand), len(hand) + 1):
            assert torch.isnan(err[p]) and counts[p].tolist() == [0, 0]
            continue
        mm = lambda a: (a * np.float32(1000.0)).astype(np.float32)  # noqa: E731
        want, c = bop_other_ref.cus_from_depths(mm(est[e_idx[p]]), mm(gt[g_idx[p]]), return_counts=True)
        assert counts[p].tolist() == c, p
        assert torch.equal(err[p], torch.tensor(want, dtype=torch.float64)), (p, err[p], want)
    assert err[0] == 1.0 and err[3] == 1.0 and counts[3].tolist() == [0, 0]
    assert err[1] == 1.0 - 16 / 72.0 and err[4] == 0.0 and counts[4].tolist() == [h * w, h * w]


def test_cus_on_rasteriser_renders(split):  # noqa: F811
    root, gt = split
    ev = bop_eval.BopEvaluator(root)
    sp = ev.split
    K = sp.K(1, 0)
    r = np.random.RandomState(0)
    poses = [_random_pose(r, z=550.0) for _ in range(6)]
    objs = [1, 2, 3, 1, 2, 3]
    d = ev.render_depth(objs, [p[0] for p in poses], [p[1] for p in poses], [K] * 6, (480, 640))
    e_idx = np.array([0, 1, 2, 3, 4, 5, 0, 3], np.int32)
    g_idx = np.array([3, 4, 5, 0, 1, 2, 0, 5], np.int32)
    err, counts = bop_eval.cus_from_depths(d, d, cuda(e_idx), cuda(g_idx))
    dm = (d.cpu().numpy() * np.float32(1000.0)).astype(np.float32)
    for p in range(len(e_idx)):
        want, c = bop_other_ref.cus_from_depths(dm[e_idx[p]], dm[g_idx[p]], return_counts=True)
        assert counts[p].tolist() == c and err[p].item() == want, p
    assert err[6].item() == 0.0 and 0 < err[:6].min() and (counts[:, 1] > 0).all()


def _rot_cases(r):
    """(R_e, R_g): identical, 180-degree turns, cosines just outside [-1, 1], small and random angles"""
    R0 = bop_split.random_rotation(r)
    out = [(R0, R0), (np.eye(3) * (1 + 4e-16), np.eye(3)), (np.diag([1.0, -1.0, -1.0]) * (1 + 4e-16), np.eye(3))]
    for axis in range(3):
        a = np.zeros(3)
        a[axis] = 1.0
        S = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
        for ang in (np.pi, 1e-3, 0.5):
            out.append((R0.dot(np.eye(3) + np.sin(ang) * S + (1 - np.cos(ang)) * S.dot(S)), R0))
    out += [(bop_split.random_rotation(r), bop_split.random_rotation(r)) for _ in range(6)]
    return out


@pytest.mark.parametrize("n_pts", [1, 31, 4097, 20000])
def test_pose_errors(n_pts):
    r = np.random.RandomState(n_pts)
    pts = r.normal(0, 30.0, (n_pts, 3))
    store = bop_eval.PointStore([pts, pts[: max(1, n_pts // 2)]], [np.zeros((1, 12))] * 2)
    cases = []
    for k, (R_e, R_g) in enumerate(_rot_cases(r)):
        t_g = np.array([r.uniform(-20, 20), r.uniform(-20, 20), 600.0])
        t_e = t_g if k < 3 else t_g + r.normal(0, 10.0, 3)
        cases.append((k % 2, R_e, t_e, R_g, t_g))
    K = np.array([[600.0, 0, 320.5], [0, 601.0, 240.25], [0, 0, 1]])
    mi = torch.tensor([c[0] for c in cases] + [2], dtype=torch.int32, device="cuda")  # the last: an unknown model
    pe = cuda(np.stack([bop_eval._pose12(c[1], c[2]) for c in cases] + [bop_eval._pose12(np.eye(3), [0, 0, 500.0])]))
    pg = cuda(np.stack([bop_eval._pose12(c[3], c[4]) for c in cases] + [bop_eval._pose12(np.eye(3), [0, 0, 503.0])]))
    Kt = cuda(np.stack([K] * (len(cases) + 1)))
    out = {k: v.cpu().numpy() for k, v in store.pose_errors(pe, pg, mi, Kt).items()}
    for p, (m, R_e, t_e, R_g, t_g) in enumerate(cases):
        P = pts if m == 0 else pts[: max(1, n_pts // 2)]
        assert out["proj"][p] == pytest.approx(bop_other_ref.proj(R_e, t_e, R_g, t_g, K, P), rel=1e-12, abs=1e-9), p
        assert out["te"][p] == pytest.approx(bop_other_ref.te(t_e, t_g), rel=1e-12, abs=0), p
        assert out["re"][p] == pytest.approx(bop_other_ref.re(R_e, R_g), rel=0, abs=2e-6), (p, out["re"][p], bop_other_ref.re(R_e, R_g))
    assert out["re"][1] == 0.0 and out["re"][2] == 180.0 and out["proj"][0] == 0.0 and out["te"][0] == 0.0
    assert np.isnan(out["proj"][-1]) and out["te"][-1] == 3.0 and out["re"][-1] == 0.0
    only = store.pose_errors(pe, pg, types=("re",))  # NULL outputs are skipped; no points, indices or K read
    assert list(only) == ["re"] and torch.equal(only["re"].cpu(), torch.from_numpy(out["re"]))


def test_refusals_before_any_launch():
    lib = _abi.lib()
    d = torch.zeros(64, dtype=torch.float64, device="cuda")
    p = d.data_ptr()
    host = np.zeros(64)
    hp = host.ctypes.data
    n0 = lib.mpx_launch_count()
    cus = lambda **kw: lib.mpx_bop_cus(*[kw.get(k, v) for k, v in dict(  # noqa: E731
        n=1, h=4, w=4, est=p, n_est=1, gt=p, n_gt=1, ei=p, gi=p, counts=p, err=p, stream=None).items()])
    assert cus(n=-1) == -1 and b"n_pairs" in lib.mpx_last_error()
    assert cus(h=0) == -1 and cus(w=-3) == -1 and cus(h=65536, w=65536) == -1
    assert cus(n_est=0) == -1 and cus(n_gt=-2) == -1
    for k in ("est", "gt", "ei", "gi", "counts", "err"):
        assert cus(**{k: None}) == -1 and b"NULL" in lib.mpx_last_error(), k
        assert cus(**{k: hp}) == -1 and b"not device memory" in lib.mpx_last_error(), k
    pose = lambda **kw: lib.mpx_bop_pose_errors(*[kw.get(k, v) for k, v in dict(  # noqa: E731
        n=1, n_models=1, pts=p, pt_off=p, n_pts=1, mi=p, pe=p, pg=p, K=p, proj=p, re=p, te=p, stream=None).items()])
    assert pose(n=-1) == -1 and b"n_pairs" in lib.mpx_last_error()
    assert pose(n_models=0) == -1 and pose(n_pts=-1) == -1
    for k in ("pts", "pt_off", "mi", "pe", "pg", "K", "proj", "re", "te"):
        if k not in ("proj", "re", "te"):
            assert pose(**{k: None}) == -1 and b"NULL" in lib.mpx_last_error(), k
        assert pose(**{k: hp}) == -1 and b"not device memory" in lib.mpx_last_error(), k
    torch.cuda.synchronize()
    assert lib.mpx_launch_count() == n0
    # without proj the point store, indices and K are not needed
    assert pose(proj=None, pts=None, pt_off=None, mi=None, K=None, n_models=0) == 0
    assert pose(proj=None, re=None, te=None) == 0  # nothing asked: no launch
    torch.cuda.synchronize()
    assert lib.mpx_launch_count() == n0 + 1


# ------------------------------------------------------------------------------------------------------------ end to end
def _oracle_render(ev):
    def render(obj_id, R, t, K, shape):
        return ev.render_depth([obj_id], R[None], np.reshape(t, (1, 3)), K[None], tuple(shape))[0].cpu().numpy()

    return render


def test_evaluate_matches_oracle(split):  # noqa: F811
    root, gt = split
    ev = bop_eval.BopEvaluator(root, max_renders_per_chunk=7)  # several render chunks
    ests = bop_eval.normalize_results(_ests(gt, "mixed"))
    render = _oracle_render(ev)
    got = ev.evaluate(ests, types=bop_eval.ERROR_TYPES)
    want = bop_ref.evaluate(ev.split, ests, render)
    want.update(bop_other_ref.evaluate_localization(ev.split, ests, render, NEW_TYPES, symmetric_obj_ids=[2, 3]))
    want["symmetric_obj_ids"] = [2, 3]
    assert got == want
    assert all(0 < got[t]["recall"] < 1 for t in ("ad", "add", "proj", "te", "rete")), {t: got[t]["recall"] for t in NEW_TYPES}
    rows = bop_other_ref.calc_other_errors(ev.split, ests, render, NEW_TYPES, [2, 3])
    df = ev.errors(ests, types=NEW_TYPES)
    assert len(df) == len(rows)
    np.testing.assert_array_equal(df["cus"].to_numpy(), [r["cus"] for r in rows])
    for t in ("ad", "add", "adi", "proj", "te"):
        np.testing.assert_allclose(df[t].to_numpy(), [r[t] for r in rows], rtol=1e-12, atol=1e-9, err_msg=t)
    np.testing.assert_allclose(df["re"].to_numpy(), [r["re"] for r in rows], rtol=0, atol=2e-6)
    assert np.isinf(df["add"]).any() and (df["cus"] == 1.0).any()  # gated pairs


def test_vsd_and_cus_share_renders(split, monkeypatch):  # noqa: F811
    root, gt = split
    ev = bop_eval.BopEvaluator(root, max_renders_per_chunk=7)
    ests = _ests(gt, "mixed")
    calls = []
    orig = ev.render_depth
    monkeypatch.setattr(ev, "render_depth", lambda *a, **k: calls.append(len(a[0])) or orig(*a, **k))
    both = ev.errors(ests, types=("vsd", "cus"))
    n_both = list(calls)
    calls.clear()
    vsd = ev.errors(ests, types=("vsd",))
    assert calls == n_both
    cus = ev.errors(ests, types=("cus",))
    vc = [f"vsd_{k}" for k in range(10)]
    np.testing.assert_array_equal(both[vc].to_numpy(), vsd[vc].to_numpy())
    np.testing.assert_array_equal(both["cus"].to_numpy(), cus["cus"].to_numpy())


def test_ground_truth_and_symmetric_flips(split):  # noqa: F811
    root, gt = split
    ev = bop_eval.BopEvaluator(root)
    sc = ev.evaluate(_ests(gt, "gt"), types=NEW_TYPES)
    for t in NEW_TYPES:
        assert sc[t]["recall"] == 1.0 and sc[t]["mean_obj_recall"] == 1.0 and sc[t]["mean_scene_recall"] == 1.0, t
        assert sc[t]["tp_count"] == sc[t]["targets_count"] > 0
    assert sc["symmetric_obj_ids"] == [2, 3]
    fl = ev.evaluate(_ests(gt, "flip"), types=("ad", "add", "adi"))
    for o in (2, 3):  # the symmetric objects: a flip is correct under ADI and AD, not under ADD
        assert fl["adi"]["obj_recalls"][o] == 1.0 and fl["ad"]["obj_recalls"][o] == 1.0
        assert fl["add"]["obj_recalls"][o] < 1.0
    assert fl["add"]["obj_recalls"][1] == 1.0
    explicit = bop_eval.BopEvaluator(root, symmetric_obj_ids=[3]).evaluate(_ests(gt, "flip"), types=("ad",))
    assert explicit["symmetric_obj_ids"] == [3]
    assert explicit["ad"]["obj_recalls"][3] == 1.0 and explicit["ad"]["obj_recalls"][2] == fl["add"]["obj_recalls"][2]


def test_te_override_and_cli(split, capsys, tmp_path):  # noqa: F811
    root, gt = split
    ev = bop_eval.BopEvaluator(root)
    ests = bop_eval.normalize_results(_ests(gt, "mixed"))
    base = ev.evaluate(ests, types=NEW_TYPES)
    ths = {"te": [50.0], "rete": [5.0, 50.0]}
    over = ev.evaluate(ests, types=NEW_TYPES, thresholds=ths)
    assert over["te"]["recall"] > base["te"]["recall"] and over["rete"] != base["rete"]
    assert all(over[t] == base[t] for t in NEW_TYPES if t not in ("te", "rete"))
    from megapose6d_b200.prediction_runner import save_bop_results

    csv = tmp_path / "res_synth-test.csv"
    save_bop_results(csv, ests)
    capsys.readouterr()
    bop_eval.main([str(root), str(csv), "--error-types", ",".join(NEW_TYPES), "--correct-th", "te=50",
                   "--correct-th", "rete=5,50", "--symmetric-obj-ids", "3"])
    line = capsys.readouterr().out.strip().splitlines()[-1]
    api = bop_eval.BopEvaluator(root, symmetric_obj_ids=[3]).evaluate(csv, types=NEW_TYPES, thresholds=ths)
    assert json.loads(line) == json.loads(json.dumps(api))
    assert set(json.loads(line)) == set(NEW_TYPES) | {"bop19_average_time_per_image", "symmetric_obj_ids"}
    for t in NEW_TYPES:
        assert set(json.loads(line)[t]) == {"recall", "obj_recalls", "mean_obj_recall", "scene_recalls",
                                            "mean_scene_recall", "gt_count", "targets_count", "tp_count"}
