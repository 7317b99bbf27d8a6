"""The TEASER++ refiner's oracle (oracle/teaser_ref.py) held against independent restatements, on the CPU: weighted Kabsch
against scipy, GNC-TLS under outliers, adaptive voting against a brute-force TLS minimisation, farthest-point sampling
against a naive loop, the point cloud against the reference's numpy expression, the max clique against networkx and
planted cliques; plus the host side of megapose6d_b200/teaserpp_refiner.py."""
import networkx as nx
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from megapose6d_b200 import teaserpp_refiner
from oracle import teaser_ref as T


def test_weighted_kabsch_matches_scipy():
    rng = np.random.RandomState(0)
    for trial in range(10):
        R = Rotation.random(random_state=trial).as_matrix()
        a = rng.randn(30, 3)
        b = a @ R.T + 0.01 * rng.randn(30, 3)
        w = rng.rand(30)
        got = T.weighted_kabsch(a, b, w)
        ref, _ = Rotation.align_vectors(b, a, weights=w)
        np.testing.assert_allclose(got, ref.as_matrix(), atol=1e-10)
        assert abs(np.linalg.det(got) - 1) < 1e-12


def test_gnc_tls_recovers_rotation_with_40_percent_outliers():
    rng = np.random.RandomState(1)
    R = Rotation.random(random_state=5).as_matrix()
    a = rng.uniform(-0.1, 0.1, (200, 3))
    b = a @ R.T + rng.uniform(-0.002, 0.002, (200, 3))
    bad = rng.rand(200) < 0.4
    b[bad] = rng.uniform(-0.1, 0.1, (bad.sum(), 3))
    got = T.gnc_tls_rotation(a, b, 0.02)
    ang = np.degrees(np.arccos(np.clip((np.trace(got.T @ R) - 1) / 2, -1, 1)))
    assert ang < 0.5
    ang_ls = np.degrees(np.arccos(np.clip((np.trace(T.weighted_kabsch(a, b, np.ones(200)).T @ R) - 1) / 2, -1, 1)))
    assert ang_ls > 5 * ang  # least squares alone is pulled away


@pytest.mark.parametrize("seed", range(12))
def test_adaptive_voting_equals_brute_force(seed):
    rng = np.random.RandomState(seed)
    x = np.concatenate([rng.normal(0.3, 0.004, rng.randint(1, 8)), rng.uniform(-1, 1, rng.randint(0, 6))])
    assert T.tls_voting(x, 0.01) == pytest.approx(T.tls_brute_force(x, 0.01), abs=1e-12)


def _fps_naive(pts, k):
    pts = pts.astype(np.float32)
    n = len(pts)
    out = [0]
    for _ in range(1, min(n, k)):
        best, bi = -1.0, -1
        for i in range(n):
            d = min(np.float32(((pts[i, 0] - pts[s, 0]) ** 2 + (pts[i, 1] - pts[s, 1]) ** 2) + (pts[i, 2] - pts[s, 2]) ** 2)
                    for s in out)
            if d > best:
                best, bi = d, i
        out.append(bi)
    return np.array(out + [n - 1] * (k - len(out)))


@pytest.mark.parametrize("n,k", [(50, 10), (7, 12), (40, 40), (1, 3)])
def test_fps_equals_naive(n, k):
    rng = np.random.RandomState(n)
    pts = rng.randint(0, 5, (n, 3)).astype(np.float32) * 0.01  # a coarse grid: many ties and duplicated points
    got = T.farthest_point_sampling(pts, k)
    np.testing.assert_array_equal(got, _fps_naive(pts, k))
    if n < k:
        assert (got[n:] == n - 1).all()


def test_pointcloud_is_the_reference_expression():
    rng = np.random.RandomState(2)
    depth = rng.uniform(0.3, 2.0, (37, 53)).astype(np.float32)
    depth[rng.rand(37, 53) < 0.2] = 0
    depth[3, 4] = np.nan
    K = np.array([[601.3, 0, 26.7], [0, 598.9, 17.1], [0, 0, 1]], np.float32)
    h, w = depth.shape
    px, py = np.meshgrid(np.linspace(0, w - 1, w), np.linspace(0, h - 1, h))
    with np.errstate(invalid="ignore"):
        px = (px - K[0, 2]) * (depth / K[0, 0])
        py = (py - K[1, 2]) * (depth / K[1, 1])
    ref = np.float32([px, py, depth]).transpose(1, 2, 0)
    got = T.get_pointcloud(depth, K)
    assert got.dtype == np.float32 and got.tobytes() == ref.tobytes()


def test_max_clique_equals_networkx():
    for s in range(24):
        n, p = 8 + 2 * s, [0.2, 0.5, 0.8, 0.95][s % 4]
        a = T.random_graph(n, p, s)
        c, _, exhausted = T.max_clique(a)
        _, size = nx.max_weight_clique(nx.from_numpy_array(a.astype(int)), weight=None)
        assert len(c) == size and T.is_clique(a, c) and not exhausted and c == sorted(c)


def test_max_clique_finds_planted_clique():
    a, planted = T.planted_clique_graph(1000, 0.3, 30, 7)
    c, _, exhausted = T.max_clique(a)
    assert c == planted and not exhausted


def test_max_clique_budget_returns_a_clique():
    a, _ = T.planted_clique_graph(200, 0.8, 12, 3)
    c, nodes, exhausted = T.max_clique(a, node_budget=3)
    assert exhausted and nodes == 3 and T.is_clique(a, c)


def test_solver_params_and_constructor_checks():
    p = teaserpp_refiner.get_solver_params(0.02)
    assert (p.cbar2, p.noise_bound, p.estimate_scaling, p.rotation_estimation_algorithm, p.rotation_gnc_factor,
            p.rotation_max_iterations, p.rotation_cost_threshold) == (1, 0.02, False, "GNC_TLS", 1.4, 100, 1e-12)
    with pytest.raises(ValueError):
        teaserpp_refiner.TeaserppRefiner(None, None, mask_type="nope")
    with pytest.raises(ValueError):
        teaserpp_refiner.TeaserppRefiner(None, None, n_points=1025)


def test_refine_one_gates():
    """Few masked pixels: skipped; min_num_inliers out of reach: solved, not accepted."""
    rng = np.random.RandomState(4)
    K = np.array([[500, 0, 20], [0, 500, 15], [0, 0, 1]], np.float32)
    d = np.zeros((30, 40), np.float32)
    d[5:25, 8:30] = 0.5 + 0.01 * rng.rand(20, 22).astype(np.float32)
    TCO = np.eye(4, dtype=np.float32)
    acc, out, info = T.refine_one(d, d, K, TCO, n_min_points=1000)
    assert not acc and not info["reached"] and (out == TCO).all()
    acc, out, info = T.refine_one(d, d, K, TCO, n_points=60, min_num_inliers=61)
    assert info["reached"] and info["valid"] and not acc and info["num_inliers"] == 60
    acc, out, info = T.refine_one(d, d, K, TCO, n_points=60, min_num_inliers=50)
    assert acc and np.allclose(out, TCO, atol=1e-6)
