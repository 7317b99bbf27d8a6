"""numpy / float64 restatement of the TEASER++ depth refiner's contract (DESIGN §4, megapose6d_b200/teaserpp_refiner.py).

Written from the contract's steps, not from any library: point clouds from a depth image, masks, farthest-point sampling
as a plain loop, the pairwise-invariant consistency graph, an exact maximum clique (the same branch-and-bound the device
runs, on Python integers as bitsets), GNC-TLS rotation, adaptive-voting TLS translation, the inlier count and the gated
pose update.  Every function works on one prediction.
"""
from __future__ import annotations

import random
from typing import List, Optional, Tuple

import numpy as np


# ---- step 2-3: masks and point clouds --------------------------------------------------------------------------------
def compute_mask(mask_type: str, rendered: np.ndarray, measured: np.ndarray, thresh: float = 0.1) -> np.ndarray:
    m = (measured > 0) & (rendered > 0)
    if mask_type == "threshold":
        with np.errstate(invalid="ignore"):
            m &= ~(np.abs(measured - rendered) > np.float32(thresh))
    elif mask_type != "simple":
        raise ValueError(mask_type)
    return m


def get_pointcloud(depth: np.ndarray, K: np.ndarray) -> np.ndarray:
    """[H, W] float32 depth, [3, 3] float32 K -> [H, W, 3] float32: x = fp32((u - cx) * fp32(z / fx)) in float64."""
    depth = np.asarray(depth, np.float32)
    K = np.asarray(K, np.float32)
    h, w = depth.shape
    u = np.arange(w, dtype=np.float64)[None, :]
    v = np.arange(h, dtype=np.float64)[:, None]
    with np.errstate(invalid="ignore"):
        x = (u - np.float64(K[0, 2])) * (depth / K[0, 0]).astype(np.float64)
        y = (v - np.float64(K[1, 2])) * (depth / K[1, 1]).astype(np.float64)
    return np.stack((x.astype(np.float32), y.astype(np.float32), depth), axis=-1)


def masked_clouds(rendered, measured, K, mask_type="simple", thresh=0.1):
    """(src [N,3], tgt [N,3]) in row-major pixel order: src from the rendered depth, tgt from the measured one."""
    m = compute_mask(mask_type, rendered, measured, thresh)
    return get_pointcloud(rendered, K)[m], get_pointcloud(measured, K)[m]


# ---- step 4: farthest-point sampling ---------------------------------------------------------------------------------
def farthest_point_sampling(pts: np.ndarray, k: int) -> np.ndarray:
    """Index 0 first, then the arg-max (lowest index on ties) of the running minimum of fp32 squared distances; when
    N < k the indices are padded with N - 1 (the last point)."""
    pts = np.asarray(pts, np.float32)
    n = len(pts)
    out = np.full(k, n - 1, np.int64)
    if n == 0:
        return out
    mind = np.full(n, np.inf, np.float32)
    sel = 0
    out[0] = 0
    for j in range(1, min(n, k)):
        d = pts - pts[sel]
        d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        mind = np.minimum(mind, d2)
        sel = int(np.argmax(mind))
        out[j] = sel
    return out


# ---- step 5: consistency graph ---------------------------------------------------------------------------------------
def consistency_graph(src: np.ndarray, tgt: np.ndarray, noise_bound: float, cbar2: float = 1.0) -> np.ndarray:
    """[m, m] bool: pair (i, j) consistent when | ||t_j - t_i|| - ||s_j - s_i|| | <= 2 noise_bound sqrt(cbar2)."""
    s = np.asarray(src, np.float32).astype(np.float64)
    t = np.asarray(tgt, np.float32).astype(np.float64)
    bound = 2.0 * noise_bound * np.sqrt(cbar2)

    def norms(p):
        a = p[None, :, :] - p[:, None, :]
        return np.sqrt((a[..., 0] * a[..., 0] + a[..., 1] * a[..., 1]) + a[..., 2] * a[..., 2])

    adj = np.abs(norms(t) - norms(s)) <= bound
    np.fill_diagonal(adj, False)
    return adj


def pack_adjacency(adj: np.ndarray, k: Optional[int] = None) -> np.ndarray:
    """[m, m] bool -> [k, 16] uint64 rows, bit j % 64 of word j // 64 (the device layout)."""
    m = adj.shape[0]
    k = m if k is None else k
    full = np.zeros((k, 1024), bool)
    full[:m, :m] = adj
    return np.packbits(full, axis=1, bitorder="little").view("<u8").reshape(k, 16)


# ---- step 5: maximum clique ------------------------------------------------------------------------------------------
def _rows(adj: np.ndarray) -> List[int]:
    return [int.from_bytes(np.packbits(r, bitorder="little").tobytes(), "little") for r in adj]


def core_numbers(adj: np.ndarray) -> np.ndarray:
    """k-core number of every vertex, by peeling all vertices of degree <= k at once."""
    m = adj.shape[0]
    deg = adj.sum(1).astype(np.int64)
    core = np.zeros(m, np.int64)
    rem = np.ones(m, bool)
    k = 0
    while rem.any():
        peel = rem & (deg <= k)
        if not peel.any():
            k = int(deg[rem].min())
            continue
        core[peel] = k
        rem &= ~peel
        deg = (adj & rem[None, :]).sum(1)
    return core


def max_clique(adj: np.ndarray, node_budget: Optional[int] = None) -> Tuple[List[int], int, bool]:
    """Exact maximum clique (the device's algorithm): vertices renumbered by core number (highest first, then index), a
    greedy clique in that order as the lower bound, vertices whose core number is below it dropped, then branch and bound
    with a greedy-colouring bound (branch on the highest colour first).  Returns (sorted clique, nodes, budget exhausted)."""
    m = adj.shape[0]
    if m == 0:
        return [], 0, False
    core = core_numbers(adj)
    perm = sorted(range(m), key=lambda v: (-core[v], v))          # new index -> vertex
    rows = _rows(adj[np.ix_(perm, perm)])
    best: List[int] = []
    cand = (1 << m) - 1
    for v in range(m):                                             # greedy lower bound in core order
        if cand >> v & 1:
            best.append(v)
            cand &= rows[v]
    p0 = sum(1 << v for v in range(m) if core[perm[v]] >= len(best))

    def colour(P: int, kmin: int) -> List[Tuple[int, int]]:
        out, U, k = [], P, 0
        while U:
            k += 1
            Q = U
            while Q:
                v = (Q & -Q).bit_length() - 1
                Q &= ~rows[v] & ~(1 << v)
                U &= ~(1 << v)
                if k >= kmin:
                    out.append((v, k))
        return out

    nodes, exhausted = 1, False
    R: List[int] = []
    stack = [(p0, colour(p0, len(best) + 1))]
    while stack:
        P, lst = stack[-1]
        if not lst or len(R) + lst[-1][1] <= len(best):
            stack.pop()
            if R:
                R.pop()
            continue
        v, _ = lst.pop()
        newP = P & rows[v]
        stack[-1] = (P & ~(1 << v), lst)
        if newP == 0:
            if len(R) + 1 > len(best):
                best = R + [v]
            continue
        if node_budget is not None and nodes >= node_budget:
            exhausted = True
            break
        nodes += 1
        nl = colour(newP, len(best) - len(R))
        if nl:
            R.append(v)
            stack.append((newP, nl))
    return sorted(perm[v] for v in best), nodes, exhausted


def planted_clique_graph(n: int, p: float, size: int, seed: int) -> Tuple[np.ndarray, List[int]]:
    """G(n, p) with a clique on `size` random vertices.  For the sizes the tests use the planted clique is the unique
    maximum (it is far above G(n, p)'s clique number)."""
    rng = np.random.RandomState(seed)
    a = rng.rand(n, n) < p
    a = np.triu(a, 1)
    a = a | a.T
    planted = sorted(rng.choice(n, size, replace=False).tolist())
    a[np.ix_(planted, planted)] = True
    np.fill_diagonal(a, False)
    return a, planted


def is_clique(adj: np.ndarray, c) -> bool:
    c = list(c)
    sub = adj[np.ix_(c, c)]
    return bool((sub | np.eye(len(c), dtype=bool)).all())


# ---- step 5: rotation (GNC-TLS) --------------------------------------------------------------------------------------
def weighted_kabsch(a: np.ndarray, b: np.ndarray, w: np.ndarray) -> np.ndarray:
    """R minimising sum w ||b - R a||^2: H = sum w a b^T = U S V^T, R = V diag(1, 1, det(V U^T)) U^T."""
    H = (a * w[:, None]).T @ b
    U, _, Vt = np.linalg.svd(H)
    V = Vt.T
    d = np.linalg.det(V @ U.T)
    return V @ np.diag([1.0, 1.0, d]) @ U.T


def gnc_tls_rotation(a: np.ndarray, b: np.ndarray, nb: float, gnc_factor: float = 1.4, max_iterations: int = 100,
                     cost_threshold: float = 1e-12) -> np.ndarray:
    nb2 = nb * nb
    w = np.ones(len(a))
    prev_cost, mu = 0.0, 1.0
    R = np.eye(3)
    for it in range(max_iterations):
        R = weighted_kabsch(a, b, w)
        d = b - a @ R.T
        r2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        if it == 0:
            mu = 1.0 / (2.0 * r2.max() / nb2 - 1.0)
            if mu <= 0:
                break
        th1 = (mu + 1.0) / mu * nb2
        th2 = mu / (mu + 1.0) * nb2
        cost = float(np.sum(w * r2))
        with np.errstate(divide="ignore", invalid="ignore"):
            mid = np.sqrt(nb2 * mu * (mu + 1.0) / r2) - mu
        w = np.where(r2 > th1, 0.0, np.where(r2 < th2, 1.0, mid))
        mu *= gnc_factor
        if abs(cost - prev_cost) < cost_threshold:
            break
        prev_cost = cost
    return R


# ---- step 5: translation (adaptive voting) ---------------------------------------------------------------------------
def tls_voting(x: np.ndarray, bound: float) -> float:
    """TLS estimate of a scalar: intervals [x_i - bound, x_i + bound]; end points sorted by (value, entering before
    leaving, index) and swept; after every end point the mean of the active set is a candidate with cost
    sum_active (x_i - mean)^2 + n_inactive bound^2 (as sx2 - sx^2 / n + (m - n) bound^2); the first minimum wins."""
    m = len(x)
    ev = sorted([(float(x[i]) - bound, 0, i) for i in range(m)] + [(float(x[i]) + bound, 1, i) for i in range(m)])
    b2 = bound * bound
    sx = sx2 = 0.0
    n = 0
    best, best_cost = 0.0, np.inf
    for _, kind, i in ev:
        xi = float(x[i])
        if kind == 0:
            sx += xi
            sx2 += xi * xi
            n += 1
        else:
            sx -= xi
            sx2 -= xi * xi
            n -= 1
        if n > 0:
            est = sx / n
            cost = (sx2 - sx * est) + (m - n) * b2
            if cost < best_cost:
                best, best_cost = est, cost
    return best


def tls_brute_force(x: np.ndarray, bound: float) -> float:
    """Minimum over every non-empty set of the form {i: |x_i - c| <= bound} of the TLS cost at that set's mean."""
    m = len(x)
    best, best_cost = 0.0, np.inf
    for c in sorted(set(np.concatenate([x - bound, x + bound]).tolist())):
        for eps in (-1e-12, 0.0, 1e-12):
            act = np.abs(x - (c + eps)) <= bound
            if not act.any():
                continue
            mean = x[act].mean()
            cost = np.sum((x[act] - mean) ** 2) + (m - act.sum()) * bound * bound
            if cost < best_cost - 1e-15:
                best, best_cost = mean, cost
    return best


# ---- step 5-6: the solve ---------------------------------------------------------------------------------------------
def solve(src: np.ndarray, tgt: np.ndarray, clique: List[int], noise_bound: float = 0.01, gnc_factor: float = 1.4,
          max_iterations: int = 100, cost_threshold: float = 1e-12):
    """(valid, R, t, num_inliers) for samples src/tgt [m, 3] float32 and a sorted max clique."""
    s = np.asarray(src, np.float32).astype(np.float64)
    t = np.asarray(tgt, np.float32).astype(np.float64)
    if len(clique) <= 1:
        return False, np.eye(3), np.zeros(3), 0
    c = np.asarray(clique)
    nxt = np.roll(c, -1)
    R = gnc_tls_rotation(s[nxt] - s[c], t[nxt] - t[c], 2.0 * noise_bound, gnc_factor, max_iterations, cost_threshold)
    v = t[c] - s[c] @ R.T
    tr = np.array([tls_voting(v[:, j], noise_bound) for j in range(3)])
    p = s @ R.T + tr - t
    n_in = int(np.count_nonzero(np.sqrt((p[:, 0] * p[:, 0] + p[:, 1] * p[:, 1]) + p[:, 2] * p[:, 2]) < noise_bound))
    return True, R, tr, n_in


def refine_one(rendered, measured, K, TCO, mask_type="simple", thresh=0.1, n_min_points=100, n_points=1000,
               noise_bound=0.01, min_num_inliers=50, clique_budget: Optional[int] = None):
    """Steps 2-6 for one prediction with farthest-point sampling: returns (accepted, new TCO float32, info)."""
    src, tgt = masked_clouds(rendered, measured, K, mask_type, thresh)
    TCO = np.asarray(TCO, np.float32)
    if len(src) < n_min_points:
        return False, TCO, dict(reached=False)
    idx = farthest_point_sampling(src, n_points)
    ss, tt = src[idx], tgt[idx]
    clique, _, _ = max_clique(consistency_graph(ss, tt, noise_bound), clique_budget)
    valid, R, tr, n_in = solve(ss, tt, clique, noise_bound)
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, tr
    info = dict(reached=True, valid=valid, T=T, num_inliers=n_in, clique=clique, idx=idx)
    if valid and n_in >= min_num_inliers:
        return True, (T @ TCO.astype(np.float64)).astype(np.float32), info
    return False, TCO, info


def random_graph(n: int, p: float, seed: int) -> np.ndarray:
    r = random.Random(seed)
    a = np.zeros((n, n), bool)
    for i in range(n):
        for j in range(i + 1, n):
            if r.random() < p:
                a[i, j] = a[j, i] = True
    return a
