"""Case builders for the hypothesis-geometry kernels (tests/test_geometry_host.py, tests/test_gpu_geometry.py).

Dyadic cases choose every operand so that each fp32 intermediate of the reference's expression is exact: signed-permutation
rotations, power-of-two focal lengths / depths / box extents / image-size ratios, points, translations and principal
points on a 2^-k grid, lamb 1 or 1.5 (with output sizes 3 * 2^k), ortho6d inputs whose norms are powers of two.  Then the
fp32 result does not depend on rounding or on FMA contraction, and a kernel must equal the float64 restatement bit for
bit.  The CPU test proves that claim for every case by evaluating oracle/geometry_ref.py in float32 and in float64.

Random cases put random operands at the same edges (point counts around warp / block multiples with the extreme point
in the last warp or a thread's second stride, several labels with padded point tables, the 0.1 z clamp, portrait shapes);
they are compared against float64 within the running error bound of geometry_ref.Bounded.
"""
from __future__ import annotations

import itertools

import numpy as np
import torch

from oracle import lib3d_ref

N_PTS = (1, 31, 32, 33, 127, 129, 255, 257, 2000)
# (image (h, w), output (h, w), lamb): landscape and portrait, power-of-two ratios; lamb 1.5 needs sizes 3 * 2^k
DYADIC_SHAPES = (((480, 960), (128, 256), 1.0), ((960, 480), (256, 128), 1.0), ((512, 512), (96, 96), 1.5),
                 ((256, 1024), (96, 192), 1.5), ((1024, 512), (192, 96), 1.5))
RANDOM_SHAPES = (((480, 640), (240, 320), 1.4), ((640, 480), (320, 240), 1.4), ((720, 540), (240, 320), 1.2),
                 ((480, 640), (320, 240), 1.0))


def signed_permutations(rs: np.random.RandomState, n: int) -> np.ndarray:
    perms = list(itertools.permutations(range(3)))
    R = np.zeros((n, 3, 3))
    for i in range(n):
        p = perms[rs.randint(6)]
        s = rs.choice([-1.0, 1.0], 3)
        for r in range(3):
            R[i, r, p[r]] = s[r]
    return R


def pad_points(point_list) -> np.ndarray:
    """[L, N_max, 3] float32 table, shorter meshes padded as MeshDataBase.batched() pads them."""
    return lib3d_ref.pad_stack_points([torch.as_tensor(np.asarray(p, np.float32)) for p in point_list]).numpy()


def extreme_slots(n_pts: int, block: int) -> list:
    """Where a block-strided min/max is easy to get wrong: index 0, the last index (last warp), a thread's second
    stride (i + block) and the last index of the first warp."""
    return sorted({0, n_pts - 1, min(block + 5, n_pts - 1), min(31, n_pts - 1)})


# ---------------------------------------------------------------------------------------------------------------------
# crop geometry
# ---------------------------------------------------------------------------------------------------------------------
def dyadic_crop_case(seed: int, n_pts: int, shape, n: int = 8) -> dict:
    """n hypotheses over two labels (n_pts and fewer points, padded).  Camera-space points are built first: their depth
    is a power of two, so u = (fx X + cx Z) / Z is exact, and one point sits exactly 2^a px from the rendering centre
    (the others closer), so the deepim box and the crop scale are powers of two (times lamb)."""
    (im_h, im_w), out_size, lamb = shape
    rs = np.random.RandomState(seed)
    r = max(im_h, im_w) // min(im_h, im_w)
    R = signed_permutations(rs, n)
    K = np.zeros((n, 3, 3))
    f = 2.0 ** rs.randint(8, 10, n)
    K[:, 0, 0], K[:, 1, 1], K[:, 2, 2] = f, f, 1.0
    K[:, 0, 2] = im_w / 2 + rs.randint(-8, 9, n) / 2
    K[:, 1, 2] = im_h / 2 + rs.randint(-8, 9, n) / 2
    tz = 2.0 ** rs.randint(-1, 2, n)
    t = np.stack([rs.randint(-16, 17, n) / 256, rs.randint(-16, 17, n) / 256, tz], 1)
    tCR = t + np.stack([rs.randint(-4, 5, n) / 256, rs.randint(-4, 5, n) / 256, np.zeros(n)], 1)
    labels = np.arange(n) % 2
    n_lab = [n_pts, max(1, n_pts - 3)]
    tables = [np.zeros((n_lab[0], 3)), np.zeros((n_lab[1], 3))]
    # one pose per label defines the points (the other hypotheses of that label see the same points through their pose)
    for lab in (0, 1):
        i = lab
        cu = (K[i, 0, 0] * tCR[i, 0] + K[i, 0, 2] * tCR[i, 2]) / tCR[i, 2]
        cv = (K[i, 1, 1] * tCR[i, 1] + K[i, 1, 2] * tCR[i, 2]) / tCR[i, 2]
        a = 2.0 ** rs.randint(3, 6)
        y_dominant = rs.rand() < 0.5
        lim_u, lim_v = (a * r, a) if y_dominant else (a, a / r)
        m = n_lab[lab]
        du = rs.randint(-int(lim_u) + 1, int(lim_u), m).astype(float)
        dv = rs.randint(-int(lim_v) + 1, int(lim_v), m).astype(float)
        slots = extreme_slots(m, 128)
        slot = slots[max(0, len(slots) - 1 - lab % 2)]
        if y_dominant:
            dv[slot] = a if rs.rand() < 0.5 else -a
        else:
            du[slot] = a if rs.rand() < 0.5 else -a
        Z = tz[i] * 2.0 ** rs.randint(-1, 2, m)
        X = (cu + du - K[i, 0, 2]) * Z / K[i, 0, 0]
        Y = (cv + dv - K[i, 1, 2]) * Z / K[i, 1, 1]
        C = np.stack([X, Y, Z], 1)
        tables[lab] = (C - t[i]) @ R[i]  # p = R^T (C - t)
    # the other hypotheses of a label: the same pose, so every box is exact (the batch still has n rows)
    for i in range(2, n):
        R[i], t[i], K[i], tCR[i] = R[i % 2], t[i % 2], K[i % 2], tCR[i % 2]
    TCO = np.tile(np.eye(4), (n, 1, 1))
    TCO[:, :3, :3], TCO[:, :3, 3] = R, t
    return dict(points=pad_points(tables), label_idx=labels.astype(np.int32), TCO=TCO.astype(np.float32),
                K=K.astype(np.float32), tCR=tCR.astype(np.float32), lamb=lamb, im_size=(im_h, im_w), out_size=out_size)


def random_rotations(rs: np.random.RandomState, n: int) -> np.ndarray:
    x = torch.as_tensor(rs.randn(n, 6), dtype=torch.float64)
    return lib3d_ref.compute_rotation_matrix_from_ortho6d(x).numpy()


def random_crop_case(seed: int, n_pts: int, shape, n: int = 12, n_labels: int = 3, z_edges: bool = False) -> dict:
    """Random poses and meshes of n_pts, n_pts - 7 and n_pts // 2 points (padded); the extreme point of each label in
    one of extreme_slots().  z_edges: points and tCR on, just under and just over the 0.1 z clamp."""
    (im_h, im_w), out_size, lamb = shape
    rs = np.random.RandomState(seed)
    tables = []
    for lab in range(n_labels):
        m = max(1, (n_pts, n_pts - 7, n_pts // 2)[lab % 3])
        p = rs.uniform(-0.05, 0.05, (m, 3))
        slot = extreme_slots(m, 128)[lab % len(extreme_slots(m, 128))]
        p[slot] = [0.09, -0.08, 0.07]
        tables.append(p)
    points = pad_points(tables)
    R = random_rotations(rs, n)
    t = np.stack([rs.uniform(-0.1, 0.1, n), rs.uniform(-0.1, 0.1, n), rs.uniform(0.3, 1.2, n)], 1)
    K = np.zeros((n, 3, 3))
    K[:, 0, 0] = rs.uniform(400, 1200, n)
    K[:, 1, 1] = K[:, 0, 0] * rs.uniform(0.98, 1.02, n)
    K[:, 0, 2], K[:, 1, 2], K[:, 2, 2] = im_w / 2 + rs.uniform(-20, 20, n), im_h / 2 + rs.uniform(-20, 20, n), 1.0
    tCR = t + rs.uniform(-0.01, 0.01, (n, 3))
    labels = (np.arange(n) % n_labels).astype(np.int32)
    if z_edges:
        # pose 0: one point at camera depth exactly float32(0.1), pose 1 just under, pose 2 just over; tCR likewise
        z01 = np.float32(0.1)
        for i, z in enumerate((float(z01), float(np.nextafter(z01, np.float32(0))), float(np.nextafter(z01, np.float32(1))))):
            R[i] = np.eye(3)
            points[labels[i], 0, 2] = 0.0  # this point's camera depth is t_z exactly
            t[i, 2] = z
            tCR[i] = [0.01, -0.01, z]
        for i in (3, 4):  # far behind the clamp
            t[i, 2] = 0.02
            tCR[i, 2] = -0.3
    TCO = np.tile(np.eye(4), (n, 1, 1))
    TCO[:, :3, :3], TCO[:, :3, 3] = R, t
    return dict(points=points.astype(np.float32), label_idx=labels, TCO=TCO.astype(np.float32), K=K.astype(np.float32),
                tCR=tCR.astype(np.float32), lamb=lamb, im_size=(im_h, im_w), out_size=out_size)


# ---------------------------------------------------------------------------------------------------------------------
# pose init
# ---------------------------------------------------------------------------------------------------------------------
def dyadic_pose_init_case(seed: int, n_pts: int, n: int = 8) -> dict:
    """Boxes with power-of-two extent + 1 (bb_dx = 2^k, among them bb_dx = 1: a zero-width box), points on a 2^-8 grid,
    signed-permutation rotations; two labels with padded point tables."""
    rs = np.random.RandomState(seed)
    tables = [rs.randint(-24, 25, (max(1, m), 3)) / 256 for m in (n_pts, n_pts - 5)]
    R = signed_permutations(rs, n)
    K = np.zeros((n, 3, 3))
    f = 2.0 ** rs.randint(8, 11, n)
    K[:, 0, 0], K[:, 1, 1], K[:, 2, 2] = f, f, 1.0
    K[:, 0, 2], K[:, 1, 2] = 320 + rs.randint(-8, 9, n) / 2, 240 + rs.randint(-8, 9, n) / 2
    bb = np.zeros((n, 4))
    bb[:, 0], bb[:, 1] = rs.randint(100, 300, n) / 2, rs.randint(100, 300, n) / 2
    wx, wy = 2.0 ** rs.randint(0, 8, n), 2.0 ** rs.randint(0, 8, n)
    wx[0] = 1.0  # zero-width box: x2 == x1
    bb[:, 2], bb[:, 3] = bb[:, 0] + wx - 1, bb[:, 1] + wy - 1
    return dict(points=pad_points(tables), label_idx=(np.arange(n) % 2).astype(np.int32), bboxes=bb.astype(np.float32),
                K=K.astype(np.float32), R=R.astype(np.float32))


def random_pose_init_case(seed: int, n_pts: int, n: int = 16, n_labels: int = 3) -> dict:
    rs = np.random.RandomState(seed)
    tables = []
    for lab in range(n_labels):
        m = max(1, (n_pts, n_pts - 7, n_pts // 2)[lab % 3])
        p = rs.uniform(-0.05, 0.05, (m, 3))
        p[extreme_slots(m, 256)[lab % len(extreme_slots(m, 256))]] = [0.08, 0.09, -0.07]
        tables.append(p)
    K = np.zeros((n, 3, 3))
    K[:, 0, 0] = rs.uniform(400, 1200, n)
    K[:, 1, 1] = K[:, 0, 0] * rs.uniform(0.98, 1.02, n)
    K[:, 0, 2], K[:, 1, 2], K[:, 2, 2] = rs.uniform(300, 340, n), rs.uniform(220, 260, n), 1.0
    x1, y1 = rs.uniform(0, 500, n), rs.uniform(0, 350, n)
    bb = np.stack([x1, y1, x1 + rs.uniform(2, 200, n), y1 + rs.uniform(2, 200, n)], 1)
    return dict(points=pad_points(tables), label_idx=(np.arange(n) % n_labels).astype(np.int32), bboxes=bb.astype(np.float32),
                K=K.astype(np.float32), R=random_rotations(rs, n).astype(np.float32))


# ---------------------------------------------------------------------------------------------------------------------
# ortho6d inputs: pose update, normalize_T
# ---------------------------------------------------------------------------------------------------------------------
def dyadic_ortho6d(rs: np.random.RandomState, n: int):
    """x_raw = 2^j * (signed unit axis), y_raw = 2^k * (another signed axis) + c * x (dyadic c): the normalised x, z and
    y are exact signed axes."""
    Rp = signed_permutations(rs, n)
    xr = Rp[:, :, 0] * (2.0 ** rs.randint(-2, 3, n))[:, None]
    yr = Rp[:, :, 1] * (2.0 ** rs.randint(-2, 3, n))[:, None] + Rp[:, :, 0] * (rs.randint(-8, 9, n) / 8)[:, None]
    return xr, yr


def dyadic_pose_update_case(seed: int, n: int = 64) -> dict:
    rs = np.random.RandomState(seed)
    xr, yr = dyadic_ortho6d(rs, n)
    pose9 = np.concatenate([xr, yr, rs.randint(-16, 17, (n, 2)) / 8, (2.0 ** rs.randint(-1, 2, n))[:, None]], 1)
    TCO = np.tile(np.eye(4), (n, 1, 1))
    TCO[:, :3, :3] = signed_permutations(rs, n)
    TCO[:, :3, 3] = np.stack([rs.randint(-32, 33, n) / 256, rs.randint(-32, 33, n) / 256, 2.0 ** rs.randint(-1, 2, n)], 1)
    TCO[:, 3] = rs.randint(-4, 5, (n, 4)) / 4  # a non-identity bottom row: the reference clones TCO, so it is kept
    tCR = TCO[:, :3, 3] + np.stack([rs.randint(-4, 5, n) / 256, rs.randint(-4, 5, n) / 256, np.zeros(n)], 1)
    K = np.zeros((n, 3, 3))
    f = 2.0 ** rs.randint(8, 11, n)
    K[:, 0, 0], K[:, 1, 1], K[:, 0, 2], K[:, 1, 2], K[:, 2, 2] = f, f * 2, 160, 120, 1
    return dict(TCO=TCO.astype(np.float32), K_crop=K.astype(np.float32), pose9=pose9.astype(np.float32),
                tCR=tCR.astype(np.float32))


def random_pose_update_case(seed: int, n: int = 300) -> dict:
    rs = np.random.RandomState(seed)
    pose9 = rs.randn(n, 9)
    pose9[:, 8] = 1 + 0.05 * pose9[:, 8]
    pose9[:, 6:8] *= 4
    TCO = np.tile(np.eye(4), (n, 1, 1))
    TCO[:, :3, :3] = random_rotations(rs, n)
    TCO[:, :3, 3] = np.stack([rs.uniform(-0.1, 0.1, n), rs.uniform(-0.1, 0.1, n), rs.uniform(0.3, 1.5, n)], 1)
    TCO[5, 3] = [0.25, -0.5, 0.125, 2.0]
    tCR = TCO[:, :3, 3] + rs.uniform(-0.01, 0.01, (n, 3))
    K = np.zeros((n, 3, 3))
    K[:, 0, 0], K[:, 1, 1] = rs.uniform(300, 3000, n), rs.uniform(300, 3000, n)
    K[:, 0, 2], K[:, 1, 2], K[:, 2, 2] = 160, 120, 1
    return dict(TCO=TCO.astype(np.float32), K_crop=K.astype(np.float32), pose9=pose9.astype(np.float32),
                tCR=tCR.astype(np.float32))


def dyadic_normalize_case(seed: int, n: int = 64) -> np.ndarray:
    rs = np.random.RandomState(seed)
    xr, yr = dyadic_ortho6d(rs, n)
    T = np.zeros((n, 4, 4))
    T[:, :3, 0], T[:, :3, 1] = xr, yr
    T[:, :3, 2] = rs.randint(-8, 9, (n, 3)) / 8  # ignored by normalize_T
    T[:, :3, 3] = rs.randint(-64, 65, (n, 3)) / 64
    T[:, 3] = rs.randint(-4, 5, (n, 4)) / 4      # replaced by (0, 0, 0, 1)
    return T.astype(np.float32)


def random_normalize_case(seed: int, n: int = 300) -> np.ndarray:
    rs = np.random.RandomState(seed)
    T = np.tile(np.eye(4), (n, 1, 1))
    T[:, :3, :3] = random_rotations(rs, n) + 0.02 * rs.randn(n, 3, 3)
    T[:, :3, 3] = rs.randn(n, 3)
    return T.astype(np.float32)
