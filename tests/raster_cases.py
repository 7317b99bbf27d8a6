"""Case builders for the float64 rasteriser tests (tests/test_raster_f64_host.py, tests/test_gpu_raster_f64.py), and a
restatement of the rasteriser's dispatch and per-triangle path choice (megapose6d_b200/csrc/raster.cu: raster_launch,
cover_triangle, raster_tiled_kernel) computed from the snapped integer coordinates.

Dyadic cases choose every operand so that the fp32 vertex stage is exact: signed-permutation rotations, power-of-two
depths and focal lengths, screen positions on the 1/256 px grid.  Every snapped vertex then equals its float64
projection, and coverage and the winning triangle must equal the float64 statement on every pixel.  Where a case also
needs exact 1/z interpolation (ties on shared edges, the depth window at 10 and 0.1) its triangles have power-of-two
areas and its samples fall on vertices and edge midpoints.  The near and far plane cases put vertices at 2^k z for the
fp32 depth z whose reciprocal rounds to 10.0f (0.1f), or to 0.1f (10.0f), and at the next fp32 depth on either side:
x * (1/z) still rounds to 2^k.

Random cases put random triangles at the same edges: more large triangles than one CTA's queue holds, tall images with
rows up to 4094 in the tiled kernel's 12-bit row fields, 128 and 129 strips, 16 and 15 rows per strip, 1 x W, H x 1 and
odd sizes, projections beyond the 2^20 px clamp, and a 10k-triangle mesh at random poses.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List

import numpy as np

SUB = 256
SMALL_EXT = 16384
BIG_AREA = 1024
BIG_QUEUE = 2048
TILE_MIN_ROWS, TILE_MAX_STRIPS, TILE_THREADS, REC_FIELDS = 16, 128, 512, 16
COVER_THREADS, MAX_PARTS = 256, 40


@dataclass
class Case:
    name: str
    meshes: List[dict]            # verts, normals, colors [nv,3] float32, faces [nf,3] int32
    labels: np.ndarray            # [n] int32
    TCO: np.ndarray               # [n,4,4] float32
    K: np.ndarray                 # [n,3,3] float32
    h: int
    w: int
    dyadic: bool
    sm_limit: int = 0             # mesh database created and rendered under mpx_set_sm_limit
    batches: tuple = (1, 17)      # view batch sizes the GPU test renders (views repeated cyclically; at least every view)
    notes: dict = field(default_factory=dict)

    def __post_init__(self):
        self.batches = tuple(max(b, len(self.labels)) for b in self.batches)

    def view(self, i):
        m = self.meshes[int(self.labels[i])]
        return m, self.TCO[i], self.K[i]


def _mesh(verts, faces, colors=None, normals=None, seed=0):
    rs = np.random.RandomState(seed)
    verts = np.asarray(verts, np.float64)
    n = len(verts)
    if colors is None:
        colors = rs.randint(0, 256, (n, 3)) / 256.0
    if normals is None:
        normals = rs.randn(n, 3)
        normals /= np.linalg.norm(normals, axis=1, keepdims=True)
    return dict(verts=np.ascontiguousarray(verts, np.float32), faces=np.ascontiguousarray(faces, np.int32),
                colors=np.ascontiguousarray(colors, np.float32), normals=np.ascontiguousarray(normals, np.float32))


def _K(f, cx, cy, fy=None):
    return np.array([[f, 0, cx], [0, f if fy is None else fy, cy], [0, 0, 1]], np.float32)


def _T(R=None, t=(0, 0, 0)):
    T = np.eye(4)
    if R is not None:
        T[:3, :3] = R
    T[:3, 3] = t
    return T.astype(np.float32)


def _model_from_screen(uvz, K, T):
    """Model-frame vertices whose camera points project to screen (u, v) at depth z (float64; exact for dyadic input)."""
    uvz = np.asarray(uvz, np.float64)
    z = uvz[:, 2]
    Pc = np.stack([(uvz[:, 0] - K[0, 2]) * z / K[0, 0], (uvz[:, 1] - K[1, 2]) * z / K[1, 1], z], 1)
    T = np.asarray(T, np.float64)
    return (Pc - T[:3, 3]) @ T[:3, :3]


# ---------------------------------------------------------------------------------------------------------------------
# dyadic cases
# ---------------------------------------------------------------------------------------------------------------------
SIGNED_PERMS = [np.eye(3), np.diag([-1.0, -1.0, 1.0]), np.array([[0, 1.0, 0], [1.0, 0, 0], [0, 0, -1.0]]),
                np.diag([-1.0, 1.0, -1.0])]


def fan_grid_case() -> Case:
    """4-px squares with vertices on pixel centres, split along alternating diagonals (fans around every other vertex),
    fronto-parallel at z = 1/2: samples on edges, shared edges and vertices, power-of-two areas.  Two faces have
    coplanar duplicates (new vertices, other colours), one listed after and one before its original."""
    h, w = 48, 64
    K = _K(512.0, 32.0, 24.0)
    T = _T(SIGNED_PERMS[2], (0.0625, -0.125, 0.25))
    uvz, faces = [], []
    nx, ny = 10, 8
    for gy in range(ny + 1):
        for gx in range(nx + 1):
            uvz.append((gx * 4 + 10.5, gy * 4 + 7.5, 0.5))
    vid = lambda gx, gy: gy * (nx + 1) + gx  # noqa: E731
    for gy in range(ny):
        for gx in range(nx):
            a, b, c, d = vid(gx, gy), vid(gx + 1, gy), vid(gx + 1, gy + 1), vid(gx, gy + 1)
            if (gx + gy) % 2 == 0:
                faces += [[a, b, c], [a, c, d]]
            else:
                faces += [[a, b, d], [b, c, d]]
    faces = np.array(faces)
    n0 = len(uvz)
    # duplicates: face 13 followed by its copy, face 40 preceded by its copy
    dup = lambda f: [n0 + k for k in range(3)] if f == 13 else [n0 + 3 + k for k in range(3)]  # noqa: E731
    uvz += [uvz[i] for i in faces[13]] + [uvz[i] for i in faces[40]]
    faces = np.concatenate([faces[:14], [dup(13)], faces[14:40], [dup(40)], faces[40:]])
    verts = _model_from_screen(uvz, K, T)
    return Case("dyadic_fan_grid", [_mesh(verts, faces, seed=1)], np.zeros(1, np.int32), T[None], K[None], h, w, True)


def extent_case() -> Case:
    """Right triangles whose snapped extents are 16384 (the last 32-bit walk) and 16385 (64-bit) sub-pixels in x, in y
    and in both; the far corner of each bounding box holds the largest edge value.  Vertex depths 1/2, 1, 2 (perspective-
    correct attributes).  Three views: the second rotates the camera by 180 degrees about its axis, moving the right
    angles (and the largest edge values) to the opposite corners and keeping the winding; a third mirrors x (winding
    flipped: two-sided)."""
    h, w = 160, 160
    K = _K(256.0, 80.0, 80.0)
    uvz, faces = [], []
    spec = [(SMALL_EXT, SMALL_EXT), (SMALL_EXT + 1, SMALL_EXT), (SMALL_EXT, SMALL_EXT + 1), (SMALL_EXT + 1, SMALL_EXT + 1)]
    origins = [(2 * SUB + 128, 2 * SUB + 128), (78 * SUB + 128, 3 * SUB + 77), (3 * SUB + 1, 78 * SUB + 128),
               (80 * SUB + 128, 80 * SUB + 128)]
    for (ex, ey), (ox, oy) in zip(spec, origins):
        base = len(uvz)
        uvz += [(ox / SUB, oy / SUB, 1.0), ((ox + ex) / SUB, oy / SUB, 0.5), (ox / SUB, (oy + ey) / SUB, 2.0)]
        faces.append([base, base + 1, base + 2])
    T0 = _T(np.eye(3), (0.0, 0.0, 0.5))
    verts = _model_from_screen(uvz, K, T0)
    # camera 2: rotate 180 degrees about the optical axis around the image centre (cx, cy map onto themselves)
    T1 = _T(np.diag([-1.0, -1.0, 1.0]), (0.0, 0.0, 0.5))
    T2 = _T(np.diag([-1.0, 1.0, 1.0]), (0.0, 0.0, 0.5))
    TCO = np.stack([T0, T1, T2])
    return Case("dyadic_extent_16384", [_mesh(verts, faces, seed=2)], np.zeros(3, np.int32), TCO, np.stack([K] * 3),
                h, w, True)


def box_area_case() -> Case:
    """Right triangles with vertices on pixel centres whose bounding boxes hold exactly 1023, 1024 (the last per-thread
    box) and 1025 pixels (the first CTA-wide one)."""
    h, w = 96, 128
    K = _K(128.0, 64.0, 48.0)
    T = _T(SIGNED_PERMS[1], (0.125, 0.0, 1.0))
    uvz, faces = [], []
    for (bw, bh), (x0, y0) in zip([(32, 32), (41, 25), (25, 41), (31, 33)], [(2, 2), (40, 2), (90, 2), (2, 50)]):
        base = len(uvz)
        uvz += [(x0 + 0.5, y0 + 0.5, 1.0), (x0 + bw - 0.5, y0 + 0.5, 1.0), (x0 + 0.5, y0 + bh - 0.5, 0.5)]
        faces.append([base, base + 1, base + 2])
    verts = _model_from_screen(uvz, K, T)
    return Case("dyadic_box_area_1024", [_mesh(verts, faces, seed=3)], np.zeros(1, np.int32), T[None], K[None], h, w, True)


def proj_min_case() -> Case:
    """A triangle with a vertex at camera z = 2^-10 (projectable: 1/z = 1024 there, so only its far edge, at 1/z = 1/2, is
    inside the depth window and drawn) and the same triangle elsewhere with that vertex at the next fp32 depth below
    (not projectable: dropped)."""
    h, w = 64, 96
    K = _K(64.0, 48.0, 32.0)
    zmin = np.float32(2.0 ** -10)
    below = np.nextafter(zmin, np.float32(0))
    P = []
    for zc, un, xf in ((float(zmin), 0.5, 40.5), (float(below), 50.5, 90.5)):
        P += [[(un - 48.0) * zc / 64.0, 0.0, zc], [(xf - 48.0) * 2.0 / 64.0, (2.5 - 32.0) * 2.0 / 64.0, 2.0],
              [(xf - 48.0) * 2.0 / 64.0, (61.5 - 32.0) * 2.0 / 64.0, 2.0]]
    faces = [[0, 1, 2], [3, 4, 5]]
    T = _T()
    return Case("dyadic_proj_min", [_mesh(np.asarray(P), faces, seed=4)], np.zeros(1, np.int32), T[None], K[None], h, w,
                True)


def _plane_patch(z: float, K, seed: int):
    """8 triangles with 2-px legs around (cx, cy) on the plane at fp32 depth z: camera x, y in {0, +-2^-7 z}, so that
    fp32 x * (1/z) rounds to +-2^-7 and u = cx + 256 x/z lands on pixel centres; every sample is a vertex or an edge
    midpoint (barycentrics 0, 1/2, 1: 1/z interpolates exactly)."""
    zf = np.float32(z)
    s = np.float32(2.0 ** -7) * zf
    g = [-float(s), 0.0, float(s)]
    verts = [[x, y, 0.0] for y in g for x in g]
    faces = []
    for gy in range(2):
        for gx in range(2):
            a, b, c, d = gy * 3 + gx, gy * 3 + gx + 1, (gy + 1) * 3 + gx + 1, (gy + 1) * 3 + gx
            faces += [[a, b, c], [a, c, d]] if (gx + gy) % 2 == 0 else [[a, b, d], [b, c, d]]
    return _mesh(verts, faces, seed=seed), _T(np.eye(3), (0.0, 0.0, float(zf)))


def depth_window_case(near: bool) -> Case:
    """Fronto-parallel patches at the fp32 depth whose reciprocal rounds to 10.0f (near) or 0.1f (far), and at the next
    fp32 depth on either side: drawn / rejected / drawn in the order below, at, above for the near plane (1/z > 10 is
    rejected), drawn / rejected for the far plane above it."""
    z0 = np.float32(0.1) if near else np.float32(10.0)
    zs = [np.nextafter(z0, np.float32(0)), z0, np.nextafter(z0, np.float32(np.inf))]
    K = _K(256.0, 16.5, 12.5)
    meshes, TCO = [], []
    for k, z in enumerate(zs):
        m, T = _plane_patch(float(z), K, seed=10 + k)
        meshes.append(m)
        TCO.append(T)
    name = "dyadic_near_plane" if near else "dyadic_far_plane"
    return Case(name, meshes, np.arange(3, dtype=np.int32), np.stack(TCO), np.stack([K] * 3), 24, 32, True,
                notes=dict(z=[float(z) for z in zs]))


def dyadic_cases() -> List[Case]:
    return [fan_grid_case(), extent_case(), box_area_case(), proj_min_case(), depth_window_case(True),
            depth_window_case(False)]


# ---------------------------------------------------------------------------------------------------------------------
# random cases
# ---------------------------------------------------------------------------------------------------------------------
def _rotation(rs):
    q = rs.randn(4)
    q /= np.linalg.norm(q)
    a, b, c, d = q
    return np.array([[a * a + b * b - c * c - d * d, 2 * (b * c - a * d), 2 * (b * d + a * c)],
                     [2 * (b * c + a * d), a * a - b * b + c * c - d * d, 2 * (c * d - a * b)],
                     [2 * (b * d - a * c), 2 * (c * d + a * b), a * a - b * b - c * c + d * d]])


def _soup(rs, n, h, w, size, z_range=(0.3, 2.0), margin=8.0):
    """n independent triangles in screen space: centres uniform over the image (plus a margin), vertices within `size`
    pixels of them, random vertex depths.  Returns uvz [3n,3], faces [n,3]."""
    cx = rs.uniform(-margin, w + margin, n)
    cy = rs.uniform(-margin, h + margin, n)
    uvz = np.zeros((n, 3, 3))
    sz = np.broadcast_to(np.asarray(size, np.float64), (2,))
    uvz[:, :, 0] = cx[:, None] + rs.uniform(-1, 1, (n, 3)) * sz[0]
    uvz[:, :, 1] = cy[:, None] + rs.uniform(-1, 1, (n, 3)) * sz[1]
    uvz[:, :, 2] = rs.uniform(*z_range, (n, 3))
    return uvz.reshape(-1, 3), np.arange(3 * n).reshape(n, 3)


def _random_view(rs, h, w, f=300.0):
    K = _K(f + rs.uniform(0, 1), w / 2 + rs.uniform(-1, 1), h / 2 + rs.uniform(-1, 1), fy=f + rs.uniform(0, 1))
    T = np.eye(4)
    T[:3, :3] = _rotation(rs)
    T[:3, 3] = rs.uniform(-0.1, 0.1, 3)
    return K, T.astype(np.float32)


def soup_case(name, h, w, n, size, seed, n_views=1, batches=(1, 17), z_range=(0.3, 2.0), extra=None) -> Case:
    rs = np.random.RandomState(seed)
    meshes, Ks, Ts = [], [], []
    for v in range(n_views):
        K, T = _random_view(rs, h, w)
        uvz, faces = _soup(rs, n, h, w, size, z_range)
        if extra is not None:
            e_uvz, e_faces = extra(rs, K)
            faces = np.concatenate([faces, e_faces + len(uvz)])
            uvz = np.concatenate([uvz, e_uvz])
        meshes.append(_mesh(_model_from_screen(uvz, K, T), faces, seed=seed + v))
        Ks.append(K)
        Ts.append(T)
    return Case(name, meshes, np.arange(n_views, dtype=np.int32), np.stack(Ts), np.stack(Ks), h, w, False,
                batches=batches)


def queue_case() -> Case:
    """Under mpx_set_sm_limit(16): the scatter kernel spreads one view over 16 CTAs, CTA p taking triangles t with
    (t // 256) % 16 == p.  CTA 0 gets 2304 triangles with boxes over 1024 px (256 more than its queue holds), CTA 1
    exactly 2048; every other triangle is degenerate.  At 32 views (one whole view per CTA) the untiled kernel queues all
    4352 of them in each CTA."""
    rs = np.random.RandomState(7)
    h, w = 64, 80
    K, T = _random_view(rs, h, w, f=200.0)
    n = 9 * 16 * 256
    t = np.arange(n)
    part = (t // 256) % 16
    big = (part == 0) | ((part == 1) & (t < 8 * 4096))
    uvz = np.zeros((n, 3, 3))
    nb = int(big.sum())
    cxy = np.stack([rs.uniform(17, w - 17, nb), rs.uniform(17, h - 17, nb)], 1)
    off = rs.uniform(-1, 1, (nb, 3, 2)) * 16.5            # boxes of 33 x 33 px or more (over 1024 px) inside the image
    off[:, 0] = -16.5
    off[:, 1, 0] = 16.5
    off[:, 2, 1] = 16.5
    uvz[big, :, :2] = cxy[:, None] + off
    uvz[big, :, 2] = rs.uniform(0.4, 3.0, (nb, 3))
    uvz[~big, :, :2] = rs.uniform(0, w, (n - nb, 1, 2))      # three equal points: area 0, dropped
    uvz[~big, :, 2] = 1.0
    faces = np.arange(3 * n).reshape(n, 3)
    m = _mesh(_model_from_screen(uvz.reshape(-1, 3), K, T), faces, seed=7)
    return Case("random_queue_overflow", [m], np.zeros(1, np.int32), T[None], K[None], h, w, False, sm_limit=16,
                batches=(1, 32), notes=dict(big=big))


def clamp_extra(rs, K):
    """Triangles with one vertex 1.5 mm in front of the eye plane and 6-12 m off axis: its projection lies beyond the
    2^20 px clamp, the other two are on screen (and only the part of the triangle beyond the near plane is drawn)."""
    uvz, faces = [], []
    for k in range(6):
        base = len(uvz)
        z = 0.0015
        X = rs.choice([-1, 1]) * rs.uniform(6.0, 12.0)
        u = K[0, 0] * X / z + K[0, 2]
        uvz += [(u, rs.uniform(0, 240), z), (rs.uniform(40, 280), rs.uniform(20, 220), 0.5),
                (rs.uniform(40, 280), rs.uniform(20, 220), 0.6)]
        faces.append([base, base + 1, base + 2])
    return np.asarray(uvz), np.asarray(faces)


def mesh_case() -> Case:
    """A 10k-triangle bumpy sphere at four random poses, 240x320, with smooth vertex normals and colours."""
    from megapose6d_b200 import procedural

    m = procedural.bumpy_sphere().with_defaults()
    v = np.asarray(m.vertices)
    mesh = _mesh(v, np.asarray(m.faces), colors=0.5 + 0.45 * v / np.abs(v).max(0), normals=np.asarray(m.vertex_normals))
    T = procedural.random_poses(4, 9, z_range=(0.25, 0.5), xy_range=0.03).astype(np.float32)
    K = np.stack([_K(600.0 + k, 160.3, 119.7) for k in range(4)])
    return Case("random_mesh_10k", [mesh], np.zeros(4, np.int32), T, K, 240, 320, False, batches=(4, 17))


def random_cases() -> List[Case]:
    return [
        mesh_case(),
        queue_case(),
        soup_case("random_tiled_4095x64", 4095, 64, 3000, (20.0, 36.0), 11,
                  extra=lambda rs, K: (np.array([[8.5, 3000.0, 1.0], [60.5, 3000.0, 1.0], [30.0, 3090.0, 1.2]]),
                                       np.array([[0, 1, 2]]))),
        soup_case("random_untiled_4096x16", 4096, 16, 1500, (8.0, 30.0), 12),
        soup_case("random_strips_128", 2048, 607, 4000, (10.0, 33.0), 13),
        soup_case("random_strips_129", 2049, 607, 4000, (10.0, 33.0), 14),
        soup_case("random_rows_16", 240, 607, 1500, (10.0, 20.0), 15),
        soup_case("random_rows_15", 240, 608, 1500, (10.0, 20.0), 16),
        soup_case("random_1x320", 1, 320, 200, (6.0, 3.0), 17),
        soup_case("random_240x1", 240, 1, 200, (3.0, 6.0), 18),
        soup_case("random_37x53", 37, 53, 300, (5.0, 5.0), 19),
        soup_case("random_clamp", 240, 320, 400, (10.0, 10.0), 20, extra=clamp_extra),
    ]


# ---------------------------------------------------------------------------------------------------------------------
# restatement of raster_launch and of the per-triangle path choice
# ---------------------------------------------------------------------------------------------------------------------
def dispatch(h, w, n_views, sm, slots, mode=7, cap_slots=True):
    """The kernel raster_launch picks, and its decomposition.  `cap_slots`: the untiled grid is capped at
    min(slots, 2 sm) (False: the grid of the parent, capped at slots alone)."""
    if (mode & 1) and n_views * 8 <= sm:
        parts = min(MAX_PARTS, sm // n_views)
        return dict(kernel="scatter", parts=parts)
    if (mode & 4) and h < 4096 and w < 4096:
        fixed = (REC_FIELDS * TILE_THREADS + TILE_THREADS + 1) * 4 + 16
        R = (110 * 1024 - fixed) // (8 * w)
        R = min(R, h)
        if R >= TILE_MIN_ROWS:
            ns = -(-h // R)
            R = -(-h // ns)
            ns = -(-h // R)
            if ns <= TILE_MAX_STRIPS and R >= TILE_MIN_ROWS:
                groups = slots // n_views if n_views < slots else 1
                groups = min(groups, ns)
                return dict(kernel="tiled", R=R, n_strips=ns, groups=groups, grid=min(n_views * groups, slots))
    s = min(slots, 2 * sm) if cap_slots else slots
    strips = min(16, s // n_views, h) if n_views < s else 1
    return dict(kernel="untiled", strips=strips, grid=min(n_views * strips, s))


def snapped_triangles(mesh, TCO, K, h, w):
    """Per triangle of one view: ok, clipped bounding box (j0, j1, i0, i1) and snapped extents."""
    from oracle.raster_f64 import snap_f32

    X, Y, _, behind = snap_f32(mesh["verts"], TCO, K)
    f = mesh["faces"].astype(np.int64)
    xa, ya = X[f], Y[f]
    area2 = (xa[:, 1] - xa[:, 0]) * (ya[:, 2] - ya[:, 0]) - (ya[:, 1] - ya[:, 0]) * (xa[:, 2] - xa[:, 0])
    ok = (area2 != 0) & ~behind[f].any(1)
    j0 = np.maximum(0, -((-(xa.min(1) - 128)) // SUB))
    j1 = np.minimum(w - 1, (xa.max(1) - 128) // SUB)
    i0 = np.maximum(0, -((-(ya.min(1) - 128)) // SUB))
    i1 = np.minimum(h - 1, (ya.max(1) - 128) // SUB)
    return dict(ok=ok, j0=j0, j1=j1, i0=i0, i1=i1, ext_x=xa.max(1) - xa.min(1), ext_y=ya.max(1) - ya.min(1),
                clamped=(np.abs(X) >= (1 << 28)) | (np.abs(Y) >= (1 << 28)), behind=behind)


def triangle_paths(case: Case, n_views: int, sm: int, slots: int, mode: int = 7) -> dict:
    """Which paths the triangles of `case` take when it is rendered `n_views` views at a time (views repeated).  Returns
    the dispatch and a dict of observations: path labels hit, the queue counts of the CTAs, extents and box areas
    met on each side of their thresholds, the largest tiled row, the strip spans."""
    d = dispatch(case.h, case.w, n_views, sm, slots, mode)
    obs = dict(paths=set(), queue=set(), ext_le=False, ext_gt_x=False, ext_gt_y=False, area=set(), max_row=-1,
               max_span=0)
    h, w = case.h, case.w
    for v in range(min(n_views, len(case.labels))):
        m, T, K = case.view(v)
        t = snapped_triangles(m, T, K, h, w)
        ok = t["ok"] & (t["j0"] <= t["j1"]) & (t["i0"] <= t["i1"])
        ex, ey = t["ext_x"], t["ext_y"]
        small = (ex <= SMALL_EXT) & (ey <= SMALL_EXT)
        obs["ext_le"] |= bool((ok & small & ((ex == SMALL_EXT) | (ey == SMALL_EXT))).any())
        obs["ext_gt_x"] |= bool((ok & (ex == SMALL_EXT + 1)).any())
        obs["ext_gt_y"] |= bool((ok & (ey == SMALL_EXT + 1)).any())
        idx = np.nonzero(ok)[0]
        if d["kernel"] == "tiled":
            R = d["R"]
            big = ~small[idx]
            if big.any():
                obs["paths"].add("tiled-big")
            if (~big).any():
                obs["paths"].add("tiled-small")
                span = t["i1"][idx][~big] // R - t["i0"][idx][~big] // R + 1
                obs["max_span"] = max(obs["max_span"], int(span.max()))
                if span.max() > 1:
                    obs["paths"].add("strip-span")
            obs["max_row"] = max(obs["max_row"], int(t["i1"][idx].max()) if idx.size else -1)
            continue
        if d["kernel"] == "scatter":
            items = [(np.nonzero(((idx // COVER_THREADS) % d["parts"]) == p)[0], 0, h - 1) for p in range(d["parts"])]
        else:
            rows = -(-h // d["strips"])
            items = [(np.arange(idx.size), s * rows, min(h, s * rows + rows) - 1) for s in range(d["strips"])]
        for sel, lo, hi in items:
            tri = idx[sel]
            i0 = np.maximum(t["i0"][tri], lo)
            i1 = np.minimum(t["i1"][tri], hi)
            live = i0 <= i1
            area = (t["j1"][tri] - t["j0"][tri] + 1) * (i1 - i0 + 1)
            obs["area"] |= set(int(a) for a in np.unique(area[live]) if BIG_AREA - 1 <= a <= BIG_AREA + 1)
            big = live & (area > BIG_AREA)
            nq = int(big.sum())
            obs["queue"].add(nq)
            if nq:
                obs["paths"].add("queued")
            if nq > BIG_QUEUE:
                obs["paths"].add("queue-full")
            walk = live & (~big | (nq > BIG_QUEUE))
            if (walk & small[tri]).any():
                obs["paths"].add("walk32")
            if (walk & ~small[tri]).any():
                obs["paths"].add("walk64")
    return dict(dispatch=d, **obs)


# ---------------------------------------------------------------------------------------------------------------------
# references
# ---------------------------------------------------------------------------------------------------------------------
def ref_render(mesh, TCO, K, h, w, flags=1):
    """One view through oracle/raster_ref.c (raster_ref_render): rgb, normals [3,h,w], depth [h,w], tri_id [h,w]."""
    import ctypes

    from oracle import pipeline_ref

    lib = pipeline_ref.raster_lib()
    out = dict(rgb=np.zeros((3, h, w), np.float32), nrm=np.zeros((3, h, w), np.float32),
               depth=np.zeros((h, w), np.float32), tri=np.zeros((h, w), np.int32))
    arr = [np.ascontiguousarray(a) for a in (mesh["verts"], mesh["normals"], mesh["colors"], mesh["faces"],
                                             np.asarray(TCO, np.float32), np.asarray(K, np.float32))]
    p = [a.ctypes.data_as(ctypes.c_void_p) for a in arr]
    o = [out[k].ctypes.data_as(ctypes.c_void_p) for k in ("rgb", "nrm", "depth", "tri")]
    rc = lib.raster_ref_render(p[0], p[1], p[2], ctypes.c_int(len(arr[0])), p[3], ctypes.c_int(len(arr[3])), p[4], p[5],
                               ctypes.c_int(h), ctypes.c_int(w), ctypes.c_uint(flags), *o)
    assert rc == 0
    return out


_CACHE = {}


def rendered(case: Case, v: int, flags: int = 1):
    """(raster_ref.c render, float64 render) of view v of `case`, computed once per process."""
    from oracle import raster_f64

    key = (case.name, v, flags)
    if key not in _CACHE:
        m, T, K = case.view(v)
        _CACHE[key] = (ref_render(m, T, K, case.h, case.w, flags),
                       raster_f64.render(m["verts"], m["normals"], m["colors"], m["faces"], T, K, case.h, case.w, flags))
    return _CACHE[key]
