"""oracle/geometry_ref.py -- numpy restatement of the hypothesis-geometry kernels (megapose6d_b200/csrc/geom.cu).

TEST INFRASTRUCTURE ONLY.  Nothing under megapose6d_b200/ may import this module.

Each function spells out the reference's expression in the reference's operation order (paths relative to
src/megapose), one scalar operation at a time, so that the same code runs in three number systems:

  * float64 numpy arrays: the high-precision value the kernels are compared against;
  * float32 numpy arrays: every operation rounded to fp32 (no fused multiply-add).  On the dyadic cases of
    tests/geometry_cases.py this equals the float64 result bit for bit, which proves that every intermediate is exact;
  * `Bounded` values: the float64 value together with a running bound on the error of ANY fp32 evaluation of the same
    expression, contracted into FMAs or not (see `Bounded`).

The operands are what the kernels receive: fp32 tensors, plus the reference's fp32 constants (the 0.1 z clamp is
float32(0.1), as torch multiplies it into a float32 tensor).  `lib3d_ref.py` (pinned to the reference) is the fp32
check of these restatements in tests/test_geometry_host.py.
"""
from __future__ import annotations

import numpy as np

from oracle import lib3d_ref

U32 = 2.0 ** -24  # unit roundoff of fp32 (round to nearest)
Z_MIN = float(np.float32(0.1))


class Bounded:
    """A float64 value `v` and a bound `e` with |fp32 evaluation - v| <= e, propagated operation by operation.

    Every fp32 operation rounds its exact result r to r (1 + d), |d| <= U32.  With inputs known to within ea, eb:
      a +- b : e = ea + eb + U32 (|a +- b| + ea + eb)
      a * b  : e = |a| eb + |b| ea + ea eb + U32 (|a b| + |a| eb + |b| ea + ea eb)
      a / b  : e = (ea + |a / b| eb) / (|b| - eb) + U32 (|a / b| + that)           (requires eb < |b|)
      sqrt a : e = ea / (sqrt(a) + sqrt(max(a - ea, 0))) + U32 (sqrt(a) + that)
      min, max, |.|, negation, constants: no rounding; min/max of a set is within the largest of the members' bounds.
    A fused a * b + c rounds once where the unfused form rounds twice, and its one rounding error U32 |a b + c| is covered
    by the unfused bound's U32 |a b + c| term, so the bound holds whatever contraction the compiler chose.  Values are far
    from the subnormal range in every case (no underflow term).  The float64 evaluation of `v` itself is off by ~1e-16
    relative, which is below every bound's rounding term."""

    __array_priority__ = 100

    def __init__(self, v, e=None):
        self.v = np.asarray(v, dtype=np.float64)
        self.e = np.zeros_like(self.v) if e is None else np.broadcast_to(np.asarray(e, np.float64), self.v.shape).copy()

    @staticmethod
    def of(x) -> "Bounded":
        return x if isinstance(x, Bounded) else Bounded(x)

    def _round(self, v, e):
        return Bounded(v, e + U32 * (np.abs(v) + e))

    def __add__(self, o):
        o = Bounded.of(o)
        return self._round(self.v + o.v, self.e + o.e)

    __radd__ = __add__

    def __sub__(self, o):
        o = Bounded.of(o)
        return self._round(self.v - o.v, self.e + o.e)

    def __rsub__(self, o):
        return Bounded.of(o) - self

    def __neg__(self):
        return Bounded(-self.v, self.e)

    def __mul__(self, o):
        o = Bounded.of(o)
        e = np.abs(self.v) * o.e + np.abs(o.v) * self.e + self.e * o.e
        return self._round(self.v * o.v, e)

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = Bounded.of(o)
        q = self.v / o.v
        assert np.all(o.e < np.abs(o.v)), "divisor not bounded away from 0"
        e = (self.e + np.abs(q) * o.e) / (np.abs(o.v) - o.e)
        return self._round(q, e)

    def __rtruediv__(self, o):
        return Bounded.of(o) / self

    def __getitem__(self, k):
        return Bounded(self.v[k], self.e[k])

    @property
    def shape(self):
        return self.v.shape


# ---- dispatch: numpy arrays (float32 / float64) or Bounded ----------------------------------------------------------
def _sqrt(a):
    if isinstance(a, Bounded):
        s = np.sqrt(a.v)
        e = a.e / (s + np.sqrt(np.maximum(a.v - a.e, 0.0)))
        return a._round(s, e)
    return np.sqrt(a)


def _abs(a):
    return Bounded(np.abs(a.v), a.e) if isinstance(a, Bounded) else np.abs(a)


def _max(a, b):
    """torch.max(a, b): NaN if either is NaN."""
    if isinstance(a, Bounded) or isinstance(b, Bounded):
        a, b = Bounded.of(a), Bounded.of(b)
        return Bounded(np.maximum(a.v, b.v), np.maximum(a.e, b.e))
    return np.maximum(a, b)


def _reduce(a, axis, fn):
    if isinstance(a, Bounded):
        return Bounded(fn(a.v, axis=axis), np.max(a.e, axis=axis))
    return fn(a, axis=axis)


def _const(x, like):
    """A constant in the number system of `like` (exact)."""
    if isinstance(like, Bounded):
        return Bounded(np.float64(x))
    return np.asarray(x, dtype=like.dtype)


def _dot3(m_row, v):
    """m_row[0] v[0] + m_row[1] v[1] + m_row[2] v[2], left to right."""
    return m_row[0] * v[0] + m_row[1] * v[1] + m_row[2] * v[2]


def _wrap(x, dtype):
    if dtype == "bounded":
        return Bounded(np.asarray(x, np.float64))
    return np.asarray(x, dtype=dtype)


# ---------------------------------------------------------------------------------------------------------------------
# TCO_init_from_boxes_autodepth_with_R (lib3d/cosypose_ops.py:169-218)
# ---------------------------------------------------------------------------------------------------------------------
def pose_init(points, label_idx, bboxes, K, R, dtype=np.float64):
    """points [L, N, 3], label_idx [n], bboxes [n, 4], K [n, 3, 3], R [n, 3, 3] -> TCO [n, 4, 4] (numpy, or the
    Bounded entries as a dict {name: Bounded} when dtype == "bounded")."""
    pts = _wrap(np.asarray(points)[np.asarray(label_idx)], dtype)  # [n, N, 3]
    bb, Kw, Rw = _wrap(bboxes, dtype), _wrap(K, dtype), _wrap(R, dtype)
    fx, fy, cx, cy = Kw[:, 0, 0], Kw[:, 1, 1], Kw[:, 0, 2], Kw[:, 1, 2]
    two, one = _const(2.0, fx), _const(1.0, fx)
    bcx, bcy = (bb[:, 0] + bb[:, 2]) / two, (bb[:, 1] + bb[:, 3]) / two
    tx, ty = ((bcx - cx) * one) / fx, ((bcy - cy) * one) / fy
    px, py, pz = pts[..., 0], pts[..., 1], pts[..., 2]
    x = Rw[:, 0, 0][:, None] * px + Rw[:, 0, 1][:, None] * py + Rw[:, 0, 2][:, None] * pz + tx[:, None]
    y = Rw[:, 1, 0][:, None] * px + Rw[:, 1, 1][:, None] * py + Rw[:, 1, 2][:, None] * pz + ty[:, None]
    dx = _reduce(x, 1, np.max) - _reduce(x, 1, np.min)
    dy = _reduce(y, 1, np.max) - _reduce(y, 1, np.min)
    bb_dx, bb_dy = (bb[:, 2] - bb[:, 0]) + one, (bb[:, 3] - bb[:, 1]) + one
    z = ((fy * dy) / bb_dy + (fx * dx) / bb_dx) / two
    t = [((bcx - cx) * z) / fx, ((bcy - cy) * z) / fy, z]
    if dtype == "bounded":
        return {"03": t[0], "13": t[1], "23": t[2]}
    n = len(label_idx)
    T = np.zeros((n, 4, 4), dtype=dtype)
    T[:, :3, :3] = Rw
    T[:, 0, 3], T[:, 1, 3], T[:, 2, 3] = t
    T[:, 3, 3] = 1
    return T


# ---------------------------------------------------------------------------------------------------------------------
# project_points_robust + boxes_from_uv (camera_geometry.py:40-64), deepim_boxes with obs = rend (cropping.py:30-67,
# pose_rigid.py:218-229), get_K_crop_resize (camera_geometry.py:67-115)
# ---------------------------------------------------------------------------------------------------------------------
def _KT(Kw, Tw):
    """P = K @ TCO[:3] as 12 entries P[r][c], each a left-to-right 3-term sum."""
    return [[Kw[:, r, 0] * Tw[:, 0, c] + Kw[:, r, 1] * Tw[:, 1, c] + Kw[:, r, 2] * Tw[:, 2, c] for c in range(4)]
            for r in range(3)]


def crop_geometry(points, label_idx, TCO, K, tCR, lamb, im_size, out_size, dtype=np.float64):
    """-> dict(boxes_rend [n,4], boxes_crop [n,4], K_crop [n,3,3] entries).  im_size / out_size are (h, w)."""
    pts = _wrap(np.asarray(points)[np.asarray(label_idx)], dtype)
    Kw, Tw, tr = _wrap(K, dtype), _wrap(TCO, dtype), _wrap(tCR, dtype)
    lamb = _const(np.float32(lamb), Kw[:, 0, 0])
    zero, one, two = (_const(v, lamb) for v in (0.0, 1.0, 2.0))
    P = _KT(Kw, Tw)
    px, py, pz = pts[..., 0], pts[..., 1], pts[..., 2]
    s = [P[r][0][:, None] * px + P[r][1][:, None] * py + P[r][2][:, None] * pz + P[r][3][:, None] for r in range(3)]
    sz = _max(_const(Z_MIN, lamb), s[2])
    u, v = s[0] / sz, s[1] / sz
    x1, y1 = _reduce(u, 1, np.min), _reduce(v, 1, np.min)
    x2, y2 = _reduce(u, 1, np.max), _reduce(v, 1, np.max)
    # the rendering centre: the origin projected through K @ [R | tCR] (deepim_crops_robust); the rotation terms are
    # multiplied by 0, which is exact for finite entries and NaN for non-finite ones
    c = [P[r][0] * zero + P[r][1] * zero + P[r][2] * zero + _dot3([Kw[:, r, k] for k in range(3)], [tr[:, k] for k in range(3)])
         for r in range(3)]
    cz = _max(_const(Z_MIN, lamb), c[2])
    xc, yc = c[0] / cz, c[1] / cz
    h, w = min(im_size), max(im_size)
    r = _const(np.float32(w / h), lamb)
    xdist = _max(_abs(x1 - xc), _abs(x2 - xc))
    ydist = _max(_abs(y1 - yc), _abs(y2 - yc))
    width = (_max(xdist, ydist * r) * two) * lamb
    height = (_max(xdist / r, ydist) * two) * lamb
    bx1, by1, bx2, by2 = xc - width / two, yc - height / two, xc + width / two, yc + height / two
    final_w, final_h = _const(float(max(out_size)), lamb), _const(float(min(out_size)), lamb)
    crop_w, crop_h = bx2 - bx1, by2 - by1
    crop_cj, crop_ci = (bx1 + bx2) / two, (by1 + by2) / two
    cxk = Kw[:, 0, 2] + (crop_w - one) / two - crop_cj
    cyk = Kw[:, 1, 2] + (crop_h - one) / two - crop_ci
    dcx, dcy = cxk - (crop_w - one) / two, cyk - (crop_h - one) / two
    sx, sy = final_w / crop_w, final_h / crop_h
    kc = dict(fx=sx * Kw[:, 0, 0], fy=sy * Kw[:, 1, 1], cx=(final_w - one) / two + sx * dcx,
              cy=(final_h - one) / two + sy * dcy)
    out = dict(x1=x1, y1=y1, x2=x2, y2=y2, bx1=bx1, by1=by1, bx2=bx2, by2=by2, **kc)
    if dtype == "bounded":
        return out
    K_crop = np.array(Kw, copy=True)
    K_crop[:, 0, 0], K_crop[:, 1, 1], K_crop[:, 0, 2], K_crop[:, 1, 2] = kc["fx"], kc["fy"], kc["cx"], kc["cy"]
    return dict(boxes_rend=np.stack([x1, y1, x2, y2], 1), boxes_crop=np.stack([bx1, by1, bx2, by2], 1), K_crop=K_crop)


def crop_geometry_bounds(points, label_idx, TCO, K, tCR, lamb, im_size, out_size):
    """(value, bound) arrays in the kernels' output layout: boxes_rend [n,4], boxes_crop [n,4], K_crop [n,3,3] (the
    copied entries of K have bound 0)."""
    b = crop_geometry(points, label_idx, TCO, K, tCR, lamb, im_size, out_size, dtype="bounded")

    def stack(names):
        return np.stack([b[k].v for k in names], 1), np.stack([b[k].e for k in names], 1)

    Kc = np.array(K, dtype=np.float64, copy=True)
    eK = np.zeros_like(Kc)
    for (i, j), k in (((0, 0), "fx"), ((1, 1), "fy"), ((0, 2), "cx"), ((1, 2), "cy")):
        Kc[:, i, j], eK[:, i, j] = b[k].v, b[k].e
    return dict(boxes_rend=stack(["x1", "y1", "x2", "y2"]), boxes_crop=stack(["bx1", "by1", "bx2", "by2"]), K_crop=(Kc, eK))


# ---------------------------------------------------------------------------------------------------------------------
# ortho6d (rotations.py:25-40), pose_update_with_reference_point (cosypose_ops.py:33-58), normalize_T
# (transform_ops.py:106-119)
# ---------------------------------------------------------------------------------------------------------------------
def _cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def _ortho6d(xr, yr):
    """-> R[i][j] (row i, column j), columns x, y, z."""
    nx = _sqrt(xr[0] * xr[0] + xr[1] * xr[1] + xr[2] * xr[2])
    x = [xr[0] / nx, xr[1] / nx, xr[2] / nx]
    z = _cross(x, yr)
    nz = _sqrt(z[0] * z[0] + z[1] * z[1] + z[2] * z[2])
    z = [z[0] / nz, z[1] / nz, z[2] / nz]
    y = _cross(z, x)
    return [[x[i], y[i], z[i]] for i in range(3)]


def _assemble(R, t, bottom, dtype, n):
    if dtype == "bounded":
        return {f"{i}{j}": (R[i][j] if j < 3 else t[i]) for i in range(3) for j in range(4)}
    T = np.zeros((n, 4, 4), dtype=dtype)
    for i in range(3):
        for j in range(3):
            T[:, i, j] = R[i][j]
        T[:, i, 3] = t[i]
    T[:, 3] = bottom
    return T


def pose_update(TCO, K_crop, pose9, tCR, dtype=np.float64):
    """models/pose_rigid.py:305-312 (update_pose).  The bottom row of TCO is kept (the reference clones TCO)."""
    Tw, Kw, o9, tr = _wrap(TCO, dtype), _wrap(K_crop, dtype), _wrap(pose9, dtype), _wrap(tCR, dtype)
    n = np.asarray(TCO).shape[0]
    dR = _ortho6d([o9[:, i] for i in range(3)], [o9[:, 3 + i] for i in range(3)])
    vx, vy, vz = o9[:, 6], o9[:, 7], o9[:, 8]
    zsrc = tr[:, 2]
    ztgt = vz * zsrc
    tox = (vx / Kw[:, 0, 0] + tr[:, 0] / zsrc) * ztgt
    toy = (vy / Kw[:, 1, 1] + tr[:, 1] / zsrc) * ztgt
    d = [Tw[:, 0, 3] - tr[:, 0], Tw[:, 1, 3] - tr[:, 1], Tw[:, 2, 3] - tr[:, 2]]
    R = [[_dot3(dR[i], [Tw[:, 0, j], Tw[:, 1, j], Tw[:, 2, j]]) for j in range(3)] for i in range(3)]
    t = [_dot3(dR[i], d) + (tox, toy, ztgt)[i] for i in range(3)]
    bottom = None if dtype == "bounded" else np.asarray(TCO, dtype=dtype)[:, 3]
    return _assemble(R, t, bottom, dtype, n)


def normalize_T(T, dtype=np.float64):
    Tw = _wrap(T, dtype)
    n = np.asarray(T).shape[0]
    R = _ortho6d([Tw[:, i, 0] for i in range(3)], [Tw[:, i, 1] for i in range(3)])
    t = [Tw[:, i, 3] for i in range(3)]
    bottom = None if dtype == "bounded" else np.array([0, 0, 0, 1], dtype=dtype)
    return _assemble(R, t, bottom, dtype, n)


def bounds_as_T(b: dict, n: int):
    """{"ij": Bounded} of the top 3x4 -> (value [n,4,4], bound [n,4,4]); the bottom row is copied (bound 0)."""
    v, e = np.zeros((n, 4, 4)), np.zeros((n, 4, 4))
    for k, x in b.items():
        v[:, int(k[0]), int(k[1])], e[:, int(k[0]), int(k[1])] = x.v, x.e
    return v, e


# ---------------------------------------------------------------------------------------------------------------------
# make_TCO_multiview (lib3d/multiview.py:165-246): the closed-form look-at of lib3d_ref, in float64 throughout
# ---------------------------------------------------------------------------------------------------------------------
def multiview(TCO, tCR, offsets):
    """TCO [n,4,4], tCR [n,3], offsets [n_extra,3] -> TCV_O [n, 1 + n_extra, 4, 4] float64; view 0 is TCO."""
    TCO = np.asarray(TCO, np.float64)
    n, V = TCO.shape[0], 1 + len(offsets)
    out = np.empty((n, V, 4, 4))
    for b in range(n):
        out[b, 0] = TCO[b]
        for v, TC0_CV in enumerate(lib3d_ref.views_TC0_CV(TCO[b], np.asarray(tCR[b], np.float64), np.asarray(offsets, np.float64))):
            R, t = TC0_CV[:3, :3], TC0_CV[:3, 3]
            inv = np.eye(4)
            inv[:3, :3], inv[:3, 3] = R.T, -R.T @ t
            # explicit sums: a non-finite entry of TCO reaches its whole column (0 * NaN = NaN), as in torch's matmul
            out[b, v + 1] = (inv[:, :, None] * TCO[b][None, :, :]).sum(1)
    return out


# ---------------------------------------------------------------------------------------------------------------------
# top-K per group (pose_estimator.py:643-667): sort_values(ascending=False) with NaN last, ties to the lower index
# ---------------------------------------------------------------------------------------------------------------------
def topk(logits, k):
    """logits [g, m] -> int64 indices [g, k]: a stable argsort of -x (numpy puts NaN last; -0 ties +0)."""
    x = np.asarray(logits, np.float64)
    return np.argsort(-x, axis=1, kind="stable")[:, :k]
