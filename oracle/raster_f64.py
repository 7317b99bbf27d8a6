"""oracle/raster_f64.py -- float64 statement of the rasteriser contract, with derived error margins.

TEST INFRASTRUCTURE ONLY: the checker of tests/test_raster_f64_host.py and tests/test_gpu_raster_f64.py.

Written from the contract in the header of megapose6d_b200/csrc/raster.cu and include/mpx.h, not from
oracle/raster_ref.c, with which it shares no code.  Per view:
  * projection: camera transform and pinhole projection in float64; a vertex is projectable iff z >= 2^-10 m; no
    snapping, no clamping;
  * coverage: pixel (i, j) is sampled at (j + 0.5, i + 0.5); two-sided; inclusive edges;
  * depth window: 1/z is linear in screen space; a sample is rejected unless 0.1 <= 1/z <= 10;
  * visibility: the largest 1/z wins, ties go to the lower triangle index;
  * outputs: depth z = 1/(1/z), 0 where d = (1/z - 10) / (0.1 - 10) > 0.999; perspective-correct vertex colour under
    ambient light 1.0; the unit eye normal in Panda axes (x right, y forward, z up) through the 32-level wrapped texture;
    both optionally quantised to k/255 (round to nearest level).

The device computes the same picture from vertices snapped to 1/256 pixel in fp32.  Each pixel therefore comes with
margins derived from that difference (no tolerance is guessed):
  * snap displacement per vertex: |snapped fp32 position - float64 projection| (the fp32 position is computed here in
    numpy fp32 following the contract's operation order: three nested fmaf per camera coordinate, 1/z, x * (1/z),
    fmaf(f, ., c), clamp, round(256 u));
  * edge ambiguity: moving edge a->b by da, db changes its edge function at p by at most
    (|da| + |db|) |p - a| + |b - a| |da| + |da| (|da| + |db|); a sample whose float64 edge value is within that (plus
    1e-9 px of float64 slack) can be covered or not;
  * visibility ambiguity: the device's 1/z differs from the float64 1/z by at most |grad 1/z| x max displacement x
    (sum |l_k| + 1) (the sample's pre-image in the moved triangle) plus the fp32 interpolation error
    16u sum |l_k| (1/z_k) (1 + S_k / z_k) (u = 2^-24, S_k = sum of |terms| of the camera z of vertex k); another covering
    or edge-ambiguous triangle within the sum of the two bounds makes the pixel ambiguous;
  * plane ambiguity: 1/z within that bound of 10 or of 0.1 (plus |0.1f - 0.1|);
  * attribute bound: the winner's attribute spread x the snap-induced shift of its perspective barycentrics, plus
    32u (1 + S/z) of fp32 rounding; a quantised channel may take another level than the float64 value only where the
    float64 value lies within this bound of a rounding boundary (its level is within bound + half a level of it).
"""
from __future__ import annotations

import numpy as np

PROJ_MIN = 2.0 ** -10
IZ_MAX, IZ_MIN = 10.0, 0.1
IZ_MIN_F32_GAP = abs(float(np.float32(0.1)) - 0.1)
CLAMP_UV = 2.0 ** 20
SUB = 256
U = 2.0 ** -24
SLACK_PX = 1e-9
TEX = np.array([((k * 255) >> 5) / 255.0 for k in range(32)])


# ---------------------------------------------------------------------------------------------------------------------
# projection
# ---------------------------------------------------------------------------------------------------------------------
def project_f64(verts, TCO, K):
    """float64 camera points [nv,3], screen (u, v) [nv], projectable flag [nv]."""
    T = np.asarray(TCO, np.float64)
    P = np.asarray(verts, np.float64) @ T[:3, :3].T + T[:3, 3]
    K = np.asarray(K, np.float64)
    z = P[:, 2]
    ok = z >= PROJ_MIN
    zs = np.where(ok, z, 1.0)
    u = K[0, 0] * P[:, 0] / zs + K[0, 2]
    v = K[1, 1] * P[:, 1] / zs + K[1, 2]
    return P, u, v, ok


def fma32(a, b, c):
    """Correctly rounded fp32 fma of fp32 operands: a*b is exact in float64; the float64 sum is rounded once and its
    exact error (TwoSum) decides fp32 midpoints, so the result has no double rounding."""
    a, b, c = (np.asarray(x, np.float32).astype(np.float64) for x in (a, b, c))
    p = a * b
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    f = s.astype(np.float32)
    f64 = f.astype(np.float64)
    toward = np.where(s > f64, np.float32(np.inf), np.float32(-np.inf)).astype(np.float32)
    other = np.nextafter(f, toward)
    tie = (s == (f64 + other.astype(np.float64)) * 0.5) & (e != 0)
    up = np.maximum(f, other)
    dn = np.minimum(f, other)
    return np.where(tie & (e > 0), up, np.where(tie & (e < 0), dn, f)).astype(np.float32)


def snap_f32(verts, TCO, K):
    """The contract's fp32 vertex stage: snapped integer (X, Y) in 1/256 px, fp32 1/z, not-projectable flag."""
    p = np.asarray(verts, np.float32)
    R = np.asarray(TCO, np.float32).reshape(-1)
    Kf = np.asarray(K, np.float32).reshape(-1)

    def row(r):
        return fma32(R[4 * r], p[:, 0], fma32(R[4 * r + 1], p[:, 1], fma32(R[4 * r + 2], p[:, 2], R[4 * r + 3])))

    xc, yc, zc = row(0), row(1), row(2)
    behind = ~(zc >= np.float32(PROJ_MIN))
    zs = np.where(behind, np.float32(1.0), zc).astype(np.float32)
    with np.errstate(all="ignore"):
        iz = (np.float32(1.0) / zs).astype(np.float32)
        u = fma32(Kf[0], (xc * iz).astype(np.float32), Kf[2])
        v = fma32(Kf[4], (yc * iz).astype(np.float32), Kf[5])
    u = np.clip(u, np.float32(-CLAMP_UV), np.float32(CLAMP_UV))
    v = np.clip(v, np.float32(-CLAMP_UV), np.float32(CLAMP_UV))
    bad = np.isnan(u) | np.isnan(v)
    u = np.where(bad, np.float32(0), u)
    v = np.where(bad, np.float32(0), v)
    X = np.rint((u * np.float32(SUB)).astype(np.float32)).astype(np.int64)
    Y = np.rint((v * np.float32(SUB)).astype(np.float32)).astype(np.int64)
    return X, Y, iz, behind | bad


def camera_z_terms(verts, TCO):
    """S_k: the sum of the absolute terms of each vertex's camera z (scales the fp32 error of z)."""
    T = np.asarray(TCO, np.float64)
    return np.abs(np.asarray(verts, np.float64)) @ np.abs(T[2, :3]) + abs(T[2, 3])


def displacement(verts, TCO, K):
    """Per-vertex snap displacement in pixels (inf where either side cannot project the vertex)."""
    _, u, v, ok = project_f64(verts, TCO, K)
    X, Y, _, behind = snap_f32(verts, TCO, K)
    d = np.hypot(X / SUB - u, Y / SUB - v)
    return np.where(ok & ~behind, d, np.inf)


# ---------------------------------------------------------------------------------------------------------------------
# rendering
# ---------------------------------------------------------------------------------------------------------------------
def normal_texture(s):
    u = 32.0 * s - 0.5
    fl = np.floor(u)
    f = u - fl
    k0 = fl.astype(np.int64) & 31
    return TEX[k0] + f * (TEX[(k0 + 1) & 31] - TEX[k0])


def _texture_lipschitz(s):
    """Largest slope of the texture on the segment holding s and its two neighbours."""
    k0 = np.floor(32.0 * s - 0.5).astype(np.int64)
    slope = 32.0 * np.abs(TEX[(np.arange(32) + 1) & 31] - TEX)
    return np.maximum(np.maximum(slope[(k0 - 1) & 31], slope[k0 & 31]), slope[(k0 + 1) & 31])


def quant8(v):
    return np.rint(np.clip(v, 0.0, 1.0) * 255.0) / 255.0


def _pairs(tri_idx, j0, j1, i0, i1):
    bw = j1 - j0 + 1
    cnt = np.where((j1 >= j0) & (i1 >= i0), bw * (i1 - i0 + 1), 0)
    t = np.repeat(tri_idx, cnt)
    start = np.repeat(np.cumsum(cnt) - cnt, cnt)
    k = np.arange(t.size) - start
    bw_r = np.repeat(bw, cnt)
    di = k // np.maximum(bw_r, 1)
    return t, np.repeat(i0, cnt) + di, np.repeat(j0, cnt) + (k - di * bw_r)


def render(verts, normals, colors, faces, TCO, K, h, w, flags=1, max_pairs=4_000_000):
    """Float64 render of one view.  Returns a dict of [h,w] / [3,h,w] float64 arrays: tri (-1 = background), iz, depth,
    rgb, rgb_q, nrm, nrm_q; and margins: amb (edge-, visibility-, plane- or projection-ambiguous pixel), bound_rgb,
    bound_nrm, bound_depth (per pixel), disp (per vertex) and clamped (per vertex: the device clamps its projection)."""
    verts = np.asarray(verts, np.float32)
    faces = np.asarray(faces, np.int64)
    T = np.asarray(TCO, np.float64)
    P, u, v, ok = project_f64(verts, TCO, K)
    X, Y, _, behind = snap_f32(verts, TCO, K)
    disp = np.where(ok & ~behind, np.hypot(X / SUB - u, Y / SUB - v), np.inf)
    S = camera_z_terms(verts, TCO)
    z = P[:, 2]
    zerr = 4 * U * S                                   # fp32 error of the camera z (three nested fmaf)
    proj_amb_v = np.abs(z - PROJ_MIN) <= zerr + 1e-300
    clamped = np.maximum(np.abs(X), np.abs(Y)) >= int(CLAMP_UV) * SUB
    npix = h * w
    out = {"disp": disp, "clamped": clamped}

    fa, fb, fc = faces[:, 0], faces[:, 1], faces[:, 2]
    # triangles that exist in float64 or may exist on the device
    tri_ok = ok[fa] & ok[fb] & ok[fc]
    tri_pamb = (proj_amb_v[fa] | proj_amb_v[fb] | proj_amb_v[fc]) & (z[fa] > 0) & (z[fb] > 0) & (z[fc] > 0)
    pos_ok = np.isfinite(u) & np.isfinite(v) & (z > 0)
    tri_any = (tri_ok | tri_pamb) & pos_ok[fa] & pos_ok[fb] & pos_ok[fc]
    A = np.stack([u, v], 1)
    iz_v = np.where(z > 0, 1.0 / np.where(z > 0, z, 1.0), 0.0)
    Lab = np.linalg.norm(A[fb] - A[fa], axis=1)
    Lbc = np.linalg.norm(A[fc] - A[fb], axis=1)
    Lca = np.linalg.norm(A[fa] - A[fc], axis=1)
    area = ((A[fb] - A[fa])[:, 0] * (A[fc] - A[fa])[:, 1] - (A[fb] - A[fa])[:, 1] * (A[fc] - A[fa])[:, 0])
    dmax = np.maximum(np.maximum(disp[fa], disp[fb]), disp[fc])
    dmax_f = np.where(np.isfinite(dmax), dmax, 0.0)
    lmin = np.maximum(np.minimum(np.minimum(Lab, Lbc), Lca), 1e-12)
    lmax = np.maximum(np.maximum(Lab, Lbc), Lca)
    pad = np.minimum(dmax_f * (2.0 + 2.0 * lmax / lmin) + 2 * dmax_f ** 2 + 1e-6, float(h + w))
    pad = np.where(tri_pamb, float(h + w), pad)
    xs, ys = A[faces][..., 0], A[faces][..., 1]
    with np.errstate(invalid="ignore"):
        j0 = np.maximum(0, np.ceil(np.nan_to_num(xs.min(1) - pad, nan=0) - 0.5)).astype(np.int64)
        j1 = np.minimum(w - 1, np.floor(np.nan_to_num(xs.max(1) + pad, nan=-1) - 0.5)).astype(np.int64)
        i0 = np.maximum(0, np.ceil(np.nan_to_num(ys.min(1) - pad, nan=0) - 0.5)).astype(np.int64)
        i1 = np.minimum(h - 1, np.floor(np.nan_to_num(ys.max(1) + pad, nan=-1) - 0.5)).astype(np.int64)
    cand_tris = np.nonzero(tri_any & ((area != 0) | tri_pamb) & (j1 >= j0) & (i1 >= i0))[0]

    keep = {k: [] for k in ("t", "pix", "iz", "b", "cov", "unc", "lam")}
    cnt = (j1 - j0 + 1) * (i1 - i0 + 1)
    csum = np.cumsum(cnt[cand_tris])
    lo = 0
    while lo < cand_tris.size:
        hi = int(np.searchsorted(csum, (csum[lo - 1] if lo else 0) + max_pairs, side="right"))
        hi = max(hi, lo + 1)
        ct = cand_tris[lo:hi]
        lo = hi
        t, ii, jj = _pairs(ct, j0[ct], j1[ct], i0[ct], i1[ct])
        if t.size == 0:
            continue
        p = np.stack([jj + 0.5, ii + 0.5], 1)
        idx = faces[t]
        Vs = A[idx]                                            # [n,3,2]
        dv = disp[idx]
        dv = np.where(np.isfinite(dv), dv, 0.0)
        wk, dw = [], []
        for k in range(3):                                     # edge opposite vertex k: e1 -> e2
            e1, e2 = Vs[:, (k + 1) % 3], Vs[:, (k + 2) % 3]
            d1, d2 = dv[:, (k + 1) % 3], dv[:, (k + 2) % 3]
            ed = e2 - e1
            L = np.hypot(ed[:, 0], ed[:, 1])
            wk.append(ed[:, 0] * (p[:, 1] - e1[:, 1]) - ed[:, 1] * (p[:, 0] - e1[:, 0]))
            dw.append((d1 + d2) * np.hypot(*(p - e1).T) + L * d1 + d1 * (d1 + d2) + SLACK_PX * L)
        W = np.stack(wk, 1)
        DW = np.stack(dw, 1)
        ar = area[t][:, None]
        with np.errstate(divide="ignore", invalid="ignore"):
            lam = W / ar
        lam = np.where(np.isfinite(lam), lam, 0.0)
        inside = (area[t] != 0) & np.all(W * np.sign(ar) >= 0, 1) & tri_ok[t]
        near_edge = np.any(np.abs(W) <= DW, 1) | tri_pamb[t]
        izk = iz_v[idx]
        iz = (lam * izk).sum(1)
        # |grad 1/z| of the float64 plane: d(lam_k)/dx = (y_{k+1} - y_{k+2}) / area, d(lam_k)/dy = (x_{k+2} - x_{k+1}) / area
        gx = (izk * np.stack([Vs[:, (k + 1) % 3, 1] - Vs[:, (k + 2) % 3, 1] for k in range(3)], 1)).sum(1)
        gy = (izk * np.stack([Vs[:, (k + 2) % 3, 0] - Vs[:, (k + 1) % 3, 0] for k in range(3)], 1)).sum(1)
        with np.errstate(divide="ignore", invalid="ignore"):
            grad = np.hypot(gx, gy) / np.abs(area[t])
        grad = np.where(np.isfinite(grad), grad, np.inf)
        suml = np.abs(lam).sum(1)
        dm = np.where(np.isfinite(dmax[t]), dmax[t], np.inf)
        with np.errstate(invalid="ignore"):
            b_geo = np.where(dm > 0, grad * dm * (suml + 1.0), 0.0)
        b_fp = 16 * U * (np.abs(lam) * izk * (1.0 + S[idx] / np.maximum(z[idx], 1e-300))).sum(1)
        b = b_geo + b_fp
        cov = inside & (iz >= IZ_MIN) & (iz <= IZ_MAX)
        win_amb = (np.abs(iz - IZ_MAX) <= b) | (np.abs(iz - IZ_MIN) <= b + IZ_MIN_F32_GAP)
        unc = near_edge | ((inside | near_edge) & win_amb)
        sel = cov | unc
        keep["t"].append(t[sel]); keep["pix"].append((ii * w + jj)[sel]); keep["iz"].append(iz[sel])
        keep["b"].append(b[sel]); keep["cov"].append(cov[sel]); keep["unc"].append(unc[sel]); keep["lam"].append(lam[sel])
    if keep["t"]:
        K_ = {k: np.concatenate(v) for k, v in keep.items()}
    else:
        K_ = {"t": np.zeros(0, np.int64), "pix": np.zeros(0, np.int64), "iz": np.zeros(0), "b": np.zeros(0),
              "cov": np.zeros(0, bool), "unc": np.zeros(0, bool), "lam": np.zeros((0, 3))}

    # winner per pixel: largest 1/z, ties to the lower triangle index
    c = np.nonzero(K_["cov"])[0]
    order = c[np.lexsort((K_["t"][c], -K_["iz"][c], K_["pix"][c]))]
    first = np.ones(order.size, bool)
    first[1:] = K_["pix"][order][1:] != K_["pix"][order][:-1]
    win = order[first]
    wpix = K_["pix"][win]
    win_iz = np.full(npix, -np.inf)
    win_b = np.zeros(npix)
    win_tri = np.full(npix, -1, np.int64)
    win_iz[wpix] = K_["iz"][win]
    win_b[wpix] = K_["b"][win]
    win_tri[wpix] = K_["t"][win]

    # ambiguity
    pix = K_["pix"]
    reach = K_["iz"] + K_["b"] >= win_iz[pix] - win_b[pix]
    threat = K_["unc"] & reach
    vis = K_["cov"] & (K_["t"] != win_tri[pix]) & (np.abs(K_["iz"] - win_iz[pix]) <= K_["b"] + win_b[pix])
    amb = np.zeros(npix, bool)
    amb[pix[threat | vis]] = True

    # shading of the winners
    iz_w = K_["iz"][win]
    lam_w = K_["lam"][win]
    tw = K_["t"][win]
    idx = faces[tw]
    izk = iz_v[idx]
    bary = lam_w * izk / iz_w[:, None]
    col = np.einsum("nk,nkc->nc", bary, np.asarray(colors, np.float64)[idx])
    nrm_o = np.einsum("nk,nkc->nc", bary, np.asarray(normals, np.float64)[idx])
    e = nrm_o @ T[:3, :3].T
    en = np.linalg.norm(e, axis=1)
    e_u = np.where(en[:, None] > 0, e / np.where(en > 0, en, 1.0)[:, None], e)
    if flags & 2:
        s = np.stack([e_u[:, 0], -e_u[:, 1], -e_u[:, 2]], 1)
    else:
        s = np.stack([e_u[:, 0], e_u[:, 2], -e_u[:, 1]], 1)
    ntex = normal_texture(s)
    zw = 1.0 / iz_w
    d = (iz_w - IZ_MAX) / (IZ_MIN - IZ_MAX)
    dep = np.where(d > 0.999, 0.0, zw)

    # attribute bounds of the winners: |d lam_k| <= |grad lam_k| x the pre-image shift, |grad lam_k| = |edge k| / |area|
    dm = dmax_f[tw]
    Lk = np.stack([Lbc[tw], Lca[tw], Lab[tw]], 1)
    suml = np.abs(lam_w).sum(1)
    dlam = Lk / np.abs(area[tw])[:, None] * (dm * (suml + 1.0))[:, None]
    b_geo = K_["b"][win] - 16 * U * (np.abs(lam_w) * izk * (1.0 + S[idx] / z[idx])).sum(1)
    sum_db = (dlam * izk).sum(1) / iz_w + np.maximum(b_geo, 0) / iz_w
    fp = 32 * U * (1.0 + (S[idx] / z[idx]).max(1))
    cidx = np.asarray(colors, np.float64)[idx]
    spread_c = cidx.max(1) - cidx.min(1)
    bnd_c = spread_c * sum_db[:, None] + fp[:, None] * (np.abs(bary)[..., None] * np.abs(cidx)).sum(1) + 4 * U
    nidx = np.asarray(normals, np.float64)[idx]
    spread_n = np.linalg.norm(nidx.max(1) - nidx.min(1), axis=1)
    eps_e = spread_n * sum_db + fp * (np.abs(bary)[..., None] * np.abs(nidx)).sum(1).sum(1)
    with np.errstate(divide="ignore", invalid="ignore"):
        eps_u = np.where(en > 0, 2 * eps_e / en, np.inf)
    bnd_n = _texture_lipschitz(s) * eps_u[:, None] + 8 * U
    bnd_d = np.maximum(b_geo, 0) / iz_w ** 2 * 2 + 32 * U * zw
    # the d > 0.999 rule: a pixel whose 1/z is within its bound of the cut is depth-ambiguous
    d_cut = IZ_MAX + 0.999 * (IZ_MIN - IZ_MAX)
    dep_amb = np.abs(iz_w - d_cut) <= K_["b"][win] + 1e-6 * d_cut

    def plane(vals, fill=0.0):
        o = np.full((vals.shape[1] if vals.ndim == 2 else 1, npix), fill)
        o[:, wpix] = vals.T if vals.ndim == 2 else vals[None]
        return o.reshape(-1, h, w)

    out["tri"] = win_tri.reshape(h, w)
    out["amb"] = amb.reshape(h, w)
    out["iz"] = plane(iz_w)[0]
    rgb = np.clip(col, 0.0, 1.0)
    nt = np.clip(ntex, 0.0, 1.0)
    out["rgb"] = plane(rgb)
    out["rgb_q"] = plane(quant8(col))
    out["nrm"] = plane(nt)
    out["nrm_q"] = plane(quant8(ntex))
    out["depth"] = plane(dep)[0]
    out["bound_rgb"] = plane(bnd_c)
    out["bound_nrm"] = plane(bnd_n)
    out["bound_depth"] = plane(bnd_d)[0]
    out["depth_amb"] = plane(dep_amb.astype(np.float64))[0] > 0
    return out


def check_outputs(ref, rgb, nrm, depth, quantised=True, mask=None):
    """Compares device-contract outputs (numpy [3,h,w], [3,h,w], [h,w]) with the float64 render on the pixels of `mask`
    (default: every unambiguous pixel).  Returns {name: (n_bad, worst error / bound)}: a float channel is bad beyond its
    bound; a quantised channel is bad when it differs from the float64 level, except by one level where the float64
    value lies within the bound of a rounding boundary."""
    m = ~ref["amb"] if mask is None else mask
    res = {}
    for name, got, exact, q, bnd in (("rgb", rgb, ref["rgb"], ref["rgb_q"], ref["bound_rgb"]),
                                     ("normals", nrm, ref["nrm"], ref["nrm_q"], ref["bound_nrm"])):
        bnd = np.maximum(bnd, 1e-30)
        if quantised:
            # the device's level rounds a value within `bnd` of the float64 one: at most half a level further off
            bad = np.abs(np.rint(got * 255.0) - exact * 255.0) > 255.0 * bnd + 0.5 + 1e-9
            ratio = 0.0
        else:
            err = np.abs(got - exact)
            bad = err > bnd
            ratio = float((err / bnd)[:, m].max()) if m.any() else 0.0
        res[name] = (int(bad[:, m].sum()), ratio)
    dm = m & ~ref["depth_amb"]
    err = np.abs(depth - ref["depth"])
    bd = np.maximum(ref["bound_depth"], 1e-30)
    res["depth"] = (int((err > bd)[dm].sum()), float((err / bd)[dm].max()) if dm.any() else 0.0)
    return res
