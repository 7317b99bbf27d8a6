"""The pose networks' input tensor `x`, element for element.

Every hypothesis enters the network through one act16 tensor in the space-to-depth layout of DESIGN §2:
`[n, H/2, W/2, 4*c_pad]`, channel `(dy*2+dx)*c_pad + c` of pixel `(2i+dy, 2j+dx)`; channels `[crop rgb(d) | view 0 |
view 1 | ...]`, each view `rgb [+ normals] [+ depth]`, then zero pad up to `c_pad`.  Three kernels write it:
`mpx_render_crop_fused` (single-view samples: the rasteriser's resolve pass crops the observation too) and
`mpx_roi_align_fused` + `mpx_raster_render_fused` (multi-view refiners), both with the depth normalisation of
PosePredictor.normalize_depth.

The expected tensor is computed once on the host from independent pieces: the crop with torchvision's roi_align in
float64 plus the reference's validity mask (`oracle.lib3d_ref.crop_images`), the renders from the C rasteriser
(`oracle.pipeline_ref.RefRenderer`, bit-exact with the device), the normalisation in fp32 (`lib3d_ref.normalize_depth`:
a correctly rounded division, like the kernels' `__fdiv_rn`), and the layout restated here (`_assemble`), rounded to the
16-bit type with saturation.  The operands are dyadic (image values k/256, depths k/256 m below 4 m, box corners on a
1/8-px grid, bins of 1/2 to 4 px), so every sample coordinate lies on a 1/16 grid, every bilinear weight on 2^-8, every
product on 2^-16 (2^-20 in the collapsed form) and every partial sum below 2^22 of those units: the kernels' fp32 sums
are exact in any order, with or without FMA contraction, and `x` must equal the expectation bit for bit.
`test_dyadic_operands_make_the_crop_exact` checks that premise on the host for every case.
"""
from __future__ import annotations

import dataclasses
import functools

import numpy as np
import pytest
import torch

from megapose6d_b200 import _abi, lib3d, procedural
from megapose6d_b200.renderer import DEPTH_NORM_KINDS, DEPTH_NORM_SHIFT, RASTER_POINT_LIGHTS
from oracle import lib3d_ref as L
from oracle import pipeline_ref
from tests import helpers

gpu = pytest.mark.gpu
DEV = "cuda"
ACT = _abi.act_dtype() if torch.cuda.is_available() else torch.float16
KIND_NAMES = {v: k for k, v in DEPTH_NORM_KINDS.items() if k is not None}
SENTINEL = -7.5          # no real channel can hold it: rgb, normals in [0, 1], normalised depths >= -2
B, H, W = 3, 480, 640    # observation frames (NHWC4 batch)
SMS_H100 = 132
AXIS_TABLE_MAX = 1024    # crop_device.cuh kAxisTableMax: oh + ow entries of collapsed weights
# per-sample tCR z: clamps of both sides under kinds 0 and 2 (negative z, z beyond the background), a z that saturates
# kind 1 (depth / 2^-16 > 65504), ordinary values
Z = [0.75, 3.5, -0.75, 2.0 ** -16, 1.3, 0.45]


# ---------------------------------------------------------------------------------------------
# layouts, from the predictor configurations
# ---------------------------------------------------------------------------------------------
CONFIGS = {
    "coarse_rgb": helpers.COARSE_CFG,
    "coarse_rgbd": dict(helpers.COARSE_CFG, input_depth=True, render_depth=True),
    "coarse_rgb_no_normals": dict(helpers.COARSE_CFG, render_normals=False),
    "refiner_1view_rgbd_no_normals": dict(helpers.REFINER_RGBD_CFG, n_rendered_views=1, multiview_type="TCO",
                                          render_normals=False),
    "refiner_rgb": helpers.REFINER_CFG,
    "refiner_rgbd": helpers.REFINER_RGBD_CFG,
    "refiner_rgb_no_normals": dict(helpers.REFINER_CFG, render_normals=False),
    "refiner_rgbd_no_normals": dict(helpers.REFINER_RGBD_CFG, render_normals=False),
    "sphere_26views": dict(helpers.REFINER_CFG, multiview_type="sphere_26views", n_rendered_views=27),
}


@dataclasses.dataclass(frozen=True)
class Layout:
    name: str
    c_in: int        # crop channels: rgb (+ depth)
    cpv: int         # channels per rendered view: rgb (+ normals) (+ depth)
    views: int
    c_pad: int
    normals: bool
    render_depth: bool

    @property
    def channels(self):
        return self.c_in + self.cpv * self.views

    @property
    def has_depth(self):
        return self.c_in == 4 or self.render_depth


def layout_of(name, cfg, c_pad=None) -> Layout:
    """What PosePredictor derives from a configuration (pose_predictor.py: _n_single_render_channels, backbone.c_pad)."""
    c = helpers.n_inputs(cfg)
    return Layout(name, 3 + int(cfg["input_depth"]), 3 + 3 * int(cfg["render_normals"]) + int(cfg["render_depth"]),
                  cfg["n_rendered_views"], c_pad or 16 * -(-c // 16), cfg["render_normals"], cfg["render_depth"])


LAYOUTS = {name: layout_of(name, cfg) for name, cfg in CONFIGS.items()}
# the fused kernel also takes c_pad 32 for 16 real channels or fewer: channels 16..31 must come out zero
LAYOUTS["coarse_rgb_pad32"] = layout_of("coarse_rgb_pad32", CONFIGS["coarse_rgb"], c_pad=32)
FUSED = [k for k, v in LAYOUTS.items() if v.views == 1]
SPLIT = [k for k, v in LAYOUTS.items() if v.views > 1]

# raster paths that resolve into x: mpx_raster_set_mode value, batch ("small": at most SMs/8 views), render size and
# the kernel that runs (raster.cu raster_launch, restated in test_case_list_reaches_every_form_and_edge)
PATHS = {
    "scatter": (7, "small", (240, 320), "raster_resolve_kernel"),
    "strips": (2, "small", (240, 320), "raster_kernel<"),
    "strips_read_then_atomic": (0, "small", (240, 320), "raster_kernel<"),
    "tiled": (7, "large", (240, 320), "raster_tiled_kernel"),
    "untiled": (3, "large", (240, 320), "raster_kernel<"),
    "odd_size_untiled_fallback": (7, "large", (64, 800), "raster_kernel<"),
    "480x640": (7, "small", (480, 640), "raster_resolve_kernel"),
}


# ---------------------------------------------------------------------------------------------
# crop cases
# ---------------------------------------------------------------------------------------------
@dataclasses.dataclass(frozen=True)
class Crop:
    name: str
    box: tuple       # x1, y1, x2, y2
    im: int          # frame index (out of range: zeros)
    exact: bool = True


def crop_cases(oh, ow):
    """Boxes for an oh x ow crop of the B frames of H x W, by sample position: bin sizes, the validity edges at -1 and
    at the size, the clamp to the last row / column, boxes outside the image, the 1 px width clamp, mixed and
    out-of-range frame indices."""
    def box(x1, y1, bw, bh):
        return (x1, y1, x1 + bw * ow, y1 + bh * oh)

    e = 0.125  # samples sit at (k + 0.5) / 4 of a 1 px bin: the first at x1 + 1/8, the last at x2 - 1/8
    return [
        Crop("bin 1/2", box(100.125, 60.25, 0.5, 0.5), 0),
        Crop("bin 1, first samples on -1", box(-1 - e, -1 - e, 1, 1), 1),
        Crop("bin 1, last samples on the size", box(W - ow + e, H - oh + e, 1, 1), 2),
        Crop("bin 1, first samples one step below -1", box(-1.25, -1.25, 1, 1), 0),
        Crop("bin 1, last samples one step past the size", box(W - ow + 0.25, H - oh + 0.25, 1, 1), 1),
        Crop("bin 2, hole grid at 15/16", box(8, 16, 2, 2), 1),
        Crop("bin 4, hole grid at 63/64", box(-300, -240, 4, 4), 2),
        Crop("bins 1/2 x 4", box(31.5, -50.375, 0.5, 4), 0),
        Crop("right of and below the image", box(W + 60, H + 20, 0.5, 0.5), 0),
        Crop("left of and above the image", box(-400, -300, 0.5, 0.5), 1),
        Crop("x2 < x1, y2 < y1: 1 px clamp", (300.0, 200.0, 250.0, 150.0), 2, exact=False),
        Crop("frame index b", box(100, 100, 1, 1), B),
        Crop("frame index -1", box(60, 40, 1, 1), -1),
    ]


@functools.lru_cache(maxsize=1)
def dyadic_frames() -> torch.Tensor:
    """[B, 4, H, W] float32: rgb k/256, depth k/256 m in (0, 4) with holes on a 16-px grid (isolated: validity 15/16 under
    2 px bins, 63/64 under 4 px bins) and a scattered pattern."""
    g = np.random.RandomState(11)
    rgb = g.randint(0, 257, size=(B, 3, H, W)) / 256.0
    depth = g.randint(1, 1024, size=(B, 1, H, W)) / 256.0
    yy, xx = np.mgrid[:H, :W]
    for f in range(B):
        holes = ((yy % 16 == 0) & (xx % 16 == 0)) | ((yy * 7 + xx * 3 + 5 * f) % 61 == 0)
        depth[f, 0][holes] = 0.0
    return torch.from_numpy(np.concatenate((rgb, depth), axis=1)).float().contiguous()


def _boxes5(cases):
    """torchvision boxes: frame index (0 for out-of-range frames; their crops are zeroed afterwards), x1, y1, x2, y2."""
    return torch.tensor([[c.im if 0 <= c.im < B else 0, *c.box] for c in cases], dtype=torch.float64)


@functools.lru_cache(maxsize=4)
def crop_reference(oh, ow):
    """Per case of crop_cases(oh, ow): (crop [n, 4, oh, ow] fp32 = the reference's crop_images in float64: rgb, depth
    masked where the validity fraction is < 0.99; validity fraction [n, oh, ow] float64)."""
    import torchvision

    cases = crop_cases(oh, ow)
    frames = dyadic_frames().double()
    boxes5 = _boxes5(cases)
    crop = L.crop_images(frames, boxes5, (oh, ow))
    valid = torchvision.ops.roi_align((frames[:, 3:] > 0).double(), boxes5, output_size=(oh, ow), sampling_ratio=4)[:, 0]
    off = torch.tensor([not 0 <= c.im < B for c in cases])
    crop[off] = 0
    valid[off] = 0
    exact = crop.float().double()
    for i, c in enumerate(cases):
        if c.exact:
            assert torch.equal(exact[i], crop[i]), f"{c.name}: the float64 crop is not an fp32 value"
    return crop.float(), valid


# ---------------------------------------------------------------------------------------------
# the expected tensor
# ---------------------------------------------------------------------------------------------
def _to_act(v: torch.Tensor) -> torch.Tensor:
    """fp32 -> the 16-bit type as `cvt.rn.satfinite`: round to nearest even, saturate at the largest finite value."""
    if ACT == torch.float16:
        return v.clamp(-65504.0, 65504.0).to(torch.float16)
    return v.to(ACT)


def _assemble(planes: torch.Tensor, c_pad: int, fill: float, act: bool = True) -> torch.Tensor:
    """planes [n, C, h, w] fp32 -> x [n, h/2, w/2, 4*c_pad]: channel (dy*2+dx)*c_pad + c holds plane c at pixel
    (2i+dy, 2j+dx); channels C..c_pad-1 of every sub-pixel hold `fill`.  Rounded to the 16-bit type unless `act` is
    False."""
    n, c, h, w = planes.shape
    out = torch.full((n, h // 2, w // 2, 4, c_pad), fill, dtype=torch.float32)
    for dy in (0, 1):
        for dx in (0, 1):
            out[:, :, :, dy * 2 + dx, :c] = planes[:, :, dy::2, dx::2].permute(0, 2, 3, 1)
    out = out.reshape(n, h // 2, w // 2, 4 * c_pad)
    return _to_act(out) if act else out


def _unpack(x: torch.Tensor, c: int) -> torch.Tensor:
    n, hs, ws, c4 = x.shape
    c_pad = c4 // 4
    return x.float().view(n, hs, ws, 2, 2, c_pad).permute(0, 5, 1, 3, 2, 4).reshape(n, c_pad, 2 * hs, 2 * ws)[:, :c]


def _norm(d: torch.Tensor, z: torch.Tensor, kind: int) -> torch.Tensor:
    """lib3d_ref.normalize_depth in fp32 with z per leading index."""
    tcr = torch.zeros(d.shape[0], 3)
    tcr[:, 2] = z
    return L.normalize_depth(d, tcr, KIND_NAMES[kind])


def _crop_planes(crop: torch.Tensor, c_in: int, z: torch.Tensor, kind: int) -> torch.Tensor:
    out = crop[:, :c_in].clone()
    if c_in == 4:
        out[:, 3:] = _norm(crop[:, 3:], z, kind)
    return out


def _render_planes(ref: dict, lay: Layout, z_views: torch.Tensor, kind: int) -> torch.Tensor:
    """[n_views, cpv, h, w] -> [n_samples, views * cpv, h, w] in the network's channel order."""
    parts = [ref["rgbs"]] + ([ref["normals"]] if lay.normals else [])
    if lay.render_depth:
        parts.append(_norm(ref["depths"], z_views, kind))
    r = torch.cat(parts, dim=1)
    return r.view(-1, lay.views * lay.cpv, *r.shape[-2:])


def _tolerance(ref: torch.Tensor, e: torch.Tensor) -> torch.Tensor:
    """|x - ref| bound for a value within e of `ref` before its rounding to the 16-bit type: e + half a unit in the last
    place of the 16-bit type at |ref| + e."""
    mag = (ref.abs() + e).clamp_min(2.0 ** -14)
    mant = 10 if ACT == torch.float16 else 7
    return e + torch.exp2(torch.floor(torch.log2(mag)) - mant - 1)


def crop_error_bound(frames: torch.Tensor, box, c_in: int, z: float, kind: int, ref: torch.Tensor) -> torch.Tensor:
    """Bound on |crop_device - crop_torchvision_fp32| per channel of one crop, before the 16-bit rounding.

    A sample coordinate x1 + p*bin + (k + 1/2)*bin/4 takes four fp32 roundings in torchvision's order; FMA contraction
    may skip up to two of them on either side, and a bin of 1/w px is itself rounded once, so the two coordinates differ
    by at most 8 u S, u = 2^-24, S = the largest |coordinate| of the box plus one bin.  A bilinear sample is continuous
    in its coordinate (also across the floor and the clamp to the last texel; only the validity cut at -1 and at the
    size is not, and the cases keep their samples off it by more than 8 u S) with slope at most G = the largest
    difference of adjacent texels, so each of the 16 samples, and their mean, moves by at most 2 * 8 u S G (two axes).
    The 64 products are summed in another order by the collapsed form: each fp32 sum of at most 80 terms whose weights
    add up to 16 is within 80 u * 16 M of its exact value (M = the largest |texel|), divided by 16, so the two sums
    differ by at most 160 u M.  Depth: normalised by division by |z| (kinds 0, 1), plus one fp32 rounding of the result.
    The validity fraction moves by the same coordinate term (G = 1): pixels within that of 0.99 may be masked on one side
    only and are not compared (returned as inf)."""
    u = 2.0 ** -24
    x1, y1, x2, y2 = box
    bin_ = max(max(x2 - x1, 1.0) / ref.shape[-1], max(y2 - y1, 1.0) / ref.shape[-2])
    s = max(abs(x1), abs(y1), abs(x2), abs(y2)) + bin_
    out = torch.empty(c_in, *ref.shape[-2:])
    for c in range(c_in):
        img = frames[:, c]
        g = max((img[:, 1:] - img[:, :-1]).abs().max().item(), (img[:, :, 1:] - img[:, :, :-1]).abs().max().item())
        m = img.abs().max().item()
        e = 16 * u * s * g + 160 * u * m
        if c == 3:
            e = e / abs(z) if kind in (0, 1) else e
            e = e + 2 * u * ref[3].abs()
        out[c] = _tolerance(ref[c], torch.as_tensor(e, dtype=torch.float32).expand_as(ref[c]))
    return out


def _assert_x(got: torch.Tensor, want: torch.Tensor, tol: torch.Tensor = None, what: str = "",
              want32: torch.Tensor = None):
    """got == want bit for bit, except where `tol` (same shape, float; nan = exact) allows |got - want32| <= tol, want32
    being the expectation before its rounding to the 16-bit type."""
    got = got.cpu()
    if tol is None:
        same = got.view(torch.int16) == want.view(torch.int16)
    else:
        exact = torch.isnan(tol)
        same = torch.where(exact, got.view(torch.int16) == want.view(torch.int16),
                           (got.float() - want32).abs() <= tol)
    if not same.all():
        bad = (~same).nonzero()
        i = tuple(bad[0].tolist())
        c_pad = got.shape[3] // 4
        chans = sorted(set((bad[:, 3] % c_pad).tolist()))
        samples = sorted(set(bad[:, 0].tolist()))
        raise AssertionError(f"{what}: {bad.shape[0]} elements differ (samples {samples}, channels {chans}), first at {i} "
                             f"(channel {i[3] % c_pad}, sub-pixel {i[3] // c_pad}): got {got[i].item()}, "
                             f"want {want[i].item()}")


# ---------------------------------------------------------------------------------------------
# host tests: the premise and the coverage
# ---------------------------------------------------------------------------------------------
def _f32(v):
    return np.asarray(v, dtype=np.float32)


def _fma(a, b, c):
    """fp32 fused multiply-add: the product of two fp32 values is exact in float64, then one rounding (of the float64
    sum, then to fp32: exact whenever the fp32 result is, which is what the premise test requires)."""
    return _f32(a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64))


def _coords(start, bin_, n, fma):
    p = np.arange(n, dtype=np.float32)[:, None]
    k = _f32(np.arange(4) + 0.5)[None, :]
    if fma:  # fma(p, bin, x1), then fma(k + 1/2, bin / 4, .)
        a = _fma(p, np.broadcast_to(bin_, p.shape), np.broadcast_to(start, p.shape))
        return _fma(np.broadcast_to(k, (n, 4)), np.broadcast_to(_f32(bin_ / _f32(4)), (n, 4)), np.broadcast_to(a, (n, 4)))
    return _f32(_f32(start + p * bin_) + _f32(k * bin_) / _f32(4))


def _axis_taps(v, size):
    """crop_device.cuh axis_tap on an array of coordinates."""
    ok = ~((v < -1.0) | (v > size))
    vv = np.maximum(v, _f32(0))
    lo = vv.astype(np.int64)
    clamp = lo >= size - 1
    lo = np.where(clamp, size - 1, lo)
    hi = np.where(clamp, size - 1, lo + 1)
    vv = np.where(clamp, _f32(lo), vv)
    l = _f32(vv - lo)
    return ok, lo, hi, l, _f32(1) - l


def _roi_params(box, oh, ow):
    x1, y1, x2, y2 = (_f32(v) for v in box)
    bw = _f32(max(_f32(x2 - x1), _f32(1))) / _f32(ow)
    bh = _f32(max(_f32(y2 - y1), _f32(1))) / _f32(oh)
    return x1, y1, _f32(bw), _f32(bh)


def roi_align_fp32(img: np.ndarray, box, oh, ow, fma: bool) -> np.ndarray:
    """The plain form's sums in fp32, img [C, H, W]: without contraction in torchvision's order
    (acc += w1 v1 + w2 v2 + w3 v3 + w4 v4, samples row-major), or with every multiply-add fused and the samples in reverse
    order."""
    x1, y1, bw, bh = _roi_params(box, oh, ow)
    cy, cx = _coords(y1, bh, oh, fma), _coords(x1, bw, ow, fma)
    acc = np.zeros((img.shape[0], oh, ow), np.float32)
    order = [(iy, ix) for iy in range(4) for ix in range(4)]
    for iy, ix in (reversed(order) if fma else order):
        oky, ly0, hy0, lyw, hyw = _axis_taps(cy[:, iy], img.shape[1])
        okx, lx0, hx0, lxw, hxw = _axis_taps(cx[:, ix], img.shape[2])
        w = [hyw[:, None] * hxw[None], hyw[:, None] * lxw[None], lyw[:, None] * hxw[None], lyw[:, None] * lxw[None]]
        v = [img[:, ly0][:, :, lx0], img[:, ly0][:, :, hx0], img[:, hy0][:, :, lx0], img[:, hy0][:, :, hx0]]
        if fma:
            new = acc
            for wk, vk in zip(w, v):
                new = _fma(np.broadcast_to(wk, vk.shape), vk, new)
        else:
            new = _f32(acc + _f32(_f32(_f32(w[0] * v[0] + w[1] * v[1]) + w[2] * v[2]) + w[3] * v[3]))
        acc = np.where((oky[:, None] & okx[None])[None], new, acc)
    return _f32(acc / _f32(16))


def collapses(box, oh, ow, h=H, w=W) -> bool:
    """crop_device.cuh axis_collapse over every output row and column: the four samples of each touch at most four
    consecutive image rows / columns."""
    x1, y1, bw, bh = _roi_params(box, oh, ow)
    for start, bin_, n, size in ((y1, bh, oh, h), (x1, bw, ow, w)):
        _, lo, hi, _, _ = _axis_taps(_coords(start, bin_, n, fma=False), size)
        if (hi[:, 3] - lo[:, 0] > 3).any():
            return False
    return True


def crop_form(c: Crop, oh, ow) -> str:
    """Which roi_align form a crop takes, in roi_align_kernel and in the rasteriser's resolve pass alike."""
    if not 0 <= c.im < B:
        return "none"
    return "collapsed" if oh + ow <= AXIS_TABLE_MAX and collapses(c.box, oh, ow) else "plain"


SIZES = sorted({p[2] for p in PATHS.values()})


@pytest.mark.parametrize("size", SIZES, ids=[f"{h}x{w}" for h, w in SIZES])
def test_dyadic_operands_make_the_crop_exact(size):
    """The premise of the exact comparisons: for every case the fp32 sums of roi_align, in two orders, with and without
    FMA contraction, equal torchvision's float64 result (rgb, depth and the validity fraction)."""
    import torchvision

    oh, ow = size
    frames = dyadic_frames()
    img = torch.cat((frames, (frames[:, 3:] > 0).float()), dim=1)
    for c in crop_cases(oh, ow):
        if not c.exact or not 0 <= c.im < B:
            continue
        want = torchvision.ops.roi_align(img[c.im:c.im + 1].double(), torch.tensor([[0.0, *c.box]], dtype=torch.float64),
                                         output_size=(oh, ow), sampling_ratio=4)[0].numpy()
        for fma in (False, True):
            got = roi_align_fp32(img[c.im].numpy(), c.box, oh, ow, fma)
            assert np.array_equal(got.astype(np.float64), want), (c.name, fma, np.abs(got - want).max())


def test_case_list_reaches_every_form_and_edge():
    """The crop cases, the raster paths and the layouts reach what the exact tests are meant to exercise (evaluated for a
    132-SM H100)."""
    reached = set()
    for oh, ow in SIZES:
        cases = crop_cases(oh, ow)
        _, valid = crop_reference(oh, ow)
        for i, c in enumerate(cases):
            form = crop_form(c, oh, ow)
            x1, y1, bw, bh = _roi_params(c.box, oh, ow)
            cx = _coords(x1, bw, ow, fma=False)
            cy = _coords(y1, bh, oh, fma=False)
            reached.add(form)
            if form == "plain":
                reached.add("plain, h + w > 1024" if oh + ow > AXIS_TABLE_MAX else "plain, h + w <= 1024")
                if max(bw, bh) == 4:
                    reached.add("plain, bin 4 px")
            for v, size in ((cx, W), (cy, H)):
                reached |= {"sample on -1"} if (v == -1).any() else set()
                reached |= {"sample on the size"} if (v == size).any() else set()
                reached |= {"sample one step below -1"} if ((v < -1) & (v >= -1.125)).any() else set()
                reached |= {"sample one step past the size"} if ((v > size) & (v <= size + 0.125)).any() else set()
                reached |= {"clamp to the last texel"} if ((v >= size - 1) & (v <= size)).any() else set()
                if ((v < -1) | (v > size)).all():
                    reached.add("box outside the image")
            if c.box[2] < c.box[0] and c.box[3] < c.box[1]:
                reached.add("x2 < x1")
            if c.im >= B:
                reached.add("frame index past the batch")
            if c.im < 0:
                reached.add("negative frame index")
            if form != "none":
                for frac, label in ((1.0, "validity 1"), (63 / 64, "validity 63/64"), (15 / 16, "validity 15/16")):
                    if (valid[i] == frac).any():
                        reached.add(label)
        if len({c.im for c in cases if 0 <= c.im < B}) == B:
            reached.add("every frame of the batch")
    # raster paths: small batches go to the coverage + resolve kernels under bit 0, large ones to the tiled kernel under
    # bit 2 unless its strips of >= 16 rows do not fit 110 KB of shared memory beside the crop's axis tables
    for mode, batch, (h, w), kern in PATHS.values():
        fixed = (16 * 512 + 512 + 1) * 4 + (20 * (h + w) if h + w <= AXIS_TABLE_MAX else 0) + 16
        rows = (110 * 1024 - fixed) // (8 * w)
        if batch == "small" and mode & 1:
            want = "raster_resolve_kernel"
        elif mode & 4 and rows >= 16:
            want = "raster_tiled_kernel"
        else:
            want = "raster_kernel<"
        assert kern == want, (mode, batch, h, w)
        reached.add(f"{kern} ({batch})")
        if rows < 16 and mode & 4:
            reached.add("untiled fallback")
    for lay in LAYOUTS.values():
        reached.add(f"c_in {lay.c_in}, {lay.cpv} per view, c_pad {lay.c_pad}, {'fused' if lay.views == 1 else 'split'}")
        if lay.channels == lay.c_pad:
            reached.add("no pad channels")
    need = {"collapsed", "plain, bin 4 px", "plain, h + w > 1024", "none", "sample on -1", "sample on the size",
            "sample one step below -1", "sample one step past the size", "clamp to the last texel",
            "box outside the image", "x2 < x1", "frame index past the batch", "negative frame index",
            "every frame of the batch", "validity 1", "validity 63/64", "validity 15/16",
            "raster_resolve_kernel (small)", "raster_kernel< (small)", "raster_tiled_kernel (large)",
            "raster_kernel< (large)", "untiled fallback", "no pad channels",
            "c_in 3, 6 per view, c_pad 16, fused", "c_in 4, 7 per view, c_pad 16, fused",
            "c_in 3, 3 per view, c_pad 16, fused", "c_in 4, 4 per view, c_pad 16, fused",
            "c_in 3, 6 per view, c_pad 32, fused", "c_in 3, 6 per view, c_pad 32, split",
            "c_in 4, 7 per view, c_pad 32, split", "c_in 3, 3 per view, c_pad 16, split",
            "c_in 4, 4 per view, c_pad 32, split", "c_in 3, 6 per view, c_pad 176, split"}
    assert need <= reached, sorted(need - reached)
    assert SMS_H100 // 8 >= len(crop_cases(240, 320)), "a small fused batch holds every crop case"


# ---------------------------------------------------------------------------------------------
# device tests
# ---------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def env():
    ds, images, K = helpers.make_scene(2, seed=8, with_depth=True)
    from megapose6d_b200.renderer import BatchRenderer

    rm = helpers.ref_meshes_from_dataset(ds)
    frames = dyadic_frames()
    return dict(ds=ds, images=images, K=K, rm=rm, renderer=BatchRenderer(object_dataset=ds),
                labels=[o.label for o in ds.list_objects],
                nhwc4={c: lib3d.image_to_nhwc4(frames[:, :c].contiguous().cuda()) for c in (3, 4)}, renders={})


@pytest.fixture
def raster_mode():
    yield lambda m: _abi.lib().mpx_raster_set_mode(m)
    _abi.lib().mpx_raster_set_mode(7)


def _renders(env, n_views, size, normals, seed):
    """Views of the scene's meshes, and the oracle's rgb / normals / depth of them."""
    key = (n_views, size, normals, seed)
    if key not in env["renders"]:
        h, w = size
        labels = [env["labels"][i % len(env["labels"])] for i in range(n_views)]
        TCO = torch.from_numpy(procedural.random_poses(n_views, seed, z_range=(0.3, 0.8))).float()
        K = torch.tensor([[2.4 * w, 0, w / 2 + 0.3], [0, 2.4 * w, h / 2 - 0.2], [0, 0, 1]]).repeat(n_views, 1, 1)
        ref = pipeline_ref.RefRenderer(env["rm"]).render(labels, TCO, K, None, size, render_depth=True,
                                                          render_normals=normals, point_lights=not normals)
        assert (ref["depths"] > 0).float().mean() > 0.02
        env["renders"][key] = (labels, TCO, K, ref)
    return env["renders"][key]




def _samples(batch, views, n_cases):
    small = (torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else SMS_H100) // 8
    if batch == "small":
        return min(n_cases, small // views)
    # every crop case once, except for views so many that one sample already fills a large batch
    return max(n_cases if views <= 4 else 1, small // views + 1)


def _crop_expectation(cases, sel, crop, valid, lay, z, kind):
    """Expected crop planes of the samples, and the tolerance (nan = exact) of each: the 1 px clamped box has bins of
    1/w px, off the dyadic grid, and is held to crop_error_bound."""
    want = _crop_planes(crop[sel], lay.c_in, z, kind)
    tol = torch.full_like(want, float("nan"))
    frames = dyadic_frames()
    for s, i in enumerate(sel):
        c = cases[i]
        if c.exact:
            continue
        t = crop_error_bound(frames[c.im:c.im + 1], c.box, lay.c_in, z[s].item(), kind, want[s])
        if lay.c_in == 4:
            e_valid = 16 * 2.0 ** -24 * max(abs(v) for v in c.box) + 2.0 ** -20
            t[3][(valid[i] - 0.99).abs() <= e_valid] = float("inf")
        tol[s] = t
    return want, tol


@gpu
@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("layout", FUSED)
def test_render_crop_fused_writes_the_exact_input(env, raster_mode, layout, path):
    """mpx_render_crop_fused into a sentinel-filled x: every real channel of every pixel (background included) equals
    the host expectation bit for bit under every depth normalisation, and channels C..c_pad are zero."""
    lay = LAYOUTS[layout]
    mode, batch, size, _ = PATHS[path]
    h, w = size
    cases = crop_cases(h, w)
    crop, valid = crop_reference(h, w)
    n = _samples(batch, 1, len(cases))
    sel = [s % len(cases) for s in range(n)]
    labels, TCO, K, ref = _renders(env, n, size, lay.normals, seed=40 + n)
    r = env["renderer"]
    lab = r.mesh_db.label_ids(labels, DEV)
    boxes = torch.tensor([cases[i].box for i in sel], dtype=torch.float32, device=DEV)
    im_idx = torch.tensor([cases[i].im for i in sel], dtype=torch.int32, device=DEV)
    z = torch.tensor([Z[s % len(Z)] for s in range(n)])
    zd = z.to(DEV)
    raster_mode(mode)
    for kind in (range(4) if lay.has_depth else [0]):
        x = torch.full((n, h // 2, w // 2, 4 * lay.c_pad), SENTINEL, dtype=ACT, device=DEV)
        flags = (0 if lay.normals else RASTER_POINT_LIGHTS) | (kind << DEPTH_NORM_SHIFT)

        def run():
            r.render_crop_fused(lab, TCO.cuda(), K.cuda(), size, env["nhwc4"][lay.c_in], im_idx, boxes, lay.c_in, x,
                                lay.c_pad, lay.cpv, zd, flags)
        run()
        want_crop, tol_crop = _crop_expectation(cases, sel, crop, valid, lay, z, kind)
        planes = torch.cat((want_crop, _render_planes(ref, lay, z, kind)), dim=1)
        tol = torch.cat((tol_crop, torch.full((n, lay.c_pad - lay.c_in, h, w), float("nan"))), dim=1)
        _assert_x(x, _assemble(planes, lay.c_pad, 0.0), _assemble_tol(tol), f"{layout} {path} kind {kind}",
                  _assemble(planes, lay.c_pad, 0.0, act=False))


def _assemble_tol(tol: torch.Tensor) -> torch.Tensor:
    """A per-plane tolerance [n, c_pad, h, w] in x's layout (float32)."""
    n, c_pad, h, w = tol.shape
    return tol.view(n, c_pad, h // 2, 2, w // 2, 2).permute(0, 2, 4, 3, 5, 1).reshape(n, h // 2, w // 2, 4 * c_pad)


SPLIT_PATHS = [(lay, p) for lay in SPLIT for p in PATHS
               if PATHS[p][1] == "large" or LAYOUTS[lay].views <= SMS_H100 // 8]


@gpu
@pytest.mark.parametrize("layout,path", SPLIT_PATHS, ids=[f"{l}-{p}" for l, p in SPLIT_PATHS])
def test_split_path_writes_the_exact_input(env, raster_mode, layout, path):
    """mpx_raster_render_fused then mpx_roi_align_fused into a sentinel-filled x: the views land in their slots
    (ch_offset + slot * ch_per_view) without touching the crop channels, the crop without touching the views, the pad
    channels keep the sentinel, and every real channel equals the host expectation bit for bit under every depth
    normalisation (each sample's z: a view normalised with another sample's z differs)."""
    lay = LAYOUTS[layout]
    mode, batch, size, _ = PATHS[path]
    h, w = size
    cases = crop_cases(h, w)
    crop, valid = crop_reference(h, w)
    n = _samples(batch, lay.views, len(cases))
    sel = [s % len(cases) for s in range(n)]
    labels, TCO, K, ref = _renders(env, n * lay.views, size, lay.normals, seed=60 + n * lay.views)
    r = env["renderer"]
    lab = r.mesh_db.label_ids(labels, DEV)
    boxes = torch.tensor([cases[i].box for i in sel], dtype=torch.float32, device=DEV)
    im_idx = torch.tensor([cases[i].im for i in sel], dtype=torch.int32, device=DEV)
    z = torch.tensor([Z[s % len(Z)] for s in range(n)])
    zd = z.to(DEV)
    z_views = z.repeat_interleave(lay.views)
    raster_mode(mode)
    for kind in (range(4) if lay.has_depth else [0]):
        x = torch.full((n, h // 2, w // 2, 4 * lay.c_pad), SENTINEL, dtype=ACT, device=DEV)
        flags = (0 if lay.normals else RASTER_POINT_LIGHTS) | (kind << DEPTH_NORM_SHIFT)

        def render():
            r.render_fused(lab, TCO.cuda(), K.cuda(), lay.views, size, x, lay.c_pad, lay.c_in, lay.cpv,
                           zd if lay.render_depth else None, flags)
        render()
        views = _render_planes(ref, lay, z_views, kind)
        sent_crop = torch.full((n, lay.c_in, h, w), SENTINEL)
        _assert_x(x, _assemble(torch.cat((sent_crop, views), dim=1), lay.c_pad, SENTINEL), None,
                  f"{layout} {path} kind {kind}, views only")
        _abi.check(_abi.lib().mpx_roi_align_fused(
            _abi.ptr(env["nhwc4"][lay.c_in]), B, H, W, _abi.ptr(im_idx), _abi.ptr(boxes), n, lay.c_in, h, w, _abi.ptr(x),
            lay.c_pad, _abi.ptr(zd if lay.c_in == 4 else None), kind, _abi.stream_ptr()))
        torch.cuda.synchronize()
        want_crop, tol_crop = _crop_expectation(cases, sel, crop, valid, lay, z, kind)
        tol = torch.cat((tol_crop, torch.full((n, lay.c_pad - lay.c_in, h, w), float("nan"))), dim=1)
        planes = torch.cat((want_crop, views), dim=1)
        _assert_x(x, _assemble(planes, lay.c_pad, SENTINEL), _assemble_tol(tol), f"{layout} {path} kind {kind}",
                  _assemble(planes, lay.c_pad, SENTINEL, act=False))


@gpu
def test_non_finite_depth_texels_do_not_depend_on_the_roi_align_form(env):
    """NaN and inf depth texels.  The collapsed form skips taps of zero weight; the plain form must do the same, so that
    a crop does not depend on which form its size selects.  The same box geometry at 240x320 (collapsed) and 480x640
    (plain: h + w > 1024) gives the same values on the shared 240x320 corner, and both equal the pinned behaviour:
    masked pixels (validity < 0.99; NaN is not > 0, inf is) are 0, otherwise NaN if a NaN texel has positive weight,
    else inf if an inf texel has, else the exact crop.  torchvision multiplies every tap, so where it finds NaN through
    a zero weight or through the mask (NaN * 0) the engine differs from the reference (DESIGN §4)."""
    import torchvision

    frames = dyadic_frames().clone()
    # samples of a 1 px bin starting 1/8 past an integer fall on integers x0 + p + 1 (weight 1 on x0 + p + 1, 0 on x0 + p + 2)
    x1, y1 = 40.125, 30.125
    for f in range(B):
        d = frames[f, 3]
        d[35:300:9, 44:600:7] = float("nan")
        d[37:300:23, 47:600:13] = float("inf")
    depth = frames[:, 3:].double()
    finite = torch.where(torch.isfinite(depth), depth, torch.zeros_like(depth))
    nhwc4 = lib3d.image_to_nhwc4(frames.contiguous().cuda())
    got = {}
    for oh, ow in ((240, 320), (480, 640)):
        box = (x1, y1, x1 + ow, y1 + oh)
        assert crop_form(Crop("", box, 1), oh, ow) == ("collapsed" if oh == 240 else "plain")
        got[oh] = lib3d.crop_images(nhwc4, torch.tensor([box], device=DEV), torch.tensor([1], dtype=torch.int32, device=DEV),
                                    4, (oh, ow))[0, 3].cpu()
        b5 = torch.tensor([[1.0, *box]], dtype=torch.float64)

        def ra(img):
            return torchvision.ops.roi_align(img, b5, output_size=(oh, ow), sampling_ratio=4)[0, 0]
        valid, w_nan, w_inf = ra((depth > 0).double()), ra(torch.isnan(depth).double()), ra(torch.isinf(depth).double())
        want = ra(finite)
        want = torch.where(w_inf > 0, torch.full_like(want, float("inf")), want)
        want = torch.where(w_nan > 0, torch.full_like(want, float("nan")), want)
        want = torch.where(valid < 0.99, torch.zeros_like(want), want).float()
        assert torch.isinf(want).any() and ((w_nan > 0) & (want == 0)).any()
        assert torch.equal(torch.isnan(got[oh]), torch.isnan(want)), f"{oh}x{ow}: NaN at {(torch.isnan(got[oh]) != torch.isnan(want)).sum()} pixels"
        fin = ~torch.isnan(want)
        assert torch.equal(got[oh][fin], want[fin]), f"{oh}x{ow}"
    small, corner = got[240], got[480][:240, :320]
    assert torch.equal(torch.isnan(small), torch.isnan(corner)) and torch.equal(small.nan_to_num(), corner.nan_to_num())


PREDICTOR_CONFIGS = ["coarse_rgb", "coarse_rgbd", "refiner_rgb", "refiner_rgbd", "refiner_rgb_no_normals",
                     "refiner_rgbd_no_normals", "sphere_26views"]


@gpu
@pytest.mark.parametrize("name", PREDICTOR_CONFIGS)
def test_predictor_input_is_rebuilt_from_its_outputs(env, name):
    """One eager PosePredictor step on ordinary inputs (smooth noise, random depth with holes, boxes and cameras from the
    device's crop geometry): its input buffer, rebuilt on the host from the step's boxes_crop, KV_crop, TCV_O and tCR.
    Render channels equal the oracle's renders (normalised with each sample's z) bit for bit, pad channels are zero, crop
    channels lie within crop_error_bound of torchvision's fp32 crop; `pack_input` of the same planes gives the same
    tensor as the layout restated here."""
    from megapose6d_b200 import load_model
    from megapose6d_b200.meshes import MeshDataBase
    from megapose6d_b200.renderer import BatchRenderer
    from workloads import weights

    cfg = load_model.Cfg(dict(CONFIGS[name], backbone_str="vanilla_resnet34", views_inplane_rotations=False))
    lay = LAYOUTS[name]
    ds, images, K0, rm = env["ds"], env["images"], env["K"], env["rm"]
    head = "pose_fc" if cfg.predict_pose_update else "views_logits_head"
    sd = weights.init_state_dict(helpers.n_inputs(cfg), head, 9 if cfg.predict_pose_update else cfg.n_rendered_views,
                                 seed=3)
    mesh_db = MeshDataBase.from_object_ds(ds).batched().cuda()
    model = load_model.create_model_pose(cfg, BatchRenderer(object_dataset=ds, mesh_db=mesh_db), mesh_db, sd)
    assert (model.backbone.c_pad, model._n_single_render_channels) == (lay.c_pad, lay.cpv)
    model.use_cuda_graphs = False
    n, (h, w) = 3, model.render_size
    labels = [env["labels"][i % 2] for i in range(n)]
    TCO = torch.from_numpy(procedural.random_poses(n, 19, z_range=(0.4, 0.8))).float()
    imgs = (images if lay.c_in == 4 else images[:, :3]).contiguous()
    K = K0.repeat(n, 1, 1)
    ids = torch.zeros(n, dtype=torch.long)
    if cfg.predict_pose_update:
        it = model(images=imgs.cuda(), K=K.cuda(), labels=labels, TCO=TCO.cuda(), n_iterations=1, batch_im_ids=ids)
        it = it["iteration=1"]
        boxes, KV, TCV_O, tCR = it.boxes_crop, it.KV_crop, it.TCV_O_input, it.tCR
    else:
        model.forward_coarse(imgs.cuda(), K.cuda(), labels, TCO.cuda(), batch_im_ids=ids)
        TCV_O = lib3d.normalize_T(TCO.cuda()).unsqueeze(1)
        tCR = TCV_O[:, 0, :3, 3].contiguous()
        _, boxes, K_crop = lib3d.crop_geometry(mesh_db.point_subset(2000), mesh_db.label_ids(labels, DEV),
                                               TCV_O[:, 0].contiguous(), K.cuda(), tCR, imgs.shape[-2:], (h, w))
        KV = K_crop.unsqueeze(1)
    x = model._input_buffer(n, h, w).cpu()
    boxes, KV, TCV_O, tCR = boxes.cpu(), KV.cpu(), TCV_O.cpu(), tCR.cpu()
    kind = DEPTH_NORM_KINDS[cfg.depth_normalization_type]
    z = tCR[:, 2]
    # renders: exact
    labels_mv = [l for l in labels for _ in range(lay.views)]
    ref = pipeline_ref.RefRenderer(rm).render(labels_mv, TCV_O.flatten(0, 1), KV.flatten(0, 1), None, (h, w),
                                              render_depth=lay.render_depth, render_normals=lay.normals,
                                              point_lights=not lay.normals)
    views = _render_planes(ref, lay, z.repeat_interleave(lay.views), kind)
    # crop: torchvision fp32
    boxes5 = torch.cat((torch.zeros(n, 1), boxes), dim=1)
    crop = L.crop_images(imgs, boxes5, (h, w))
    want_crop = _crop_planes(crop, lay.c_in, z, kind)
    tol = torch.full((n, lay.c_pad, h, w), float("nan"))
    if lay.c_in == 4:
        import torchvision
        valid = torchvision.ops.roi_align((imgs[:, 3:] > 0).float(), boxes5, output_size=(h, w), sampling_ratio=4)[:, 0]
    for s in range(n):
        b = boxes[s].tolist()
        tol[s, :lay.c_in] = crop_error_bound(imgs, b, lay.c_in, z[s].item(), kind, want_crop[s])
        if lay.c_in == 4:
            e_valid = 16 * 2.0 ** -24 * (max(abs(v) for v in b) + 4) + 2.0 ** -20
            tol[s, 3][(valid[s] - 0.99).abs() <= e_valid] = float("inf")
    planes = torch.cat((want_crop, views), dim=1)
    want = _assemble(planes, lay.c_pad, 0.0)
    _assert_x(x, want, _assemble_tol(tol), name, _assemble(planes, lay.c_pad, 0.0, act=False))
    assert torch.equal(model.backbone.pack_input(planes.cuda()).cpu().view(torch.int16), want.view(torch.int16))
    got_crop = _unpack(x, lay.c_in)
    print(f"{name}: max |crop - torchvision fp32| = {(got_crop - want_crop).abs().max():.3g}")
