"""The C_out = 64 pixel-major kernel (conv64_wgmma_kernel in conv_wgmma.cu): 256-pixel tiles on the wgmma N dimension,
two consumer warpgroups taking alternate tiles, an epilogue staged through shared memory and stored by TMA, and the skipped
k16 steps of the space-to-depth stem.

Bit-exact cases run with mode bit 26 (every convolution the kernel can serve takes it) on the integer operands of
test_gpu_conv_exact, inside NaN guards a full tile of rows wide.  _uses_conv64 restates the dispatch rule of conv_forward;
test_dispatch_rule_covers_the_cases (no GPU) checks that the case list reaches each of its edges.
"""
from __future__ import annotations

import dataclasses

import pytest
import torch

from megapose6d_b200 import _abi
from tests.test_gpu_conv_exact import (ACT, DEFAULT_CONV_MODE, FORCE_C64, NEVER_C64, P0, P1, SMS_H100, STEM, TINY, UNIT,
                                       Conv, _conv64, _gen, _guarded, _guards_intact, _launch, _out_dim, _problem, _to_act,
                                       device_kernels, mode_fixture)

gpu = pytest.mark.gpu
C64_PIXELS = 256
C64_STAGES = 4


def _uses_conv64(c: Conv, mode: int, sms: int, out_aligned: bool = True) -> bool:
    """conv_forward's choice of conv64_wgmma_kernel for mpx_conv2d (no K split)."""
    if c.cout != 64 or c.block_n != 0 or c.splits is not None or not out_aligned or mode & NEVER_C64:
        return False
    P, Q = _out_dim(c.h, c.pads[0], c.pads[2], c.r, c.stride), _out_dim(c.w, c.pads[1], c.pads[3], c.s, c.stride)
    tiles = -(-c.n * P * Q // C64_PIXELS)
    return bool(mode & FORCE_C64) or tiles >= 2 * (c.max_ctas or sms)


def _c64(name, n, h, w, cin, r, s, **kw):
    return Conv(name, n, h, w, cin, 64, r, s, **kw)


CASES = [
    # M and the partial last tile
    _c64("m1", 1, 1, 1, 64, 1, 1, relu=True, res=True),
    _c64("m255", 1, 15, 17, 64, 3, 3, pads=P1, relu=True),
    _c64("m256", 1, 16, 16, 64, 3, 3, pads=P1, res=True),
    _c64("m257_1x1", 1, 1, 257, 64, 1, 1),
    _c64("m513_last_tile_one_row", 1, 27, 19, 64, 3, 3, pads=P1, relu=True, res=True),
    _c64("m129_second_half_one_row", 1, 3, 43, 64, 3, 3, pads=P1, res=True),
    _c64("pq63_n9_tiles_span_images", 9, 7, 9, 64, 3, 3, pads=P1, relu=True, res=True),
    # persistent loop: warpgroup 1 gets one tile more than warpgroup 2, or warpgroup 2 none
    _c64("ctas1_5tiles", 5, 16, 16, 64, 3, 3, pads=P1, relu=True, res=True, max_ctas=1),
    _c64("ctas2_3tiles", 3, 16, 16, 64, 3, 3, pads=P1, res=True, max_ctas=2),
    _c64("ctas3_7tiles", 7, 16, 16, 128, 1, 1, relu=True, max_ctas=3),
    _c64("ctas3_2tiles", 2, 16, 16, 64, 1, 3, pads=(0, 1, 0, 1), max_ctas=3),
    # k-block counts around the ring depth (4) and far beyond it
    _c64("kb1", 2, 20, 20, 64, 1, 1, res=True, max_ctas=2),
    _c64("kb3", 2, 20, 20, 64, 3, 1, pads=(1, 0, 1, 0), relu=True, max_ctas=2),
    _c64("kb4", 2, 20, 20, 256, 1, 1, relu=True, res=True, max_ctas=2),
    _c64("kb5", 2, 20, 20, 320, 1, 1, max_ctas=2),
    _c64("kb9", 2, 20, 20, 64, 3, 3, pads=P1, relu=True, res=True, max_ctas=2),
    _c64("kb72", 2, 12, 14, 512, 3, 3, pads=P1, res=True, max_ctas=1),
    # im2col geometry
    _c64("s2_3x3", 3, 31, 40, 64, 3, 3, stride=2, pads=P1, relu=True, res=True),
    _c64("s2_1x1_pad0", 3, 31, 41, 128, 1, 1, stride=2),
    _c64("stem_4x4_c64", 2, 24, 32, 64, 4, 4, pads=STEM, relu=True),
    # rounding families
    _c64("ties", 2, 20, 26, 64, 3, 3, pads=P1, res=True, family="ties"),
    _c64("ties_relu", 2, 20, 26, 64, 1, 1, relu=True, family="ties"),
    _c64("saturate", 2, 20, 26, 64, 3, 3, pads=P1, res=True, family="saturate"),
    _c64("saturate_relu", 2, 20, 26, 64, 1, 1, relu=True, family="saturate"),
]
assert len({c.name for c in CASES}) == len(CASES)


forced = mode_fixture(FORCE_C64 | DEFAULT_CONV_MODE)


def _ran_conv64(names):
    return any("conv64_wgmma_kernel" in n for n in names)


@gpu
@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_conv64_bit_exact(case, forced):
    if case.family == "saturate" and ACT != torch.float16:
        pytest.skip("saturation at +-65504 is the fp16 conversion")
    x, w, b, r, want = _problem(case, _gen(case.name))
    got, names = device_kernels(lambda: _launch(case, x, w, b, r), "conv64_wgmma_kernel")
    assert _ran_conv64(names) and not any("conv_wgmma_kernel" in n for n in names), names
    bad = got.float() != want.float()
    assert not bad.any(), f"{int(bad.sum())} of {bad.numel()} outputs differ, first at {bad.nonzero()[0].tolist()}"


def _run(c: Conv, x, w, b, r, flags):
    """mpx_conv2d with relu `flags`, the output between NaN guards of a tile of rows."""
    lib = _abi.lib()
    P, Q = _out_dim(c.h, c.pads[0], c.pads[2], c.r, c.stride), _out_dim(c.w, c.pads[1], c.pads[3], c.s, c.stride)
    guard = C64_PIXELS * 64
    obuf, out = _guarded((c.n, P, Q, 64), guard, float("nan"))
    xv = x.to(ACT).contiguous()
    rv = r.to(ACT).contiguous() if r is not None else None
    _abi.check(lib.mpx_conv2d(_abi.ptr(xv), c.n, c.h, c.w, c.cin, _abi.ptr(w.reshape(64, -1).to(ACT).contiguous()),
                              _abi.ptr(b.float().contiguous()), 64, c.r, c.s, c.stride, *c.pads, flags, _abi.ptr(rv),
                              _abi.ptr(out), 0, c.max_ctas, _abi.stream_ptr()))
    torch.cuda.synchronize()
    assert _guards_intact(obuf, guard, float("nan")), "write outside the output tensor"
    return out


@gpu
def test_misaligned_output_is_refused_before_any_kernel(forced):
    """The TMA store needs a 16-byte-aligned output.  mpx_conv2d refuses any pointer that is not 16-byte aligned before
    it reaches the kernel choice (as it always has), so an output 4 bytes off alignment is an error even with bit 26, and
    nothing is launched; the network's workspace buffers are 256-byte aligned."""
    c = _c64("misaligned_out", 2, 20, 26, 64, 3, 3, pads=P1, relu=True)
    x, w, b, _, _ = _problem(c, _gen(c.name))
    lib = _abi.lib()
    obuf = torch.full((2 * 20 * 26 * 64 + 8,), float("nan"), dtype=ACT, device="cuda")
    out = obuf[2:2 + 2 * 20 * 26 * 64]  # 4-byte aligned only
    assert out.data_ptr() % 16 == 4
    xv = x.to(ACT).contiguous()
    launches = lib.mpx_launch_count()
    rc = lib.mpx_conv2d(_abi.ptr(xv), c.n, c.h, c.w, c.cin, _abi.ptr(w.reshape(64, -1).to(ACT).contiguous()),
                        _abi.ptr(b.float().contiguous()), 64, c.r, c.s, c.stride, *c.pads, 1, None, _abi.ptr(out), 0, 0,
                        _abi.stream_ptr())
    torch.cuda.synchronize()
    assert rc == -1 and b"16-byte aligned" in lib.mpx_last_error(), (rc, lib.mpx_last_error())
    assert lib.mpx_launch_count() == launches
    assert torch.isnan(obuf).all()


def _stem_zero_slices(cin):
    """[4, 4, cin] mask of the weight columns that are structurally zero in the space-to-depth form of a 7x7 / s2 stem
    (backbone._stem_s2d): column (r, s, (dy*2+dx)*c_pad + c) holds the 7x7 tap (2r+dy-1, 2s+dx-1)."""
    c_pad = cin // 4
    m = torch.zeros(4, 4, cin, dtype=torch.bool)
    for r in range(4):
        for s in range(4):
            for sl in range(4):
                ky, kx = 2 * r + sl // 2 - 1, 2 * s + sl % 2 - 1
                m[r, s, sl * c_pad:(sl + 1) * c_pad] = not (0 <= ky <= 6 and 0 <= kx <= 6)
    return m


@gpu
@pytest.mark.parametrize("cin", [64, 128], ids=["c_pad16", "c_pad32"])
def test_stem_skips_structural_zero_slices(cin, forced):
    """Stem-shaped weights with non-zero garbage in the structurally zero slices: with relu bit 1 (space-to-depth stem
    weights) the result equals the convolution with those slices zeroed, so their MMAs were not issued; without it the
    garbage counts."""
    c = _c64(f"stem_skip_{cin}", 2, 24, 32, cin, 4, 4, pads=STEM, relu=True)
    g = _gen(c.name)
    x, w, b, r, want = _problem(c, g)
    zero = _stem_zero_slices(cin).to(w.device)
    assert int(zero[:, :, ::cin // 4].sum()) == 15  # 64 - 7 * 7 slices
    w_clean = torch.where(zero, torch.zeros_like(w), w)
    garbage = torch.where(zero, torch.randint(1, 4, w.shape, generator=g, device=w.device).double(), torch.zeros_like(w))
    want_clean = _to_act(torch.relu(_conv64(x, w_clean, 1, STEM) + b))
    want_garbage = _to_act(torch.relu(_conv64(x, w_clean + garbage, 1, STEM) + b))
    assert not torch.equal(want_clean, want_garbage)
    got, names = device_kernels(lambda: _run(c, x, w_clean + garbage, b, None, flags=1 | 2), "conv64_wgmma_kernel")
    assert _ran_conv64(names) and torch.equal(got, want_clean)
    got, names = device_kernels(lambda: _run(c, x, w_clean + garbage, b, None, flags=1), "conv64_wgmma_kernel")
    assert _ran_conv64(names) and torch.equal(got, want_garbage)


GAUSS_CASES = [  # batch >= 64 at the coarse network's shapes (240x320 renders)
    _c64("gauss_stem", 64, 120, 160, 64, 4, 4, pads=STEM, relu=True),
    _c64("gauss_layer1_conv2_res", 64, 60, 80, 64, 3, 3, pads=P1, relu=True, res=True),
]


@gpu
@pytest.mark.parametrize("case", GAUSS_CASES, ids=[c.name for c in GAUSS_CASES])
def test_conv64_gaussian_data_within_rounding_bound(case):
    """Gaussian operands at the default mode (the size selects the kernel), per element within the bound of
    test_gpu_conv_exact:  |y - y64| <= u |y64| + tiny + (K + 2) 2^-23 (conv(|x|, |w|) + |b| + |r|)."""
    assert _uses_conv64(case, DEFAULT_CONV_MODE, _abi.lib().mpx_sm_count())
    g = _gen(case.name)
    k = case.r * case.s * case.cin
    P, Q = _out_dim(case.h, case.pads[0], case.pads[2], case.r, 1), _out_dim(case.w, case.pads[1], case.pads[3], case.s, 1)
    x = torch.randn(case.n, case.h, case.w, case.cin, device="cuda", generator=g).to(ACT).double()
    w = (torch.randn(64, case.r, case.s, case.cin, device="cuda", generator=g) / k ** 0.5).to(ACT).double()
    b = torch.randn(64, device="cuda", generator=g).double()
    r = torch.randn(case.n, P, Q, 64, device="cuda", generator=g).to(ACT).double() if case.res else None
    y64 = _conv64(x, w, case.stride, case.pads) + b + (r if r is not None else 0)
    if case.relu:
        y64 = torch.relu(y64)
    mag = _conv64(x.abs(), w.abs(), case.stride, case.pads) + b.abs() + (r.abs() if r is not None else 0)
    got, names = device_kernels(lambda: _run(case, x, w, b, r, flags=int(case.relu)), "conv64_wgmma_kernel")
    assert _ran_conv64(names), names
    got = got.double()
    err = (got - y64).abs()
    bound = UNIT * y64.abs() + TINY + (k + 2) * 2.0 ** -23 * mag
    assert (err <= bound).all(), (err - bound).max().item()


@gpu
def test_network_forward_with_and_without_conv64():
    """A coarse forward at a batch whose stem and layer1 take the pixel-major kernel, against the same forward with mode
    bit 22 (the 128-row kernel everywhere): within the act16 bound of test_gpu_net."""
    from megapose6d_b200.backbone import ResNet34Engine
    from oracle import resnet_ref
    from tests import helpers

    n = 16  # layer1: 16 * 60 * 80 / 256 = 300 tiles >= 2 * 132
    assert _uses_conv64(_c64("layer1", n, 60, 80, 64, 3, 3, pads=P1), DEFAULT_CONV_MODE, _abi.lib().mpx_sm_count())
    cfg = helpers.COARSE_CFG
    sd = helpers.make_state_dict(cfg, seed=4)
    eng = ResNet34Engine(sd, n_inputs=helpers.n_inputs(cfg), head="views_logits_head")
    xc = helpers._calibration_batch(helpers.n_inputs(cfg), 6, n=n)
    x = eng.pack_input(xc.cuda())
    lib = _abi.lib()
    try:
        lib.mpx_net_set_graphs(0)
        lib.mpx_conv_set_mode(DEFAULT_CONV_MODE | NEVER_C64)
        old, names_old = device_kernels(lambda: eng.forward(x, 240, 320).clone())
        lib.mpx_conv_set_mode(DEFAULT_CONV_MODE)
        new, names_new = device_kernels(lambda: eng.forward(x, 240, 320).clone(), "conv64_wgmma_kernel", 7)
    finally:
        lib.mpx_net_set_graphs(1)
        lib.mpx_conv_set_mode(DEFAULT_CONV_MODE)
    # stem + 6 layer1 convolutions on the pixel-major kernel by default, none under bit 22
    assert sum("conv64_wgmma_kernel" in n for n in names_new) == 7 and not _ran_conv64(names_old)
    with torch.no_grad():
        bound = resnet_ref.act16_forward_error_bound(sd, xc, dtype=ACT).cuda()
    err = (new - old).abs()
    print(f"conv64 network: max |new - old| = {err.max().item():.3g}, bit-identical: {torch.equal(new, old)}")
    assert torch.isfinite(new).all()
    assert (err <= 0.5 * bound + 1e-6).all(), (err.max(), bound.min())


def test_dispatch_rule_covers_the_cases():
    """The case list reaches every edge of the pixel-major kernel, evaluated for a 132-SM H100."""
    for c in CASES:
        assert _uses_conv64(c, FORCE_C64, SMS_H100), c.name
    plans = []
    for c in CASES:
        P, Q = _out_dim(c.h, c.pads[0], c.pads[2], c.r, c.stride), _out_dim(c.w, c.pads[1], c.pads[3], c.s, c.stride)
        m = c.n * P * Q
        tiles = -(-m // C64_PIXELS)
        grid = min(tiles, c.max_ctas or SMS_H100)
        plans.append((c, dict(M=m, tiles=tiles, grid=grid, pq=P * Q, nkb=c.r * c.s * c.cin // 64,
                              last_rows=m - (tiles - 1) * C64_PIXELS)))
    need = {
        "M = 1": lambda c, p: p["M"] == 1,
        "M = 255": lambda c, p: p["M"] == 255,
        "M = 256": lambda c, p: p["M"] == 256,
        "M = 257": lambda c, p: p["M"] == 257,
        "last tile with one row, several tiles": lambda c, p: p["last_rows"] == 1 and p["tiles"] > 2,
        "second 128-pixel half with one row": lambda c, p: p["last_rows"] == 129,
        "tiles spanning images": lambda c, p: p["pq"] < C64_PIXELS and c.n > 2,
        "one CTA, warpgroup 1 one tile more": lambda c, p: p["grid"] == 1 and p["tiles"] % 2 == 1 and p["tiles"] >= 3,
        "a CTA whose warpgroup 2 has no tile": lambda c, p: c.max_ctas >= 2 and p["tiles"] < 2 * p["grid"],
        "max_ctas 3 over uneven tiles": lambda c, p: c.max_ctas == 3 and p["tiles"] % 3 != 0,
        "1x1": lambda c, p: (c.r, c.s) == (1, 1),
        "3x3 pad 1": lambda c, p: (c.r, c.s, c.pads) == (3, 3, P1),
        "stride 2": lambda c, p: c.stride == 2,
        "1x1 stride 2 pad 0": lambda c, p: (c.r, c.s, c.stride, c.pads) == (1, 1, 2, P0),
        "4x4 stem geometry": lambda c, p: c.pads == STEM,
    }
    for nkb in (1, C64_STAGES - 1, C64_STAGES, C64_STAGES + 1, 2 * C64_STAGES + 1, 72):
        need[f"{nkb} k-blocks"] = lambda c, p, nkb=nkb: p["nkb"] == nkb
    for relu in (False, True):
        for res in (False, True):
            need[f"relu {relu}, residual {res}"] = lambda c, p, relu=relu, res=res: c.relu == relu and c.res == res
    for fam in ("exact", "ties", "saturate"):
        need[f"family {fam}"] = lambda c, p, fam=fam: c.family == fam
    missing = [what for what, pred in need.items() if not any(pred(c, p) for c, p in plans)]
    assert not missing, missing
    # the rule itself: size threshold, and what keeps the 128-row kernel
    stem = _c64("stem", 1, 120, 160, 64, 4, 4, pads=STEM, relu=True)
    layer1 = _c64("layer1", 1, 60, 80, 64, 3, 3, pads=P1, relu=True, res=True)
    assert not _uses_conv64(stem, DEFAULT_CONV_MODE, SMS_H100)  # 75 tiles
    assert _uses_conv64(dataclasses.replace(stem, n=4), DEFAULT_CONV_MODE, SMS_H100)  # 300 tiles
    assert not _uses_conv64(dataclasses.replace(layer1, n=14), DEFAULT_CONV_MODE, SMS_H100)  # 263 tiles
    assert _uses_conv64(dataclasses.replace(layer1, n=15), DEFAULT_CONV_MODE, SMS_H100)  # 282 tiles
    assert _uses_conv64(dataclasses.replace(layer1, n=576), DEFAULT_CONV_MODE, SMS_H100)
    assert not _uses_conv64(dataclasses.replace(layer1, n=576), DEFAULT_CONV_MODE | NEVER_C64, SMS_H100)
    assert not _uses_conv64(dataclasses.replace(layer1, n=576), FORCE_C64 | NEVER_C64, SMS_H100)
    for other in (dict(cout=128), dict(block_n=64), dict(splits=1)):
        assert not _uses_conv64(dataclasses.replace(layer1, n=576, **other), FORCE_C64, SMS_H100), other
    assert not _uses_conv64(dataclasses.replace(layer1, n=576), FORCE_C64, SMS_H100, out_aligned=False)
