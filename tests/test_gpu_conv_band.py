"""The band producer of the C_out = 64 pixel-major kernel (conv64_wgmma_kernel<stem, N> with N = 160 or 256 in
conv_wgmma.cu): for a stride-1 convolution a tile is whole output rows of one image, each (filter row, 64 channels) of it
is one tiled TMA load of a band of padded input rows, and filter tap s reads that band s pixel rows further on.

Bit-exact cases use the integer operands of test_gpu_conv_exact (torch.equal against a float64 convolution) with mode
bit 26, so that small shapes reach the kernel, and compare with the im2col producer (mode bit 23) as well.  Every case
checks by name, with torch.profiler, which instantiation ran.  _band_plan restates the producer choice and tile shape of
conv64_forward; test_band_rule_covers_the_cases (no GPU) checks that the cases reach each of its edges and that the coarse
network's stem and layer1 take the band producer at both render sizes.
"""
from __future__ import annotations

import dataclasses
import re
import types

import pytest
import torch

from megapose6d_b200 import _abi
from tests.test_gpu_conv64 import C64_PIXELS, _c64, _stem_zero_slices, _uses_conv64
from tests.test_gpu_conv_exact import (ACT, DEFAULT_CONV_MODE, FORCE_C64, FORCE_IM2COL, NEVER_C64, P1, SMS_H100, STEM, Conv,
                                       _conv64, _gen, _guarded, _guards_intact, _launch, _out_dim, _problem, _to_act,
                                       device_kernels, mode_fixture, set_mode)

gpu = pytest.mark.gpu
BAND_SLOTS = 3
LAYOUT_BYTES = 227 * 1024 - 1536  # shared memory less alignment slack, barriers and bias


def _band_plan(c: Conv):
    """conv64_forward's producer for a convolution that reaches the pixel-major kernel without bit 23: None for im2col,
    else the band tile (rows per tile, tiles per image, wgmma N)."""
    wp = c.w + c.pads[1] + c.pads[3]
    if c.stride != 1 or wp > C64_PIXELS or c.cin // 64 > BAND_SLOTS - 1:
        return None
    P, Q = _out_dim(c.h, c.pads[0], c.pads[2], c.r, 1), _out_dim(c.w, c.pads[1], c.pads[3], c.s, 1)
    rows = min(P, C64_PIXELS // wp)
    tiles = -(-P // rows)
    cols = (rows - 1) * wp + Q  # the columns a tile's MMAs must cover
    n = 160 if cols <= 160 else 256
    # shared-memory layout (conv64_band_layout): all weights resident beside the most band slots that fit, else a ring
    r1k = lambda b: -(-b // 1024) * 1024  # noqa: E731
    cblocks = c.cin // 64
    slot, staging, weights = r1k(wp * rows * 128), r1k(rows * Q * 128), c.r * c.s * cblocks * 8192
    slots = next((k for k in range(BAND_SLOTS, cblocks, -1) if k * slot + weights + 2 * staging <= LAYOUT_BYTES
                  and (k - 1) * slot + (n + c.s - 1) * 128 <= LAYOUT_BYTES), None)
    return types.SimpleNamespace(wp=wp, P=P, Q=Q, rows=rows, tiles_per_img=tiles, last_rows=P - (tiles - 1) * rows, n=n,
                                 resident=slots is not None, slots=slots or BAND_SLOTS)


def _conv64_instances(names):
    """(stem cblocks, band N) of every conv64_wgmma_kernel launch in `names`; band N = 0 is the im2col producer."""
    out = []
    for n in names:
        m = re.search(r"conv64_wgmma_kernel<(\d+), (\d+)>", n)
        if m:
            out.append((int(m.group(1)), int(m.group(2))))
    return out


restore_mode = mode_fixture()


# geometry of the coarse network at the two render sizes: stem over the space-to-depth input, layer1 after the max-pool
STEM_240, L1_240 = (120, 160), (60, 80)
STEM_224, L1_224 = (112, 112), (56, 56)

CASES = [
    # the network's shapes: Q = 160 (one row per tile, n160), 80 (3 rows), 112 (2 rows), 56 (4 rows)
    _c64("stem_240x320", 2, *STEM_240, 64, 4, 4, pads=STEM, relu=True),
    _c64("stem_224x224", 2, *STEM_224, 64, 4, 4, pads=STEM, relu=True),
    _c64("stem_c_pad32_240x320", 2, *STEM_240, 128, 4, 4, pads=STEM, relu=True),
    _c64("layer1_240x320", 2, *L1_240, 64, 3, 3, pads=P1, relu=True),
    _c64("layer1_240x320_res", 2, *L1_240, 64, 3, 3, pads=P1, relu=True, res=True),
    _c64("layer1_224x224", 3, *L1_224, 64, 3, 3, pads=P1, relu=True),
    _c64("layer1_224x224_res", 3, *L1_224, 64, 3, 3, pads=P1, relu=True, res=True),
    # an image's last tile shorter than the others (19 rows in tiles of 6), consecutive images, several tiles per CTA
    _c64("last_tile_one_row_3_images", 3, 19, 40, 64, 3, 3, pads=P1, relu=True, res=True),
    _c64("one_cta_odd_tiles", 3, 19, 40, 64, 3, 3, pads=P1, res=True, max_ctas=1),
    _c64("two_ctas", 5, 13, 60, 64, 3, 3, pads=P1, relu=True, max_ctas=2),
    # padding on one side only: top + left, bottom + right, and none
    _c64("pad_top_left", 2, 20, 30, 64, 3, 3, pads=(2, 2, 0, 0), relu=True, res=True),
    _c64("pad_bottom_right", 2, 20, 30, 64, 3, 3, pads=(0, 0, 2, 2), res=True),
    _c64("pad_none_5x5", 2, 20, 30, 64, 5, 5),
    _c64("filter_1x3", 2, 20, 30, 64, 1, 3, pads=(0, 1, 0, 1), relu=True),
    _c64("filter_3x1", 2, 20, 30, 64, 3, 1, pads=(1, 0, 1, 0)),
    # M = 1, 255, 256, 257 (257 = one 257 x 1 image: 85 rows per tile, a last tile of two rows)
    _c64("m1", 1, 1, 1, 64, 1, 1, relu=True, res=True),
    _c64("m255", 1, 15, 17, 64, 3, 3, pads=P1, relu=True),
    _c64("m256", 1, 16, 16, 64, 3, 3, pads=P1, res=True),
    _c64("m257", 1, 257, 1, 64, 3, 3, pads=P1, relu=True, res=True),
    # widest band (Wp = 256), several rows on the n160 chain, two bands per filter row
    _c64("wp256", 2, 5, 254, 64, 3, 3, pads=P1, res=True),
    _c64("n160_two_rows", 3, 2, 64, 64, 3, 3, pads=P1, relu=True),
    _c64("cin128_3x3", 2, 20, 30, 128, 3, 3, pads=P1, relu=True, res=True),
    _c64("cin128_1x1_one_cta", 5, 16, 16, 128, 1, 1, relu=True, max_ctas=1),
    # rounding families
    _c64("ties", 2, 20, 26, 64, 3, 3, pads=P1, res=True, family="ties"),
    _c64("ties_relu", 2, 20, 26, 64, 1, 1, relu=True, family="ties"),
    _c64("saturate", 2, 20, 26, 64, 3, 3, pads=P1, res=True, family="saturate"),
    _c64("saturate_relu", 2, 20, 26, 64, 1, 1, relu=True, family="saturate"),
]
assert len({c.name for c in CASES}) == len(CASES)


@gpu
@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_band_bit_exact(case, restore_mode):
    if case.family == "saturate" and ACT != torch.float16:
        pytest.skip("saturation at +-65504 is the fp16 conversion")
    plan = _band_plan(case)
    assert plan is not None
    x, w, b, r, want = _problem(case, _gen(case.name))
    set_mode(DEFAULT_CONV_MODE | FORCE_C64)
    got, names = device_kernels(lambda: _launch(case, x, w, b, r), "conv64_wgmma_kernel")
    assert _conv64_instances(names) == [(0, plan.n)], names
    bad = got.float() != want.float()
    assert not bad.any(), f"{int(bad.sum())} of {bad.numel()} outputs differ, first at {bad.nonzero()[0].tolist()}"
    set_mode(DEFAULT_CONV_MODE | FORCE_C64 | FORCE_IM2COL)
    old, names = device_kernels(lambda: _launch(case, x, w, b, r), "conv64_wgmma_kernel")
    assert _conv64_instances(names) == [(0, 0)], names
    assert torch.equal(old, got)


def _run_stem(c: Conv, x, w, b):
    """mpx_conv2d with relu bits 0 and 1 (ReLU, space-to-depth stem weights), the output between NaN guards.  The 16-bit
    operands stay referenced until the launch has finished: a temporary freed while the kernel is queued can be handed to
    the next allocation and overwritten before the kernel reads it."""
    lib = _abi.lib()
    P, Q = _out_dim(c.h, c.pads[0], c.pads[2], c.r, 1), _out_dim(c.w, c.pads[1], c.pads[3], c.s, 1)
    guard = C64_PIXELS * 64
    obuf, out = _guarded((c.n, P, Q, 64), guard, float("nan"))
    xv = x.to(ACT).contiguous()
    wv = w.reshape(64, -1).to(ACT).contiguous()
    bv = b.float().contiguous()
    _abi.check(lib.mpx_conv2d(_abi.ptr(xv), c.n, c.h, c.w, c.cin, _abi.ptr(wv), _abi.ptr(bv), 64, c.r, c.s, 1, *c.pads,
                              1 | 2, None, _abi.ptr(out), 0, c.max_ctas, _abi.stream_ptr()))
    torch.cuda.synchronize()
    assert _guards_intact(obuf, guard, float("nan")), "write outside the output tensor"
    return out


@gpu
@pytest.mark.parametrize("cin,size", [(64, STEM_240), (64, STEM_224), (128, STEM_240)],
                         ids=["c_pad16_240x320", "c_pad16_224x224", "c_pad32_240x320"])
def test_band_stem_skips_structural_zero_slices(cin, size, restore_mode):
    """Space-to-depth stem weights (relu bit 1) with non-zero garbage in the structurally zero slices: the unrolled stem
    instantiation of the band producer equals the convolution with those slices zeroed, as the im2col producer does."""
    c = _c64(f"band_stem_skip_{cin}_{size[0]}", 2, *size, cin, 4, 4, pads=STEM, relu=True)
    g = _gen(c.name)
    x, w, b, _, _ = _problem(c, g)
    zero = _stem_zero_slices(cin).to(w.device)
    w_clean = torch.where(zero, torch.zeros_like(w), w)
    garbage = torch.where(zero, torch.randint(1, 4, w.shape, generator=g, device=w.device).double(), torch.zeros_like(w))
    want = _to_act(torch.relu(_conv64(x, w_clean, 1, STEM) + b))
    assert not torch.equal(want, _to_act(torch.relu(_conv64(x, w_clean + garbage, 1, STEM) + b)))
    set_mode(DEFAULT_CONV_MODE | FORCE_C64)
    got, names = device_kernels(lambda: _run_stem(c, x, w_clean + garbage, b), "conv64_wgmma_kernel")
    assert _conv64_instances(names) == [(cin // 64, _band_plan(c).n)], names
    assert torch.equal(got, want)
    set_mode(DEFAULT_CONV_MODE | FORCE_C64 | FORCE_IM2COL)
    old, names = device_kernels(lambda: _run_stem(c, x, w_clean + garbage, b), "conv64_wgmma_kernel")
    assert _conv64_instances(names) == [(cin // 64, 0)], names
    assert torch.equal(old, got)


@gpu
@pytest.mark.parametrize("size,n", [((240, 320), 16), ((224, 224), 24)], ids=["240x320", "224x224"])
def test_network_forward_band_and_im2col_identical(size, n, restore_mode):
    """A coarse forward at a batch whose stem and layer1 reach the pixel-major kernel: all 7 of those launches take the band
    producer by default and the im2col producer under bit 23, and the network's outputs are bit-identical."""
    from megapose6d_b200.backbone import ResNet34Engine
    from tests import helpers

    h, w = size
    assert _uses_conv64(_c64("layer1", n, h // 4, w // 4, 64, 3, 3, pads=P1), DEFAULT_CONV_MODE, _abi.lib().mpx_sm_count())
    cfg = helpers.COARSE_CFG
    sd = helpers.make_state_dict(cfg, seed=4)
    eng = ResNet34Engine(sd, n_inputs=helpers.n_inputs(cfg), head="views_logits_head")
    g = torch.Generator(device="cuda").manual_seed(5)
    x = eng.pack_input(torch.rand(n, helpers.n_inputs(cfg), h, w, device="cuda", generator=g) * 2 - 1)
    lib = _abi.lib()
    try:
        lib.mpx_net_set_graphs(0)
        set_mode(DEFAULT_CONV_MODE)
        eng.forward(x, h, w)  # workspace and first launches outside the profiled window
        torch.cuda.synchronize()
        new, names_new = device_kernels(lambda: eng.forward(x, h, w).clone(), "conv64_wgmma_kernel", 7)
        set_mode(DEFAULT_CONV_MODE | FORCE_IM2COL)
        old, names_old = device_kernels(lambda: eng.forward(x, h, w).clone(), "conv64_wgmma_kernel", 7)
    finally:
        lib.mpx_net_set_graphs(1)
    inst_new, inst_old = _conv64_instances(names_new), _conv64_instances(names_old)
    assert len(inst_new) == 7 and all(bn > 0 for _, bn in inst_new), (inst_new, len(names_new), names_new[:3])
    assert len(inst_old) == 7 and all(bn == 0 for _, bn in inst_old), (inst_old, len(names_old), names_old[:3])
    assert torch.isfinite(new).all()
    assert torch.equal(new, old)


def test_band_rule_covers_the_cases():
    """The producer rule and the case list, evaluated for a 132-SM H100 (no GPU)."""
    for c in CASES:
        assert _uses_conv64(c, FORCE_C64, SMS_H100) and _band_plan(c) is not None, c.name
    plans = [(c, _band_plan(c)) for c in CASES]
    need = {
        "n160, one row per tile": lambda c, p: p.n == 160 and p.rows == 1,
        "n160, several rows per tile": lambda c, p: p.n == 160 and p.rows > 1,
        "n256, several rows per tile": lambda c, p: p.n == 256 and p.rows > 1,
        "an image's last tile shorter": lambda c, p: p.last_rows < p.rows,
        "one tile per image, several images": lambda c, p: p.tiles_per_img == 1 and c.n > 1,
        "Wp = 256": lambda c, p: p.wp == C64_PIXELS,
        "resident weights, 2 band slots": lambda c, p: p.resident and p.slots == 2,
        "resident weights, 3 band slots": lambda c, p: p.resident and p.slots == 3,
        "weight ring": lambda c, p: not p.resident,
        "weight ring, two bands per filter row": lambda c, p: not p.resident and c.cin == 128 and c.r > 1,
        "two bands per filter row": lambda c, p: c.cin == 128 and c.r > 1,
        "one CTA": lambda c, p: c.max_ctas == 1,
        "top and left padding only": lambda c, p: c.pads[:2] != (0, 0) and c.pads[2:] == (0, 0),
        "bottom and right padding only": lambda c, p: c.pads[:2] == (0, 0) and c.pads[2:] != (0, 0),
        "stem geometry": lambda c, p: c.pads == STEM,
    }
    for m in (1, 255, 256, 257):
        need[f"M = {m}"] = lambda c, p, m=m: c.n * p.P * p.Q == m
    for q in (160, 80, 112, 56):
        need[f"Q = {q}"] = lambda c, p, q=q: p.Q == q
    for relu in (False, True):
        for res in (False, True):
            need[f"relu {relu}, residual {res}"] = lambda c, p, relu=relu, res=res: c.relu == relu and c.res == res
    for fam in ("exact", "ties", "saturate"):
        need[f"family {fam}"] = lambda c, p, fam=fam: c.family == fam
    missing = [what for what, pred in need.items() if not any(pred(c, p) for c, p in plans)]
    assert not missing, missing
    # every convolution of the coarse forward that reaches the pixel-major kernel takes the band producer at both render
    # sizes, as does the refiner's c_pad 32 stem
    for (sh, sw), (lh, lw) in ((STEM_240, L1_240), (STEM_224, L1_224)):
        for cin in (64, 128):
            stem = _c64("stem", 576, sh, sw, cin, 4, 4, pads=STEM, relu=True)
            assert _uses_conv64(stem, DEFAULT_CONV_MODE, SMS_H100) and _band_plan(stem) is not None
        for res in (False, True):
            l1 = _c64("layer1", 576, lh, lw, 64, 3, 3, pads=P1, relu=True, res=res)
            assert _uses_conv64(l1, DEFAULT_CONV_MODE, SMS_H100) and _band_plan(l1) is not None
    assert (_band_plan(_c64("s", 1, *STEM_240, 64, 4, 4, pads=STEM)).rows, _band_plan(_c64("s", 1, *STEM_240, 64, 4, 4,
                                                                                          pads=STEM)).n) == (1, 160)
    assert (_band_plan(_c64("l", 1, *L1_240, 64, 3, 3, pads=P1)).rows, _band_plan(_c64("l", 1, *L1_240, 64, 3, 3,
                                                                                       pads=P1)).n) == (3, 256)
    # the 240x320 stem and layer1 keep their weights resident
    assert _band_plan(_c64("s", 1, *STEM_240, 64, 4, 4, pads=STEM)).resident
    assert _band_plan(_c64("l", 1, *L1_240, 64, 3, 3, pads=P1)).resident
    # what stays on the im2col producer: stride 2, a padded row wider than a TMA box, more than two 64-channel blocks
    layer1 = _c64("layer1", 576, *L1_240, 64, 3, 3, pads=P1, relu=True)
    assert _band_plan(dataclasses.replace(layer1, stride=2)) is None
    assert _band_plan(dataclasses.replace(layer1, h=1, w=255)) is None  # Wp = 257
    assert _band_plan(dataclasses.replace(layer1, h=1, w=254)) is not None  # Wp = 256
    assert _band_plan(dataclasses.replace(layer1, cin=192)) is None
    assert not _uses_conv64(layer1, DEFAULT_CONV_MODE | NEVER_C64, SMS_H100)
