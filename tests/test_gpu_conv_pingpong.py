"""The C_out = 128 .. 512 ping-pong kernel (convpp_wgmma_kernel in conv_wgmma.cu): each of two consumer warpgroups owns a
whole 128 x 128 tile, they take alternate tiles of the CTA's persistent sequence, and the epilogue is staged through
shared memory (residual TMA-loaded, result TMA-stored).

Bit-exact cases run with mode bit 28 (every convolution the kernel can serve takes it) on the integer operands of
test_gpu_conv_exact, inside NaN guards a full tile of rows wide.  _uses_pp restates the dispatch rule of conv_forward;
test_dispatch_rule_covers_the_cases (no GPU) checks that the case list reaches each of its edges.
"""
from __future__ import annotations

import dataclasses

import pytest
import torch

from megapose6d_b200 import _abi
from tests.test_gpu_conv_exact import (ACT, CAP, DEFAULT_CONV_MODE, FORCE_PP, NEVER_PP, NO_PDL, P0, P1, SMS_H100, TINY,
                                       UNIT, Conv, _conv64, _gen, _guarded, _ints, _launch, _out_dim, _problem, _to_act,
                                       _weights, device_kernels, mode_fixture, set_mode)

gpu = pytest.mark.gpu
BLOCK_M = 128
PP_STAGES = 4


def _items(c: Conv) -> int:
    P, Q = _out_dim(c.h, c.pads[0], c.pads[2], c.r, c.stride), _out_dim(c.w, c.pads[1], c.pads[3], c.s, c.stride)
    return -(-c.n * P * Q // BLOCK_M) * (c.cout // 128)


def _uses_pp(c: Conv, mode: int, sms: int, out_aligned: bool = True) -> bool:
    """conv_forward's choice of convpp_wgmma_kernel for mpx_conv2d (no K split): by default C_out = 128 only."""
    if c.cout % 128 or c.cout > 512 or c.block_n != 0 or c.splits is not None or not out_aligned:
        return False
    if mode & NEVER_PP:
        return False
    return bool(mode & FORCE_PP) or (c.cout == 128 and _items(c) >= 2 * (c.max_ctas or sms))


def _pp(name, n, h, w, cin, cout, r, s, **kw):
    return Conv(name, n, h, w, cin, cout, r, s, **kw)


CASES = [
    # M and the partial last tile
    _pp("m1", 1, 1, 1, 64, 128, 1, 1, relu=True, res=True),
    _pp("m127", 1, 1, 127, 64, 256, 1, 3, pads=(0, 1, 0, 1), relu=True),
    _pp("m128", 1, 8, 16, 128, 128, 3, 3, pads=P1, res=True),
    _pp("m129", 1, 3, 43, 64, 512, 3, 3, pads=P1, relu=True, res=True),
    _pp("m255", 1, 15, 17, 64, 128, 3, 3, pads=P1, res=True),
    _pp("m257_1x1", 1, 1, 257, 128, 256, 1, 1, relu=True),
    _pp("pq63_n9_tiles_span_images", 9, 7, 9, 64, 128, 3, 3, pads=P1, relu=True, res=True),
    # persistent loop: consumer 1 one tile more than consumer 2, a CTA whose second consumer has no tile, 1-3 CTAs
    _pp("ctas1_5tiles", 5, 8, 16, 64, 128, 3, 3, pads=P1, relu=True, res=True, max_ctas=1),
    _pp("ctas2_3tiles", 3, 8, 16, 64, 128, 3, 3, pads=P1, res=True, max_ctas=2),
    _pp("ctas3_8tiles_c512", 2, 8, 16, 64, 512, 3, 3, pads=P1, relu=True, max_ctas=3),
    _pp("ctas3_1tile", 1, 4, 16, 128, 128, 1, 1, relu=True, res=True, max_ctas=3),
    # k-block counts around the ring depth (4) and far beyond it, several tiles per consumer
    _pp("kb1", 2, 20, 20, 64, 256, 1, 1, res=True, max_ctas=2),
    _pp("kb3", 2, 20, 20, 64, 128, 3, 1, pads=(1, 0, 1, 0), relu=True, max_ctas=2),
    _pp("kb4", 2, 20, 20, 256, 128, 1, 1, relu=True, res=True, max_ctas=2),
    _pp("kb5", 2, 20, 20, 320, 256, 1, 1, max_ctas=2),
    _pp("kb9", 2, 20, 20, 64, 512, 3, 3, pads=P1, relu=True, res=True, max_ctas=2),
    _pp("kb72", 2, 12, 14, 512, 512, 3, 3, pads=P1, res=True, max_ctas=1),
    # the network's geometries: 3x3 s1, 3x3 s2, 1x1 s2 at every width
    _pp("s1_3x3_c256", 3, 15, 20, 256, 256, 3, 3, pads=P1, relu=True, res=True),
    _pp("s2_3x3_c128", 3, 31, 40, 64, 128, 3, 3, stride=2, pads=P1, relu=True),
    _pp("s2_3x3_c256", 3, 15, 20, 128, 256, 3, 3, stride=2, pads=P1, relu=True),
    _pp("s2_3x3_c512", 3, 15, 20, 256, 512, 3, 3, stride=2, pads=P1, relu=True),
    _pp("s2_1x1_c128", 3, 31, 41, 64, 128, 1, 1, stride=2),
    _pp("s2_1x1_c256", 3, 15, 20, 128, 256, 1, 1, stride=2),
    _pp("s2_1x1_c512", 3, 15, 20, 256, 512, 1, 1, stride=2),
    _pp("c384", 2, 9, 13, 64, 384, 3, 3, pads=P1, relu=True, res=True),
    # rounding families
    _pp("ties", 2, 9, 11, 64, 256, 3, 3, pads=P1, res=True, family="ties"),
    _pp("ties_relu", 2, 9, 11, 64, 128, 1, 1, relu=True, family="ties"),
    _pp("saturate", 2, 8, 10, 64, 512, 3, 3, pads=P1, res=True, family="saturate"),
    _pp("saturate_relu", 2, 8, 10, 64, 128, 1, 1, relu=True, family="saturate"),
]
assert len({c.name for c in CASES}) == len(CASES)


forced = mode_fixture(FORCE_PP | DEFAULT_CONV_MODE)


def _ran_pp(names):
    return any("convpp_wgmma_kernel" in n for n in names)


def _ran_128row(names):
    return any("conv_wgmma_kernel" in n for n in names)


@gpu
@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_convpp_bit_exact(case, forced):
    if case.family == "saturate" and ACT != torch.float16:
        pytest.skip("saturation at +-65504 is the fp16 conversion")
    x, w, b, r, want = _problem(case, _gen(case.name))
    got, names = device_kernels(lambda: _launch(case, x, w, b, r), "convpp_wgmma_kernel")
    assert _ran_pp(names) and not _ran_128row(names), names
    bad = got.float() != want.float()
    assert not bad.any(), f"{int(bad.sum())} of {bad.numel()} outputs differ, first at {bad.nonzero()[0].tolist()}"


def _chain_problem(g, n, h, w):
    """Integer operands of conv1 (3x3, 128 -> 128, ReLU) -> conv2 (3x3, + conv1's input, ReLU) -> conv3 (1x1 / s2,
    128 -> 256) and the exact result of each stage; the precondition is checked at every layer."""
    x0 = _ints((n, h, w, 128), 2, 0.8, g)
    w1 = _weights(128, 3, 3, 128, x0, 32, g, hi=1)
    b1 = _ints((128,), 8, 1.0, g)
    y1 = torch.relu(_conv64(x0, w1, 1, P1) + b1)
    w2 = _weights(128, 3, 3, 128, y1, 64, g, hi=1)
    b2 = _ints((128,), 8, 1.0, g)
    y2 = torch.relu(_conv64(y1, w2, 1, P1) + b2 + x0)
    w3 = _weights(256, 1, 1, 128, y2, 128, g, hi=1)
    b3 = _ints((256,), 8, 1.0, g)
    y3 = _conv64(y2, w3, 2, P0) + b3
    for xi, wi, bi, extra, stride, pads in ((x0, w1, b1, 0, 1, P1), (y1, w2, b2, x0.abs(), 1, P1), (y2, w3, b3, 0, 2, P0)):
        bound = _conv64(xi.abs(), wi.abs(), stride, pads) + bi.abs() + extra
        assert bound.max().item() <= CAP, "generator precondition"
    return x0, (w1, b1, y1), (w2, b2, y2), (w3, b3, y3)


@gpu
@pytest.mark.parametrize("mode", [DEFAULT_CONV_MODE, DEFAULT_CONV_MODE | NO_PDL], ids=["pdl", "no_pdl"])
def test_dependent_chain_on_one_stream(mode):
    """conv1 -> conv2 (+ conv1's input as residual) -> 1x1 / s2 on the ping-pong kernel, launched back to back without a
    host synchronisation into NaN-filled intermediates: every stage equals the float64 chain."""
    n, h, w = 2, 16, 20
    x0, (w1, b1, y1), (w2, b2, y2), (w3, b3, y3) = _chain_problem(_gen("pp_chain"), n, h, w)
    lib = _abi.lib()
    _, xv = _guarded(x0.shape, 64, float("nan"))
    xv.copy_(x0)
    _, a1 = _guarded(y1.shape, 64, float("nan"))
    _, a2 = _guarded(y2.shape, 64, float("nan"))
    _, a3 = _guarded(y3.shape, 64, float("nan"))
    ws = [wi.reshape(wi.shape[0], -1).to(ACT).contiguous() for wi in (w1, w2, w3)]
    bs = [bi.float().contiguous() for bi in (b1, b2, b3)]
    torch.cuda.synchronize()
    s = _abi.stream_ptr()

    def chain():
        _abi.check(lib.mpx_conv2d(_abi.ptr(xv), n, h, w, 128, _abi.ptr(ws[0]), _abi.ptr(bs[0]), 128, 3, 3, 1, *P1, 1,
                                  None, _abi.ptr(a1), 0, 0, s))
        _abi.check(lib.mpx_conv2d(_abi.ptr(a1), n, h, w, 128, _abi.ptr(ws[1]), _abi.ptr(bs[1]), 128, 3, 3, 1, *P1, 1,
                                  _abi.ptr(xv), _abi.ptr(a2), 0, 0, s))
        _abi.check(lib.mpx_conv2d(_abi.ptr(a2), n, h, w, 128, _abi.ptr(ws[2]), _abi.ptr(bs[2]), 256, 1, 1, 2, *P0, 0,
                                  None, _abi.ptr(a3), 0, 0, s))

    try:
        set_mode(mode | FORCE_PP)
        _, names = device_kernels(chain, "convpp_wgmma_kernel", 3)
    finally:
        set_mode(DEFAULT_CONV_MODE)
    assert sum("convpp_wgmma_kernel" in nm for nm in names) == 3, names
    for got, want in ((a1, y1), (a2, y2), (a3, y3)):
        assert torch.equal(got, _to_act(want))


GAUSS_CASES = [  # batch 32 of the coarse network's layer2 at 240x320 (300 tiles), and deeper layers under bit 28
    (_pp("gauss_layer2_conv2_res", 32, 30, 40, 128, 128, 3, 3, pads=P1, relu=True, res=True), DEFAULT_CONV_MODE),
    (_pp("gauss_layer3_conv1_s2", 8, 30, 40, 128, 256, 3, 3, stride=2, pads=P1, relu=True), FORCE_PP | DEFAULT_CONV_MODE),
    (_pp("gauss_layer4_conv2_res", 8, 8, 10, 512, 512, 3, 3, pads=P1, relu=True, res=True), FORCE_PP | DEFAULT_CONV_MODE),
]


@gpu
@pytest.mark.parametrize("case,mode", GAUSS_CASES, ids=[c.name for c, _ in GAUSS_CASES])
def test_convpp_gaussian_data_within_rounding_bound(case, mode):
    """Gaussian operands, per element within the bound of test_gpu_conv_exact:
    |y - y64| <= u |y64| + tiny + (K + 2) 2^-23 (conv(|x|, |w|) + |b| + |r|)."""
    assert _uses_pp(case, mode, _abi.lib().mpx_sm_count())
    g = _gen(case.name)
    k = case.r * case.s * case.cin
    P = _out_dim(case.h, case.pads[0], case.pads[2], case.r, case.stride)
    Q = _out_dim(case.w, case.pads[1], case.pads[3], case.s, case.stride)
    x = torch.randn(case.n, case.h, case.w, case.cin, device="cuda", generator=g).to(ACT).double()
    w = (torch.randn(case.cout, case.r, case.s, case.cin, device="cuda", generator=g) / k ** 0.5).to(ACT).double()
    b = torch.randn(case.cout, device="cuda", generator=g).double()
    r = torch.randn(case.n, P, Q, case.cout, device="cuda", generator=g).to(ACT).double() if case.res else None
    y64 = _conv64(x, w, case.stride, case.pads) + b + (r if r is not None else 0)
    if case.relu:
        y64 = torch.relu(y64)
    mag = _conv64(x.abs(), w.abs(), case.stride, case.pads) + b.abs() + (r.abs() if r is not None else 0)
    try:
        set_mode(mode)
        got, names = device_kernels(lambda: _launch(case, x.to(ACT), w, b, r.to(ACT) if r is not None else None),
                                      "convpp_wgmma_kernel")
    finally:
        set_mode(DEFAULT_CONV_MODE)
    assert _ran_pp(names), names
    err = (got.double() - y64).abs()
    bound = UNIT * y64.abs() + TINY + (k + 2) * 2.0 ** -23 * mag
    assert (err <= bound).all(), (err - bound).max().item()


def _network_convs(n, h, w):
    """The 29 convolutions of layers 2-4 of the ResNet-34 backbone for n renders of h x w (the stem is 7x7 / s2 and a
    3x3 / s2 max-pool follows it)."""
    H, W = ((h // 2) + 1) // 2, ((w // 2) + 1) // 2
    out, c = [], 64
    for li, (nb, width) in enumerate(zip([4, 6, 3], [128, 256, 512])):
        out.append(_pp(f"layer{li + 2}.0.conv1", n, H, W, c, width, 3, 3, stride=2, pads=P1, relu=True))
        out.append(_pp(f"layer{li + 2}.0.downsample", n, H, W, c, width, 1, 1, stride=2))
        H, W = (H + 1) // 2, (W + 1) // 2
        out += [_pp(f"layer{li + 2}.conv1", n, H, W, width, width, 3, 3, pads=P1, relu=True)] * (nb - 1)
        out += [_pp(f"layer{li + 2}.conv2", n, H, W, width, width, 3, 3, pads=P1, relu=True, res=True)] * nb
        c = width
    return out


@gpu
def test_network_forward_bit_identical_without_pingpong():
    """The coarse forward at batch 576, 240x320 (the benchmark's shape: layer2 on the ping-pong kernel), and with mode
    bit 28 (layers 2-4 on it), against the same forward under mode bit 27 (the 128-row kernel for all of them): every
    output's k16 sum order is the same in both kernels, so the logits are bit-identical."""
    from megapose6d_b200.backbone import ResNet34Engine
    from tests import helpers

    n, h, w = 576, 240, 320
    sms = _abi.lib().mpx_sm_count()
    want_pp = sum(_uses_pp(c, DEFAULT_CONV_MODE, sms) for c in _network_convs(n, h, w))
    assert want_pp == 9  # layer2
    cfg = helpers.COARSE_CFG
    sd = helpers.make_state_dict(cfg, seed=5)
    eng = ResNet34Engine(sd, n_inputs=helpers.n_inputs(cfg), head="views_logits_head")
    x = eng.alloc_input(n, h, w)
    x.copy_(torch.rand(x.shape, device="cuda", generator=_gen("pp_net")).to(x.dtype))
    lib = _abi.lib()
    try:
        lib.mpx_net_set_graphs(0)
        lib.mpx_conv_set_mode(DEFAULT_CONV_MODE | NEVER_PP)
        old, names_old = device_kernels(lambda: eng.forward(x, h, w).clone())
        lib.mpx_conv_set_mode(DEFAULT_CONV_MODE)
        new, names_new = device_kernels(lambda: eng.forward(x, h, w).clone(), "convpp_wgmma_kernel", want_pp)
        lib.mpx_conv_set_mode(DEFAULT_CONV_MODE | FORCE_PP)
        forced, names_forced = device_kernels(lambda: eng.forward(x, h, w).clone(), "convpp_wgmma_kernel", 29)
    finally:
        lib.mpx_net_set_graphs(1)
        lib.mpx_conv_set_mode(DEFAULT_CONV_MODE)
    assert sum("convpp_wgmma_kernel" in nm for nm in names_new) == want_pp and not _ran_pp(names_old)
    assert sum("convpp_wgmma_kernel" in nm for nm in names_forced) == 29
    assert torch.isfinite(new).all()
    assert torch.equal(new, old), (new - old).abs().max().item()
    assert torch.equal(forced, old), (forced - old).abs().max().item()


def test_dispatch_rule_covers_the_cases():
    """The case list reaches every edge of the ping-pong kernel, evaluated for a 132-SM H100."""
    for c in CASES:
        assert _uses_pp(c, FORCE_PP, SMS_H100), c.name
    plans = []
    for c in CASES:
        P, Q = _out_dim(c.h, c.pads[0], c.pads[2], c.r, c.stride), _out_dim(c.w, c.pads[1], c.pads[3], c.s, c.stride)
        m = c.n * P * Q
        items = _items(c)
        grid = min(items, c.max_ctas or SMS_H100)
        per_cta = [len(range(b, items, grid)) for b in range(grid)]
        plans.append((c, dict(M=m, items=items, grid=grid, per_cta=per_cta, pq=P * Q, nkb=c.r * c.s * c.cin // 64,
                              m_tiles=-(-m // BLOCK_M))))
    need = {
        "M = 1": lambda c, p: p["M"] == 1,
        "M = 127": lambda c, p: p["M"] == 127,
        "M = 128": lambda c, p: p["M"] == 128,
        "M = 129": lambda c, p: p["M"] == 129,
        "M = 255": lambda c, p: p["M"] == 255,
        "M = 257": lambda c, p: p["M"] == 257,
        "tiles spanning images": lambda c, p: p["pq"] < BLOCK_M and c.n > 2,
        "a CTA whose first consumer has one tile more": lambda c, p: any(k % 2 == 1 and k >= 3 for k in p["per_cta"]),
        "a CTA with a single tile (second consumer idle)": lambda c, p: 1 in p["per_cta"] and p["grid"] > 1,
        "one CTA, several tiles": lambda c, p: c.max_ctas == 1 and p["items"] >= 3,
        "two CTAs": lambda c, p: c.max_ctas == 2,
        "three CTAs over uneven tiles": lambda c, p: c.max_ctas == 3 and p["items"] % 3 != 0 and p["items"] > 3,
        "several n-tiles per m-tile, several m-tiles": lambda c, p: c.cout > 128 and p["m_tiles"] > 1,
        "3x3 stride 1": lambda c, p: (c.r, c.s, c.stride, c.pads) == (3, 3, 1, P1),
        "1x1 stride 2 pad 0": lambda c, p: (c.r, c.s, c.stride, c.pads) == (1, 1, 2, P0),
    }
    for cout in (128, 256, 512):
        need[f"3x3 stride 2, C_out {cout}"] = lambda c, p, co=cout: (c.r, c.stride, c.cout) == (3, 2, co)
        need[f"1x1 stride 2, C_out {cout}"] = lambda c, p, co=cout: (c.r, c.stride, c.cout) == (1, 2, co)
    for nkb in (1, PP_STAGES - 1, PP_STAGES, PP_STAGES + 1, 2 * PP_STAGES + 1, 72):
        need[f"{nkb} k-blocks, several tiles per consumer"] = \
            lambda c, p, nkb=nkb: p["nkb"] == nkb and max(p["per_cta"]) >= 3
    for relu in (False, True):
        for res in (False, True):
            need[f"relu {relu}, residual {res}"] = lambda c, p, relu=relu, res=res: c.relu == relu and c.res == res
    for fam in ("exact", "ties", "saturate"):
        need[f"family {fam}"] = lambda c, p, fam=fam: c.family == fam
    missing = [what for what, pred in need.items() if not any(pred(c, p) for c, p in plans)]
    assert not missing, missing
    # the rule itself: size threshold, and what keeps the 128-row kernel
    layer2 = _pp("layer2", 1, 30, 40, 128, 128, 3, 3, pads=P1, relu=True, res=True)  # 10 tiles per image
    assert not _uses_pp(dataclasses.replace(layer2, n=28), DEFAULT_CONV_MODE, SMS_H100)  # 263 tiles
    assert _uses_pp(dataclasses.replace(layer2, n=29), DEFAULT_CONV_MODE, SMS_H100)  # 272 tiles
    assert not _uses_pp(dataclasses.replace(layer2, n=29, max_ctas=137), DEFAULT_CONV_MODE, SMS_H100)
    assert _uses_pp(dataclasses.replace(layer2, n=29, max_ctas=136), DEFAULT_CONV_MODE, SMS_H100)
    assert _uses_pp(dataclasses.replace(layer2, n=576), DEFAULT_CONV_MODE, SMS_H100)
    assert not _uses_pp(dataclasses.replace(layer2, n=576), DEFAULT_CONV_MODE | NEVER_PP, SMS_H100)
    assert not _uses_pp(dataclasses.replace(layer2, n=576), FORCE_PP | NEVER_PP, SMS_H100)
    assert _uses_pp(dataclasses.replace(layer2, n=1), FORCE_PP, SMS_H100)
    for other in (dict(cout=64), dict(cout=192), dict(cout=640), dict(block_n=128), dict(splits=1)):
        assert not _uses_pp(dataclasses.replace(layer2, n=576, **other), FORCE_PP, SMS_H100), other
    assert not _uses_pp(dataclasses.replace(layer2, n=576), FORCE_PP, SMS_H100, out_aligned=False)
    for other in (dict(cout=256), dict(cout=512)):  # served under bit 28 only
        assert not _uses_pp(dataclasses.replace(layer2, n=576, **other), DEFAULT_CONV_MODE, SMS_H100), other
        assert _uses_pp(dataclasses.replace(layer2, n=576, **other), FORCE_PP, SMS_H100), other
    # the benchmark's coarse forward: layer2 on the ping-pong kernel at batch 576, layers 3 and 4 under bit 28
    convs = _network_convs(576, 240, 320)
    assert [c.name for c in convs if _uses_pp(c, DEFAULT_CONV_MODE, SMS_H100)] == [c.name for c in convs[:9]]
    assert all(_uses_pp(c, FORCE_PP, SMS_H100) for c in convs)
