"""The pose networks (mpx_net_forward, both backbone families) bit for bit against the float64 plan of
oracle/net_plan_ref.py on integer operands, at the batches where the convolutions change kernel, under every kernel-
selection mode, at sizes down to a 1-pixel layer-4 map, eager and under graph replay, inside a workspace and input /
output guards; the max-pool and pooled-linear kernels at their own edges.

Operands (workloads/weights.integer_state_dict): integer folded weights and biases, inputs 0..3, so every value of the plan
is an integer and fp32 accumulation is exact in any order; the oracle asserts it per convolution.  What remains are the
roundings to the 16-bit type, which the oracle makes in the same places.  The read-out head (fc = I, a signed permutation
scaled by powers of two) makes every pooled channel visible bit for bit; the real heads (views logits 1, pose 9) are held
to net_plan_ref.fp32_head_bound, their fp32 dot-product order.

The case list is chosen from a restatement of conv_forward's dispatch (`route`); tests/test_net_exact_host.py checks on the
host that it reaches every kernel path, and that the workspace layout (`workspace_layout`) holds every map.
"""
from __future__ import annotations

import math

import pytest
import torch
import torch.nn.functional as F

from megapose6d_b200 import _abi
from oracle import net_plan_ref as R
from tests import helpers
from tests.test_gpu_conv_exact import (ACT, DEFAULT_CONV_MODE, FORCE_C64, FORCE_IM2COL, FORCE_PP, NEVER_C64, NEVER_PP,
                                       SMS_H100, _guarded, device_kernels)
from workloads.weights import integer_state_dict

gpu = pytest.mark.gpu
SPLITK_CAP2, SPLITK_CAP1 = 262144, 524288  # MPX_CONV_SPLITK_CAP2 / _CAP1
WIDTHS = (64, 128, 256, 512)
BLOCKS = {"vanilla_resnet34": (3, 4, 6, 3), "resnet34": (3, 4, 6, 3), "resnet18": (2, 2, 2, 2)}

# name -> (input channels, backbone, real head, its dimension)
CONFIGS = {
    "coarse": (helpers.n_inputs(helpers.COARSE_CFG), "vanilla_resnet34", "views_logits_head", 1),  # c_pad 16
    "refiner": (helpers.n_inputs(helpers.REFINER_CFG), "vanilla_resnet34", "pose_fc", 9),  # c_pad 32
    "refiner_rgbd": (helpers.n_inputs(helpers.REFINER_RGBD_CFG), "vanilla_resnet34", "pose_fc", 9),  # 32
    "views6": (helpers.n_inputs(dict(helpers.REFINER_CFG, n_rendered_views=6)), "vanilla_resnet34", "pose_fc", 9),  # 48
    "views41": (helpers.n_inputs(dict(helpers.REFINER_CFG, n_rendered_views=41)), "vanilla_resnet34", "pose_fc", 9),  # 256
    "wide34": (helpers.n_inputs(helpers.REFINER_CFG), "resnet34", "pose_fc", 9),
    "wide18": (helpers.n_inputs(helpers.REFINER_CFG), "resnet18", "pose_fc", 9),
}


def c_pad(config: str) -> int:
    return 16 * ((CONFIGS[config][0] + 15) // 16)


def is_preact(config: str) -> bool:
    return CONFIGS[config][1] != "vanilla_resnet34"


# ---------------------------------------------------------------------------------------------
# host-side restatement of the plan: the convolutions of net_forward_direct / net_forward_preact and conv_forward's choice
# ---------------------------------------------------------------------------------------------
def _pool(v: int) -> int:
    return (v + 2 - 3) // 2 + 1


def net_convs(config: str, n: int, h: int, w: int, mode: int = DEFAULT_CONV_MODE):
    """(name, n, H, W, C_in, C_out, R, S, stride, pad_lo + pad_hi (the same on both axes), splitk) of every convolution,
    in launch order."""
    sk = -1 if (mode & 8) and n <= 64 else 0
    hs, ws = h // 2, w // 2
    out = []
    if is_preact(config):
        out.append(("stem", n, hs, ws, 4 * c_pad(config), 64, 3, 3, 1, 2, 0))
    else:
        out.append(("stem", n, hs, ws, 4 * c_pad(config), 64, 4, 4, 1, 3, 0))
    H, W, C = _pool(hs), _pool(ws), 64
    for layer, (nb, width) in enumerate(zip(BLOCKS[CONFIGS[config][1]], WIDTHS)):
        for blk in range(nb):
            stride = 2 if blk == 0 and layer > 0 else 1
            Ho, Wo = (H + 2 - 3) // stride + 1, (W + 2 - 3) // stride + 1
            out.append((f"layer{layer + 1}.{blk}.conv1", n, H, W, C, width, 3, 3, stride, 2, sk))
            if blk == 0 and layer > 0:
                out.append((f"layer{layer + 1}.{blk}.downsample", n, H, W, C, width, 1, 1, stride, 0, sk))
            out.append((f"layer{layer + 1}.{blk}.conv2", n, Ho, Wo, width, width, 3, 3, 1, 2, sk))
            H, W, C = Ho, Wo, width
    return out


def route(conv, mode: int = DEFAULT_CONV_MODE, sms: int = SMS_H100):
    """conv_forward's kernel for one convolution of the network: (kernel, K splits, activation producer)."""
    _, n, H, W, cin, cout, r, s, stride, pads, sk = conv
    P, Q = (H + pads - r) // stride + 1, (W + pads - s) // stride + 1
    M = n * P * Q
    m_tiles = -(-M // 128)
    bn = 256 if cout % 256 == 0 else (128 if cout % 128 == 0 else 64)
    while bn > 64 and m_tiles * (cout // bn) < 32:
        bn //= 2
    nkb = r * s * cin // 64
    if cout == 64 and sk <= 0 and not mode & NEVER_C64 and (mode & FORCE_C64 or -(-M // 256) >= 2 * sms):
        if not (sk < 0 and m_tiles * 2 <= sms and nkb >= 8):
            band = stride == 1 and W + pads <= 256 and cin // 64 <= 2 and not mode & FORCE_IM2COL
            return "conv64_wgmma_kernel", 1, "band" if band else "im2col"
    if cout % 128 == 0 and cout <= 512 and sk <= 0 and not mode & NEVER_PP and (
            mode & FORCE_PP or (cout == 128 and m_tiles >= 2 * sms)):
        if not (sk < 0 and m_tiles * (cout // bn) * 2 <= sms and nkb >= 8):
            return "convpp_wgmma_kernel", 1, None
    splits = 1
    if sk != 0:
        tiles = m_tiles * (cout // bn)
        want = 1
        if tiles * 2 <= sms and nkb >= 8:
            want = min(nkb // 4, sms // tiles)
        cap = 1 if mode & SPLITK_CAP1 else (2 if mode & SPLITK_CAP2 else 8)
        while splits * 2 <= want and splits * 2 <= cap and splits * 2 <= nkb:
            splits *= 2
    return "conv_wgmma_kernel", splits, None


def layer_maps(n: int, h: int, w: int):
    """Elements of the pooled stem map and of the layer 1-4 maps."""
    H, W = _pool(h // 2), _pool(w // 2)
    maps = [n * H * W * 64]
    for layer, width in enumerate(WIDTHS):
        if layer:
            H, W = (H - 1) // 2 + 1, (W - 1) // 2 + 1
        maps.append(n * H * W * width)
    return maps


def _a256(v: int) -> int:
    return (v + 255) // 256 * 256


def workspace_layout(n: int, h: int, w: int, preact: bool):
    """The workspace layout of net.cu: (stem map bytes, rotating buffer bytes, buffer count, total bytes)."""
    stem = _a256(n * (h // 2) * (w // 2) * 64 * 2)
    buf = _a256(max(layer_maps(n, h, w)) * 2)
    count = 5 if preact else 3
    return stem, buf, count, stem + count * buf + 1024


def buffer_writes(n: int, h: int, w: int, preact: bool, blocks=(3, 4, 6, 3)):
    """(buffer written, bytes written, buffers read) of every step after the stem, following the buffer rotation of
    run_layers (3 buffers) / net_forward_preact (5 buffers)."""
    H, W, C = _pool(h // 2), _pool(w // 2), 64
    steps = [(0, n * H * W * C * 2, ("stem",))]  # max-pool into buffer 0
    cur = 0
    for layer, (nb, width) in enumerate(zip(blocks, WIDTHS)):
        for blk in range(nb):
            stride = 2 if blk == 0 and layer > 0 else 1
            ds = blk == 0 and layer > 0
            Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
            out_bytes = n * Ho * Wo * width * 2
            if preact:
                ia, iy, ir, io = ((cur + k) % 5 for k in (1, 2, 3, 4))
                steps.append((ia, n * H * W * C * 2, (cur,)))
                steps.append((iy, out_bytes, (ia,)))
                if ds:
                    steps.append((ir, out_bytes, (ia,)))
                steps.append((io, out_bytes, (iy, ir if ds else cur)))
                cur = io
            else:
                t1, t2 = (cur + 1) % 3, (cur + 2) % 3
                steps.append((t1, out_bytes, (cur,)))
                if ds:
                    steps.append((t2, out_bytes, (cur,)))
                out = cur if ds else t2
                steps.append((out, out_bytes, (t1, t2 if ds else cur)))
                cur = out
            H, W, C = Ho, Wo, width
    return steps


# ---------------------------------------------------------------------------------------------
# cases
# ---------------------------------------------------------------------------------------------
def _first_batch(pred, lo=1, hi=512):
    return next(n for n in range(lo, hi) if pred(n))


def _kernels(config, n, h, w, mode=DEFAULT_CONV_MODE):
    return [route(c, mode) for c in net_convs(config, n, h, w, mode)]


# the smallest batch at 240x320 whose stem and layer 1 run on the pixel-major kernel and layer 2 on the ping-pong kernel
N_ALL_KERNELS = _first_batch(lambda n: {k for k, _, _ in _kernels("coarse", n, 240, 320)} ==
                             {"conv64_wgmma_kernel", "convpp_wgmma_kernel", "conv_wgmma_kernel"}
                             and all(k == "conv64_wgmma_kernel" for k, _, _ in _kernels("coarse", n, 240, 320)[:7]))
BATCHES = sorted({1, 2, 64, 65, N_ALL_KERNELS, max(N_ALL_KERNELS, 72)})
TINY_SIZES = [(2, 2), (4, 4), (4, 130), (8, 8), (8, 12)]
SIZES = [(64, 96), (66, 130)] + TINY_SIZES

EXACT_CASES = (
    [(cfg, 4, 240, 320) for cfg in CONFIGS]
    + [("coarse", n, 240, 320) for n in BATCHES if n != 4]
    + [("wide34", n, 240, 320) for n in (1, 65)]
    + [("refiner", 1, 240, 320)]
    + [(cfg, 2, h, w) for cfg in ("coarse", "wide34") for h, w in SIZES]
    + [("wide18", 3, 66, 130), ("wide18", 1, 4, 4), ("refiner_rgbd", 3, 8, 12)]
)
MODES = [DEFAULT_CONV_MODE, 0, NEVER_PP | 8, FORCE_PP | 8, NEVER_C64 | 8, FORCE_C64 | 8, FORCE_IM2COL | 8,
         SPLITK_CAP2 | 8, SPLITK_CAP1 | 8]
MODE_CASES = [("coarse", 2, 240, 320), ("coarse", N_ALL_KERNELS, 240, 320), ("wide34", 2, 240, 320)]


def _case_id(c):
    return f"{c[0]}-n{c[1]}-{c[2]}x{c[3]}"


# ---------------------------------------------------------------------------------------------
# engines, oracle and the guarded harness
# ---------------------------------------------------------------------------------------------
_state_dicts, _engines, _oracle = {}, {}, {}


def _state_dict(config: str, readout: bool = True):
    key = (config, readout)
    if key not in _state_dicts:
        c, backbone, head, dim = CONFIGS[config]
        _state_dicts[key] = integer_state_dict(c, head=head, head_dim=512 if readout else dim, readout=readout, seed=11,
                                               backbone_str=backbone)
    return _state_dicts[key]


def _engine(config: str, readout: bool = True):
    from megapose6d_b200.backbone import ResNet34Engine

    key = (config, readout)
    if key not in _engines:
        c, _, head, _ = CONFIGS[config]
        _engines[key] = ResNet34Engine(_state_dict(config, readout), n_inputs=c, head=head)
    return _engines[key]


def _input(config: str, n: int, h: int, w: int, seed: int = 0) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed * 100003 + n * 1009 + h * 31 + w)
    return torch.randint(0, 4, (n, CONFIGS[config][0], h, w), generator=g).float()


def oracle(config: str, n: int, h: int, w: int, seed: int = 0):
    """(read-out output [n, 512] fp32, Stats) of the float64 plan, cached per case."""
    key = (config, n, h, w, seed)
    if key not in _oracle:
        if len(_oracle) > 8:
            _oracle.clear()
        with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
            out, stats = R.forward(_state_dict(config), _input(config, n, h, w, seed).cuda(), ACT)
        want = out.float()
        assert torch.equal(want.double(), out)  # the read-out head is exact in fp32
        _oracle[key] = (want, stats)
    return _oracle[key]


WS_FILL = 0xA5
GUARD = 4096  # bytes


class Harness:
    """An engine's mpx_net_forward on persistent buffers: the input inside NaN guards of 4 KiB, the output inside NaN guards,
    and a workspace of exactly mpx_net_workspace_bytes followed by a tail filled with WS_FILL.  The tail is at least 4 KiB
    and reaches past the end of the layout an overflowing buffer could write to (workspace_layout's total)."""

    def __init__(self, eng, n: int, h: int, w: int):
        self.eng, self.n, self.h, self.w = eng, n, h, w
        lib = _abi.lib()
        shape = (n, h // 2, w // 2, 4 * eng.c_pad)
        self.in_buf, self.x = _guarded(shape, GUARD // 2, float("nan"))
        self.out_buf, self.out = _guarded((n, eng.out_dim), GUARD // 4, float("nan"), dtype=torch.float32)
        self.need = lib.mpx_net_workspace_bytes(eng._handle, n, h, w)
        mirror = workspace_layout(n, h, w, bool(getattr(eng, "_affines", None)))[3]
        self.ws = torch.full((self.need + GUARD + max(0, mirror - self.need),), WS_FILL, dtype=torch.uint8, device="cuda")
        assert self.ws.data_ptr() % 256 == 0

    def run(self, x_nchw: torch.Tensor) -> torch.Tensor:
        self.x.copy_(self.eng.pack_input(x_nchw.cuda()))
        self.out.fill_(float("nan"))
        return self.forward()

    def forward(self) -> torch.Tensor:
        _abi.check(_abi.lib().mpx_net_forward(self.eng._handle, _abi.ptr(self.x), self.n, self.h, self.w,
                                              _abi.ptr(self.out), _abi.ptr(self.ws), self.need, _abi.stream_ptr()))
        torch.cuda.synchronize()
        self.check_guards()
        return self.out.clone()

    def check_guards(self):
        tail = self.ws[self.need:]
        assert bool((tail == WS_FILL).all()), f"{int((tail != WS_FILL).sum())} bytes written past the workspace"
        g_in, g_out = GUARD // 2, GUARD // 4
        assert bool(torch.isnan(torch.cat([self.in_buf[:g_in], self.in_buf[-g_in:]]).float()).all()), "input guard"
        assert bool(torch.isnan(torch.cat([self.out_buf[:g_out], self.out_buf[-g_out:]])).all()), "output guard"


def _equal(got: torch.Tensor, want: torch.Tensor, what: str):
    assert got.shape == want.shape, what
    bad = got != want
    assert not bool(bad.any()), (f"{what}: {int(bad.sum())} of {got.numel()} outputs differ, first at "
                                 f"{bad.nonzero()[0].tolist()}: {got[bad][0].item()} != {want[bad][0].item()}")


@pytest.fixture(autouse=True)
def _eager_default_mode():
    """Eager launches (a replayed graph keeps the kernels of the mode it was captured under) and the default mode."""
    lib = _abi.lib() if torch.cuda.is_available() else None
    if lib is not None:
        lib.mpx_net_set_graphs(0)
        lib.mpx_conv_set_mode(DEFAULT_CONV_MODE)
    try:
        yield
    finally:
        if lib is not None:
            lib.mpx_net_set_graphs(1)
            lib.mpx_conv_set_mode(DEFAULT_CONV_MODE)


# ---------------------------------------------------------------------------------------------
# the network
# ---------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("case", EXACT_CASES, ids=_case_id)
def test_network_equals_the_float64_plan(case):
    config, n, h, w = case
    want, stats = oracle(config, n, h, w)
    harness = Harness(_engine(config), n, h, w)
    expect = {k for k, _, _ in _kernels(config, n, h, w)}
    got, names = device_kernels(lambda: harness.run(_input(config, n, h, w)), kernel=sorted(expect)[0])
    _equal(got, want, _case_id(case))
    ran = {k for k in expect if any(k in name for name in names)}
    splits = sorted({s for _, s, _ in _kernels(config, n, h, w)})
    print(f"[{_case_id(case)}] max |value| before rounding {stats.max_abs:.0f}, saturated {stats.saturated_fraction:.4f}, "
          f"kernels {sorted(ran)}, K splits {splits}")
    assert ran == expect, (ran, expect)
    if h * w >= 64 * 96:
        assert stats.max_abs > 2048, stats.max_abs  # values were rounded (fp16 integers above 2048 are even)
        assert stats.saturated_fraction < 0.05, stats.saturated_fraction


@gpu
@pytest.mark.parametrize("case", MODE_CASES, ids=_case_id)
def test_every_kernel_mode_equals_the_float64_plan(case):
    config, n, h, w = case
    want, _ = oracle(config, n, h, w)
    harness = Harness(_engine(config), n, h, w)
    x = _input(config, n, h, w)
    lib = _abi.lib()
    try:
        for mode in MODES:
            lib.mpx_conv_set_mode(mode)
            _equal(harness.run(x), want, f"mode {mode}")
    finally:
        lib.mpx_conv_set_mode(DEFAULT_CONV_MODE)


@gpu
@pytest.mark.parametrize("case", [("coarse", 2, 240, 320), ("wide18", 3, 64, 96), ("refiner", 2, 4, 130)], ids=_case_id)
def test_graph_capture_and_replay_equal_the_plan_and_follow_the_input(case):
    config, n, h, w = case
    want, _ = oracle(config, n, h, w)
    want2, _ = oracle(config, n, h, w, seed=1)
    harness = Harness(_engine(config), n, h, w)
    lib = _abi.lib()
    lib.mpx_net_set_graphs(1)
    x = _input(config, n, h, w)
    harness.run(x)  # a first call of its own buffers: a shape seen before may already have a graph
    for i in range(3):  # eager first sight (or replay), capture, replay
        _equal(harness.run(x), want, f"call {i}")
    l0 = lib.mpx_launch_count()
    harness.x.copy_(harness.eng.pack_input(_input(config, n, h, w, seed=1).cuda()))  # new contents, same buffer
    _equal(harness.forward(), want2, "replay after the input changed in place")
    assert lib.mpx_launch_count() - l0 == len(net_convs(config, n, h, w)) + 2 + (
        sum(BLOCKS[CONFIGS[config][1]]) if is_preact(config) else 0)  # convolutions, max-pool, tail, affine passes


@gpu
@pytest.mark.parametrize("case", [("coarse", 4, 240, 320), ("refiner", 2, 66, 130), ("wide34", 4, 240, 320),
                                  ("wide18", 2, 8, 8)], ids=_case_id)
def test_real_heads_within_the_fp32_dot_product_bound(case):
    """The integer backbone with the real heads (Gaussian fc and head): the pooled features are exact, the fp32 dot
    product differs from float64 by at most net_plan_ref.fp32_head_bound."""
    config, n, h, w = case
    _, stats = oracle(config, n, h, w)
    sd = _state_dict(config, readout=False)
    want = R.head(sd, stats.pooled)
    bound = R.fp32_head_bound(sd, stats.pooled)
    got = Harness(_engine(config, readout=False), n, h, w).run(_input(config, n, h, w)).double()
    err = (got - want).abs()
    print(f"[{_case_id(case)}] max |err| {err.max().item():.3g}, bound {bound.min().item():.3g}..{bound.max().item():.3g}")
    assert bool((err <= bound).all()), (err - bound).max()


@gpu
def test_workspace_bytes_cover_the_layout():
    """mpx_net_workspace_bytes is at least the mirrored layout's total (every rotating buffer holds every map) for
    n in {1, 2, 3, 64} and every even h, w <= 128, for both schedules."""
    lib = _abi.lib()
    short = []
    for config in ("coarse", "wide18"):
        handle = _engine(config)._handle
        for n in (1, 2, 3, 64):
            for h in range(2, 129, 2):
                for w in range(2, 129, 2):
                    need = workspace_layout(n, h, w, is_preact(config))[3]
                    got = lib.mpx_net_workspace_bytes(handle, n, h, w)
                    if got < need:
                        short.append((config, n, h, w, got, need))
    assert not short, f"{len(short)} shapes short, e.g. {short[:4]}"


# ---------------------------------------------------------------------------------------------
# standalone kernels
# ---------------------------------------------------------------------------------------------
def _maxpool(x: torch.Tensor):
    n, h, w, c = x.shape
    ho, wo = _pool(h), _pool(w)
    buf, out = _guarded((n, ho, wo, c), 64, float("nan"))
    _abi.check(_abi.lib().mpx_maxpool3x3s2(_abi.ptr(x), n, h, w, c, _abi.ptr(out), _abi.stream_ptr()))
    torch.cuda.synchronize()
    assert bool(torch.isnan(torch.cat([buf[:64], buf[-64:]]).float()).all()), "output guard"
    want = F.max_pool2d(x.double().permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1).to(ACT)
    return out, want


MAXPOOL_SHAPES = [(n, h, w, c) for c in (8, 24, 64, 512) for h in (1, 2, 3, 7, 10) for w in (1, 2, 3, 9, 12)
                  for n in (2,)] + [
    (3, 9, 130, 64),  # wo * c / 8 = 520 channel groups: two passes per row
    (2, 5, 257, 512),  # 8256 groups: 512 threads, 17 passes
    (40, 240, 4, 8),  # n * ho = 4800 rows > 32 * 132: the persistent row loop
]


@gpu
def test_maxpool_equals_float64_at_its_edges():
    g = torch.Generator(device="cuda").manual_seed(3)
    for i, (n, h, w, c) in enumerate(MAXPOOL_SHAPES):
        x = (torch.randn(n, h, w, c, device="cuda", generator=g) * 3000).clamp(-65504, 65504).to(ACT)
        if i % 3 == 1:
            x = -x.abs() - 1  # all negative: the -inf padding must never win
        if i % 3 == 2:
            x.view(-1)[::7] = 65504
            x.view(-1)[3::11] = -65504
        got, want = _maxpool(x)
        _equal(got, want, f"maxpool {n}x{h}x{w}x{c}")


AVGPOOL_C = (4, 12, 64, 512, 1000, 2048, 2052, 4096)
AVGPOOL_HW = (1, 6, 80, 300)
AVGPOOL_OUT = (1, 9, 16, 17, 512)


def _avgpool_cases():
    """Every C with every hw; the output widths spread over them; n from 1 to a few hundred."""
    out = []
    for i, c in enumerate(AVGPOOL_C):
        for j, hw in enumerate(AVGPOOL_HW):
            k = i * len(AVGPOOL_HW) + j
            out.append(((1, 3, 37, 300)[k % 4] if c * hw <= 512 * 300 else (1, 2, 5)[k % 3], hw, c,
                        AVGPOOL_OUT[k % len(AVGPOOL_OUT)]))
    return out


def _avgpool(x, w, b, out_dim):
    n, hw, c = x.shape
    buf, out = _guarded((n, out_dim), 64, float("nan"), dtype=torch.float32)
    _abi.check(_abi.lib().mpx_avgpool_linear(_abi.ptr(x), n, hw, c, _abi.ptr(w), _abi.ptr(b), out_dim, _abi.ptr(out),
                                             _abi.stream_ptr()))
    torch.cuda.synchronize()
    assert bool(torch.isnan(torch.cat([buf[:64], buf[-64:]])).all()), "output guard"
    return out


def _groups(c: int) -> int:
    nq = c // 4
    return 1 if nq >= 512 else 512 // nq


@gpu
@pytest.mark.parametrize("n,hw,c,out_dim", _avgpool_cases())
def test_avgpool_linear_exact_on_integers_and_bounded_on_gaussians(n, hw, c, out_dim):
    g = torch.Generator(device="cuda").manual_seed(n * 7 + hw * 13 + c)
    # integers below 2^24 / hw: the pooled sums are exact in any order; one-hot power-of-two rows, integer bias
    x = torch.randint(-2000, 2001, (n, hw, c), device="cuda", generator=g).to(ACT)
    cols = torch.randint(0, c, (out_dim,), device="cuda", generator=g)
    w = torch.zeros(out_dim, c, device="cuda")
    w[torch.arange(out_dim, device="cuda"), cols] = 2.0 ** torch.randint(-2, 3, (out_dim,), device="cuda", generator=g).float()
    b = torch.randint(-3, 4, (out_dim,), device="cuda", generator=g).float()
    s = x.double().sum(dim=1).float()  # exact
    pooled = s * torch.tensor(1.0 / hw, dtype=torch.float32, device="cuda")  # fp32(fp32(sum) * fp32(1 / hw))
    want = pooled[:, cols] * w[torch.arange(out_dim, device="cuda"), cols] + b  # one product, one rounding of the sum
    _equal(_avgpool(x, w, b, out_dim), want, "integers")
    # Gaussian: each term x_pk W_jk / hw passes through at most a = ceil(hw / G) + G + 2 roundings in the pooling
    # (per-thread sum over every G-th pixel, the G group sums, 1 / hw and the product) and d = ceil(c / 32) + 6 in the dot
    # product (fmas per lane, 5 shuffle levels, the bias): |err| <= gamma_(a+d) * (sum_k |W_jk| mean_p |x_pk| + |b_j|)
    x = torch.randn(n, hw, c, device="cuda", generator=g).to(ACT)
    w = torch.randn(out_dim, c, device="cuda", generator=g)
    b = torch.randn(out_dim, device="cuda", generator=g)
    want = x.double().mean(dim=1) @ w.double().t() + b.double()
    G = _groups(c)
    m = -(-hw // G) + G + 2 + -(-c // 32) + 6
    u = 2.0 ** -24
    bound = m * u / (1 - m * u) * (x.double().abs().mean(dim=1) @ w.double().abs().t() + b.double().abs())
    err = (_avgpool(x, w, b, out_dim).double() - want).abs()
    assert bool((err <= bound).all()), ((err - bound).max().item(), bound.min().item())
    # one pixel less moves some output by far more than the bound
    lost = (x[:, 1:].double().sum(dim=1) / hw) @ w.double().t() + b.double() if hw > 1 else b.double().expand_as(want)
    assert bool(((lost - want).abs() > bound).any())


@gpu
def test_pooling_kernels_refuse_unsupported_channels_and_launch_nothing():
    lib = _abi.lib()
    x = torch.zeros(2 * 9 * 9 * 4104, device="cuda", dtype=ACT)
    out = torch.zeros(2 * 5 * 5 * 4104, device="cuda", dtype=ACT)
    w = torch.zeros(9 * 4104, device="cuda")
    b = torch.zeros(9, device="cuda")
    o = torch.zeros(2, 9, device="cuda")
    cases = [
        ("maxpool c=12", lambda: lib.mpx_maxpool3x3s2(_abi.ptr(x), 2, 9, 9, 12, _abi.ptr(out), _abi.stream_ptr()),
         "multiple of 8"),
        ("maxpool c=4", lambda: lib.mpx_maxpool3x3s2(_abi.ptr(x), 2, 9, 9, 4, _abi.ptr(out), _abi.stream_ptr()),
         "multiple of 8"),
        ("avgpool c=6", lambda: lib.mpx_avgpool_linear(_abi.ptr(x), 2, 9, 6, _abi.ptr(w), _abi.ptr(b), 9, _abi.ptr(o),
                                                       _abi.stream_ptr()), "unsupported"),
        ("avgpool c=4100", lambda: lib.mpx_avgpool_linear(_abi.ptr(x), 2, 9, 4100, _abi.ptr(w), _abi.ptr(b), 9,
                                                          _abi.ptr(o), _abi.stream_ptr()), "unsupported"),
    ]
    for name, call, msg in cases:
        before = lib.mpx_launch_count()
        assert call() != 0, name
        assert msg in lib.mpx_last_error().decode(), (name, lib.mpx_last_error())
        assert lib.mpx_launch_count() == before, name
    torch.cuda.synchronize()
    assert math.isfinite(o.sum().item()) and o.abs().sum().item() == 0  # nothing was written
