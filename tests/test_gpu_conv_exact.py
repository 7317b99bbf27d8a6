"""The wgmma convolution (conv_wgmma.cu) held bit-exactly to a float64 reference at its tile, pipeline, split-K and im2col
edges; the max-pool and pooled-linear kernels against plain references.

Exact operands.  Activations and weights are small integers stored in the library's 16-bit type, the bias is an fp32
integer and the residual a 16-bit integer.  Every product is then exact on the tensor core and every fp32 partial sum is an
integer below 2^24, exact in any order and under any K split: the result is one known integer whatever the tile width, CTA
count, split count or accumulation order.  The reference is a float64 convolution (exact as well: every partial sum is an
integer below 2^53) rounded once to the 16-bit type, round-to-nearest-even and saturating at the largest finite value as
the kernel's cvt.rn.satfinite does, and the kernel must equal it (torch.equal).  Three families of outputs:
  * exact:    |y| <= 2048 (256 in a bf16 build), no rounding at all: one missing, duplicated or misplaced product changes
              an output;
  * ties:     y in (2048, 8192); the odd integers in [2048, 4096) are exact round-to-nearest-even ties;
  * saturate: |y| at and beyond 65504; +-65504 is the answer, never +-inf.
The generator asserts its own precondition on the host (conv(|x|, |w|) + |b| + |r| within the family's cap).

_plan restates the host-side choices of conv_forward / launch_conv (tile width, ring depth, grid, tiles per CTA, K split,
images per tile, driver fix-up); test_plan_covers_every_decision_point (no GPU) checks that CASES reaches each of them.

The mpx_conv_set_mode bits, set_mode, mode_fixture and device_kernels are defined here for every convolution test.
"""
from __future__ import annotations

import dataclasses
import math
import types
import zlib
from typing import Optional

import pytest
import torch
import torch.nn.functional as F

from megapose6d_b200 import _abi

gpu = pytest.mark.gpu
ACT = _abi.act_dtype() if torch.cuda.is_available() else torch.float16
CAP = 2048 if ACT == torch.float16 else 256  # every integer up to CAP is exact in ACT
ACT_MAX = torch.finfo(ACT).max
UNIT = 2.0 ** -11 if ACT == torch.float16 else 2.0 ** -8  # unit roundoff of ACT
TINY = 2.0 ** -25 if ACT == torch.float16 else 2.0 ** -134  # half the smallest subnormal step of ACT
STAGES = {64: 8, 128: 6, 256: 4}  # ConvCfg<BLOCK_N>::kStages
BLOCK_M = 128
SMS_H100 = 132
P0, P1, STEM = (0, 0, 0, 0), (1, 1, 1, 1), (2, 2, 1, 1)


@dataclasses.dataclass(frozen=True)
class Conv:
    name: str
    n: int
    h: int
    w: int
    cin: int
    cout: int
    r: int
    s: int
    stride: int = 1
    pads: tuple = P0  # pad_lo_h, pad_lo_w, pad_hi_h, pad_hi_w
    relu: bool = False
    res: bool = False
    block_n: int = 0  # 0: automatic
    max_ctas: int = 0  # 0: one CTA per SM
    splits: Optional[int] = None  # None: mpx_conv2d; else mpx_conv2d_splitk with this split count (0: heuristic)
    family: str = "exact"  # exact | ties | saturate


# ---------------------------------------------------------------------------------------------
# kernel selection: the mpx_conv_set_mode bits of include/mpx.h (MPX_CONV_*)
# ---------------------------------------------------------------------------------------------
DEFAULT_CONV_MODE = 8  # MPX_CONV_NET_SPLITK, the library's default
NO_PDL = 512  # MPX_CONV_NO_PDL: launch without programmatic dependent launch
NEVER_C64 = 4194304  # MPX_CONV_NEVER_C64: never the pixel-major C_out = 64 kernel
FORCE_IM2COL = 8388608  # MPX_CONV_FORCE_IM2COL: the pixel-major kernel loads by im2col for every shape
FORCE_C64 = 67108864  # MPX_CONV_FORCE_C64: the pixel-major kernel for every convolution it can serve
NEVER_PP = 134217728  # MPX_CONV_NEVER_PP: never the ping-pong kernel
FORCE_PP = 268435456  # MPX_CONV_FORCE_PP: the ping-pong kernel for every convolution it can serve


def set_mode(mode):
    _abi.lib().mpx_conv_set_mode(mode)


def mode_fixture(mode=None):
    """A fixture that sets `mode` (when given) for the test and restores DEFAULT_CONV_MODE after it."""
    @pytest.fixture
    def fixture():
        if mode is not None:
            set_mode(mode)
        yield
        set_mode(DEFAULT_CONV_MODE)
    return fixture


def device_kernels(fn, kernel=None, launches=1):
    """Runs `fn` under torch.profiler (CUDA activities) and returns its result and the names of the kernels it launched:
    the proof that a case ran on the kernel it is meant for, since every kernel gives the same bits.  With `kernel`, `fn`
    is captured again (at most three captures) until the capture holds `launches` launches whose name contains it:
    torch.profiler can drop device activity from one of many short captures, while a launch it does record always names
    the kernel that ran."""
    from torch.profiler import ProfilerActivity, profile

    for _ in range(3 if kernel else 1):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            out = fn()
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        if kernel is None or sum(kernel in n for n in names) >= launches:
            break
    return out, names


# ---------------------------------------------------------------------------------------------
# host-side plan: a plain restatement of conv_forward / launch_conv
# ---------------------------------------------------------------------------------------------
def _out_dim(size, lo, hi, k, stride):
    return (size + lo + hi - k) // stride + 1


def _auto_block_n(cout, m_tiles):
    """Automatic tile width: the widest of 256 / 128 / 64 that divides C_out, halved while the layer has fewer than 32
    output tiles."""
    bn = 256 if cout % 256 == 0 else (128 if cout % 128 == 0 else 64)
    while bn > 64 and m_tiles * (cout // bn) < 32:
        bn //= 2
    return bn


def _plan(c: Conv, sms: int):
    P = _out_dim(c.h, c.pads[0], c.pads[2], c.r, c.stride)
    Q = _out_dim(c.w, c.pads[1], c.pads[3], c.s, c.stride)
    M = c.n * P * Q
    m_tiles = -(-M // BLOCK_M)
    bn = c.block_n or _auto_block_n(c.cout, m_tiles)
    nkb = c.r * c.s * c.cin // 64
    n_tiles = c.cout // bn
    tiles = m_tiles * n_tiles
    splits = 1
    if c.splits is not None:  # mpx_conv2d_splitk: max_ctas = 0, K split cap 8 (default mode)
        want = c.splits if c.splits > 0 else 1
        if c.splits == 0 and tiles * 2 <= sms and nkb >= 8:
            want = min(nkb // 4, sms // tiles)
        while splits * 2 <= want and splits * 2 <= 8 and splits * 2 <= nkb:
            splits *= 2
    items = tiles * splits
    grid = items if splits > 1 else min(items, c.max_ctas or sms)
    pq = P * Q

    def images(m0):
        return (min(m0 + BLOCK_M, M) - 1) // pq - m0 // pq + 1

    in_bytes = c.n * c.h * c.w * c.cin * 2
    return types.SimpleNamespace(
        P=P, Q=Q, M=M, block_n=bn, stages=STAGES[bn], num_k_blocks=nkb, m_tiles=m_tiles, n_tiles=n_tiles, tiles=tiles,
        grid=grid, tiles_per_cta=-(-items // grid), splits=splits,
        k_ranges=[(sp * nkb // splits, (sp + 1) * nkb // splits) for sp in range(splits)],
        first_tile_images=images(0), last_tile_images=images((m_tiles - 1) * BLOCK_M),
        last_tile_rows=M - (m_tiles - 1) * BLOCK_M, input_bytes=in_bytes,
        driver_fixup=in_bytes < 131072)  # (applied by drivers up to 13.1)


# ---------------------------------------------------------------------------------------------
# case matrix
# ---------------------------------------------------------------------------------------------
def _ring_cases():
    """num_k_blocks 1, stages - 1, stages, stages + 1, 2 stages + 1 and 72 at each tile width; 3 m-tiles over 2 CTAs."""
    shapes = {  # num_k_blocks -> (r, s, cin, pads)
        1: (1, 1, 64, P0), 3: (3, 1, 64, (1, 0, 1, 0)), 4: (1, 1, 256, P0), 5: (1, 1, 320, P0), 6: (1, 3, 128, (0, 1, 0, 1)),
        8: (1, 1, 512, P0), 9: (3, 3, 64, P1), 13: (1, 1, 832, P0), 17: (1, 1, 1088, P0), 72: (3, 3, 512, P1),
    }
    out = []
    for bn, st in STAGES.items():
        for nkb in (1, st - 1, st, st + 1, 2 * st + 1, 72):
            if nkb == 7:  # 1x7 at BLOCK_N 64, 7x1 at BLOCK_N 128
                r, s, cin, pads = (1, 7, 64, (0, 3, 0, 3)) if bn == 64 else (7, 1, 64, (3, 0, 3, 0))
            else:
                r, s, cin, pads = shapes[nkb]
            out.append(Conv(f"ring_bn{bn}_kb{nkb}", 3, 9, 13, cin, min(2 * bn, 256), r, s, pads=pads, relu=nkb % 2 == 1,
                            res=nkb % 3 == 0, block_n=bn, max_ctas=2))
    return out


def _cout_cases():
    out = []
    for cout in range(64, 513, 64):
        out.append(Conv(f"auto_cout{cout}_few_tiles", 1, 8, 10, 64, cout, 1, 1, relu=True))
        out.append(Conv(f"auto_cout{cout}_many_tiles", 1, 64, 80, 64, cout, 1, 1, res=True))
    return out


def _splitk_epilogue_cases():
    """Residual on / off and ReLU on / off through the split-K reduction at every tile width (18 k-blocks: uneven ranges
    over 4 and 8 splits)."""
    out = []
    for bn in (64, 128, 256):
        for i, (relu, res) in enumerate(((False, False), (True, False), (False, True), (True, True))):
            out.append(Conv(f"splitk_bn{bn}_relu{int(relu)}_res{int(res)}", 1, 9, 11, 128, bn, 3, 3, pads=P1, relu=relu,
                            res=res, block_n=bn, splits=(2, 4, 8, 4)[i]))
    return out


CASES = _ring_cases() + [
    # persistent loop: tile counts not a multiple of the CTA count, k-block counts not a multiple of the ring depth
    Conv("persist_ctas1", 3, 12, 20, 64, 64, 3, 3, pads=P1, relu=True, res=True, block_n=64, max_ctas=1),
    Conv("persist_ctas2", 1, 15, 21, 64, 256, 5, 5, pads=(2, 2, 2, 2), relu=True, block_n=256, max_ctas=2),
    Conv("persist_ctas3", 3, 15, 20, 128, 128, 1, 7, pads=(0, 3, 0, 3), res=True, block_n=128, max_ctas=3),
    Conv("persist_ctas7", 4, 17, 23, 64, 192, 3, 3, pads=P1, relu=True, block_n=64, max_ctas=7),
    # M layout
    Conv("pq63_n5_three_images_per_tile", 5, 7, 9, 64, 64, 3, 3, pads=P1, relu=True, res=True),
    Conv("pq128", 3, 8, 16, 64, 128, 3, 3, pads=P1, res=True),
    Conv("pq129", 2, 3, 43, 64, 64, 3, 3, pads=P1, relu=True),
    Conv("m_128k_plus_1", 1, 5, 77, 128, 64, 3, 3, pads=P1, res=True, max_ctas=2),
    Conv("m_129_1x1", 1, 1, 129, 64, 128, 1, 1, relu=True),
    # im2col geometry
    Conv("s2_h_even_w_odd", 2, 15, 20, 64, 128, 3, 3, stride=2, pads=P1, relu=True),
    Conv("s2_h_odd_w_even", 2, 16, 21, 64, 128, 3, 3, stride=2, pads=P1, res=True),
    Conv("s2_1x1_pad0", 3, 15, 20, 128, 256, 1, 1, stride=2),
    Conv("pads_2211_4x4", 2, 24, 32, 128, 64, 4, 4, pads=STEM, relu=True, max_ctas=3),
    Conv("pads_0110_3x3", 2, 10, 14, 64, 64, 3, 3, pads=(0, 1, 1, 0), res=True),
    Conv("taps_1x3", 2, 11, 13, 64, 64, 1, 3, pads=(0, 1, 0, 1), relu=True),
    Conv("taps_3x1", 2, 11, 13, 64, 64, 3, 1, pads=(1, 0, 1, 0)),
    Conv("taps_7x7_p3", 1, 14, 18, 64, 64, 7, 7, pads=(3, 3, 3, 3), relu=True),
    Conv("taps_8x8", 2, 12, 15, 64, 64, 8, 8, pads=(4, 4, 3, 3), res=True),
    Conv("taps_8x8_s2_pad0", 1, 20, 19, 64, 64, 8, 8, stride=2),
    Conv("taps_3x3_pad3_bias_only_border", 1, 6, 7, 64, 64, 3, 3, pads=(3, 3, 3, 3), res=True),
    # driver fix-up of small im2col maps (< 131072 bytes of input)
    Conv("fixup_off_32x32", 1, 32, 32, 64, 64, 3, 3, pads=P1, relu=True),
    Conv("fixup_on_31x33", 1, 31, 33, 64, 64, 3, 3, pads=P1, relu=True),
    Conv("fixup_off_32x32_s2", 1, 32, 32, 64, 128, 3, 3, stride=2, pads=P1),
    Conv("fixup_on_31x33_s2", 1, 31, 33, 64, 128, 3, 3, stride=2, pads=P1),
    # wide K: the space-to-depth stem at the largest c_pad (256): 4x4 over 1024 channels, 256 k-blocks
    Conv("stem_c1024", 1, 6, 8, 1024, 64, 4, 4, pads=STEM, relu=True),
] + _cout_cases() + [
    # split-K
    Conv("splitk_9kb_over_8", 1, 8, 10, 64, 128, 3, 3, pads=P1, relu=True, res=True, block_n=64, splits=8),
    Conv("splitk_9kb_over_4", 1, 8, 10, 64, 128, 3, 3, pads=P1, res=True, block_n=128, splits=4),
    Conv("splitk_9kb_over_2", 1, 8, 10, 64, 256, 3, 3, pads=P1, relu=True, block_n=256, splits=2),
    Conv("splitk_clamped_1kb", 1, 8, 10, 64, 64, 1, 1, block_n=64, splits=8),
    Conv("splitk_clamped_3kb", 1, 8, 10, 64, 128, 1, 3, pads=(0, 1, 0, 1), res=True, block_n=128, splits=8),
    Conv("splitk_heuristic", 1, 8, 10, 512, 512, 3, 3, pads=P1, relu=True, res=True, block_n=64, splits=0),
    Conv("splitk_heuristic_declines", 7, 32, 40, 64, 64, 3, 3, pads=P1, relu=True, block_n=64, splits=0),
    Conv("splitk_two_mtiles", 2, 10, 10, 128, 256, 3, 3, pads=P1, relu=True, res=True, block_n=128, splits=4),
    Conv("splitk_s2", 1, 30, 40, 128, 256, 3, 3, stride=2, pads=P1, relu=True, block_n=64, splits=4),
] + _splitk_epilogue_cases() + [
    # rounding: round-to-nearest-even ties, and saturation at the largest finite value
    Conv("ties_direct", 2, 9, 11, 64, 128, 3, 3, pads=P1, family="ties"),
    Conv("ties_direct_relu_res", 2, 9, 11, 64, 256, 3, 3, pads=P1, relu=True, res=True, family="ties"),
    Conv("ties_splitk", 1, 9, 11, 128, 128, 3, 3, pads=P1, res=True, block_n=128, splits=4, family="ties"),
    Conv("saturate_direct", 2, 8, 10, 64, 64, 3, 3, pads=P1, res=True, family="saturate"),
    Conv("saturate_direct_relu", 2, 8, 10, 64, 128, 1, 1, relu=True, family="saturate"),
    Conv("saturate_splitk", 1, 8, 10, 64, 128, 3, 3, pads=P1, res=True, block_n=64, splits=8, family="saturate"),
    Conv("saturate_splitk_bn256", 1, 8, 10, 128, 256, 3, 3, pads=P1, block_n=256, splits=2, family="saturate"),
]
assert len({c.name for c in CASES}) == len(CASES)


# ---------------------------------------------------------------------------------------------
# operands and references
# ---------------------------------------------------------------------------------------------
def _ints(shape, hi, density, gen):
    """float64 integers in [-hi, hi]: non-zero with probability `density`, then uniform over +-1 .. +-hi."""
    dev = gen.device
    mag = torch.randint(1, hi + 1, shape, generator=gen, device=dev)
    sign = torch.randint(0, 2, shape, generator=gen, device=dev) * 2 - 1
    keep = torch.rand(shape, generator=gen, device=dev) < density
    return (mag * sign * keep).double()


def _weights(cout, r, s, cin, x, target, gen, hi=3):
    """Integer weights whose products with `x` sum to about `target` per output (density scaled by 1 / K)."""
    k = r * s * cin
    density = min(1.0, target / (k * max(x.abs().mean().item(), 1e-3) * (hi + 1) / 2))
    return _ints((cout, r, s, cin), hi, density, gen)


def _conv64(x, w, stride, pads):
    """NHWC float64 convolution with asymmetric zero padding, one matrix product per filter tap: x [n, H, W, C_in],
    w [C_out, R, S, C_in] -> [n, P, Q, C_out]."""
    n, H, W, _ = x.shape
    _, R, S, _ = w.shape
    P, Q = _out_dim(H, pads[0], pads[2], R, stride), _out_dim(W, pads[1], pads[3], S, stride)
    xp = F.pad(x, (0, 0, pads[1], pads[3], pads[0], pads[2]))
    y = x.new_zeros(n, P, Q, w.shape[0])
    for r in range(R):
        for s in range(S):
            y += xp[:, r:r + stride * (P - 1) + 1:stride, s:s + stride * (Q - 1) + 1:stride, :] @ w[:, r, s, :].T
    return y


def _to_act(y):
    """float64 -> ACT: round to nearest even, saturating at the largest finite value (cvt.rn.satfinite)."""
    t = y.to(ACT)
    return torch.where(torch.isinf(t), torch.sign(y).to(ACT) * ACT_MAX, t)


def _problem(c: Conv, gen):
    """Integer operands for `c` and the exact result, rounded to ACT.  Asserts the generator's precondition."""
    dev = gen.device
    P, Q = _out_dim(c.h, c.pads[0], c.pads[2], c.r, c.stride), _out_dim(c.w, c.pads[1], c.pads[3], c.s, c.stride)
    small = CAP // 32
    x = _ints((c.n, c.h, c.w, c.cin), 2, 0.8, gen)
    w = _weights(c.cout, c.r, c.s, c.cin, x, CAP // 4, gen)
    if c.family == "exact":
        b = _ints((c.cout,), small, 1.0, gen)
    elif c.family == "ties":  # |b| in [CAP, 2 CAP): with a small conv term, y lands on (CAP, 4 CAP)
        b = (CAP + torch.randint(0, CAP, (c.cout,), generator=gen, device=dev)).double() * _ints((c.cout,), 1, 1.0, gen)
    else:  # around the largest finite value: below it, in the round-down band, on the 65520 tie, far beyond
        delta = torch.tensor([-100.0, -17, -1, 0, 1, 7, 15, 16, 17, 100, 5000, 2 ** 20], device=dev)
        b = (ACT_MAX + delta[torch.randint(0, len(delta), (c.cout,), generator=gen, device=dev)]) * \
            _ints((c.cout,), 1, 1.0, gen)
    r = _ints((c.n, P, Q, c.cout), small, 0.5, gen) if c.res else None
    y = _conv64(x, w, c.stride, c.pads) + b
    bound = _conv64(x.abs(), w.abs(), c.stride, c.pads) + (r.abs() if r is not None else 0)
    if c.family == "exact":
        assert (bound + b.abs()).max().item() <= CAP, "generator precondition: |y| <= CAP"
    else:
        assert bound.max().item() <= CAP and (bound + b.abs()).max().item() < 2 ** 24, "generator precondition"
    if r is not None:
        y = y + r
    if c.relu:
        y = torch.relu(y)
    return x, w, b, r, _to_act(y)


def _guarded(shape, guard, fill, dtype=None):
    """A contiguous view of `shape` at element offset `guard` inside a buffer filled with `fill`, with `guard` elements
    after it as well (16-byte aligned when guard * itemsize is a multiple of 16)."""
    numel = math.prod(shape)
    buf = torch.full((2 * guard + numel,), fill, dtype=dtype or ACT, device="cuda")
    return buf, buf[guard:guard + numel].view(shape)


def _guards_intact(buf, guard, fill):
    ends = torch.cat([buf[:guard], buf[-guard:]])
    return bool(torch.isnan(ends).all()) if math.isnan(fill) else bool((ends == fill).all())


def _run_conv(c: Conv, x, w, b, r, out, lib):
    args = (_abi.ptr(x), c.n, c.h, c.w, c.cin, _abi.ptr(w), _abi.ptr(b), c.cout, c.r, c.s, c.stride, *c.pads,
            int(c.relu), _abi.ptr(r), _abi.ptr(out))
    if c.splits is None:
        return lib.mpx_conv2d(*args, c.block_n, c.max_ctas, _abi.stream_ptr())
    return lib.mpx_conv2d_splitk(*args, c.block_n, c.splits, _abi.stream_ptr())


def _launch(c: Conv, x, w, b, r):
    """One launch with the input and residual at an offset inside NaN-filled buffers and the output inside NaN guards of a
    full tile of rows before and after; returns the output after checking that the guards are untouched."""
    plan = _plan(c, _abi.lib().mpx_sm_count())
    lib = _abi.lib()
    xbuf, xv = _guarded(x.shape, 64, float("nan"))
    xv.copy_(x)
    rv = None
    if r is not None:
        rbuf, rv = _guarded(r.shape, 64, float("nan"))
        rv.copy_(r)
    wv = w.reshape(c.cout, -1).to(ACT).contiguous()
    bv = b.float().contiguous()
    guard = BLOCK_M * c.cout
    obuf, out = _guarded((c.n, plan.P, plan.Q, c.cout), guard, float("nan"))
    launches = lib.mpx_launch_count()
    _abi.check(_run_conv(c, xv, wv, bv, rv, out, lib))
    torch.cuda.synchronize()
    assert lib.mpx_launch_count() == launches + 1
    assert _guards_intact(obuf, guard, float("nan")), "write outside the output tensor"
    return out


def _gen(name):
    return torch.Generator(device="cuda").manual_seed(zlib.crc32(name.encode()))


# ---------------------------------------------------------------------------------------------
# convolution tests
# ---------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_conv_bit_exact(case):
    if case.family == "saturate" and ACT != torch.float16:
        pytest.skip("saturation at +-65504 is the fp16 conversion")
    x, w, b, r, want = _problem(case, _gen(case.name))
    got = _launch(case, x, w, b, r)
    bad = got.float() != want.float()
    assert not bad.any(), f"{int(bad.sum())} of {bad.numel()} outputs differ, first at {bad.nonzero()[0].tolist()}"


@gpu
def test_every_tile_width_gives_the_same_bits():
    """The same inputs at every legal BLOCK_N (and the automatic choice), directly and split over K."""
    base = Conv("widths", 2, 15, 20, 128, 256, 3, 3, pads=P1, relu=True, res=True)
    x, w, b, r, want = _problem(base, _gen(base.name))
    for bn in (0, 64, 128, 256):
        assert torch.equal(_launch(dataclasses.replace(base, block_n=bn), x, w, b, r), want), bn
    small = dataclasses.replace(base, name="widths_splitk", n=1, h=6, w=7)
    x, w, b, r, want = _problem(small, _gen(small.name))
    for bn in (64, 128, 256):
        assert torch.equal(_launch(dataclasses.replace(small, block_n=bn, splits=4), x, w, b, r), want), bn


def _chain_problem(g, n, h, w):
    """Integer operands of conv1 (3x3, ReLU) -> conv2 (3x3, + conv1's input, ReLU) -> conv3 (1x1 / s2) and the exact
    result of each stage; the precondition is checked at every layer."""
    x0 = _ints((n, h, w, 64), 2, 0.8, g)
    w1 = _weights(64, 3, 3, 64, x0, 32, g, hi=1)
    b1 = _ints((64,), 8, 1.0, g)
    y1 = torch.relu(_conv64(x0, w1, 1, P1) + b1)
    w2 = _weights(64, 3, 3, 64, y1, 64, g, hi=1)
    b2 = _ints((64,), 8, 1.0, g)
    y2 = torch.relu(_conv64(y1, w2, 1, P1) + b2 + x0)
    w3 = _weights(128, 1, 1, 64, y2, 128, g, hi=1)
    b3 = _ints((128,), 8, 1.0, g)
    y3 = _conv64(y2, w3, 2, P0) + b3
    for xi, wi, bi, extra, stride, pads in ((x0, w1, b1, 0, 1, P1), (y1, w2, b2, x0.abs(), 1, P1), (y2, w3, b3, 0, 2, P0)):
        bound = _conv64(xi.abs(), wi.abs(), stride, pads) + bi.abs() + extra
        assert bound.max().item() <= CAP, "generator precondition"
    return x0, (w1, b1, y1), (w2, b2, y2), (w3, b3, y3)


@gpu
@pytest.mark.parametrize("mode", [DEFAULT_CONV_MODE, DEFAULT_CONV_MODE | NO_PDL], ids=["pdl", "no_pdl"])
def test_dependent_chain_on_one_stream(mode):
    """conv1 -> conv2 (+ conv1's input as residual) -> 1x1 / s2, launched back to back without a host synchronisation into
    NaN-filled intermediates: every stage equals the float64 chain."""
    n, h, w = 2, 16, 20
    x0, (w1, b1, y1), (w2, b2, y2), (w3, b3, y3) = _chain_problem(_gen("chain"), n, h, w)
    lib = _abi.lib()
    xbuf, xv = _guarded(x0.shape, 64, float("nan"))
    xv.copy_(x0)
    _, a1 = _guarded(y1.shape, 64, float("nan"))
    _, a2 = _guarded(y2.shape, 64, float("nan"))
    _, a3 = _guarded(y3.shape, 64, float("nan"))
    ws = [wi.reshape(wi.shape[0], -1).to(ACT).contiguous() for wi in (w1, w2, w3)]
    bs = [bi.float().contiguous() for bi in (b1, b2, b3)]
    torch.cuda.synchronize()
    s = _abi.stream_ptr()
    try:
        set_mode(mode)
        _abi.check(lib.mpx_conv2d(_abi.ptr(xv), n, h, w, 64, _abi.ptr(ws[0]), _abi.ptr(bs[0]), 64, 3, 3, 1, *P1, 1, None,
                                  _abi.ptr(a1), 0, 0, s))
        _abi.check(lib.mpx_conv2d(_abi.ptr(a1), n, h, w, 64, _abi.ptr(ws[1]), _abi.ptr(bs[1]), 64, 3, 3, 1, *P1, 1,
                                  _abi.ptr(xv), _abi.ptr(a2), 0, 0, s))
        _abi.check(lib.mpx_conv2d(_abi.ptr(a2), n, h, w, 64, _abi.ptr(ws[2]), _abi.ptr(bs[2]), 128, 1, 1, 2, *P0, 0, None,
                                  _abi.ptr(a3), 0, 0, s))
        torch.cuda.synchronize()
    finally:
        set_mode(DEFAULT_CONV_MODE)
    for got, want in ((a1, y1), (a2, y2), (a3, y3)):
        assert torch.equal(got, _to_act(want))


def _contract_cases():
    ok = dict(n=1, h=8, w=8, cin=64, cout=64, r=1, s=1, stride=1, pads=P0, relu=0, res=False, block_n=0, extra=0,
              splitk=False, misalign=0)
    cases = [
        ("cin_48", dict(cin=48), "C_in=48 must be a multiple of 64"),
        ("cout_96", dict(cout=96), "C_out=96 must be a multiple of 64"),
        ("cout_576", dict(cout=576), "C_out=576 must be a multiple of 64, at most 512"),
        ("stride_3", dict(stride=3), "stride 3 unsupported"),
        ("filter_9x1", dict(r=9, pads=(4, 0, 4, 0)), "filter 9x1 unsupported"),
        ("filter_1x9", dict(s=9, pads=(0, 4, 0, 4)), "filter 1x9 unsupported"),
        ("filter_0x1", dict(r=0), "filter 0x1 unsupported"),
        ("block_n_96", dict(block_n=96), "BLOCK_N=96 invalid for C_out=64"),
        ("block_n_256_cout_192", dict(cout=192, block_n=256), "BLOCK_N=256 invalid for C_out=192"),
        ("block_n_128_cout_64", dict(block_n=128), "BLOCK_N=128 invalid for C_out=64"),
        ("empty_output", dict(h=2, r=3), "empty output"),
        ("empty_input", dict(n=0), "empty input"),
        ("misaligned_input", dict(misalign=2), "16-byte aligned"),
        ("splitk_splits_3", dict(splitk=True, block_n=64, extra=3), "splits=3 must be 0 (heuristic), 1, 2, 4 or 8"),
        ("splitk_splits_16", dict(splitk=True, block_n=64, extra=16), "splits=16"),
        ("splitk_block_n_0", dict(splitk=True, block_n=0, extra=2), "block_n must be 64|128|256"),
        ("splitk_cin_48", dict(splitk=True, block_n=64, extra=2, cin=48), "C_in=48 must be a multiple of 64"),
        ("splitk_block_n_256_cout_192", dict(splitk=True, cout=192, block_n=256, extra=2), "BLOCK_N=256 invalid"),
    ]
    for relu in (4, 5, 8):  # relu flags: bits 0 (ReLU) and 1 (space-to-depth stem weights) only
        cases.append((f"relu_flags_{relu}", dict(relu=relu), f"relu flags 0x{relu:x}: only bits 0 and 1 are defined"))
        cases.append((f"splitk_relu_flags_{relu}", dict(splitk=True, block_n=64, extra=2, relu=relu),
                      f"relu flags 0x{relu:x}: only bits 0 and 1 are defined"))
    # bit 2 beside a residual or an explicit tile width: refused by the flag check before anything else
    cases.append(("relu_flags_5_with_residual", dict(relu=5, res=True), "relu flags 0x5: only bits 0 and 1 are defined"))
    cases.append(("relu_flags_5_with_block_n_64", dict(relu=5, block_n=64), "relu flags 0x5: only bits 0 and 1 are defined"))
    return [(name, {**ok, **kw}, msg) for name, kw, msg in cases]


CONTRACT_CASES = _contract_cases()


@gpu
@pytest.mark.parametrize("name,a,msg", CONTRACT_CASES, ids=[c[0] for c in CONTRACT_CASES])
def test_conv_refuses_unsupported_arguments(name, a, msg):
    """Every refusal returns non-zero with its message and launches nothing."""
    lib = _abi.lib()
    x = torch.zeros(1 << 16, device="cuda", dtype=ACT)
    w = torch.zeros(1 << 20, device="cuda", dtype=ACT)
    b = torch.zeros(1024, device="cuda")
    res = torch.zeros(1 << 16, device="cuda", dtype=ACT) if a["res"] else None
    out = torch.zeros(1 << 16, device="cuda", dtype=ACT)
    torch.cuda.synchronize()
    # a known message first, so that a message left by an earlier call cannot pass for this refusal's
    assert lib.mpx_conv2d(_abi.ptr(x), 1, 8, 8, 32, _abi.ptr(w), _abi.ptr(b), 64, 1, 1, 1, *P0, 0, None, _abi.ptr(out),
                          0, 0, _abi.stream_ptr()) == -1
    launches = lib.mpx_launch_count()
    fn = lib.mpx_conv2d_splitk if a["splitk"] else lib.mpx_conv2d
    rc = fn(_abi.ptr(x) + a["misalign"], a["n"], a["h"], a["w"], a["cin"], _abi.ptr(w), _abi.ptr(b), a["cout"], a["r"],
            a["s"], a["stride"], *a["pads"], a["relu"], _abi.ptr(res), _abi.ptr(out), a["block_n"],
            a["extra"] if a["splitk"] else 0, _abi.stream_ptr())
    torch.cuda.synchronize()
    assert lib.mpx_launch_count() == launches
    assert rc == -1 and msg.encode() in lib.mpx_last_error(), (rc, lib.mpx_last_error())


GAUSS_CASES = [
    Conv("gauss_bn64", 2, 15, 20, 128, 256, 3, 3, pads=P1, relu=True, res=True, block_n=64),
    Conv("gauss_bn128", 2, 15, 20, 128, 256, 3, 3, pads=P1, relu=True, res=True, block_n=128),
    Conv("gauss_bn256", 2, 15, 20, 128, 256, 3, 3, pads=P1, relu=True, res=True, block_n=256),
    Conv("gauss_splitk_bn64", 1, 8, 10, 512, 128, 3, 3, pads=P1, res=True, block_n=64, splits=8),
]


@gpu
@pytest.mark.parametrize("case", GAUSS_CASES, ids=[c.name for c in GAUSS_CASES])
def test_conv_gaussian_data_within_rounding_bound(case):
    """Real activations are not integers: Gaussian operands, checked per element against the float64 result y64 on the same
    16-bit operands:  |y - y64| <= u |y64| + tiny + (K + 2) 2^-23 (conv(|x|, |w|) + |b| + |r|),  u the unit roundoff of
    the 16-bit type; 2^-23 per term covers tensor-core adders that truncate."""
    g = _gen(case.name)
    k = case.r * case.s * case.cin
    P, Q = _out_dim(case.h, case.pads[0], case.pads[2], case.r, 1), _out_dim(case.w, case.pads[1], case.pads[3], case.s, 1)
    x = torch.randn(case.n, case.h, case.w, case.cin, device="cuda", generator=g).to(ACT).double()
    w = (torch.randn(case.cout, case.r, case.s, case.cin, device="cuda", generator=g) / k ** 0.5).to(ACT).double()
    b = torch.randn(case.cout, device="cuda", generator=g).double()
    r = torch.randn(case.n, P, Q, case.cout, device="cuda", generator=g).to(ACT).double() if case.res else None
    y64 = _conv64(x, w, case.stride, case.pads) + b + (r if r is not None else 0)
    if case.relu:
        y64 = torch.relu(y64)
    mag = _conv64(x.abs(), w.abs(), case.stride, case.pads) + b.abs() + (r.abs() if r is not None else 0)
    got = _launch(case, x.to(ACT), w, b, r.to(ACT) if r is not None else None).double()
    err = (got - y64).abs()
    bound = UNIT * y64.abs() + TINY + (k + 2) * 2.0 ** -23 * mag
    assert (err <= bound).all(), (err - bound).max().item()


def test_auto_tile_width_unchanged_for_network_widths():
    """Automatic BLOCK_N divides every accepted C_out, and for the widths the network uses (64, 128, 256, 512) it is the
    width the previous rule (start from min(C_out, 256)) chose."""
    def previous(cout, m_tiles):
        bn = 256 if cout >= 256 else cout
        while bn > 64 and m_tiles * (cout // bn) < 32:
            bn //= 2
        return bn

    for m_tiles in range(1, 300):
        for cout in range(64, 513, 64):
            bn = _auto_block_n(cout, m_tiles)
            assert bn in STAGES and cout % bn == 0
        for cout in (64, 128, 256, 512):
            assert _auto_block_n(cout, m_tiles) == previous(cout, m_tiles)
    assert [_auto_block_n(c, 40) for c in (192, 320, 384, 448)] == [64, 64, 128, 64]


def test_plan_covers_every_decision_point():
    """Evaluates _plan over CASES for a 132-SM H100 and checks that every edge of the kernel is reached by some case."""
    plans = [(c, _plan(c, SMS_H100)) for c in CASES]
    need = {}
    for bn, st in STAGES.items():
        for nkb in sorted({1, st - 1, st, st + 1, 2 * st + 1, 72}):
            need[f"BLOCK_N {bn} with {nkb} k-blocks"] = lambda c, p, bn=bn, nkb=nkb: p.block_n == bn and p.num_k_blocks == nkb
    for mc in (1, 2, 3, 7):
        need[f"max_ctas {mc}: uneven tiles per CTA, ring wraps inside a tile"] = (
            lambda c, p, mc=mc: c.max_ctas == mc and (mc == 1 or p.tiles % mc != 0) and p.num_k_blocks % p.stages != 0
            and p.tiles_per_cta >= 2)
    need[">= 3 tiles per CTA with num_k_blocks % stages != 0"] = \
        lambda c, p: p.splits == 1 and p.tiles_per_cta >= 3 and p.num_k_blocks % p.stages != 0
    need["a tile spanning three images"] = lambda c, p: p.first_tile_images >= 3
    need["P*Q = 128"] = lambda c, p: p.P * p.Q == 128 and c.n > 1
    need["P*Q = 129"] = lambda c, p: p.P * p.Q == 129 and c.n > 1
    need["last tile with one valid row (M = 128k + 1)"] = lambda c, p: p.last_tile_rows == 1 and p.m_tiles > 1
    for size, k, lo, hi in (("h", "r", 0, 2), ("w", "s", 1, 3)):
        for parity in (0, 1):
            need[f"stride 2, {size.upper()} + pads - {k.upper()} {'odd' if parity else 'even'}"] = (
                lambda c, p, size=size, k=k, lo=lo, hi=hi, parity=parity: c.stride == 2 and
                (getattr(c, size) + c.pads[lo] + c.pads[hi] - getattr(c, k)) % 2 == parity)
    need["1x1 stride 2 pad 0"] = lambda c, p: (c.r, c.s, c.stride, c.pads) == (1, 1, 2, P0)
    for pads in (STEM, (0, 1, 1, 0)):
        need[f"pads {pads}"] = lambda c, p, pads=pads: c.pads == pads
    for rs, pads in (((1, 3), None), ((3, 1), None), ((5, 5), (2, 2, 2, 2)), ((7, 7), (3, 3, 3, 3)), ((8, 8), None)):
        need[f"filter {rs}"] = lambda c, p, rs=rs, pads=pads: (c.r, c.s) == rs and (pads is None or c.pads == pads)
    need["3x3 pad 3 (bias-only border)"] = lambda c, p: (c.r, c.s, c.pads) == (3, 3, (3, 3, 3, 3))
    for stride in (1, 2):
        need[f"driver fix-up off at exactly 131072 B, stride {stride}"] = \
            lambda c, p, st=stride: c.stride == st and p.input_bytes == 131072 and not p.driver_fixup
        need[f"driver fix-up on just below, stride {stride}"] = \
            lambda c, p, st=stride: c.stride == st and 131072 - 128 * 64 < p.input_bytes < 131072 and p.driver_fixup
    need["256 k-blocks"] = lambda c, p: p.num_k_blocks == 256
    for cout in range(64, 513, 64):
        need[f"automatic BLOCK_N, C_out {cout}, few tiles"] = \
            lambda c, p, co=cout: c.cout == co and c.block_n == 0 and c.splits is None and p.tiles < 32
        need[f"automatic BLOCK_N, C_out {cout}, many tiles"] = \
            lambda c, p, co=cout: c.cout == co and c.block_n == 0 and c.splits is None and p.m_tiles >= 32
    for sp in (2, 4, 8):
        need[f"{sp} splits over a k-block count they do not divide"] = \
            lambda c, p, sp=sp: p.splits == sp and p.num_k_blocks % sp != 0
    need["k-ranges of 1 and 2 blocks"] = lambda c, p: {e - b for b, e in p.k_ranges} == {1, 2}
    need["splits clamped to 1 (1 k-block)"] = lambda c, p: c.splits and c.splits > 1 and p.splits == 1
    need["splits clamped below the request"] = lambda c, p: c.splits and 1 < p.splits < c.splits
    need["heuristic split"] = lambda c, p: c.splits == 0 and p.splits > 1
    need["heuristic declines (many tiles)"] = lambda c, p: c.splits == 0 and p.splits == 1
    need["split, M < 128"] = lambda c, p: p.splits > 1 and p.M < BLOCK_M
    need["split, partial second m-tile"] = lambda c, p: p.splits > 1 and p.m_tiles == 2 and p.M % BLOCK_M != 0
    for bn in STAGES:
        for relu in (False, True):
            for res in (False, True):
                need[f"split at BLOCK_N {bn}, relu {relu}, residual {res}"] = (
                    lambda c, p, bn=bn, relu=relu, res=res: p.splits > 1 and p.block_n == bn and c.relu == relu and
                    c.res == res)
    for fam in ("ties", "saturate"):
        need[f"{fam}, direct epilogue"] = lambda c, p, fam=fam: c.family == fam and p.splits == 1
        need[f"{fam}, split-K reduction"] = lambda c, p, fam=fam: c.family == fam and p.splits > 1
    missing = [what for what, pred in need.items() if not any(pred(c, p) for c, p in plans)]
    assert not missing, missing


# ---------------------------------------------------------------------------------------------
# max-pool and pooled linear
# ---------------------------------------------------------------------------------------------
POOL_SHAPES = [(h, w, c) for h, w in ((1, 1), (2, 3), (17, 23), (31, 40), (60, 80)) for c in (8, 64, 136)]
POOL_SHAPES += [(3, 250, 64), (2, 400, 64)]  # 1000 and 1600 items per output row: 512 threads, several passes


@gpu
@pytest.mark.parametrize("h,w,c", POOL_SHAPES, ids=[f"{h}x{w}x{c}" for h, w, c in POOL_SHAPES])
def test_maxpool3x3s2_bit_exact(h, w, c):
    n = 3
    g = _gen(f"maxpool{h}x{w}x{c}")
    x = torch.randn(n, h, w, c, device="cuda", generator=g).to(ACT)
    want = F.max_pool2d(x.double().permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1).to(ACT)
    xbuf, xv = _guarded(x.shape, 64, 60000.0)  # a read outside the input wins every maximum
    xv.copy_(x)
    guard = 64 * c
    obuf, out = _guarded(tuple(want.shape), guard, float("nan"))
    _abi.check(_abi.lib().mpx_maxpool3x3s2(_abi.ptr(xv), n, h, w, c, _abi.ptr(out), _abi.stream_ptr()))
    torch.cuda.synchronize()
    assert _guards_intact(obuf, guard, float("nan"))
    assert torch.equal(out, want)


AVG_CASES = [  # n, hw, c, out_dim: every C with every hw; each out_dim and n at several C
    (1, 1, 4, 1), (7, 6, 4, 9), (300, 49, 4, 33), (7, 80, 4, 512),
    (7, 1, 12, 9), (1, 6, 12, 33), (7, 49, 12, 512), (300, 80, 12, 1),
    (300, 1, 64, 33), (7, 6, 64, 512), (1, 49, 64, 1), (7, 80, 64, 9),
    (7, 1, 512, 512), (300, 6, 512, 1), (7, 49, 512, 9), (1, 80, 512, 33),
    (1, 1, 2048, 1), (7, 6, 2048, 9), (300, 49, 2048, 33), (7, 80, 2048, 512),
    (300, 1, 4096, 9), (7, 6, 4096, 33), (1, 49, 4096, 512), (7, 80, 4096, 1),
]


@gpu
@pytest.mark.parametrize("n,hw,c,out_dim", AVG_CASES, ids=[f"n{a}_hw{b}_c{c}_o{d}" for a, b, c, d in AVG_CASES])
def test_avgpool_linear_within_rounding_bound(n, hw, c, out_dim):
    """Spatial mean then linear, fp32 on the device, against float64 per element:
    |y - y64| <= (hw + C + 2) 2^-23 (|W| mean|x| + |b|)."""
    g = _gen(f"avg{n}_{hw}_{c}_{out_dim}")
    x = torch.randn(n, hw, c, device="cuda", generator=g).to(ACT)
    W = torch.randn(out_dim, c, device="cuda", generator=g) * 0.05
    b = torch.randn(out_dim, device="cuda", generator=g)
    xd = x.double()
    y64 = xd.mean(dim=1) @ W.double().T + b.double()
    mag = xd.abs().mean(dim=1) @ W.double().abs().T + b.double().abs()
    obuf, out = _guarded((n, out_dim), 64, float("nan"), torch.float32)
    _abi.check(_abi.lib().mpx_avgpool_linear(_abi.ptr(x), n, hw, c, _abi.ptr(W), _abi.ptr(b), out_dim, _abi.ptr(out),
                                             _abi.stream_ptr()))
    torch.cuda.synchronize()
    assert _guards_intact(obuf, 64, float("nan"))
    err = (out.double() - y64).abs()
    bound = (hw + c + 2) * 2.0 ** -23 * mag
    assert (err <= bound).all(), (err - bound).max().item()
