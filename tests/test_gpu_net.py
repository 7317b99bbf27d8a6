"""GPU parity of the wgmma convolution and of the whole ResNet-34 engine.

The kernel-selection values of mpx_conv_set_mode that chose between kernel variants (window kernels, CTA pairs, staged
epilogues) are accepted and have no effect in this build: one kernel serves every shape.  The tests that run a shape under
several of those values keep checking that the result does not depend on them, and each result against fp32 torch.

Tolerances (stated, floating point):
  * single conv vs fp32 torch conv on the same 16-bit-rounded operands: |err| <= ULP * max|ref| + ATOL, one rounding
    of the output in the library's 16-bit type (fp16: ULP = 2^-10, ATOL = 2e-3; bf16 build: 2^-7, 1e-2; accumulation
    is fp32 on both sides);
  * full network vs the fp32 oracle: |err_j| <= ACT16_EPS * sum_i |W_ji| |pooled_i| (fp16: 2^-13 of the folded head's
    absolute-value condition bound ~ 0.14 logit standard deviations, about 3x the observed error;
    oracle/resnet_ref.py:act16_forward_error_bound); vs the emulated oracle (same quantisation points, only the
    accumulation order differs): half of that.  The reference itself was trained under fp16 autocast
    (train_megapose.py:299).
"""
import pytest
import torch
import torch.nn.functional as F

from megapose6d_b200 import _abi
from megapose6d_b200.backbone import ResNet34Engine
from oracle import resnet_ref
from tests import helpers

pytestmark = pytest.mark.gpu
ACT = _abi.act_dtype() if torch.cuda.is_available() else torch.float16
ULP, ATOL = (2 ** -10, 2e-3) if ACT == torch.float16 else (2 ** -7, 1e-2)
SINGLE_CTA_MODE = 11  # kernel-variant bits 0, 1 and split-K in the network (bit 3)
DEFAULT_CONV_MODE = 8  # the library's default (include/mpx.h): split-K in the network for small batches
RELOAD_MODE = DEFAULT_CONV_MODE | 32768  # a kernel-variant bit: no effect


def _conv_ref(x, w, bias, stride, pads, relu, residual):
    xf = F.pad(x.float().permute(0, 3, 1, 2), (pads[1], pads[3], pads[0], pads[2]))
    y = F.conv2d(xf, w.float().permute(0, 3, 1, 2), bias=bias, stride=stride).permute(0, 2, 3, 1)
    if residual is not None:
        y = y + residual.float()
    return torch.relu(y) if relu else y


CASES = [
    # name, n, h, w, cin, cout, r, s, stride, (pad_lo_h, pad_lo_w, pad_hi_h, pad_hi_w), relu, residual, block_n, max_ctas
    ("gemm1x1", 1, 8, 16, 64, 64, 1, 1, 1, (0, 0, 0, 0), False, False, 0, 0),
    ("c3x3_relu_res", 2, 12, 20, 64, 64, 3, 3, 1, (1, 1, 1, 1), True, True, 0, 0),
    ("c3x3_s2", 2, 30, 40, 64, 128, 3, 3, 2, (1, 1, 1, 1), True, False, 0, 0),
    ("odd_s2", 3, 15, 20, 128, 256, 3, 3, 2, (1, 1, 1, 1), True, False, 0, 0),
    ("odd_1x1_s2", 3, 15, 20, 128, 256, 1, 1, 2, (0, 0, 0, 0), False, False, 0, 0),
    ("stem4x4", 2, 24, 32, 64, 64, 4, 4, 1, (2, 2, 1, 1), True, False, 0, 0),
    ("stem4x4_c128", 2, 24, 32, 128, 64, 4, 4, 1, (2, 2, 1, 1), True, False, 0, 0),
    ("l4_bn256", 3, 8, 10, 512, 512, 3, 3, 1, (1, 1, 1, 1), True, True, 0, 0),
    ("l4_bn128", 3, 8, 10, 512, 512, 3, 3, 1, (1, 1, 1, 1), True, True, 128, 0),
    ("l3_bn64", 3, 15, 20, 256, 256, 3, 3, 1, (1, 1, 1, 1), True, True, 64, 0),
    ("persist_fewctas", 4, 60, 80, 64, 64, 3, 3, 1, (1, 1, 1, 1), True, True, 0, 7),
    ("ragged_m", 1, 7, 9, 64, 64, 3, 3, 1, (1, 1, 1, 1), False, False, 0, 0),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_conv_vs_torch(case):
    torch.backends.cudnn.allow_tf32 = False
    name, n, h, w, cin, cout, r, s, stride, pads, relu, use_res, block_n, max_ctas = case
    g = torch.Generator(device="cuda").manual_seed(sum(map(ord, name)) % 1000)
    x = torch.randn(n, h, w, cin, device="cuda", generator=g).to(ACT)
    wt = (torch.randn(cout, r, s, cin, device="cuda", generator=g) / (r * s * cin) ** 0.5).to(ACT)
    bias = torch.randn(cout, device="cuda", generator=g)
    p = (h + pads[0] + pads[2] - r) // stride + 1
    q = (w + pads[1] + pads[3] - s) // stride + 1
    res = torch.randn(n, p, q, cout, device="cuda", generator=g).to(ACT) if use_res else None
    out = torch.full((n, p, q, cout), float("nan"), device="cuda", dtype=ACT)
    _abi.check(_abi.lib().mpx_conv2d(_abi.ptr(x), n, h, w, cin, _abi.ptr(wt.view(cout, -1)), _abi.ptr(bias), cout, r, s,
                                          stride, pads[0], pads[1], pads[2], pads[3], int(relu), _abi.ptr(res),
                                          _abi.ptr(out), block_n, max_ctas, _abi.stream_ptr()))
    torch.cuda.synchronize()
    ref = _conv_ref(x, wt, bias, stride, pads, relu, res)
    err = (out.float() - ref).abs().max().item()
    assert not torch.isnan(out.float()).any()
    assert err <= ULP * ref.abs().max().item() + ATOL, err


SPLITK_CASES = [
    # name, n, h, w, cin, cout, r, s, stride, pads, relu, use_res, block_n, splits (0 = heuristic)
    ("layer4_b1", 1, 8, 10, 512, 512, 3, 3, 1, (1, 1, 1, 1), True, True, 64, 8),
    ("layer4_b1_heur", 1, 8, 10, 512, 512, 3, 3, 1, (1, 1, 1, 1), True, True, 64, 0),
    ("layer3_s2", 1, 30, 40, 128, 256, 3, 3, 2, (1, 1, 1, 1), True, False, 64, 4),
    ("layer3_ds_1x1", 2, 30, 40, 128, 256, 1, 1, 2, (0, 0, 0, 0), False, False, 128, 2),
    ("layer2_b2", 2, 30, 40, 128, 128, 3, 3, 1, (1, 1, 1, 1), True, True, 128, 4),
    ("wide_tile", 1, 15, 20, 256, 256, 3, 3, 1, (1, 1, 1, 1), False, True, 256, 8),
    ("many_tiles", 3, 8, 10, 512, 512, 3, 3, 1, (1, 1, 1, 1), True, True, 64, 8),
    ("single_split", 1, 8, 10, 256, 256, 3, 3, 1, (1, 1, 1, 1), True, True, 64, 1),
]


@pytest.mark.parametrize("case", SPLITK_CASES, ids=[c[0] for c in SPLITK_CASES])
def test_conv_splitk_matches_unsplit_and_reference(case):
    """K loop split over a thread-block cluster, partial tiles reduced through distributed shared memory."""
    name, n, h, w, cin, cout, r, s, stride, pads, relu, use_res, block_n, splits = case
    g = torch.Generator(device="cuda").manual_seed(sum(map(ord, name)) % 1000)
    x = torch.randn(n, h, w, cin, device="cuda", generator=g).to(ACT)
    wt = (torch.randn(cout, r, s, cin, device="cuda", generator=g) / (r * s * cin) ** 0.5).to(ACT)
    bias = torch.randn(cout, device="cuda", generator=g)
    p = (h + pads[0] + pads[2] - r) // stride + 1
    q = (w + pads[1] + pads[3] - s) // stride + 1
    res = torch.randn(n, p, q, cout, device="cuda", generator=g).to(ACT) if use_res else None
    lib = _abi.lib()
    outs = []
    for rep in range(2):
        out = torch.full((n, p, q, cout), float("nan"), device="cuda", dtype=ACT)
        _abi.check(lib.mpx_conv2d_splitk(_abi.ptr(x), n, h, w, cin, _abi.ptr(wt.view(cout, -1)), _abi.ptr(bias), cout, r,
                                              s, stride, pads[0], pads[1], pads[2], pads[3], int(relu), _abi.ptr(res),
                                              _abi.ptr(out), block_n, splits, _abi.stream_ptr()))
        torch.cuda.synchronize()
        outs.append(out.float())
    unsplit = torch.full((n, p, q, cout), float("nan"), device="cuda", dtype=ACT)
    _abi.check(lib.mpx_conv2d(_abi.ptr(x), n, h, w, cin, _abi.ptr(wt.view(cout, -1)), _abi.ptr(bias), cout, r, s, stride,
                                   pads[0], pads[1], pads[2], pads[3], int(relu), _abi.ptr(res), _abi.ptr(unsplit), block_n, 0,
                                   _abi.stream_ptr()))
    torch.cuda.synchronize()
    ref = _conv_ref(x, wt, bias, stride, pads, relu, res)
    tol = ULP * ref.abs().max().item() + ATOL
    assert not torch.isnan(outs[0]).any()
    assert (outs[0] - ref).abs().max() <= tol
    # fp32 partial sums are combined in a different (fixed) order than the unsplit K loop: one bf16 rounding at most
    assert (outs[0] - unsplit.float()).abs().max() <= ULP * ref.abs().max().item()
    assert torch.equal(outs[0], outs[1])  # partial tiles are summed in rank order: deterministic


def test_conv_splitk_rejects_bad_split_count():
    x = torch.zeros(1, 8, 8, 64, device="cuda", dtype=ACT)
    w = torch.zeros(64, 64, device="cuda", dtype=ACT)
    b = torch.zeros(64, device="cuda")
    out = torch.zeros(1, 8, 8, 64, device="cuda", dtype=ACT)
    rc = _abi.lib().mpx_conv2d_splitk(_abi.ptr(x), 1, 8, 8, 64, _abi.ptr(w), _abi.ptr(b), 64, 1, 1, 1, 0, 0, 0, 0, 0, None,
                                           _abi.ptr(out), 64, 3, _abi.stream_ptr())
    assert rc != 0 and b"splits" in _abi.lib().mpx_last_error()


def test_conv_rejects_bad_arguments():
    x = torch.zeros(1, 8, 8, 48, device="cuda", dtype=ACT)
    w = torch.zeros(64, 48, device="cuda", dtype=ACT)
    b = torch.zeros(64, device="cuda")
    out = torch.zeros(1, 8, 8, 64, device="cuda", dtype=ACT)
    rc = _abi.lib().mpx_conv2d(_abi.ptr(x), 1, 8, 8, 48, _abi.ptr(w), _abi.ptr(b), 64, 1, 1, 1, 0, 0, 0, 0, 0, None,
                                    _abi.ptr(out), 0, 0, _abi.stream_ptr())
    assert rc != 0 and b"multiple of 64" in _abi.lib().mpx_last_error()


def test_maxpool_and_tail():
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(3, 30, 40, 64, device="cuda", generator=g).to(ACT)
    out = torch.empty(3, 15, 20, 64, device="cuda", dtype=ACT)
    _abi.check(_abi.lib().mpx_maxpool3x3s2(_abi.ptr(x), 3, 30, 40, 64, _abi.ptr(out), _abi.stream_ptr()))
    ref = F.max_pool2d(x.float().permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1)
    assert torch.equal(out.float(), ref)
    f = torch.randn(5, 80, 512, device="cuda", generator=g).to(ACT)
    W = torch.randn(9, 512, device="cuda", generator=g) * 0.05
    b = torch.randn(9, device="cuda", generator=g)
    o = torch.empty(5, 9, device="cuda")
    _abi.check(_abi.lib().mpx_avgpool_linear(_abi.ptr(f), 5, 80, 512, _abi.ptr(W), _abi.ptr(b), 9, _abi.ptr(o), _abi.stream_ptr()))
    ref = f.float().mean(dim=1) @ W.t() + b
    assert torch.allclose(o, ref, rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("cfg_name", ["coarse", "refiner", "refiner_rgbd"])
def test_resnet34_engine_vs_oracle(cfg_name):
    cfg = dict(coarse=helpers.COARSE_CFG, refiner=helpers.REFINER_CFG, refiner_rgbd=helpers.REFINER_RGBD_CFG)[cfg_name]
    sd = helpers.make_state_dict(cfg, seed=2)
    c = helpers.n_inputs(cfg)
    head = resnet_ref.head_name(sd)
    eng = ResNet34Engine(sd, n_inputs=c, head=head)
    x = helpers._calibration_batch(c, 40, n=5)
    got = eng(x.cuda()).cpu()
    emu = resnet_ref.forward_act16_emulated(sd, x.cuda(), ACT).cpu()
    with torch.no_grad():
        fp32 = resnet_ref.forward(sd, x)
        bound = resnet_ref.act16_forward_error_bound(sd, x, dtype=ACT)
    e_emu = (got - emu).abs()
    e_fp = (got - fp32).abs()
    print(f"[{cfg_name}] max|engine-emulated|={e_emu.max():.4g} max|engine-fp32|={e_fp.max():.4g} "
          f"bound={bound.min():.4g}..{bound.max():.4g} out std={fp32.std():.4g}")
    assert (e_emu <= 0.5 * bound + 1e-4).all()   # same quantisation points: only accumulation order differs
    assert (e_fp <= bound + 1e-4).all()           # stated 16-bit-vs-fp32 tolerance (resnet_ref.act16_forward_error_bound)
    # small input as well (stem / pooling edge handling): 64x96
    x2 = helpers._calibration_batch(c, 41, n=3, h=64, w=96)
    got2 = eng(x2.cuda()).cpu()
    emu2 = resnet_ref.forward_act16_emulated(sd, x2.cuda(), ACT).cpu()
    with torch.no_grad():
        bound2 = resnet_ref.act16_forward_error_bound(sd, x2, dtype=ACT)
    assert ((got2 - emu2).abs() <= 0.5 * bound2 + 1e-4).all()


WINDOW_CASES = [
    # the 64 -> 64 stride-1 "same" convolutions of the stem and layer1, under mode bit 0 set and cleared
    ("win_3x3", 3, 60, 80, 3, 3, (1, 1, 1, 1), True, True),
    ("win_3x3_tiny", 5, 7, 9, 3, 3, (1, 1, 1, 1), False, False),
    ("win_stem", 2, 120, 160, 4, 4, (2, 2, 1, 1), True, False),
    ("win_stem_small", 2, 24, 32, 4, 4, (2, 2, 1, 1), True, False),
]


@pytest.mark.parametrize("case", WINDOW_CASES, ids=[c[0] for c in WINDOW_CASES])
def test_window_and_im2col_kernels_agree(case):
    """The same products accumulated in fp32 under either mode value: outputs agree to one 16-bit ulp,
    and each is within the stated tolerance of the fp32 reference."""
    name, n, h, w, r, s, pads, relu, use_res = case
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn(n, h, w, 64, device="cuda", generator=g).to(ACT)
    wt = (torch.randn(64, r, s, 64, device="cuda", generator=g) / (r * s * 64) ** 0.5).to(ACT)
    bias = torch.randn(64, device="cuda", generator=g)
    res = torch.randn(n, h, w, 64, device="cuda", generator=g).to(ACT) if use_res else None
    outs = []
    try:
        for mode in (1, 0):
            _abi.lib().mpx_conv_set_mode(mode)
            out = torch.full((n, h, w, 64), float("nan"), device="cuda", dtype=ACT)
            _abi.check(_abi.lib().mpx_conv2d(_abi.ptr(x), n, h, w, 64, _abi.ptr(wt.view(64, -1)), _abi.ptr(bias), 64, r, s, 1,
                                                  pads[0], pads[1], pads[2], pads[3], int(relu), _abi.ptr(res), _abi.ptr(out), 0, 0,
                                                  _abi.stream_ptr()))
            torch.cuda.synchronize()
            outs.append(out.float())
    finally:
        _abi.lib().mpx_conv_set_mode(DEFAULT_CONV_MODE)
    ref = _conv_ref(x, wt, bias, 1, pads, relu, res)
    tol = ULP * ref.abs().max().item() + ATOL
    assert (outs[0] - ref).abs().max() <= tol and (outs[1] - ref).abs().max() <= tol
    assert (outs[0] - outs[1]).abs().max() <= tol


@pytest.mark.parametrize("cfg_name,n", [("refiner", 1), ("coarse", 2), ("refiner", 5)])
def test_small_batch_splitk_network_matches_unsplit(cfg_name, n):
    """Small batches run layers 2-4 with split-K (mode bit 3).  Same logits as the unsplit network up to fp32
    summation order, stable over repeated calls (the scratch is left zeroed) and under graph replay."""
    cfg = helpers.REFINER_CFG if cfg_name == "refiner" else helpers.COARSE_CFG
    c = helpers.n_inputs(cfg)
    head = "pose_fc" if cfg["predict_pose_update"] else "views_logits_head"
    sd = helpers.make_state_dict(cfg, seed=3)
    eng = ResNet34Engine(sd, n_inputs=c, head=head)
    x = eng.pack_input(helpers._calibration_batch(c, 5, n=n).cuda())
    lib = _abi.lib()
    try:
        lib.mpx_net_set_graphs(0)
        lib.mpx_conv_set_mode(3)
        unsplit = eng.forward(x, 240, 320)
        lib.mpx_conv_set_mode(DEFAULT_CONV_MODE)
        split = [eng.forward(x, 240, 320) for _ in range(3)]
        lib.mpx_net_set_graphs(1)
        graphed = [eng.forward(x, 240, 320) for _ in range(4)]
    finally:
        lib.mpx_net_set_graphs(1)
        lib.mpx_conv_set_mode(DEFAULT_CONV_MODE)
    with torch.no_grad():
        bound = resnet_ref.act16_forward_error_bound(sd, helpers._calibration_batch(c, 5, n=n), dtype=ACT).cuda()
    for o in split + graphed:
        assert torch.isfinite(o).all()
        assert ((o - unsplit).abs() <= 0.5 * bound + 1e-6).all(), ((o - unsplit).abs().max(), bound.min())
        assert torch.equal(o, split[0])  # deterministic


WIN2_CASES = [
    # name, n, h, w, relu, use_res, max_ctas
    ("l2_res", 4, 30, 40, True, True, 4),
    ("l2_nores_many_per_cta", 9, 30, 40, True, False, 3),
    ("odd_size", 3, 17, 23, False, True, 2),
    ("tiny_images", 11, 5, 7, True, True, 2),
    ("one_super_tile", 1, 12, 16, True, False, 1),
]


@pytest.mark.parametrize("case", WIN2_CASES, ids=[c[0] for c in WIN2_CASES])
def test_layer2_window_kernel_agrees_with_im2col_and_torch(case):
    """The layer2 shape (128 -> 128, 3x3) with few CTAs for many tiles (persistent loop), under mode bit 8 cleared and
    set, vs fp32 torch."""
    name, n, h, w, relu, use_res, max_ctas = case
    g = torch.Generator(device="cuda").manual_seed(23)
    x = torch.randn(n, h, w, 128, device="cuda", generator=g).to(ACT)
    wt = (torch.randn(128, 3, 3, 128, device="cuda", generator=g) / (9 * 128) ** 0.5).to(ACT)
    bias = torch.randn(128, device="cuda", generator=g)
    res = torch.randn(n, h, w, 128, device="cuda", generator=g).to(ACT) if use_res else None
    outs = []
    try:
        for mode in (SINGLE_CTA_MODE, SINGLE_CTA_MODE | 256):
            _abi.lib().mpx_conv_set_mode(mode)
            out = torch.full((n, h, w, 128), float("nan"), device="cuda", dtype=ACT)
            _abi.check(_abi.lib().mpx_conv2d(_abi.ptr(x), n, h, w, 128, _abi.ptr(wt.view(128, -1)), _abi.ptr(bias), 128, 3, 3,
                                                  1, 1, 1, 1, 1, int(relu), _abi.ptr(res), _abi.ptr(out), 0, max_ctas,
                                                  _abi.stream_ptr()))
            torch.cuda.synchronize()
            outs.append(out.float())
    finally:
        _abi.lib().mpx_conv_set_mode(DEFAULT_CONV_MODE)
    ref = _conv_ref(x, wt, bias, 1, (1, 1, 1, 1), relu, res)
    tol = ULP * ref.abs().max().item() + ATOL
    assert not torch.isnan(outs[0]).any()
    assert (outs[0] - ref).abs().max() <= tol and (outs[1] - ref).abs().max() <= tol
    # equal up to one 16-bit rounding
    assert (outs[0] - outs[1]).abs().max() <= ULP * ref.abs().max().item()


def test_graph_replay_equals_eager_launches():
    cfg = helpers.COARSE_CFG
    sd = helpers.make_state_dict(cfg, seed=2)
    eng = ResNet34Engine(sd, n_inputs=9, head="views_logits_head")
    x = eng.pack_input(helpers._calibration_batch(9, 3, n=3).cuda())
    try:
        _abi.lib().mpx_net_set_graphs(0)
        eager = eng.forward(x, 240, 320)
        _abi.lib().mpx_net_set_graphs(1)
        outs = [eng.forward(x, 240, 320) for _ in range(3)]  # eager warm-up, capture, replay
    finally:
        _abi.lib().mpx_net_set_graphs(1)
    for o in outs:
        assert torch.equal(o, eager)


PAIR_CASES = [
    ("pair_l3", 5, 15, 20, 256, 256, 3, 3, 1, (1, 1, 1, 1), True, True),
    ("pair_l4_two_ntiles", 3, 8, 10, 512, 512, 3, 3, 1, (1, 1, 1, 1), True, True),
    ("pair_s2", 3, 30, 40, 128, 256, 3, 3, 2, (1, 1, 1, 1), True, False),
    ("pair_ds_1x1", 3, 30, 40, 128, 256, 1, 1, 2, (0, 0, 0, 0), False, False),
    ("pair_single_tile", 1, 8, 10, 256, 256, 3, 3, 1, (1, 1, 1, 1), False, False),
    ("pair_forced_128", 4, 30, 40, 128, 128, 3, 3, 1, (1, 1, 1, 1), True, True),
    ("pair_l3_all_sms", 96, 15, 20, 256, 256, 3, 3, 1, (1, 1, 1, 1), True, True),
    ("pair_l4_all_sms_ragged", 61, 8, 10, 512, 512, 3, 3, 1, (1, 1, 1, 1), True, True),
    ("pair_l3_no_residual", 40, 15, 20, 256, 256, 3, 3, 1, (1, 1, 1, 1), True, False),
]


@pytest.mark.parametrize("case", PAIR_CASES, ids=[c[0] for c in PAIR_CASES])
def test_cta_pair_kernel_vs_torch_and_single_cta(case):
    """The shapes of layers 3-4 under three kernel-variant values of the mode (bits 1, 2, 25) vs fp32 torch; the results
    are bit-identical."""
    name, n, h, w, cin, cout, r, s, stride, pads, relu, use_res = case
    g = torch.Generator(device="cuda").manual_seed(11)
    x = torch.randn(n, h, w, cin, device="cuda", generator=g).to(ACT)
    wt = (torch.randn(cout, r, s, cin, device="cuda", generator=g) / (r * s * cin) ** 0.5).to(ACT)
    bias = torch.randn(cout, device="cuda", generator=g)
    p = (h + pads[0] + pads[2] - r) // stride + 1
    q = (w + pads[1] + pads[3] - s) // stride + 1
    res = torch.randn(n, p, q, cout, device="cuda", generator=g).to(ACT) if use_res else None
    outs = []
    try:
        for mode in (7, 1, 7 | 33554432):  # pair kernel | single-CTA kernel | pair kernel with the staged epilogue (bit 25)
            _abi.lib().mpx_conv_set_mode(mode)
            out = torch.full((n, p, q, cout), float("nan"), device="cuda", dtype=ACT)
            _abi.check(_abi.lib().mpx_conv2d(_abi.ptr(x), n, h, w, cin, _abi.ptr(wt.view(cout, -1)), _abi.ptr(bias), cout, r, s,
                                                  stride, pads[0], pads[1], pads[2], pads[3], int(relu), _abi.ptr(res),
                                                  _abi.ptr(out), 0, 0, _abi.stream_ptr()))
            torch.cuda.synchronize()
            outs.append(out.float())
    finally:
        _abi.lib().mpx_conv_set_mode(DEFAULT_CONV_MODE)
    ref = _conv_ref(x, wt, bias, stride, pads, relu, res)
    tol = ULP * ref.abs().max().item() + ATOL
    assert (outs[0] - ref).abs().max() <= tol and (outs[1] - ref).abs().max() <= tol
    assert torch.equal(outs[0], outs[1])  # same products, same K order, fp32 accumulation
    assert torch.equal(outs[0], outs[2])  # staged epilogue (residual by TMA, bias from global memory): same arithmetic


PAIR_WINDOW_CASES = [
    # conv_window2q_kernel (bit 14 = 16384, default): the layer2 window kernel on CTA pairs, two issuers
    # name, n, h, w, c_in, c_out, relu, use_res, max_ctas
    ("l2_pairs_odd_super_tiles", 4, 30, 40, 128, 128, True, True, 4),
    ("l2_pairs_many_per_pair", 9, 30, 40, 128, 128, True, False, 2),
    ("l2_pairs_odd_size", 3, 17, 23, 128, 128, False, True, 2),
    ("l2_pairs_tiny_images", 11, 5, 7, 128, 128, True, True, 2),
    ("l2_pairs_one_item_peer_idle", 1, 12, 16, 128, 128, True, False, 1),
    ("l2_pairs_all_sms_residual", 96, 30, 40, 128, 128, True, True, 0),
    ("l2_pairs_all_sms", 80, 30, 40, 128, 128, True, False, 0),
    ("l2_pairs_224", 24, 28, 28, 128, 128, True, True, 0),
]


@pytest.mark.parametrize("case", PAIR_WINDOW_CASES, ids=[c[0] for c in PAIR_WINDOW_CASES])
def test_layer2_pair_window_kernel(case):
    """conv_window2q_kernel (the layer2 window kernel on CTA pairs, default since r02) vs the single-CTA window kernel and
    fp32 torch."""
    name, n, h, w, cin, cout, relu, use_res, max_ctas = case
    g = torch.Generator(device="cuda").manual_seed(29)
    x = torch.randn(n, h, w, cin, device="cuda", generator=g).to(ACT)
    wt = (torch.randn(cout, 3, 3, cin, device="cuda", generator=g) / (9 * cin) ** 0.5).to(ACT)
    bias = torch.randn(cout, device="cuda", generator=g)
    res = torch.randn(n, h, w, cout, device="cuda", generator=g).to(ACT) if use_res else None
    outs = []
    try:
        for mode in (DEFAULT_CONV_MODE, DEFAULT_CONV_MODE ^ 16777216, SINGLE_CTA_MODE):  # bit 24 flipped: the other epilogue form
            _abi.lib().mpx_conv_set_mode(mode)
            out = torch.full((n, h, w, cout), float("nan"), device="cuda", dtype=ACT)
            _abi.check(_abi.lib().mpx_conv2d(_abi.ptr(x), n, h, w, cin, _abi.ptr(wt.view(cout, -1)), _abi.ptr(bias), cout, 3,
                                             3, 1, 1, 1, 1, 1, int(relu), _abi.ptr(res), _abi.ptr(out), 0, max_ctas,
                                             _abi.stream_ptr()))
            torch.cuda.synchronize()
            outs.append(out.float())
    finally:
        _abi.lib().mpx_conv_set_mode(DEFAULT_CONV_MODE)
    ref = _conv_ref(x, wt, bias, 1, (1, 1, 1, 1), relu, res)
    tol = ULP * ref.abs().max().item() + ATOL
    for o in outs:
        assert not torch.isnan(o).any()
        assert (o - ref).abs().max() <= tol
        assert (o - outs[-1]).abs().max() <= ULP * ref.abs().max().item()
    assert torch.equal(outs[0], outs[1])  # staged (TMA residual, coalesced stores) vs row-per-thread epilogue: same arithmetic


PAIR_WINDOW64_CASES = [
    # name, n, h, w, r, pads (lo_h, lo_w, hi_h, hi_w), relu, use_res, max_ctas
    ("layer1", 7, 60, 80, 3, (1, 1, 1, 1), True, False, 6),
    ("layer1_residual", 5, 60, 80, 3, (1, 1, 1, 1), True, True, 4),
    ("stem_4x4", 3, 120, 160, 4, (2, 2, 1, 1), True, False, 6),
    ("odd_size_odd_tiles", 3, 17, 23, 3, (1, 1, 1, 1), False, True, 2),
    ("two_tiles_one_pair", 1, 12, 16, 3, (1, 1, 1, 1), True, False, 2),
    ("one_by_one_taps", 4, 20, 24, 1, (0, 0, 0, 0), False, False, 4),
    ("layer1_all_sms", 40, 60, 80, 3, (1, 1, 1, 1), True, True, 0),
    ("stem_all_sms", 12, 120, 160, 4, (2, 2, 1, 1), True, False, 0),
    ("ragged_runs", 9, 33, 47, 3, (1, 1, 1, 1), True, True, 10),
]


@pytest.mark.parametrize("case", PAIR_WINDOW64_CASES, ids=[c[0] for c in PAIR_WINDOW64_CASES])
def test_pair_window64_kernel(case):
    """conv_windowq_kernel (bit 15 = 32768, default since r02: the 64 -> 64 window kernel on CTA pairs) vs the single-CTA
    window kernel and fp32 torch."""
    name, n, h, w, r, pads, relu, use_res, max_ctas = case
    g = torch.Generator(device="cuda").manual_seed(37)
    x = torch.randn(n, h, w, 64, device="cuda", generator=g).to(ACT)
    wt = (torch.randn(64, r, r, 64, device="cuda", generator=g) / (r * r * 64) ** 0.5).to(ACT)
    bias = torch.randn(64, device="cuda", generator=g)
    res = torch.randn(n, h, w, 64, device="cuda", generator=g).to(ACT) if use_res else None
    outs = []
    try:
        for mode in (DEFAULT_CONV_MODE, RELOAD_MODE, SINGLE_CTA_MODE):
            _abi.lib().mpx_conv_set_mode(mode)
            out = torch.full((n, h, w, 64), float("nan"), device="cuda", dtype=ACT)
            _abi.check(_abi.lib().mpx_conv2d(_abi.ptr(x), n, h, w, 64, _abi.ptr(wt.view(64, -1)), _abi.ptr(bias), 64, r, r,
                                             1, pads[0], pads[1], pads[2], pads[3], int(relu), _abi.ptr(res), _abi.ptr(out),
                                             0, max_ctas, _abi.stream_ptr()))
            torch.cuda.synchronize()
            outs.append(out.float())
    finally:
        _abi.lib().mpx_conv_set_mode(DEFAULT_CONV_MODE)
    ref = _conv_ref(x, wt, bias, 1, pads, relu, res)
    tol = ULP * ref.abs().max().item() + ATOL
    for o in outs:
        assert not torch.isnan(o).any()
        assert (o - ref).abs().max() <= tol
        assert (o - outs[-1]).abs().max() <= ULP * ref.abs().max().item()
    assert torch.equal(outs[0], outs[1])  # sliding window: the same MMAs in the same order per output row


@pytest.mark.parametrize("mode", [DEFAULT_CONV_MODE, SINGLE_CTA_MODE], ids=["cta_pairs", "single_cta"])
def test_stem_space_to_depth_skips_zero_slices(mode):
    """The 7x7 / stride-2 stem runs as a 4x4 convolution over the space-to-depth input; 15 of its 64 (tap, sub-pixel) weight
    slices are zero by construction.  With or without the space-to-depth flag (relu bit 1) and mode bit 17 the output is
    bit-identical, and it matches torch's 7x7 / stride-2 convolution."""
    from megapose6d_b200.backbone import _stem_s2d

    n, h, w, c, c_pad = 5, 96, 128, 9, 16
    g = torch.Generator(device="cuda").manual_seed(41)
    w7 = (torch.randn(64, c, 7, 7, device="cuda", generator=g) / (49 * c) ** 0.5).to(ACT)
    x = torch.rand(n, c, h, w, device="cuda", generator=g).to(ACT)
    bias = torch.randn(64, device="cuda", generator=g)
    ws2d = _stem_s2d(w7.float().cpu(), c_pad).to(ACT).cuda().contiguous()
    xp = torch.zeros(n, c_pad, h, w, device="cuda", dtype=ACT)
    xp[:, :c] = x
    xs = xp.view(n, c_pad, h // 2, 2, w // 2, 2).permute(0, 2, 4, 3, 5, 1).reshape(n, h // 2, w // 2, 4 * c_pad).contiguous()
    outs = []
    try:
        for flags, m in ((3, mode), (1, mode), (3, mode | 131072)):
            _abi.lib().mpx_conv_set_mode(m)
            out = torch.full((n, h // 2, w // 2, 64), float("nan"), device="cuda", dtype=ACT)
            _abi.check(_abi.lib().mpx_conv2d(_abi.ptr(xs), n, h // 2, w // 2, 4 * c_pad, _abi.ptr(ws2d), _abi.ptr(bias), 64, 4, 4, 1,
                                             2, 2, 1, 1, flags, None, _abi.ptr(out), 0, 6, _abi.stream_ptr()))
            torch.cuda.synchronize()
            outs.append(out)
    finally:
        _abi.lib().mpx_conv_set_mode(DEFAULT_CONV_MODE)
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])
    ref = torch.relu(F.conv2d(x.float(), w7.float(), bias=bias, stride=2, padding=3)).permute(0, 2, 3, 1)
    assert (outs[0].float() - ref).abs().max() <= ULP * ref.abs().max().item() + ATOL


@pytest.mark.parametrize("backbone_str", ["resnet34", "resnet18"])
def test_wide_resnet_engine_vs_oracle(backbone_str):
    """Pre-activation backbones (models/wide_resnet.py, backbone_str "resnet34" / "resnet18"): 5x5 stem as a 3x3 convolution
    over the space-to-depth input, affine + ReLU pass per block, bare downsample, spatial mean into the head."""
    cfg = dict(helpers.REFINER_CFG, backbone_str=backbone_str)
    sd = helpers.make_state_dict(cfg, seed=4)
    c = helpers.n_inputs(cfg)
    eng = ResNet34Engine(sd, n_inputs=c, head="pose_fc")
    for n, hh, ww in ((5, 240, 320), (3, 64, 96), (70, 64, 96)):
        x = helpers._calibration_batch(c, 42 + n, n=n, h=hh, w=ww)
        got = eng(x.cuda()).cpu()
        emu = resnet_ref.forward_wide_act16_emulated(sd, x.cuda(), ACT).cpu()
        with torch.no_grad():
            fp32 = resnet_ref.forward_wide(sd, x)
            bound = resnet_ref.act16_forward_error_bound(sd, x, dtype=ACT)
        print(f"[{backbone_str} n={n}] max|engine-emulated|={(got - emu).abs().max():.4g} max|engine-fp32|={(got - fp32).abs().max():.4g} "
              f"bound={bound.min():.4g}..{bound.max():.4g}")
        assert ((got - emu).abs() <= 0.5 * bound + 2e-4).all()  # same quantisation points; 2e-4 = a fifth of an fp16 ulp at 1
        assert ((got - fp32).abs() <= bound + 1e-4).all()


SEPARATE_POOL_MODE = DEFAULT_CONV_MODE & ~2097152  # without bit 21: stem output stored, max-pool as its own kernel
FUSED_POOL_MODE = DEFAULT_CONV_MODE | 2097152  # bit 21: the stem's epilogue max-pools
POOL_CASES = [
    # name, n, h, w, r, pads, max_ctas
    ("stem_4x4", 3, 120, 160, 4, (2, 2, 1, 1), 6),
    ("stem_224", 2, 112, 112, 4, (2, 2, 1, 1), 0),
    ("odd_rows_odd_cols", 3, 17, 23, 3, (1, 1, 1, 1), 2),
    ("odd_rows", 2, 31, 40, 3, (1, 1, 1, 1), 4),
    ("two_tiles_one_pair", 1, 12, 16, 3, (1, 1, 1, 1), 2),
    ("stem_all_sms", 10, 120, 160, 4, (2, 2, 1, 1), 0),
]


@pytest.mark.parametrize("case", POOL_CASES, ids=[c[0] for c in POOL_CASES])
def test_fused_maxpool_epilogue_equals_conv_then_maxpool(case):
    """mpx_conv2d with relu bit 2 (the pooled epilogue: vector max-reductions into the zeroed pooled tensor) against the
    stored convolution followed by mpx_maxpool3x3s2: the maximum is exact, so the two agree value for value (torch.equal on
    floats: +0 == -0), for even and odd sizes, image borders and tile borders."""
    name, n, h, w, r, pads, max_ctas = case
    g = torch.Generator(device="cuda").manual_seed(43)
    x = torch.randn(n, h, w, 64, device="cuda", generator=g).to(ACT)
    wt = (torch.randn(64, r, r, 64, device="cuda", generator=g) / (r * r * 64) ** 0.5).to(ACT)
    bias = torch.randn(64, device="cuda", generator=g)
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    lib = _abi.lib()
    full = torch.full((n, h, w, 64), float("nan"), device="cuda", dtype=ACT)
    _abi.check(lib.mpx_conv2d(_abi.ptr(x), n, h, w, 64, _abi.ptr(wt.view(64, -1)), _abi.ptr(bias), 64, r, r, 1, *pads, 1, None,
                              _abi.ptr(full), 0, max_ctas, _abi.stream_ptr()))
    want = torch.empty(n, ho, wo, 64, device="cuda", dtype=ACT)
    _abi.check(lib.mpx_maxpool3x3s2(_abi.ptr(full), n, h, w, 64, _abi.ptr(want), _abi.stream_ptr()))
    assert not torch.isnan(want.float()).any()
    try:
        for mode in (DEFAULT_CONV_MODE, RELOAD_MODE):
            lib.mpx_conv_set_mode(mode)
            got = torch.zeros(n, ho, wo, 64, device="cuda", dtype=ACT)
            _abi.check(lib.mpx_conv2d(_abi.ptr(x), n, h, w, 64, _abi.ptr(wt.view(64, -1)), _abi.ptr(bias), 64, r, r, 1, *pads, 1 | 4,
                                      None, _abi.ptr(got), 0, max_ctas, _abi.stream_ptr()))
            torch.cuda.synchronize()
            assert torch.equal(got.float(), want.float()), mode
    finally:
        lib.mpx_conv_set_mode(DEFAULT_CONV_MODE)
    # shapes without the epilogue are refused without launching anything (the network then runs conv + max-pool)
    assert lib.mpx_conv2d(_abi.ptr(x), n, h, w, 64, _abi.ptr(wt.view(64, -1)), _abi.ptr(bias), 64, r, r, 1, *pads, 4, None,
                          _abi.ptr(got), 0, max_ctas, _abi.stream_ptr()) == -3  # no ReLU


@pytest.mark.parametrize("cfg_name,n", [("coarse", 7), ("refiner", 1)])
def test_network_with_fused_maxpool_equals_unfused(cfg_name, n):
    """The whole forward with mode bit 21 (the stem's epilogue pools) against the stem followed by the max-pool kernel:
    every later layer sees the same pooled tensor, so the outputs are identical."""
    cfg = dict(coarse=helpers.COARSE_CFG, refiner=helpers.REFINER_CFG)[cfg_name]
    sd = helpers.make_state_dict(cfg, seed=3)
    c = helpers.n_inputs(cfg)
    x = helpers._calibration_batch(c, 42, n=n).cuda()
    outs = []
    try:
        for mode in (SEPARATE_POOL_MODE, FUSED_POOL_MODE, FUSED_POOL_MODE):
            _abi.lib().mpx_conv_set_mode(mode)
            eng = ResNet34Engine(sd, n_inputs=c, head=resnet_ref.head_name(sd))
            outs.append(eng(x).clone())  # first sight of a shape runs eagerly
            outs.append(eng(x).clone())  # ... the second captures a graph (memset node + kernels), the third replays it
            outs.append(eng(x).clone())
            torch.cuda.synchronize()
    finally:
        _abi.lib().mpx_conv_set_mode(DEFAULT_CONV_MODE)
    for o in outs[1:]:
        assert torch.equal(outs[0], o)
