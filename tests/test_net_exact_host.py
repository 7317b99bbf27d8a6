"""Host checks (no GPU) of the pose networks' exact tests (tests/test_gpu_net_exact.py): the float64 plan of
oracle/net_plan_ref.py computes the reference network, the integer state dicts meet its exactness preconditions, the case
list reaches every kernel path of conv_forward on a 132-SM H100, and the workspace layout holds every map of both
schedules."""
from __future__ import annotations

import pytest
import torch

from oracle import net_plan_ref as R
from oracle import resnet_ref
from tests import test_gpu_net_exact as T


def _double(sd):
    return {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}


@pytest.mark.parametrize("family", ["vanilla_resnet34", "resnet34", "resnet18"])
@pytest.mark.parametrize("n_inputs,h,w", [(9, 64, 96), (27, 38, 50)], ids=["9ch-64x96", "27ch-38x50"])
def test_plan_without_rounding_equals_the_reference_network(family, n_inputs, h, w):
    """With rounding turned off the plan (folded BatchNorm, the stems as 7x7 / 5x5 convolutions, the folded head) is the
    reference network evaluated in float64."""
    if family == "vanilla_resnet34":
        sd = _double(resnet_ref.init_state_dict(n_inputs, "pose_fc", 9, seed=3))
        ref = resnet_ref.forward
    else:
        sd = _double(resnet_ref.init_state_dict_wide(n_inputs, "pose_fc", 9, seed=3, backbone_str=family))
        ref = resnet_ref.forward_wide
    x = torch.rand(2, n_inputs, h, w, generator=torch.Generator().manual_seed(4), dtype=torch.float64)
    got, _ = R.forward(sd, x, exact=False)
    want = ref(sd, x)
    assert got.dtype == torch.float64
    err = (got - want).abs().max().item()
    assert err <= 1e-10 * want.abs().max().item(), err


def test_plan_rounds_where_the_engine_rounds():
    """The same network with rounding on differs from the float64 network by 16-bit roundings, not more."""
    sd = _double(resnet_ref.init_state_dict(9, "views_logits_head", 1, seed=5))
    x = torch.rand(2, 9, 64, 96, generator=torch.Generator().manual_seed(6), dtype=torch.float64)
    exact, _ = R.forward(sd, x, exact=False)
    rounded, stats = R.forward(sd, x, check=False)
    bound = resnet_ref.act16_forward_error_bound(sd, x).double()
    assert 0 < (rounded - exact).abs().max().item() and bool(((rounded - exact).abs() <= bound).all())
    assert stats.convs == 36 and stats.saturated == 0


SIZES_USED = sorted({(c[0], c[2], c[3]) for c in T.EXACT_CASES + T.MODE_CASES})


@pytest.mark.parametrize("config,h,w", SIZES_USED, ids=lambda v: str(v))
def test_integer_state_dicts_meet_the_exactness_preconditions(config, h, w):
    """On every configuration and size of the GPU file the oracle's assertions hold (every partial sum and pooled sum below
    2^24 at the operands' granularity), values above 2048 are rounded, and saturation stays a small minority."""
    sd = T._state_dict(config)
    out, stats = R.forward(sd, T._input(config, 1, h, w), torch.float16)
    assert torch.equal(out.float().double(), out)  # the read-out head is exact
    assert (stats.pooled != 0).float().mean().item() > 0.5  # most channels reach the head
    if h * w >= 64 * 96:
        assert stats.max_abs > 2048 and stats.saturated_fraction < 0.05, (stats.max_abs, stats.saturated_fraction)


def test_integer_head_is_a_scaled_signed_permutation():
    for config in ("coarse", "wide34"):
        W, b = R._Plan(T._state_dict(config), torch.float16, "cpu", True, False).head()
        assert bool((b == 0).all())
        nz = W != 0
        assert bool((nz.sum(0) == 1).all()) and bool((nz.sum(1) == 1).all())
        assert set(W[nz].abs().tolist()) <= {0.5, 1.0, 2.0}


def test_case_list_reaches_every_kernel_path():
    """conv_forward's dispatch restated for a 132-SM H100 (test_gpu_net_exact.route): the GPU cases reach split-K 8/4/2/1,
    the unsplit 128-row kernel, the ping-pong kernel, the pixel-major kernel with band loading and with im2col, odd maps
    at every layer and a 1-pixel layer-4 map."""
    reached = set()
    for config, n, h, w in T.EXACT_CASES:
        for conv in T.net_convs(config, n, h, w):
            kernel, splits, producer = T.route(conv)
            reached.add((kernel, splits if kernel == "conv_wgmma_kernel" and conv[-1] < 0 else "unsplit", producer))
        maps = [(T._pool(h // 2), T._pool(w // 2))]
        for _ in range(3):
            maps.append(((maps[-1][0] - 1) // 2 + 1, (maps[-1][1] - 1) // 2 + 1))
        if all(a % 2 and b % 2 for a, b in maps):
            reached.add("odd maps at every layer")
        if maps[-1] == (1, 1):
            reached.add("1-pixel layer-4 map")
        if n == 64 and (n, h, w) == (64, 240, 320):
            reached.add("last split-K batch")
        if n == 65:
            reached.add("first unsplit batch")
    for config, n, h, w in T.MODE_CASES:
        for mode in T.MODES:
            for conv in T.net_convs(config, n, h, w, mode):
                kernel, splits, producer = T.route(conv, mode)
                reached.add(("mode", kernel, producer))
    need = {("conv_wgmma_kernel", s, None) for s in (1, 2, 4, 8)} | {
        ("conv_wgmma_kernel", "unsplit", None), ("convpp_wgmma_kernel", "unsplit", None),
        ("conv64_wgmma_kernel", "unsplit", "band"), ("conv64_wgmma_kernel", "unsplit", "im2col"),
        ("mode", "conv64_wgmma_kernel", "im2col"), ("mode", "convpp_wgmma_kernel", None),
        "odd maps at every layer", "1-pixel layer-4 map", "last split-K batch", "first unsplit batch"}
    assert need <= reached, need - reached
    # the batch whose stem and layer 1 run on the pixel-major kernel and layer 2 on the ping-pong kernel is a case
    assert T.N_ALL_KERNELS in T.BATCHES and ("coarse", T.N_ALL_KERNELS, 240, 320) in T.EXACT_CASES
    kernels = T._kernels("coarse", T.N_ALL_KERNELS, 240, 320)
    assert all(k == "conv64_wgmma_kernel" for k, _, _ in kernels[:7])
    assert kernels[7][0] == "convpp_wgmma_kernel"  # layer2.0.conv1 (stride 2) -- and the stride-1 layer-2 convolutions
    assert {k for k, _, _ in kernels[8:16]} >= {"convpp_wgmma_kernel"}


@pytest.mark.parametrize("preact", [False, True], ids=["post-activation", "pre-activation"])
def test_workspace_layout_holds_every_map(preact):
    """Every step of the buffer rotation writes at most one rotating buffer's bytes, never into a buffer it reads, for n in
    {1, 2, 3, 64} and every even h, w <= 128."""
    blocks = (3, 4, 6, 3)
    for n in (1, 2, 3, 64):
        for h in range(2, 129, 2):
            for w in range(2, 129, 2):
                _, buf, count, _ = T.workspace_layout(n, h, w, preact)
                for out, nbytes, reads in T.buffer_writes(n, h, w, preact, blocks):
                    assert 0 <= out < count and nbytes <= buf, (n, h, w, out, nbytes, buf)
                    assert out not in reads, (n, h, w, out, reads)


def test_workspace_layout_exceeds_the_layer1_sizing_at_small_inputs():
    """The sizes where a rotating buffer of the layer-1 map's size is too small, e.g. 2 images of 4x4: a 256-byte buffer
    for a 2048-byte layer-4 map."""
    _, buf, _, _ = T.workspace_layout(2, 4, 4, False)
    assert buf == 2048 and T._a256(T.layer_maps(2, 4, 4)[1] * 2) == 256
    for h, w in T.TINY_SIZES:
        maps = T.layer_maps(2, h, w)
        assert max(maps) > maps[1], (h, w)
