"""Seeded random network weights in the reference's checkpoint layout (no checkpoint is available offline).

Workload generation for bench.py, tools/ and tests/ -- neither the product (megapose6d_b200/) nor the oracle.  The
state dicts follow `resnet34(num_classes=512, n_input_channels=C)` + the single linear head
(models/torchvision_resnet.py:181-316, models/pose_rigid.py:120-130); the head is conditioned on a calibration batch
(plain torch fp32 on the host, run once per configuration) so that random weights give O(1) logits and small pose
updates.
"""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn.functional as F

LAYERS = [3, 4, 6, 3]
WIDTHS = [64, 128, 256, 512]
BN_EPS = 1e-5

COARSE_CFG = dict(n_rendered_views=1, multiview_type="TCO", render_normals=True, render_depth=False, input_depth=False,
                  predict_rendered_views_logits=True, predict_pose_update=False, remove_TCO_rendering=False,
                  depth_normalization_type="tCR_scale_clamp_center")
REFINER_CFG = dict(n_rendered_views=4, multiview_type="TCO+front_3views", render_normals=True, render_depth=False,
                   input_depth=False, predict_rendered_views_logits=False, predict_pose_update=True,
                   remove_TCO_rendering=False, depth_normalization_type="tCR_scale_clamp_center")
REFINER_RGBD_CFG = dict(REFINER_CFG, render_depth=True, input_depth=True)


def n_inputs(cfg) -> int:
    per_view = 3 + (3 if cfg.get("render_normals", True) else 0) + int(cfg["render_depth"])  # pose_models_cfg.py:95-103
    return (3 + int(cfg["input_depth"])) + per_view * cfg["n_rendered_views"]


def init_state_dict(n_inputs: int, head: str, head_dim: int, seed: int = 0) -> Dict[str, torch.Tensor]:
    """Seeded random weights in the reference checkpoint layout (kaiming fan_out convs as
    torchvision_resnet.py:232-237, non-trivial BN statistics so that folding is exercised)."""
    g = torch.Generator().manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}

    def conv(name, co, ci, k):
        std = (2.0 / (co * k * k)) ** 0.5
        sd[name + ".weight"] = torch.randn(co, ci, k, k, generator=g) * std

    def bn(name, c):
        sd[name + ".weight"] = 0.5 + torch.rand(c, generator=g)
        sd[name + ".bias"] = 0.2 * torch.randn(c, generator=g)
        sd[name + ".running_mean"] = 0.2 * torch.randn(c, generator=g)
        sd[name + ".running_var"] = 0.5 + torch.rand(c, generator=g)
        sd[name + ".num_batches_tracked"] = torch.tensor(1)

    conv("backbone.conv1", 64, n_inputs, 7)
    bn("backbone.bn1", 64)
    inplanes = 64
    for li, (nb, width) in enumerate(zip(LAYERS, WIDTHS)):
        for b in range(nb):
            p = f"backbone.layer{li + 1}.{b}"
            stride = 2 if (b == 0 and li > 0) else 1
            conv(p + ".conv1", width, inplanes, 3)
            bn(p + ".bn1", width)
            conv(p + ".conv2", width, width, 3)
            bn(p + ".bn2", width)
            if stride != 1 or inplanes != width:
                conv(p + ".downsample.0", width, inplanes, 1)
                bn(p + ".downsample.1", width)
            inplanes = width
    sd["backbone.fc.weight"] = torch.randn(512, 512, generator=g) * (1.0 / 512) ** 0.5
    sd["backbone.fc.bias"] = 0.1 * torch.randn(512, generator=g)
    sd[head + ".weight"] = torch.randn(head_dim, 512, generator=g) * (1.0 / 512) ** 0.5
    sd[head + ".bias"] = 0.1 * torch.randn(head_dim, generator=g)
    return sd



def _bn(x, sd, name):
    return F.batch_norm(x, sd[name + ".running_mean"], sd[name + ".running_var"], sd[name + ".weight"],
                        sd[name + ".bias"], training=False, eps=BN_EPS)


def _pooled_features(sd: Dict[str, torch.Tensor], x: torch.Tensor) -> torch.Tensor:
    """fp32 backbone up to the global average pool [b, 512] (calibration only)."""
    x = F.conv2d(x, sd["backbone.conv1.weight"], stride=2, padding=3)
    x = F.relu(_bn(x, sd, "backbone.bn1"))
    x = F.max_pool2d(x, kernel_size=3, stride=2, padding=1)
    for li, nb in enumerate(LAYERS):
        for b in range(nb):
            p = f"backbone.layer{li + 1}.{b}"
            stride = 2 if (b == 0 and li > 0) else 1
            identity = x
            out = F.relu(_bn(F.conv2d(x, sd[p + ".conv1.weight"], stride=stride, padding=1), sd, p + ".bn1"))
            out = _bn(F.conv2d(out, sd[p + ".conv2.weight"], stride=1, padding=1), sd, p + ".bn2")
            if (p + ".downsample.0.weight") in sd:
                identity = _bn(F.conv2d(x, sd[p + ".downsample.0.weight"], stride=stride), sd, p + ".downsample.1")
            x = F.relu(out + identity)
    return torch.flatten(F.adaptive_avg_pool2d(x, (1, 1)), 1)


WIDE_LAYERS = {"resnet34": [3, 4, 6, 3], "resnet18": [2, 2, 2, 2]}


def init_state_dict_wide(n_inputs: int, head: str, head_dim: int, seed: int = 0, backbone_str: str = "resnet34"):
    """Seeded random weights in the checkpoint layout of a WideResNet backbone (models/wide_resnet.py:59-126) + head."""
    g = torch.Generator().manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}

    def conv(name, co, ci, k):
        sd[name + ".weight"] = torch.randn(co, ci, k, k, generator=g) * (2.0 / (co * k * k)) ** 0.5

    def bn(name, c):
        sd[name + ".weight"] = 0.5 + torch.rand(c, generator=g)
        sd[name + ".bias"] = 0.2 * torch.randn(c, generator=g)
        sd[name + ".running_mean"] = 0.2 * torch.randn(c, generator=g)
        sd[name + ".running_var"] = 0.5 + torch.rand(c, generator=g)
        sd[name + ".num_batches_tracked"] = torch.tensor(1)

    conv("backbone.conv1", 64, n_inputs, 5)
    bn("backbone.bn1", 64)
    inplanes = 64
    for li, (nb, width) in enumerate(zip(WIDE_LAYERS[backbone_str], WIDTHS)):
        for b in range(nb):
            p = f"backbone.layer{li + 1}.{b}"
            stride = 2 if (b == 0 and li > 0) else 1
            bn(p + ".bn1", inplanes)
            conv(p + ".conv1", width, inplanes, 3)
            bn(p + ".bn2", width)
            conv(p + ".conv2", width, width, 3)
            if stride != 1 or inplanes != width:
                conv(p + ".downsample", width, inplanes, 1)
            inplanes = width
    sd[head + ".weight"] = torch.randn(head_dim, 512, generator=g) * (1.0 / 512) ** 0.5
    sd[head + ".bias"] = 0.1 * torch.randn(head_dim, generator=g)
    return sd


def _pooled_features_wide(sd: Dict[str, torch.Tensor], x: torch.Tensor) -> torch.Tensor:
    """fp32 pre-activation backbone up to the spatial mean [b, 512] (calibration only)."""
    x = F.relu(_bn(F.conv2d(x, sd["backbone.conv1.weight"], stride=2, padding=2), sd, "backbone.bn1"))
    x = F.max_pool2d(x, kernel_size=3, stride=2, padding=1)
    li = 0
    while f"backbone.layer{li + 1}.0.conv1.weight" in sd:
        b = 0
        while f"backbone.layer{li + 1}.{b}.conv1.weight" in sd:
            p = f"backbone.layer{li + 1}.{b}"
            stride = 2 if (b == 0 and li > 0) else 1
            a = F.relu(_bn(x, sd, p + ".bn1"))
            res = F.conv2d(a, sd[p + ".downsample.weight"], stride=stride) if (p + ".downsample.weight") in sd else x
            y = F.relu(_bn(F.conv2d(a, sd[p + ".conv1.weight"], stride=stride, padding=1), sd, p + ".bn2"))
            x = F.conv2d(y, sd[p + ".conv2.weight"], stride=1, padding=1) + res
            b += 1
        li += 1
    return x.flatten(2).mean(dim=-1)


def calibration_batch(c, seed, n=4, h=240, w=320):
    """Smooth images in [0,1]; half of them with the render channels masked to a blob on black, like real inputs."""
    g = torch.Generator().manual_seed(1000 + seed)
    x = torch.rand(n, c, h // 8, w // 8, generator=g)
    x = torch.nn.functional.interpolate(x, size=(h, w), mode="bilinear", align_corners=False)
    yy, xx = torch.meshgrid(torch.linspace(-1, 1, h), torch.linspace(-1, 1, w), indexing="ij")
    blob = ((xx ** 2 + yy ** 2) < 0.4).float()
    x[n // 2:, 3:] *= blob
    return x.clamp(0, 1)


_SD_CACHE = {}


def make_state_dict(cfg, seed=0):
    """Seeded random weights in the checkpoint layout with a conditioned head: the head is made orthogonal to the
    dominant feature direction of a calibration batch and scaled so that coarse logits are O(1) and pose updates are
    small (R ~ I, v_z ~ 1) -- random heads otherwise produce |logit| ~ 300 and 20x depth jumps."""
    key = (tuple(sorted(cfg.items())), seed)
    if key in _SD_CACHE:
        return dict(_SD_CACHE[key])
    head = "pose_fc" if cfg["predict_pose_update"] else "views_logits_head"
    dim = 9 if cfg["predict_pose_update"] else cfg["n_rendered_views"]
    c = n_inputs(cfg)
    wide = cfg.get("backbone_str", "vanilla_resnet34") in ("resnet34", "resnet18")
    if wide:
        sd = init_state_dict_wide(c, head, dim, seed=seed, backbone_str=cfg["backbone_str"])
        with torch.no_grad():
            feats = _pooled_features_wide(sd, calibration_batch(c, seed))
    else:
        sd = init_state_dict(c, head, dim, seed=seed)
        with torch.no_grad():
            pooled = _pooled_features(sd, calibration_batch(c, seed))
            feats = torch.nn.functional.linear(pooled, sd["backbone.fc.weight"], sd["backbone.fc.bias"])
    v = torch.linalg.svd(feats, full_matrices=False)[2][0]
    W = sd[head + ".weight"]
    W = W - (W @ v).unsqueeze(1) * v.unsqueeze(0)
    raw = feats @ W.t()
    W = W * ((0.02 if cfg["predict_pose_update"] else 1.5) / (raw - raw.mean(0)).std().clamp_min(1e-12))
    sd[head + ".weight"] = W
    offset = (feats @ W.t()).mean(0)
    if cfg["predict_pose_update"]:
        sd[head + ".bias"] = torch.tensor([1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0]) - offset
    else:
        sd[head + ".bias"] = -offset
    _SD_CACHE[key] = dict(sd)
    return sd


def integer_state_dict(n_inputs: int, head: str = "views_logits_head", head_dim: int = 512, readout: bool = True,
                       seed: int = 0, backbone_str: str = "vanilla_resnet34", nnz: int = 2,
                       stem_nnz: int = 4) -> Dict[str, torch.Tensor]:
    """A state dict in the checkpoint layout (either backbone family) on which every value of the engine's plan is an
    integer, so that its fp32 accumulation is exact in any order and it must equal the float64 plan of
    oracle/net_plan_ref.py bit for bit on inputs of small integers:
      * every convolution: `nnz` non-zero weights per output channel (`stem_nnz` for the stem, on real taps of real input
        channels), the rest zero;
      * every BatchNorm folded into a convolution (stored in float64): gamma = 2^e sqrt(var + eps) with e in {-1, 0, 1} per
        channel, so that the folded scale is exactly 2^e, an integer beta and an even integer mean.  The raw weights are
        +-1, and +-2 where e = -1: the folded weights are integers (+-1, +-2), and so is the folded bias;
      * the pre-activation affine (WideResNet bn1): scale in {0.5, 1, 2} and an integer shift, both varying by channel.  The
        channels scaled by 0.5 are a fixed set per layer on which every producer of the residual stream writes even values
        (folded stem weights +-2 and an even bias, conv2 and downsample weights +-2), so that the affine stays integral;
      * `readout` (head_dim 512): fc = I with zero bias (post-activation), and the head a signed permutation scaled by 2^e
        per row with zero bias -- every pooled channel reaches one output unchanged up to a power of two.  Otherwise the
        head (and the fc) get Gaussian weights, as init_state_dict.
    net_plan_ref.forward asserts for every convolution and the pooled sums that the partial sums stay below 2^24."""
    g = torch.Generator().manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}
    wide = backbone_str in WIDE_LAYERS

    def ints(lo, hi, shape):
        return torch.randint(lo, hi + 1, shape, generator=g).double()

    def conv(name, co, ci, k, nz, mag=None):
        """+-mag[o] at nz random taps of output channel o (mag: per channel, default 1)."""
        w = torch.zeros(co, ci * k * k, dtype=torch.float64)
        idx = torch.stack([torch.randperm(ci * k * k, generator=g)[:nz] for _ in range(co)])
        sign = ints(0, 1, (co, nz)) * 2 - 1
        w.scatter_(1, idx, sign * (mag.view(-1, 1) if mag is not None else 1.0))
        sd[name + ".weight"] = w.view(co, ci, k, k)

    def folded_conv(name, bn_name, co, ci, k, nz, even=None):
        """Convolution + BatchNorm with integer folded weights and bias; `even` channels get even outputs (e = 1)."""
        e = ints(-1, 1, (co,))
        beta = ints(-2, 2, (co,))
        if even is not None:
            e[even] = 1.0
            beta[even] = 2 * torch.round(beta[even] / 2)
        conv(name, co, ci, k, nz, mag=torch.where(e < 0, 2.0, 1.0))
        var = 0.5 + torch.rand(co, generator=g, dtype=torch.float64)
        sd[bn_name + ".weight"] = 2.0 ** e * torch.sqrt(var + BN_EPS)
        sd[bn_name + ".bias"] = beta
        sd[bn_name + ".running_mean"] = 2 * ints(-1, 1, (co,))
        sd[bn_name + ".running_var"] = var
        sd[bn_name + ".num_batches_tracked"] = torch.tensor(1)

    def affine(name, c, halved):
        """bn1 of a pre-activation block: scale 0.5 on `halved`, else 1 or 2; integer shift."""
        scale = torch.where(ints(0, 1, (c,)) > 0, 2.0, 1.0).double()
        scale[halved] = 0.5
        var = 0.5 + torch.rand(c, generator=g, dtype=torch.float64)
        sd[name + ".weight"] = scale * torch.sqrt(var + BN_EPS)
        sd[name + ".bias"] = ints(-3, 3, (c,))
        sd[name + ".running_mean"] = torch.zeros(c, dtype=torch.float64)
        sd[name + ".running_var"] = var
        sd[name + ".num_batches_tracked"] = torch.tensor(1)

    inplanes = 64
    if wide:
        halved = {w: torch.randperm(w, generator=g)[:w // 3] for w in WIDTHS}  # per stream width
        folded_conv("backbone.conv1", "backbone.bn1", 64, n_inputs, 5, stem_nnz, even=halved[64])
        for li, (nb, width) in enumerate(zip(WIDE_LAYERS[backbone_str], WIDTHS)):
            two = torch.ones(width, dtype=torch.float64)
            two[halved[width]] = 2.0
            for b in range(nb):
                p = f"backbone.layer{li + 1}.{b}"
                stride = 2 if (b == 0 and li > 0) else 1
                affine(p + ".bn1", inplanes, halved[inplanes])
                folded_conv(p + ".conv1", p + ".bn2", width, inplanes, 3, nnz)
                conv(p + ".conv2", width, width, 3, nnz, mag=two)
                if stride != 1 or inplanes != width:
                    conv(p + ".downsample", width, inplanes, 1, 1, mag=two)
                inplanes = width
    else:
        folded_conv("backbone.conv1", "backbone.bn1", 64, n_inputs, 7, stem_nnz)
        for li, (nb, width) in enumerate(zip(LAYERS, WIDTHS)):
            for b in range(nb):
                p = f"backbone.layer{li + 1}.{b}"
                stride = 2 if (b == 0 and li > 0) else 1
                folded_conv(p + ".conv1", p + ".bn1", width, inplanes, 3, nnz)
                folded_conv(p + ".conv2", p + ".bn2", width, width, 3, nnz)
                if stride != 1 or inplanes != width:
                    folded_conv(p + ".downsample.0", p + ".downsample.1", width, inplanes, 1, 1)
                inplanes = width
    if readout:
        assert head_dim == 512
        if not wide:
            sd["backbone.fc.weight"] = torch.eye(512, dtype=torch.float64)
            sd["backbone.fc.bias"] = torch.zeros(512, dtype=torch.float64)
        perm = torch.randperm(512, generator=g)
        scale = (2.0 ** ints(-1, 1, (512,))) * (ints(0, 1, (512,)) * 2 - 1)
        sd[head + ".weight"] = torch.zeros(512, 512, dtype=torch.float64).index_put_((torch.arange(512), perm), scale)
        sd[head + ".bias"] = torch.zeros(512, dtype=torch.float64)
    else:
        if not wide:
            sd["backbone.fc.weight"] = torch.randn(512, 512, generator=g, dtype=torch.float64) * (1.0 / 512) ** 0.5
            sd["backbone.fc.bias"] = 0.1 * torch.randn(512, generator=g, dtype=torch.float64)
        sd[head + ".weight"] = torch.randn(head_dim, 512, generator=g, dtype=torch.float64) * (1.0 / 512) ** 0.5
        sd[head + ".bias"] = 0.1 * torch.randn(head_dim, generator=g, dtype=torch.float64)
    return sd
