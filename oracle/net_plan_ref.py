"""float64 oracle of the pose networks' engine plan (megapose6d_b200/backbone.py: ResNet34Engine, csrc/net.cu:
mpx_net_forward), for both backbone families, evaluated from a state dict in the layout ResNet34Engine reads: the function
the engine computes, with its quantisation points and nothing else.

  * BatchNorm folded into the convolution before it in float64 with BN_EPS (backbone._fold), the folded weights rounded
    once to act16 and the biases to fp32, as the engine stores them; the post-activation head is fc and head folded into
    one matrix in float64, rounded to fp32 (the WideResNet head is stored as is, rounded to fp32);
  * the input rounded to act16 (the engine's space-to-depth input tensor);
  * every convolution evaluated in float64 -- the 7x7/s2 (post-activation) and 5x5/s2 (pre-activation) stems as such,
    not in the engine's space-to-depth form -- and its output rounded ONCE to act16, saturating, after bias, residual
    and ReLU;
  * the pre-activation pass fp32(x * scale + shift), ReLU, one rounding;
  * max-pool with -inf padding (exact);
  * the tail pooled = fp32(fp32(sum_p x) * fp32(1 / hw)) and the linear map in float64.
With `exact=False` nothing is rounded: the plan in float64, which must equal resnet_ref's forward.

On integer operands (workloads/weights.integer_state_dict) the engine's fp32 accumulation is exact in any order, so only
the roundings above remain and the engine must equal this oracle bit for bit.  `forward` asserts that precondition on
every call: the operands of every convolution are multiples of 2^-g and every partial sum stays below 2^(24-g) (bounded by
max|x| * max_row sum|w| + max|b| + max|residual|), and every pooled sum below 2^(24-g) (hw * max|x|).  The statistics it
returns (largest magnitude before rounding, saturated elements) show that rounding and saturation happened.

Runs on x.device: cuDNN double convolutions on the GPU, torch's CPU convolutions on the host.
"""
from __future__ import annotations

from typing import Dict, Tuple

import torch
import torch.nn.functional as F

LAYERS = [3, 4, 6, 3]
WIDE_LAYERS = {"resnet34": [3, 4, 6, 3], "resnet18": [2, 2, 2, 2]}
BN_EPS = 1e-5
EXACT_LIMIT = 2.0 ** 24  # fp32 integers are exact below this


def is_wide(sd) -> bool:
    return "backbone.layer1.0.bn1.weight" in sd and "backbone.fc.weight" not in sd


def head_name(sd) -> str:
    return "pose_fc" if "pose_fc.weight" in sd else "views_logits_head"


def wide_layers(sd):
    return [sum(1 for k in sd if k.startswith(f"backbone.layer{li}.") and k.endswith(".conv1.weight")) for li in (1, 2, 3, 4)]


def _granularity(t: torch.Tensor, limit: int = 24) -> int:
    """Smallest g with every element of t a multiple of 2^-g."""
    for g in range(limit + 1):
        s = t * (2.0 ** g)
        if bool((s == torch.floor(s)).all()):
            return g
    raise AssertionError(f"operands are not multiples of 2^-{limit}")


class Stats:
    """What the roundings did: the largest magnitude before a rounding, the elements rounded to the largest finite value."""

    def __init__(self):
        self.max_abs = 0.0
        self.saturated = 0
        self.rounded_elements = 0
        self.convs = 0
        self.pooled = None

    @property
    def saturated_fraction(self) -> float:
        return self.saturated / max(self.rounded_elements, 1)


class _Plan:
    def __init__(self, sd: Dict[str, torch.Tensor], dtype: torch.dtype, device, exact: bool, check: bool):
        self.sd, self.dtype, self.dev, self.exact, self.check = sd, dtype, device, exact, check
        self.lim = float(torch.finfo(dtype).max)
        self.stats = Stats()

    # --- quantisation points -------------------------------------------------------------------
    def q(self, t: torch.Tensor) -> torch.Tensor:
        """Round to act16 through fp32 (saturating, round to nearest even), back to float64."""
        if not self.exact:
            return t
        self.stats.max_abs = max(self.stats.max_abs, t.abs().max().item() if t.numel() else 0.0)
        self.stats.rounded_elements += t.numel()
        self.stats.saturated += int((t.abs() >= self.lim).sum().item())
        return t.to(torch.float32).clamp(-self.lim, self.lim).to(self.dtype).to(torch.float64)

    def f32(self, t: torch.Tensor) -> torch.Tensor:
        return t.to(torch.float32).to(torch.float64) if self.exact else t

    def qw(self, w: torch.Tensor) -> torch.Tensor:
        """Folded weights as the engine stores them: float64 -> fp32 -> act16."""
        return w.to(torch.float32).to(self.dtype).to(torch.float64) if self.exact else w

    # --- parameters ----------------------------------------------------------------------------
    def _t(self, name):
        return self.sd[name].detach().to(torch.float64).cpu()

    def folded(self, conv: str, bn) -> Tuple[torch.Tensor, torch.Tensor]:
        w = self._t(conv + ".weight")
        if bn is None:
            b = torch.zeros(w.shape[0], dtype=torch.float64)
        else:
            scale = self._t(bn + ".weight") / torch.sqrt(self._t(bn + ".running_var") + BN_EPS)
            w = w * scale.view(-1, 1, 1, 1)
            b = self._t(bn + ".bias") - self._t(bn + ".running_mean") * scale
        return self.qw(w).to(self.dev), self.f32(b).to(self.dev)

    def affine(self, bn: str) -> Tuple[torch.Tensor, torch.Tensor]:
        scale = self._t(bn + ".weight") / torch.sqrt(self._t(bn + ".running_var") + BN_EPS)
        shift = self._t(bn + ".bias") - self._t(bn + ".running_mean") * scale
        return self.f32(scale).view(1, -1, 1, 1).to(self.dev), self.f32(shift).view(1, -1, 1, 1).to(self.dev)

    # --- operations ----------------------------------------------------------------------------
    def conv(self, x, conv, bn, stride, padding, relu, residual=None):
        w, b = self.folded(conv, bn)
        if self.exact and self.check:
            self._assert_exact(x, w, b, residual)
        y = F.conv2d(x, w, b, stride=stride, padding=padding)
        if residual is not None:
            y = y + residual
        if relu:
            y = F.relu(y)
        self.stats.convs += 1
        return self.q(y)

    def _assert_exact(self, x, w, b, residual):
        g = max(_granularity(x) + _granularity(w), _granularity(b), _granularity(residual) if residual is not None else 0)
        bound = x.abs().max().item() * w.abs().flatten(1).sum(1).max().item() + b.abs().max().item()
        if residual is not None:
            bound += residual.abs().max().item()
        assert bound * 2.0 ** g < EXACT_LIMIT, f"convolution {self.stats.convs}: partial sums up to {bound} at 2^-{g}"

    def pre_activation(self, x, bn):
        scale, shift = self.affine(bn)
        if self.exact and self.check:
            g = max(_granularity(x) + _granularity(scale), _granularity(shift))
            bound = x.abs().max().item() * scale.abs().max().item() + shift.abs().max().item()
            assert bound * 2.0 ** g < EXACT_LIMIT, f"pre-activation affine: values up to {bound} at 2^-{g}"
        return self.q(F.relu(self.f32(x * scale + shift)))

    def tail(self, x: torch.Tensor) -> torch.Tensor:
        n, c, h, w = x.shape
        flat = x.flatten(2)
        if not self.exact:
            pooled = flat.mean(dim=-1)
        else:
            if self.check:
                g = _granularity(flat)
                assert h * w * flat.abs().max().item() * 2.0 ** g < EXACT_LIMIT, "pooled sums are not exact in fp32"
            s = flat.sum(dim=-1).to(torch.float32)
            pooled = (s * torch.tensor(1.0 / (h * w), dtype=torch.float32)).to(torch.float64)
        self.stats.pooled = pooled
        return self.linear(pooled)

    def linear(self, pooled: torch.Tensor) -> torch.Tensor:
        W, bias = self.head()
        return pooled @ W.to(pooled.device).t() + bias.to(pooled.device)

    def head(self):
        h = head_name(self.sd)
        Wh, bh = self._t(h + ".weight"), self._t(h + ".bias")
        if not is_wide(self.sd):
            Wf, bf = self._t("backbone.fc.weight"), self._t("backbone.fc.bias")
            Wh, bh = Wh @ Wf, Wh @ bf + bh
        return self.f32(Wh), self.f32(bh)

    # --- schedules -----------------------------------------------------------------------------
    def post_activation(self, x):
        x = self.conv(x, "backbone.conv1", "backbone.bn1", 2, 3, True)
        x = F.max_pool2d(x, kernel_size=3, stride=2, padding=1)
        for li, nb in enumerate(LAYERS):
            for bi in range(nb):
                p = f"backbone.layer{li + 1}.{bi}"
                stride = 2 if (bi == 0 and li > 0) else 1
                t = self.conv(x, p + ".conv1", p + ".bn1", stride, 1, True)
                identity = x
                if (p + ".downsample.0.weight") in self.sd:
                    identity = self.conv(x, p + ".downsample.0", p + ".downsample.1", stride, 0, False)
                x = self.conv(t, p + ".conv2", p + ".bn2", 1, 1, True, residual=identity)
        return x

    def pre_activation_net(self, x):
        x = self.conv(x, "backbone.conv1", "backbone.bn1", 2, 2, True)
        x = F.max_pool2d(x, kernel_size=3, stride=2, padding=1)
        for li, nb in enumerate(wide_layers(self.sd)):
            for bi in range(nb):
                p = f"backbone.layer{li + 1}.{bi}"
                stride = 2 if (bi == 0 and li > 0) else 1
                a = self.pre_activation(x, p + ".bn1")
                res = x
                if (p + ".downsample.weight") in self.sd:
                    res = self.conv(a, p + ".downsample", None, stride, 0, False)
                y = self.conv(a, p + ".conv1", p + ".bn2", stride, 1, True)
                x = self.conv(y, p + ".conv2", None, 1, 1, False, residual=res)
        return x


@torch.no_grad()
def forward(sd: Dict[str, torch.Tensor], x: torch.Tensor, dtype: torch.dtype = torch.float16, exact: bool = True,
            check: bool = True):
    """x [n, C, h, w] (any float type, on the device to compute on) -> (out [n, out_dim] float64, Stats); Stats.pooled
    holds the pooled features [n, 512].  `exact=False` rounds nothing; `check=False` skips the exactness assertions."""
    plan = _Plan(sd, dtype, x.device, exact, check)
    x = plan.q(x.to(torch.float64))
    plan.stats = Stats()  # the input's rounding is not the network's
    x = plan.pre_activation_net(x) if is_wide(sd) else plan.post_activation(x)
    return plan.tail(x), plan.stats


def head(sd: Dict[str, torch.Tensor], pooled: torch.Tensor) -> torch.Tensor:
    """The engine's linear map (fp32 weights and bias) applied to pooled features [n, 512] in float64."""
    return _Plan(sd, torch.float16, pooled.device, True, False).linear(pooled)


def fp32_head_bound(sd: Dict[str, torch.Tensor], pooled: torch.Tensor) -> torch.Tensor:
    """Bound on |engine - oracle| for a head with real (non-dyadic) weights on exactly pooled features: the engine's dot
    product (avgpool_linear_kernel) is 16 fused multiply-adds per lane (512 / 32, each one rounding), a 5-level warp
    shuffle tree and the bias addition, at most 22 fp32 roundings on the way of any term: |err| <= gamma_22 * (sum_k
    |W_jk| |pooled_k| + |b_j|), gamma_n = n u / (1 - n u), u = 2^-24.  The oracle evaluates the same fp32 weights and
    pooled values in float64.  pooled: [n, 512] float64 -> [n, out_dim]."""
    plan = _Plan(sd, torch.float16, pooled.device, True, False)
    W, b = plan.head()
    u = 2.0 ** -24
    gamma = 22 * u / (1 - 22 * u)
    return gamma * (pooled.abs() @ W.abs().to(pooled.device).t() + b.abs().to(pooled.device))
