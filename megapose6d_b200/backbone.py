"""ResNet-34 backbone + head as a libmpx network handle.

Takes the parameters of the reference's `vanilla_resnet34` backbone
(src/megapose/models/torchvision_resnet.py:181-316, created by
training/pose_models_cfg.py:106-109 with `num_classes=512, n_input_channels=C`) and of the head
(`pose_fc` or `views_logits_head`, models/pose_rigid.py:120-130) in the reference's state-dict
layout and repacks them once for the wgmma kernels:
  * eval-mode BatchNorm folded into the preceding conv (w' = w*g/sqrt(var+eps), b' = beta - mean*g/sqrt(var+eps));
  * conv weights OIHW fp32 -> [C_out, R*S*C_in] in the library's 16-bit type (`_abi.act_dtype()`: fp16 unless the
    library was built for bf16), K ordered (r, s, c);
  * the 7x7/s2 stem rewritten as a 4x4/s1 conv over the space-to-depth input (channels padded to
    c_pad = a multiple of 16 (16 | 32 for the released models), four sub-pixels -> 4 * c_pad input channels);
  * avgpool -> fc(512x512) -> head(512 x 1|9) folded into one linear map (there is no
    non-linearity between fc and the head, models/pose_rigid.py:323-334).
"""
from __future__ import annotations

import ctypes
from typing import Dict, List, Optional, Tuple

import torch

from . import _abi

LAYERS = [3, 4, 6, 3]
BN_EPS = 1e-5


def _fold(sd: Dict[str, torch.Tensor], conv: str, bn: str) -> Tuple[torch.Tensor, torch.Tensor]:
    w = sd[conv + ".weight"].detach().double().cpu()
    g = sd[bn + ".weight"].detach().double().cpu()
    beta = sd[bn + ".bias"].detach().double().cpu()
    mean = sd[bn + ".running_mean"].detach().double().cpu()
    var = sd[bn + ".running_var"].detach().double().cpu()
    scale = g / torch.sqrt(var + BN_EPS)
    return w * scale.view(-1, 1, 1, 1), beta - mean * scale


def _pack(w: torch.Tensor) -> torch.Tensor:
    """[co, ci, r, s] -> [co, r*s*ci] with k = (r, s, c)."""
    co = w.shape[0]
    return w.permute(0, 2, 3, 1).reshape(co, -1).contiguous()


def _stem_s2d(w: torch.Tensor, c_pad: int) -> torch.Tensor:
    """7x7/s2/p3 weights [64, C, 7, 7] -> 4x4/s1 (pad 2 low, 1 high) weights over the s2d input:
    w2[co, by, bx, (dy*2+dx)*c_pad + c] = w[co, c, 2*by+dy-1, 2*bx+dx-1] (zero outside 0..6)."""
    co, c, _, _ = w.shape
    w2 = torch.zeros(co, 4, 4, 4 * c_pad, dtype=w.dtype)
    for by in range(4):
        for dy in range(2):
            kh = 2 * by + dy - 1
            if not 0 <= kh <= 6:
                continue
            for bx in range(4):
                for dx in range(2):
                    kw = 2 * bx + dx - 1
                    if not 0 <= kw <= 6:
                        continue
                    base = (dy * 2 + dx) * c_pad
                    w2[:, by, bx, base:base + c] = w[:, :, kh, kw]
    return w2.reshape(co, -1).contiguous()


def _stem_s2d_5x5(w: torch.Tensor, c_pad: int) -> torch.Tensor:
    """5x5/s2/p2 weights [64, C, 5, 5] (WideResNet stem, models/wide_resnet.py:66-68) -> 3x3/s1/p1 weights over the s2d
    input: w2[co, by+1, bx+1, (dy*2+dx)*c_pad + c] = w[co, c, 2*by+dy+2, 2*bx+dx+2] for by, bx in {-1, 0, 1} (zero outside
    0..4)."""
    co, c, _, _ = w.shape
    w2 = torch.zeros(co, 3, 3, 4 * c_pad, dtype=w.dtype)
    for by in (-1, 0, 1):
        for dy in range(2):
            kh = 2 * by + dy + 2
            if not 0 <= kh <= 4:
                continue
            for bx in (-1, 0, 1):
                for dx in range(2):
                    kw = 2 * bx + dx + 2
                    if not 0 <= kw <= 4:
                        continue
                    base = (dy * 2 + dx) * c_pad
                    w2[:, by + 1, bx + 1, base:base + c] = w[:, :, kh, kw]
    return w2.reshape(co, -1).contiguous()


def is_wide_resnet(sd: Dict[str, torch.Tensor]) -> bool:
    """Checkpoint of a WideResNet backbone (backbone_str "resnet34" / "resnet18", models/wide_resnet.py): pre-activation
    blocks with their own bn1, no fc layer."""
    return "backbone.layer1.0.bn1.weight" in sd and "backbone.fc.weight" not in sd


class ResNet34Engine:
    """Owns the repacked device weights and the mpx_net handle; `forward(x)` runs the whole network.  Serves both backbone
    families of training/pose_models_cfg.py:106-116: `vanilla_resnet34` (all released models) and the pre-activation
    WideResNet34 / WideResNet18 of width 1."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], n_inputs: int, head: str, device="cuda"):
        sd = state_dict
        self.n_inputs = n_inputs
        self.n_features = 512
        if is_wide_resnet(sd):
            self._init_wide(sd, n_inputs, head, device)
            return
        self.c_pad = 16 * ((n_inputs + 15) // 16)  # 16 (coarse), 32 (refiner) for the released models
        assert n_inputs <= 256, f"n_inputs={n_inputs} > 256 is not supported"
        assert sd["backbone.conv1.weight"].shape[1] == n_inputs, "checkpoint / config channel mismatch"
        self.device = torch.device(device)
        self.act_dtype = _abi.act_dtype()
        self._weights: List[torch.Tensor] = []
        self._biases: List[torch.Tensor] = []

        def add(wmat: torch.Tensor, bias: torch.Tensor) -> None:
            self._weights.append(wmat.to(torch.float32).to(self.device).to(self.act_dtype).contiguous())
            self._biases.append(bias.to(torch.float32).to(self.device).contiguous())

        w, b = _fold(sd, "backbone.conv1", "backbone.bn1")
        add(_stem_s2d(w, self.c_pad), b)
        for li, nb in enumerate(LAYERS):
            for bi in range(nb):
                p = f"backbone.layer{li + 1}.{bi}"
                w, b = _fold(sd, p + ".conv1", p + ".bn1")
                add(_pack(w), b)
                w, b = _fold(sd, p + ".conv2", p + ".bn2")
                add(_pack(w), b)
                if (p + ".downsample.0.weight") in sd:
                    w, b = _fold(sd, p + ".downsample.0", p + ".downsample.1")
                    add(_pack(w), b)
        Wh, bh = sd[head + ".weight"].detach().double().cpu(), sd[head + ".bias"].detach().double().cpu()
        Wf, bf = sd["backbone.fc.weight"].detach().double().cpu(), sd["backbone.fc.bias"].detach().double().cpu()
        self.out_dim = Wh.shape[0]
        self.head_w = (Wh @ Wf).float().to(self.device).contiguous()
        self.head_b = (Wh @ bf + bh).float().to(self.device).contiguous()

        n = len(self._weights)
        wp = (ctypes.c_void_p * n)(*[t.data_ptr() for t in self._weights])
        bp = (ctypes.c_void_p * n)(*[t.data_ptr() for t in self._biases])
        handle = ctypes.c_void_p()
        _abi.check(_abi.lib().mpx_net_create(self.c_pad, self.out_dim, wp, bp, n, _abi.ptr(self.head_w),
                                             _abi.ptr(self.head_b), ctypes.byref(handle)))
        self._handle = handle
        self._workspace: Optional[torch.Tensor] = None
        # workspaces that were outgrown: CUDA graphs captured by the callers (PosePredictor._iterate_graphed,
        # PoseEstimator._coarse_stage_graphed) have their addresses baked in, so they are kept alive, never freed;
        # growth is geometric, the retired ones therefore sum to less than the live one
        self._retired_workspaces: List[torch.Tensor] = []
        self._out_cache: Dict[int, torch.Tensor] = {}

    def _init_wide(self, sd, n_inputs, head, device) -> None:
        self.c_pad = 16 * ((n_inputs + 15) // 16)
        assert n_inputs <= 256 and sd["backbone.conv1.weight"].shape[1] == n_inputs, "checkpoint / config channel mismatch"
        assert sd["backbone.conv1.weight"].shape[0] == 64, "WideResNet width != 1 is not supported (C_out <= 512)"
        self.device = torch.device(device)
        self.act_dtype = _abi.act_dtype()
        self._weights, self._biases, self._affines = [], [], []

        def add(wmat, bias):
            self._weights.append(wmat.to(torch.float32).to(self.device).to(self.act_dtype).contiguous())
            self._biases.append(bias.to(torch.float32).to(self.device).contiguous())

        w, b = _fold(sd, "backbone.conv1", "backbone.bn1")
        add(_stem_s2d_5x5(w, self.c_pad), b)
        layers = []
        for li in range(4):
            nb = 0
            while f"backbone.layer{li + 1}.{nb}.conv1.weight" in sd:
                p = f"backbone.layer{li + 1}.{nb}"
                g, beta = sd[p + ".bn1.weight"].double().cpu(), sd[p + ".bn1.bias"].double().cpu()
                mean, var = sd[p + ".bn1.running_mean"].double().cpu(), sd[p + ".bn1.running_var"].double().cpu()
                scale = g / torch.sqrt(var + BN_EPS)
                self._affines.append(torch.stack((scale, beta - mean * scale)).float().to(self.device).contiguous())
                w, b = _fold(sd, p + ".conv1", p + ".bn2")
                add(_pack(w), b)
                w2 = sd[p + ".conv2.weight"].detach().double().cpu()
                add(_pack(w2), torch.zeros(w2.shape[0], dtype=torch.float64))
                if (p + ".downsample.weight") in sd:
                    wd = sd[p + ".downsample.weight"].detach().double().cpu()
                    add(_pack(wd), torch.zeros(wd.shape[0], dtype=torch.float64))
                nb += 1
            layers.append(nb)
        self.head_w = sd[head + ".weight"].detach().float().to(self.device).contiguous()
        self.head_b = sd[head + ".bias"].detach().float().to(self.device).contiguous()
        self.out_dim = self.head_w.shape[0]
        assert self.head_w.shape[1] == 512
        n = len(self._weights)
        wp = (ctypes.c_void_p * n)(*[t.data_ptr() for t in self._weights])
        bp = (ctypes.c_void_p * n)(*[t.data_ptr() for t in self._biases])
        ap = (ctypes.c_void_p * len(self._affines))(*[t.data_ptr() for t in self._affines])
        lb = (ctypes.c_int32 * 4)(*layers)
        handle = ctypes.c_void_p()
        _abi.check(_abi.lib().mpx_net_create_preact(self.c_pad, self.out_dim, lb, wp, bp, n, ap, len(self._affines),
                                                    _abi.ptr(self.head_w), _abi.ptr(self.head_b), ctypes.byref(handle)))
        self._handle = handle
        self._workspace = None
        self._retired_workspaces = []
        self._out_cache = {}

    def __del__(self):
        try:
            if getattr(self, "_handle", None) is not None:
                _abi.lib().mpx_net_destroy(self._handle)
        except Exception:  # noqa: BLE001
            pass

    def alloc_input(self, n: int, h: int, w: int) -> torch.Tensor:
        """Zero-initialised network input tensor [n, h/2, w/2, 4*c_pad] fp16|bf16 (pad channels stay 0)."""
        return torch.zeros(n, h // 2, w // 2, 4 * self.c_pad, device=self.device, dtype=self.act_dtype)

    def pack_input(self, x_nchw: torch.Tensor) -> torch.Tensor:
        """[n, C, h, w] float -> space-to-depth 16-bit input (for tests and the non-fused API path)."""
        n, c, h, w = x_nchw.shape
        assert c == self.n_inputs
        x = torch.zeros(n, self.c_pad, h, w, device=self.device, dtype=torch.float32)
        x[:, :c] = x_nchw.to(self.device).float()
        x = x.view(n, self.c_pad, h // 2, 2, w // 2, 2).permute(0, 2, 4, 3, 5, 1)  # n, h/2, w/2, dy, dx, c
        return x.reshape(n, h // 2, w // 2, 4 * self.c_pad).clamp(-65504.0, 65504.0).to(self.act_dtype).contiguous()

    def forward(self, x: torch.Tensor, h: int, w: int) -> torch.Tensor:
        """x: network input tensor for n samples of size h x w -> [n, out_dim] float32."""
        n = x.shape[0]
        assert x.dtype == self.act_dtype and x.is_contiguous() and x.shape == (n, h // 2, w // 2, 4 * self.c_pad)
        need = _abi.lib().mpx_net_workspace_bytes(self._handle, n, h, w)
        if self._workspace is None or self._workspace.numel() < need:
            if self._workspace is not None:
                self._retired_workspaces.append(self._workspace)
                need = max(need, 2 * self._workspace.numel())
            self._workspace = torch.empty(need, dtype=torch.uint8, device=self.device)
        # persistent output buffer per batch size: (x, out, workspace, shape) identify the cached CUDA graph
        out = self._out_cache.get(n)
        if out is None:
            out = self._out_cache[n] = torch.empty(n, self.out_dim, device=self.device, dtype=torch.float32)
        _abi.check(_abi.lib().mpx_net_forward(self._handle, _abi.ptr(x), n, h, w, _abi.ptr(out),
                                              _abi.ptr(self._workspace), self._workspace.numel(), _abi.stream_ptr()))
        return out.clone()

    def __call__(self, x_nchw: torch.Tensor) -> torch.Tensor:
        n, c, h, w = x_nchw.shape
        return self.forward(self.pack_input(x_nchw), h, w)
