"""The reference's network through stock PyTorch (cuDNN / cuBLAS) -- the vendor-library bar of SURVEY 8(d).

`TorchResNet34` is `resnet34(num_classes=512, n_input_channels=C)` + the single linear head
(models/torchvision_resnet.py:181-316, models/pose_rigid.py:120-130, 314-334) as a plain nn.Module loaded from a
reference-format state dict.  Measurement aid for bench.py / tools/gpu_layer_table.py only: nothing in the product
package imports it.
"""
from __future__ import annotations

from typing import Dict, List

import torch
from torch import nn

LAYERS = [3, 4, 6, 3]
WIDTHS = [64, 128, 256, 512]


class _Block(nn.Module):
    def __init__(self, cin, cout, stride):
        super().__init__()
        self.conv1 = nn.Conv2d(cin, cout, 3, stride, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(cout)
        self.conv2 = nn.Conv2d(cout, cout, 3, 1, 1, bias=False)
        self.bn2 = nn.BatchNorm2d(cout)
        self.downsample = None
        if stride != 1 or cin != cout:
            self.downsample = nn.Sequential(nn.Conv2d(cin, cout, 1, stride, bias=False), nn.BatchNorm2d(cout))

    def forward(self, x):
        idt = x if self.downsample is None else self.downsample(x)
        out = torch.relu(self.bn1(self.conv1(x)))
        out = self.bn2(self.conv2(out))
        return torch.relu(out + idt)


class _Backbone(nn.Module):
    def __init__(self, c_in):
        super().__init__()
        self.conv1 = nn.Conv2d(c_in, 64, 7, 2, 3, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        self.maxpool = nn.MaxPool2d(3, 2, 1)
        cin = 64
        for li, (nb, width) in enumerate(zip(LAYERS, WIDTHS)):
            blocks: List[nn.Module] = []
            for b in range(nb):
                blocks.append(_Block(cin, width, 2 if (b == 0 and li > 0) else 1))
                cin = width
            setattr(self, f"layer{li + 1}", nn.Sequential(*blocks))
        self.avgpool = nn.AdaptiveAvgPool2d((1, 1))
        self.fc = nn.Linear(512, 512)

    def forward(self, x):
        x = self.maxpool(torch.relu(self.bn1(self.conv1(x))))
        x = self.layer4(self.layer3(self.layer2(self.layer1(x))))
        return self.fc(torch.flatten(self.avgpool(x), 1))


class TorchResNet34(nn.Module):
    def __init__(self, state_dict: Dict[str, torch.Tensor]):
        super().__init__()
        head = "pose_fc" if "pose_fc.weight" in state_dict else "views_logits_head"
        self.backbone = _Backbone(state_dict["backbone.conv1.weight"].shape[1])
        setattr(self, head, nn.Linear(512, state_dict[head + ".weight"].shape[0]))
        self._head = head
        self.load_state_dict(state_dict)
        self.eval()

    def forward(self, x):
        return getattr(self, self._head)(self.backbone(x))


PRECISIONS = {
    # name -> (dtype, channels_last, allow_tf32)
    "fp32_strict": (torch.float32, False, False),       # what the oracle computes (TF32 off)
    "fp32_tf32": (torch.float32, False, True),          # what the reference's pinned torch 1.11 ran on Ampere by default
    "bf16_channels_last": (torch.bfloat16, True, True),
    "fp16_channels_last": (torch.float16, True, True),  # this engine's number format through cuDNN
}


@torch.no_grad()
def time_forward(sd: Dict[str, torch.Tensor], n: int, h: int, w: int, precision: str, iters: int = 5, warmup: int = 3,
                 chunk: int = 0, graph: bool = False) -> float:
    """Milliseconds per forward of n samples (CUDA events, cudnn.benchmark on); `chunk` > 0 splits the batch like the
    reference's bsz_images loop (inference/pose_estimator.py:362-364); `graph` replays a CUDA graph (small batches)."""
    dtype, cl, tf32 = PRECISIONS[precision]
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.benchmark)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = tf32
    torch.backends.cudnn.benchmark = True
    try:
        net = TorchResNet34(sd).cuda().to(dtype)
        c = sd["backbone.conv1.weight"].shape[1]
        x = torch.rand(n, c, h, w, device="cuda").to(dtype)
        if cl:
            net = net.to(memory_format=torch.channels_last)
            x = x.contiguous(memory_format=torch.channels_last)
        chunks = [x] if chunk <= 0 or chunk >= n else list(x.split(chunk))

        def run():
            return [net(xc) for xc in chunks]

        for _ in range(warmup):
            run()
        torch.cuda.synchronize()
        if graph:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                run()
            run = g.replay
            run()
            torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            run()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.benchmark = old
