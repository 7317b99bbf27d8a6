"""Per-layer table: every distinct convolution of the ResNet-34 coarse forward at batch 576, this library's wgmma
kernel next to stock torch / cuDNN on the same GPU (the vendor-library bar of SURVEY 8d).

    python tools/gpu_layer_table.py --out gpurun_out/layer_table.json [--batch 576] [--render-size 240x320]

torch side: F.conv2d + folded-BN bias + (residual) + ReLU as separate ops is what eager PyTorch runs, but to give cuDNN
its best case only the convolution itself is timed (bias / residual / ReLU / BN are free for it); the mpx side times the
whole fused layer (conv + bias + residual + ReLU + 16-bit store).  CUDA events, L2 flushed by size (the activation
tensors of every layer at batch 576 are as large as the 50 MB L2 or larger).  Also prints the whole-network forward of
both sides (workloads/torch_resnet.py vs ResNet34Engine)."""
import argparse
import json
import sys
from pathlib import Path

import torch
import torch.nn.functional as F

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from megapose6d_b200 import _abi  # noqa: E402
from megapose6d_b200.backbone import ResNet34Engine  # noqa: E402
from workloads import torch_resnet as T  # noqa: E402
from workloads import weights as W  # noqa: E402


def layers(h, w, c_in):
    """(name, count, H, W, C_in, C_out, R, stride, pad, residual) per distinct conv of the backbone."""
    hs, ws = h // 2, w // 2
    h1, w1 = (hs + 1) // 2, (ws + 1) // 2
    out = [("stem7x7s2", 1, h, w, c_in, 64, 7, 2, 3, False)]
    H, Wd, C = h1, w1, 64
    for li, (nb, width) in enumerate(zip([3, 4, 6, 3], [64, 128, 256, 512])):
        if li > 0:
            out.append((f"layer{li + 1}.0.conv1_s2", 1, H, Wd, C, width, 3, 2, 1, False))
            out.append((f"layer{li + 1}.0.downsample", 1, H, Wd, C, width, 1, 2, 0, False))
            H, Wd = (H + 1) // 2, (Wd + 1) // 2
            n_c1, n_c2 = nb - 1, nb
        else:
            n_c1, n_c2 = nb, nb
        out.append((f"layer{li + 1}.conv1", n_c1, H, Wd, width, width, 3, 1, 1, False))
        out.append((f"layer{li + 1}.conv2+res", n_c2, H, Wd, width, width, 3, 1, 1, True))
        C = width
    return out


def time_ms(fn, iters=10, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=576)
    ap.add_argument("--render-size", default="240x320")
    ap.add_argument("--out", type=Path, default=Path("gpurun_out/layer_table.json"))
    ap.add_argument("--mpx-only", action="store_true", help="skip the torch / cuDNN columns")
    ap.add_argument("--conv-modes", default="", help="comma-separated mpx_conv_set_mode values to time side by side")
    args = ap.parse_args()
    h, w = (int(v) for v in args.render_size.split("x"))
    n = args.batch
    lib = _abi.lib()
    act = _abi.act_dtype()
    torch.backends.cudnn.benchmark = True
    import os
    default_mode = int(os.environ.get("MPX_CONV_MODE", "60866571"))
    rows = []
    g = torch.Generator(device="cuda").manual_seed(0)
    for name, count, H, Wd, cin, cout, r, stride, pad, use_res in layers(h, w, 9):
        P, Q = (H + 2 * pad - r) // stride + 1, (Wd + 2 * pad - r) // stride + 1
        flops = 2.0 * n * P * Q * cout * r * r * cin
        rec = dict(layer=name, count=count, M=n * P * Q, N=cout, K=r * r * cin, gflop=flops / 1e9)
        x_nchw = torch.randn(n, cin, H, Wd, device="cuda", generator=g)
        wt = torch.randn(cout, cin, r, r, device="cuda", generator=g) / (r * r * cin) ** 0.5
        for prec, (dt, cl, tf32) in ({} if args.mpx_only else T.PRECISIONS).items():
            torch.backends.cudnn.allow_tf32 = tf32
            xx, ww = x_nchw.to(dt), wt.to(dt)
            if cl:
                xx, ww = xx.contiguous(memory_format=torch.channels_last), ww.contiguous(memory_format=torch.channels_last)
            ms = time_ms(lambda: F.conv2d(xx, ww, stride=stride, padding=pad))
            rec[f"torch_{prec}_ms"] = ms
            rec[f"torch_{prec}_tflops"] = flops / ms / 1e9
            del xx, ww
        # this library: the fused layer as the network runs it (the 7x7/s2 stem as 4x4/s1 over the space-to-depth input)
        if name.startswith("stem"):
            c_pad = 16
            xm = torch.randn(n, H // 2, Wd // 2, 4 * c_pad, device="cuda", generator=g).to(act)
            wm = (torch.randn(64, 16 * 4 * c_pad, device="cuda", generator=g) / 21.0).to(act)
            geom = (H // 2, Wd // 2, 4 * c_pad, 4, 4, 1, 2, 2, 1, 1)
            relu_flags = 3  # ReLU + "space-to-depth stem weights" (structurally zero slices are skipped, as in the network)
        else:
            xm = x_nchw.permute(0, 2, 3, 1).contiguous().to(act)
            wm = wt.permute(0, 2, 3, 1).reshape(cout, -1).contiguous().to(act)
            geom = (H, Wd, cin, r, r, stride, pad, pad, pad, pad)
            relu_flags = 1
        del x_nchw, wt
        bias = torch.randn(cout, device="cuda", generator=g)
        res = torch.randn(n, P, Q, cout, device="cuda", generator=g).to(act) if use_res else None
        out = torch.empty(n, P, Q, cout, device="cuda", dtype=act)
        hh, ww_, cc, rr, ss, st, p0, p1, p2, p3 = geom
        stream = _abi.stream_ptr()

        def run_mpx():
            _abi.check(lib.mpx_conv2d(_abi.ptr(xm), n, hh, ww_, cc, _abi.ptr(wm), _abi.ptr(bias), cout, rr, ss, st, p0, p1, p2, p3,
                                      relu_flags, _abi.ptr(res), _abi.ptr(out), 0, 0, stream))

        ms = time_ms(run_mpx)
        rec["mpx_ms"], rec["mpx_tflops"] = ms, flops / ms / 1e9
        for mode in [int(m) for m in args.conv_modes.split(",") if m]:
            lib.mpx_conv_set_mode(mode)
            rec[f"mpx_mode{mode}_ms"] = time_ms(run_mpx)
        lib.mpx_conv_set_mode(default_mode)
        if not args.mpx_only:
            best = min(rec[f"torch_{p}_ms"] for p in T.PRECISIONS)
            rec["speedup_vs_best_torch"] = best / ms
            rec["speedup_vs_torch_fp32_strict"] = rec["torch_fp32_strict_ms"] / ms
        rows.append(rec)
        print(json.dumps(rec), flush=True)
        del xm, wm, out, res
        torch.cuda.empty_cache()
    # whole network forward at this batch
    sd = W.make_state_dict(W.COARSE_CFG, 1)
    net = {} if args.mpx_only else {p: T.time_forward(sd, n, h, w, p) for p in T.PRECISIONS}
    eng = ResNet34Engine(sd, n_inputs=9, head="views_logits_head")
    x = eng.alloc_input(n, h, w)
    x.copy_(torch.rand(x.shape, device="cuda").to(act))
    net["mpx"] = time_ms(lambda: eng.forward(x, h, w), iters=5)
    total = dict(batch=n, render_size=[h, w], whole_network_forward_ms=net,
                 sum_of_layers_ms={k: sum(r[k] * r["count"] for r in rows) for k in rows[0] if k.endswith("_ms")})
    print(json.dumps(total), flush=True)
    args.out.parent.mkdir(parents=True, exist_ok=True)
    args.out.write_text(json.dumps(dict(rows=rows, total=total), indent=1))


if __name__ == "__main__":
    main()
