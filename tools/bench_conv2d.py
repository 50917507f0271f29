"""Micro-benchmark of the tensor-core conv kernel on the UNet 3x3 shapes (CUDA events).
usage: python tools/bench_conv2d.py [--C 32 --H 1024 --W 127 --B 8 --kind f|r]"""
import argparse, os, sys, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from gpu_util import conv_gemm
ap = argparse.ArgumentParser()
ap.add_argument("--C", type=int, default=32); ap.add_argument("--H", type=int, default=1024)
ap.add_argument("--W", type=int, default=127); ap.add_argument("--B", type=int, default=8)
ap.add_argument("--iters", type=int, default=3); ap.add_argument("--kind", default="both")
args = ap.parse_args()
dev = "cuda:0"; C, H, W, B = args.C, args.H, args.W, args.B
a = (torch.randn(B, H, W, C, device=dev) * 0.5).bfloat16()
w = (torch.randn(9, C, C, device=dev) * 0.05).bfloat16()
bias = torch.randn(C, device=dev); X = torch.randn(B, H, W, C, device=dev)
out_act = torch.empty(B, H, W, C, device=dev, dtype=torch.bfloat16)
taps = [(kh - 1, kw - 1) for kh in range(3) for kw in range(3)]
for kind in ("f", "r"):
    if args.kind not in ("both", kind): continue
    def run():
        if kind == "f":   # conv1 with folded BN: bias + act only
            conv_gemm(a, w, taps, bias=bias, want_raw=False, want_act=True, act="lrelu", act_param=0.01, precision="bf16", impl=1, out_act=out_act)
        else:             # conv2: residual + raw (+ fused next-BN operand)
            conv_gemm(a, w, taps, residual=X, want_raw=True, want_act=True, act="lrelu", act_param=0.01, precision="bf16", impl=1, out_raw=X, out_act=out_act)
    run(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.iters): run()
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.iters
    flops = 2.0 * 9 * C * C * H * W * B; byts = B * H * W * C * (4 if kind == "f" else 12)
    print(f"conv3x3 C={C} {H}x{W} B={B} {kind}: {ms:8.3f} ms {flops/ms/1e9:8.1f} TF/s {byts/ms/1e6:8.1f} GB/s (algorithmic)", flush=True)
