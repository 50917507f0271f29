"""Micro-benchmark of the conv-GEMM kernels on the vocoder ResStack shapes (CUDA events).
usage: python tools/bench_conv.py [--only C] [--B 8] [--iters 5] [--impl 1]"""
import argparse, os, sys, ctypes
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from gpu_util import conv_gemm

ap = argparse.ArgumentParser()
ap.add_argument("--only", type=int, default=0)
ap.add_argument("--B", type=int, default=8)
ap.add_argument("--iters", type=int, default=5)
ap.add_argument("--impl", type=int, default=1)
ap.add_argument("--kind", default="both")
ap.add_argument("--taps", type=int, default=3)
ap.add_argument("--dil", type=int, default=3)
ap.add_argument("--prec", default="bf16")
args = ap.parse_args()
dev = "cuda:0"
shapes = [(512, 7042), (256, 49294), (128, 147882), (64, 443646)]
for C, L in shapes:
    if args.only and C != args.only:
        continue
    B = args.B
    odt = {"bf16": torch.bfloat16, "fp16": torch.float16}.get(args.prec, torch.float32)   # tf32: fp32 storage
    a = (torch.randn(B, 1, L, C, device=dev) * 0.5).to(odt)
    w = (torch.randn(3, C, C, device=dev) * 0.05).to(odt)
    bias = torch.randn(C, device=dev)
    X = torch.randn(B, 1, L, C, device=dev)
    out_act = torch.empty(B, 1, L, C, device=dev, dtype=odt)
    for kind in ("c1", "c2", "c2enc", "raw", "rawact", "actnone"):
        if args.kind == "pairenc":
            if kind not in ("c1", "c2enc"):
                continue
        elif (args.kind == "both" and kind not in ("c1", "c2")) or args.kind not in ("both", "all", kind):
            continue
        def run():
            taps1 = [(0, -args.dil), (0, 0), (0, args.dil)][:args.taps] if args.taps < 3 else [(0, -args.dil), (0, 0), (0, args.dil)]
            if kind == "c1":
                conv_gemm(a, w, taps1, bias=bias, want_raw=False, want_act=True, act="lrelu",
                          act_param=0.01, precision=args.prec, impl=args.impl, out_act=out_act)
            elif kind == "c2":
                conv_gemm(a, w, [(0, -1), (0, 0), (0, 1)], bias=bias, residual=X, want_raw=True, want_act=True,
                          act="lrelu", act_param=0.01, precision=args.prec, impl=args.impl, out_raw=X, out_act=out_act)
            elif kind == "c2enc":     # tf32 encoded stream: residual decoded, result encoded in place, no separate operand copy
                conv_gemm(a, w, [(0, -1), (0, 0), (0, 1)], bias=bias, residual=X, want_raw=True, want_act=False,
                          precision=args.prec, impl=args.impl, out_raw=X, res_enc=1, raw_enc=1, enc_slope=0.01)
            elif kind == "raw":
                conv_gemm(a, w, taps1, bias=bias, want_raw=True, want_act=False, precision=args.prec, impl=args.impl, out_raw=X)
            elif kind == "rawact":
                conv_gemm(a, w, taps1, bias=bias, want_raw=True, want_act=True, act="lrelu", act_param=0.01,
                          precision=args.prec, impl=args.impl, out_raw=X, out_act=out_act)
            elif kind == "actnone":
                conv_gemm(a, w, taps1, bias=bias, want_raw=False, want_act=True, act="none", precision=args.prec,
                          impl=args.impl, out_act=out_act)
        run()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            run()
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.iters
        flops = 2.0 * 3 * C * C * L * B
        e = 2 if odt != torch.float32 else 4
        byts = B * L * C * {"c1": 2 * e, "c2": 2 * e + 8, "c2enc": e + 8, "raw": e + 4, "rawact": 2 * e + 4, "actnone": 2 * e}[kind]
        print(f"C={C:4d} L={L:7d} B={B} {kind}: {ms:8.3f} ms  {flops/ms/1e9:8.1f} TF/s  {byts/ms/1e6:8.1f} GB/s (algorithmic)", flush=True)
