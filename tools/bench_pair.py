"""The fused ResStack pair (vfx_resstack_pair, resstack_pair.cu) at the restore step's shapes: B = 32 items of 10 s,
C = 64 at L = 443 646 rows and C = 128 at L = 147 882, every dilation of a stack (1, 3, ... 2187), every precision that
fuses them (tf32 C = 64 on the encoded stream; bf16 / fp16 at C = 64 and 128), with the outputs the step writes (x' as
the encoded stream or in place, and the next layer's operand).

From the shapes alone (--dry, no GPU): tiles of 126 output rows, HBM bytes (the operand read once, the fp32 residual
read in the 16-bit modes, x' written, the operand written), tensor FLOP (two k3 convolutions over 128 rows per tile,
halo included), and the least time each takes at the H100 SXM data-sheet rates (3.35 TB/s; 495 TFLOP/s tf32, 989
bf16 / fp16).  With a GPU: the time per pair by CUDA events over --iters launches after a warm-up, per tile and CTA
(time x CTAs / tiles, CTAs = min(tiles, SMs)), and the achieved share of each bound.
usage: python tools/bench_pair.py [--dry] [--iters 5] [--prec tf32,bf16,fp16]"""
import argparse
import ctypes
import os
import subprocess
import sys

ap = argparse.ArgumentParser()
ap.add_argument("--dry", action="store_true", help="print the counting model only (needs no GPU)")
ap.add_argument("--iters", type=int, default=5)
ap.add_argument("--prec", default="tf32,bf16,fp16")
ap.add_argument("--B", type=int, default=32)
ap.add_argument("--sms", type=int, default=132, help="SM count for --dry (read from the device otherwise)")
args = ap.parse_args()

HBM, TC = 3.35e12, {"tf32": 495e12, "bf16": 989e12, "fp16": 989e12}
ROWS = 126
SHAPES = [(64, 443646), (128, 147882)]
DILS = [3 ** i for i in range(8)]


def model(prec, C, L, B, sms):
    esz = 4 if prec == "tf32" else 2
    tiles = B * -(-L // ROWS)
    if prec == "tf32":      # the encoded stream: read once (operand and residual), S' written
        hbm = B * L * C * (4 + 4)
    else:                   # operand read, x read and written, next operand written
        hbm = B * L * C * (esz + 4 + 4 + esz)
    flop = tiles * 2 * (2 * 128 * C * 3 * C)
    return dict(tiles=tiles, ctas=min(tiles, sms), hbm=hbm, flop=flop, t_hbm=hbm / HBM, t_tc=flop / TC[prec])


if not args.dry:
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_pair: no CUDA device (use --dry for the counting model)")
    ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, ROOT)
    from voicefixer_b200 import _lib
    lib = _lib.load()
    p = torch.cuda.get_device_properties(0)
    args.sms = p.multi_processor_count
    try:
        info = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        info = f"nvidia-smi unavailable ({e})"
    print(f"# {p.name}, {args.sms} SMs; {info}; B = {args.B}", flush=True)

total = {}
for prec in args.prec.split(","):
    for C, L in SHAPES:
        if prec == "tf32" and C != 64:
            continue
        m = model(prec, C, L, args.B, args.sms)
        print(f"{prec} C={C} L={L}: {m['tiles']} tiles on {m['ctas']} CTAs, HBM {m['hbm'] / 1e9:.2f} GB ({m['t_hbm'] * 1e3:.2f} ms "
              f"at 3.35 TB/s), {m['flop'] / 1e12:.3f} TFLOP ({m['t_tc'] * 1e3:.2f} ms at {TC[prec] / 1e12:.0f} TFLOP/s)", flush=True)
        if args.dry:
            continue
        g = torch.Generator(device="cuda:0").manual_seed(C)
        dt = {"bf16": torch.bfloat16, "fp16": torch.float16}.get(prec, torch.float32)
        x = torch.randn(args.B, L, C, device="cuda:0", generator=g)
        w = (torch.randn(2, 3, C, C, device="cuda:0", generator=g) / (3 * C) ** 0.5).to(dt)
        bias = torch.randn(2, C, device="cuda:0", generator=g) * 0.1
        if prec == "tf32":
            s = torch.where(x > 0, x, x * 0.01).view(torch.int32).add_(0x1000).view(torch.float32)
            a, xs, out, act = s, s, torch.empty_like(s), torch.empty_like(s)
        else:
            a, xs, out, act = torch.where(x > 0, x, x * 0.01).to(dt), x, None, torch.empty(args.B, L, C, device="cuda:0", dtype=dt)
        del x
        st = torch.cuda.current_stream()
        group = 0.0
        for dil in DILS:
            d = _lib.PairDesc()
            d.a, d.x = a.data_ptr(), xs.data_ptr()
            d.w1, d.b1, d.dilation = w[0].data_ptr(), bias[0].data_ptr(), dil
            d.w2, d.b2 = w[1].data_ptr(), bias[1].data_ptr()
            d.B, d.L, d.C, d.write_raw = args.B, L, C, 1
            d.out_act, d.act, d.act_param = act.data_ptr(), _lib.ACT["lrelu"], 0.01
            d.precision = _lib.PREC[prec]
            if prec == "tf32":
                d.x_out, d.stream_enc, d.stream_enc_out = out.data_ptr(), 1, 1
            run = lambda: _lib.check(lib.vfx_resstack_pair(ctypes.byref(d), ctypes.c_void_p(st.cuda_stream)), "pair")
            run()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.iters):
                run()
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / args.iters
            group += ms
            print(f"    dil {dil:5d}: {ms:7.3f} ms  {ms * 1e3 * m['ctas'] / m['tiles']:6.2f} us per tile and CTA  "
                  f"HBM {m['hbm'] / ms / 1e9:5.2f} TB/s ({m['t_hbm'] * 1e3 / ms:.2f} of the bound)  "
                  f"tensor {m['flop'] / ms / 1e9:6.1f} TFLOP/s ({m['t_tc'] * 1e3 / ms:.2f})", flush=True)
        total[(prec, C)] = group
        print(f"    8 pairs: {group:.2f} ms", flush=True)
        del a, xs, out, act
        torch.cuda.empty_cache()
