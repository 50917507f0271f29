"""Operand feed of the tensor-core convolution (conv_gemm_tc.cu): a counting model and, on a GPU, what it comes to.

From the shapes alone (--dry, no GPU): the kernel's tiling (BN, the TMA tile box, tiles, K slices per tile), the bytes it
brings from L2 into shared memory (per K slice one A box of 128 rows x 128 bytes, fewer rows where the tile box
holds fewer, and one BN x 128-byte weight box; whole boxes, zero fill included), and the FLOP the tensor cores execute per slice (2 * 128 * BN * channels per
slice, padding included).  With a GPU: the kernel time by CUDA events, and from it the L2 -> shared-memory rate, the
executed TFLOP/s and the time one CTA spends per slice (time * CTAs / slices; the CTAs are min(tiles, SMs)).
Each shape is timed twice: with a light epilogue (raw output only) and with the restore step's (bias, an fp32 residual,
raw output and the activated operand for the next layer); the difference, per tile and CTA, is what the epilogue costs.
The ResStack C = 128 shape is also timed as the tf32 step runs its second convolution: the encoded stream read as the
residual and overwritten in place.
Shapes: the four ResStack widths, the UNet's 32- and 64-channel 3x3 on 127 bins, one up-sampler phase group.
usage: python tools/bench_conv_feed.py [--dry] [--prec tf32|bf16|fp16] [--B 8] [--iters 5]"""
import argparse, os, sys

ap = argparse.ArgumentParser()
ap.add_argument("--dry", action="store_true", help="print the counting model only (needs no GPU)")
ap.add_argument("--prec", default="tf32", choices=["tf32", "bf16", "fp16"])
ap.add_argument("--B", type=int, default=8)
ap.add_argument("--iters", type=int, default=5)
ap.add_argument("--sms", type=int, default=132, help="SM count for --dry (read from the device otherwise)")
args = ap.parse_args()

ESZ = 4 if args.prec == "tf32" else 2
BK = 128 // ESZ
# name, H, W, Cin, N, taps [(dh, dw)], first weight offsets in [N][Cin] matrices (None: tap t is matrix t)
SHAPES = [(f"resstack C={C}", 1, L, C, C, [(0, -3), (0, 0), (0, 3)], None)
          for C, L in ((512, 7042), (256, 49294), (128, 147882), (64, 443646))]
TAPS9 = [(kh - 1, kw - 1) for kh in range(3) for kw in range(3)]
SHAPES += [("unet 3x3 C=32", 1024, 127, 32, 32, TAPS9, None), ("unet 3x3 C=64", 512, 63, 64, 64, TAPS9, None),
           # ConvTranspose1d(512 -> 256, k = 14, stride 7), phase group 0: 3 phases, taps at matrices 4 and 11 of 14
           ("up-sampler 512->256 u=7 grp 0", 1, 7042, 512, 3 * 256, [(0, 0), (0, -1)], [4, 11])]


def model(B, H, W, Cin, N, taps, sms):
    bn = 32 if N <= 32 else 64 if N <= 64 else 128
    tw = min(W, 128)
    th = 1 if tw < W else min(H, 128 // tw)
    tb = 1 if (th < H or tw < W) else min(B, 128 // (tw * th))
    mtiles = -(-W // tw) * -(-H // th) * -(-B // tb)
    tiles = mtiles * -(-N // bn)
    slices = len(taps) * -(-Cin // BK)
    rows = tw * th * tb                     # of the 128 rows of a tile; the others are not loaded
    stage = rows * 128 + bn * 128
    return dict(bn=bn, box=(tw, th, tb), tiles=tiles, ctas=min(tiles, sms), slices=slices, tile_bytes=slices * stage,
                bytes=tiles * slices * stage, a_bytes=tiles * slices * rows * 128, slice_flop=2 * 128 * bn * BK,
                flop=tiles * slices * 2 * 128 * bn * BK, useful_flop=2 * B * H * W * N * Cin * len(taps))


if not args.dry:
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_conv_feed: no CUDA device (use --dry for the counting model)")
    ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
    from gpu_util import conv_gemm
    p = torch.cuda.get_device_properties(0)
    args.sms = p.multi_processor_count
    print(f"# {p.name}, {args.sms} SMs, {args.prec}, B = {args.B}")

for name, H, W, Cin, N, taps, mats in SHAPES:
    m = model(args.B, H, W, Cin, N, taps, args.sms)
    print(f"{name}: BN {m['bn']} box {m['box']} tiles {m['tiles']} slices/tile {m['slices']}  L2->smem {m['tile_bytes'] / 1024:.0f} KB/tile "
          f"{m['bytes'] / 1e9:.2f} GB/launch (A {m['a_bytes'] / 1e9:.2f})  {m['slice_flop'] / 1e6:.2f} MFLOP/slice "
          f"{m['flop'] / 1e12:.3f} TFLOP/launch executed ({m['useful_flop'] / 1e12:.3f} useful)", flush=True)
    if args.dry:
        continue
    odt = {"bf16": torch.bfloat16, "fp16": torch.float16}.get(args.prec, torch.float32)
    a = (torch.randn(args.B, H, W, Cin, device="cuda:0") * 0.5).to(odt)
    nmat = max(mats) + 1 if mats else len(taps)
    w = (torch.randn(nmat, N, Cin, device="cuda:0") * 0.05).to(odt)
    w_off = [i * N * Cin for i in mats] if mats else None
    raw = torch.empty(args.B, H, W, N, device="cuda:0")
    bias = torch.randn(N, device="cuda:0") * 0.1
    res = torch.randn(args.B, H, W, N, device="cuda:0")
    act = torch.empty(args.B, H, W, N, device="cuda:0", dtype=odt)
    runs = [("light", lambda: conv_gemm(a, w, taps, N=N, w_off=w_off, precision=args.prec, impl=1, out_raw=raw)),
            ("step", lambda: conv_gemm(a, w, taps, N=N, w_off=w_off, precision=args.prec, impl=1, out_raw=raw, bias=bias,
                                       residual=res, want_act=True, out_act=act, act="lrelu", act_param=0.01))]
    if name == "resstack C=128":
        enc = res.clone()
        runs.append(("step, encoded stream in place",
                     lambda: conv_gemm(a, w, taps, N=N, w_off=w_off, precision=args.prec, impl=1, out_raw=enc, bias=bias,
                                       residual=enc, res_enc=1, raw_enc=1, enc_slope=0.01, want_act=True, out_act=act,
                                       act="lrelu", act_param=0.01)))
    light = None
    for label, run in runs:
        run()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            run()
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.iters
        per_slice = ms * 1e3 * m['ctas'] / (m['tiles'] * m['slices'])
        extra = "" if light is None else f"  epilogue {(per_slice - light) * m['slices']:6.2f} us per tile per CTA over light"
        light = per_slice if light is None else light
        print(f"    {label:30s} {ms:8.3f} ms  L2->smem {m['bytes'] / ms / 1e9:6.2f} TB/s  executed {m['flop'] / ms / 1e9:6.1f} TFLOP/s  "
              f"{per_slice:6.3f} us per slice per CTA{extra}", flush=True)
