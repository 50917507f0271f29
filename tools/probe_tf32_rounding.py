"""What does wgmma tf32 do with fp32 operand bits below the tf32 mantissa?  Runs the tensor-core conv kernel (1 tap,
C = 64) on UN-rounded fp32 operands and compares with fp32 references computed from (a) truncated, (b) round-to-nearest
tf32 operands.  The engine relies on the answer (operands are pre-rounded by their producers so that either way is exact)."""
import os, sys, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from gpu_util import conv_gemm
from voicefixer_b200.weights import round_tf32

torch.backends.cuda.matmul.allow_tf32 = False
g = torch.Generator().manual_seed(0)
B, L, C = 1, 4096, 64
x = torch.randn(B, 1, L, C, generator=g).cuda()
w = (torch.randn(1, C, C, generator=g) * 0.1).cuda()


def trunc(t):
    return (t.contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)


raw, _ = conv_gemm(x, w, [(0, 0)], precision="tf32", impl=1)
got = raw[0, 0].double()
for name, f in (("truncate", trunc), ("round-to-nearest", lambda t: round_tf32(t.cpu()).cuda())):
    ref = f(x)[0, 0].double() @ f(w)[0].double().t()
    err = float(((got - ref) ** 2).mean().sqrt() / (ref ** 2).mean().sqrt())
    print(f"wgmma tf32 on raw fp32 operands vs {name:17s} reference: rel-rms {err:.3e}")
