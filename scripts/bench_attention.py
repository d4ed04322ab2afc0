"""Micro-benchmark of the fused attention kernel alone: `python scripts/bench_attention.py`.  The shape comes from
the environment: B frames (default 8), H heads (default 6) and N tokens (default 3137), so the defaults are ViT-S/8
@448 and `B=128 H=12 N=4097` is the c5 shape (ViT-B/8, 64x64 tokens).  Prints accuracy vs fp32 torch and TFLOP/s
(algorithmic 4*N^2*64 per (frame, head))."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from wild_visual_navigation_b200 import ops  # noqa: E402

B, H, N = int(os.environ.get("B", 8)), int(os.environ.get("H", 6)), int(os.environ.get("N", 3137))
npad = (N + 127) // 128 * 128
g = torch.Generator(device="cuda").manual_seed(0)
S = float(os.environ.get("QK_STD", 1.2))   # std of q and k: the logits have std S^2 (1.2: bland; 1.8: the bench ViT's spread)
q = (torch.randn(B, H, npad, 64, device="cuda", generator=g) * S).bfloat16()
k = (torch.randn(B, H, npad, 64, device="cuda", generator=g) * S).bfloat16()
v = torch.randn(B, H, npad, 64, device="cuda", generator=g).bfloat16()
vt = v.transpose(2, 3).contiguous()
out = ops.attention(q, k, vt, N, 0.125)
torch.cuda.synchronize()
# accuracy on one (b, h)
att = torch.softmax(q[0, 0].float() @ k[0, 0, :N].float().T * 0.125, dim=-1)
ref = att @ v[0, 0, :N].float()
got = out[0, :, :64].float()
rel = ((got[:N] - ref[:N]).norm() / ref[:N].norm()).item()
for _ in range(3):
    ops.attention(q, k, vt, N, 0.125)
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
iters = 20
torch.cuda.synchronize()
e0.record()
for _ in range(iters):
    ops.attention(q, k, vt, N, 0.125)
e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / iters
tf = 4.0 * N * N * 64 * B * H / (ms * 1e-3) / 1e12
print(f"B={B} H={H} N={N} ms={ms:.3f} TFLOP/s={tf:.1f} rel_l2={rel:.2e}")
