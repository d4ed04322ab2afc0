"""Timing of the LinearRnvp anomaly-detection learner on the GPU (CUDA events): the fp32 train step at R labelled rows
(latency-bound: reported in microseconds per step) and the fp32 row forward (rows/s and achieved TFLOP/s from the
shape-derived count of 4 nets x 2 x (D h + h h + h D) FLOP per row).  Prints the card name and power limit with the
numbers.  Per pixel: frames/s of the anomaly map at B = 32, 448 x 448 from ViT-S/8 tokens (56 x 56 x 384), and of the ViT
forward followed by the map, with TFLOP/s from the dense shape count of the padded GEMMs the path runs."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                            text=True, timeout=10).stdout.strip().splitlines()[0]
    except Exception:
        pl = "unknown"
    return name, pl


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters * 1e3   # us per call


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dim", type=int, default=384)
    ap.add_argument("--hidden", type=int, default=200)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    from wild_visual_navigation_b200 import LinearRnvp, ops

    torch.manual_seed(42)
    m = LinearRnvp(args.dim, [args.hidden], use_permutation=True).cuda()
    D, h = args.dim, args.hidden
    flop_row = 4 * 2 * (D * h + h * h + h * D)
    name, pl = card()
    out = {"card": name, "power_limit": pl, "dim": D, "hidden": h, "train_step_us": {}, "rows_forward": {}}
    tr = ops.FlowTrainer(m, max_rows=4096)
    for R in (128, 1024, 4096):
        x = torch.randn(R, D, device="cuda") * 0.5
        out["train_step_us"][R] = round(timed(lambda: tr.step(x), args.iters, args.warmup), 1)
    fi = ops.FlowInference(D, h, max_rows=65536)
    for R in (4096, 65536):
        x = torch.randn(R, D, device="cuda") * 0.5
        us = timed(lambda: fi.rows(m, x, want_logprob=False), max(args.iters // 10, 5), 3)
        out["rows_forward"][R] = {"us": round(us, 1), "rows_per_s": round(R / us * 1e6),
                                  "tflops": round(R * flop_row / us * 1e-6, 2)}
    # per-pixel map from ViT-S/8 tokens at 448 (B = 32), and ViT + map end to end
    from oracle.dino_vit import ViTConfig, synthetic_state_dict
    from wild_visual_navigation_b200 import ConfidenceGenerator, TraversabilityInference
    from wild_visual_navigation_b200.feature_extractor import DinoInterface

    B, S = 32, 448
    di = DinoInterface("cuda", input_size=S, backbone_type="vit_small", patch_size=8,
                       state_dict=synthetic_state_dict(ViTConfig.from_name("vit_small", 8, S), seed=1), max_batch=B)
    cg = ConfidenceGenerator(0.5, "latest_measurement").cuda()
    ti = TraversabilityInference(di, m, cg)
    img = torch.rand(B, 3, S, S, device="cuda")
    tokens = di.inference_tokens(img)
    hp, dp = (h + 63) // 64 * 64, (D + 63) // 64 * 64
    flop_pix = 2 * 2 * (dp * 2 * hp + 2 * hp * hp + 2 * hp * dp)   # two couplings, s and t, padded GEMM shapes
    us = timed(lambda: ti.predict_from_tokens(tokens, S), 5, 2)
    out["pixels_448_b32"] = {"ms": round(us / 1e3, 2), "frames_per_s": round(B / us * 1e6, 1),
                             "tflops": round(B * S * S * flop_pix / us * 1e-6, 1), "gflop_per_frame": round(S * S * flop_pix / 1e9, 1)}
    us = timed(lambda: ti.predict(img), 5, 2)
    out["vit_plus_pixels_448_b32"] = {"ms": round(us / 1e3, 2), "frames_per_s": round(B / us * 1e6, 1)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
