"""STEGO's dense CRF (csrc/dense_crf.cu) on the GPU, timed with CUDA events, with the card's name and power limit:
ms per frame at 448 x 448 for B in {1, 32} and 27 / 32 classes, the extra time FeatureExtractor.extract_batch takes
at B = 32 with run_crf=True over run_crf=False, and the numpy oracle's CPU time per frame at 224 x 224 (10 iterations;
at 448 it needs about a minute per frame).  Prints one JSON line."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    name, power = (q.stdout.strip().splitlines() or ["?, ?"])[0].split(", ")
    return name, power


def timed(fn, warmup, steps):
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--size", type=int, default=448)
    args = ap.parse_args()
    from oracle import dense_crf as dc
    from oracle.dino_vit import ViTConfig, synthetic_state_dict
    from oracle.slic import synthetic_image
    from oracle.stego_head import synthetic_head
    from wild_visual_navigation_b200 import ops
    from wild_visual_navigation_b200.feature_extractor import FeatureExtractor

    S = args.size
    g = S // 8
    npad = (1 + g * g + 7) // 8 * 8
    out = {"size": S}
    imgs = torch.from_numpy(np.stack([synthetic_image(S, S, s) for s in range(32)])).cuda()
    for K in (27, 32):
        crf = ops.DenseCrf(S, K, chunk=2)
        out[f"workspace_bytes_k{K}"] = crf.workspace_bytes
        for B in (1, 32):
            head = torch.randn(B * npad, 256, device="cuda")
            ms = timed(lambda: crf.run(imgs[:B], head, npad, g, 192, K), args.warmup, args.steps)
            out[f"crf_ms_per_frame_b{B}_k{K}"] = round(ms / B, 3)
        del crf
    cfg = ViTConfig.from_name("vit_small", 8, S)
    sd, hd = synthetic_state_dict(cfg, seed=6), synthetic_head(384, 90, 32, 27, seed=3)
    for crf_on in (False, True):
        fe = FeatureExtractor("cuda", segmentation_type="stego", feature_type="stego", input_size=S, state_dict=sd,
                              head_state_dict=hd, flip_tta=False, max_batch=32, run_crf=crf_on, run_clustering=False)
        out[f"extract_batch_ms_b32_crf_{'on' if crf_on else 'off'}"] = round(
            timed(lambda: fe.extract_batch(imgs), args.warmup, args.steps), 2)
        del fe
    out["extract_batch_crf_extra_ms_b32"] = round(out["extract_batch_ms_b32_crf_on"] - out["extract_batch_ms_b32_crf_off"], 2)
    s0 = 224
    img0 = synthetic_image(s0, s0, 0)
    U = dc.unary_from_logits(np.random.default_rng(0).normal(size=(s0 * s0, 27)).astype(np.float32) * 2)
    t = time.perf_counter()
    dc.mean_field(U, dc.crf_image_bytes(img0))
    out["oracle_cpu_ms_per_frame_224"] = round(1e3 * (time.perf_counter() - t), 1)
    out["gpu"], out["power_limit"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
