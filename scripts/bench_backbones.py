"""Backbone forward throughput: DINO ViT-S/8, DINOv2 ViT-S/14 / ViT-B/14 and their register variants (4 register
tokens) at 448 x 448, B = 32 frames per call,
seeded weights.  `python scripts/bench_backbones.py [--steps 20] [--warmup 3] [--repeats 5] [--batch 32]`.

For each backbone: frames/s from CUDA events around `--steps` back-to-back forward calls (median of `--repeats`
windows after `--warmup` calls), GFLOP/frame from the shapes (below), the achieved TFLOP/s, and the card's name,
power limit and max SM clock read in the same run.  Prints one JSON line per backbone.  Needs an sm_90a GPU; without
one it fails.

GFLOP/frame counts the algorithmic work on the n = grid^2 + 1 + R real tokens (R register tokens; padding rows are not
counted):
patch embed 2 P (3 p^2) D; per block 2 n (3 D^2 + D^2 + 2 D M) for QKV / out-projection / MLP and 4 n^2 D for
Q K^T and P V."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import warnings

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

BACKBONES = [("dino_vit_s8", "dino", "vit_small", 8), ("dinov2_vit_s14", "dinov2", "vit_small", 14),
             ("dinov2_vit_b14", "dinov2", "vit_base", 14), ("dinov2_reg_vit_s14", "dinov2_reg", "vit_small", 14),
             ("dinov2_reg_vit_b14", "dinov2_reg", "vit_base", 14)]


def gflop_per_frame(dim, depth, mlp_dim, patch, image_size, registers=0):
    g = image_size // patch
    P, n = g * g, g * g + 1 + registers
    flop = 2 * P * 3 * patch * patch * dim
    flop += depth * (2 * n * (4 * dim * dim + 2 * dim * mlp_dim) + 4 * n * n * dim)
    return flop / 1e9


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (s.strip() for s in q.split(","))
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--image-size", type=int, default=448)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_backbones: no CUDA device (this benchmark only runs on the GPU)")
    from wild_visual_navigation_b200.feature_extractor import DinoInterface
    from wild_visual_navigation_b200.feature_extractor.weights import VIT_SHAPES

    info = card()
    S, B = args.image_size, args.batch
    img = torch.rand(B, 3, S, S, generator=torch.Generator().manual_seed(0)).cuda()
    for name, backbone, backbone_type, patch in BACKBONES:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")   # seeded weights: timing only
            di = DinoInterface("cuda", backbone=backbone, input_size=S, backbone_type=backbone_type, patch_size=patch,
                               max_batch=B, chunk=B)
        for _ in range(args.warmup):
            di.inference_tokens(img)
        torch.cuda.synchronize()
        rates = []
        for _ in range(args.repeats):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                di.inference_tokens(img)
            e1.record()
            torch.cuda.synchronize()
            rates.append(B * args.steps / (e0.elapsed_time(e1) * 1e-3))
        shp = VIT_SHAPES[backbone_type]
        gf = gflop_per_frame(shp["dim"], shp["depth"], shp["mlp_dim"], patch, S, di._model.registers)
        fps = statistics.median(rates)
        print(json.dumps({"backbone": name, "image_size": S, "batch": B, "grid": S // patch, "registers": di._model.registers,
                          "npad": di._model.npad,
                          "frames_per_s": round(fps, 1), "frames_per_s_runs": [round(r, 1) for r in rates],
                          "gflop_per_frame": round(gf, 1), "tflop_per_s": round(fps * gf / 1e3, 1), **info}),
              flush=True)
        del di
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
