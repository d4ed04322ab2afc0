"""DINOv2 ViT-g/14 forward throughput (``backbone_type="vit_giant"``, plain and with 4 register tokens), seeded weights.
`python scripts/bench_vit_giant.py [--steps 10] [--warmup 2] [--repeats 3] [--sizes 448 224] [--batches 32 1]`.

For each variant, image size and batch: frames/s of the handle's eager forward (``DinoInterface.inference_tokens``)
from CUDA events around `--steps` back-to-back calls (median of `--repeats` windows after `--warmup` calls), the
GFLOP/frame from the shapes and the achieved TFLOP/s.  Then the kernel time of one w12 GEMM with the fused SwiGLU
epilogue alone (M = B * npad rows of the 448 layout, N = 8192, K = 1536), timed the same way.  The card's name, power
limit and max SM clock are read in the same run.  One JSON line per measurement.  Needs an sm_90a GPU.

GFLOP/frame counts the algorithmic work on the n = grid^2 + 1 + R real tokens: patch embed 2 P (3 p^2) D, and per
block 2 n (4 D^2 + 3 D H) for QKV, the out-projection, w12 (D -> 2 H) and w3 (H -> D), plus 4 n^2 D for Q K^T and
P V.  At 448 (n = 1025) that is 64.5 GFLOP per block and 2.58 TFLOP per frame.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import warnings

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

VARIANTS = [("dinov2_vit_g14", "dinov2"), ("dinov2_reg_vit_g14", "dinov2_reg")]


def gflop_per_frame(dim, depth, hidden, patch, image_size, registers=0):
    g = image_size // patch
    P, n = g * g, g * g + 1 + registers
    block = 2 * n * (4 * dim * dim + 3 * dim * hidden) + 4 * n * n * dim
    return (2 * P * 3 * patch * patch * dim + depth * block) / 1e9, block / 1e9


def time_calls(fn, warmup, repeats, steps):
    """Median milliseconds per call over `repeats` windows of `steps` calls, and the windows' values."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1) / steps)
    return statistics.median(ms), ms


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (s.strip() for s in q.split(","))
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def swiglu_gemm_ms(rows, dim, hidden, warmup, repeats, steps):
    """One w12 GEMM with the SwiGLU epilogue (wvn_gemm_bf16_ex, epi 7) on rows x dim bf16 activations."""
    from ctypes import byref, c_void_p

    from wild_visual_navigation_b200 import _C

    g = torch.Generator(device="cuda").manual_seed(0)
    a = torch.randn(rows, dim, generator=g, device="cuda").bfloat16()
    w = (torch.randn(2 * hidden, dim, generator=g, device="cuda") / dim**0.5).bfloat16()
    bias = torch.randn(2 * hidden, generator=g, device="cuda")
    out = torch.empty(rows, hidden, dtype=torch.bfloat16, device="cuda")
    args = _C.GemmExArgs()
    args.m, args.n, args.k, args.epi = rows, 2 * hidden, dim, 7
    args.a, args.lda, args.w, args.bias = c_void_p(a.data_ptr()), dim, c_void_p(w.data_ptr()), c_void_p(bias.data_ptr())
    args.out, args.ldo = c_void_p(out.data_ptr()), hidden
    run = lambda: _C.check(_C.lib().wvn_gemm_bf16_ex(byref(args), _C.stream()))  # noqa: E731
    return time_calls(run, warmup, repeats, steps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--sizes", type=int, nargs="*", default=[448, 224])
    ap.add_argument("--batches", type=int, nargs="*", default=[32, 1])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_vit_giant: no CUDA device (this benchmark only runs on the GPU)")
    from wild_visual_navigation_b200.feature_extractor import DinoInterface
    from wild_visual_navigation_b200.feature_extractor.weights import VIT_SHAPES

    shp = VIT_SHAPES["vit_giant"]
    info = card()
    for name, backbone in VARIANTS:
        for S in args.sizes:
            Bmax = max(args.batches)
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")   # seeded weights: timing only
                di = DinoInterface("cuda", backbone=backbone, input_size=S, backbone_type="vit_giant", patch_size=14,
                                   max_batch=Bmax, chunk=Bmax)
            for B in args.batches:
                img = torch.rand(B, 3, S, S, generator=torch.Generator().manual_seed(0)).cuda()
                ms, runs = time_calls(lambda: di.inference_tokens(img), args.warmup, args.repeats, args.steps)
                gf, gf_block = gflop_per_frame(shp["dim"], shp["depth"], shp["mlp_dim"], 14, S, di._model.registers)
                fps = B / (ms * 1e-3)
                print(json.dumps({"backbone": name, "image_size": S, "batch": B, "registers": di._model.registers,
                                  "npad": di._model.npad, "frames_per_s": round(fps, 2),
                                  "frames_per_s_runs": [round(B / (m * 1e-3), 2) for m in runs],
                                  "gflop_per_frame": round(gf, 1), "gflop_per_block": round(gf_block, 2),
                                  "tflop_per_s": round(fps * gf / 1e3, 1), **info}), flush=True)
            npad = di._model.npad
            del di
            torch.cuda.empty_cache()
            if backbone == "dinov2" and S == max(args.sizes):
                rows = Bmax * npad
                ms, runs = swiglu_gemm_ms(rows, shp["dim"], shp["mlp_dim"], args.warmup, args.repeats, args.steps)
                flop = 2.0 * rows * shp["dim"] * 2 * shp["mlp_dim"]
                print(json.dumps({"kernel": "w12 GEMM + SwiGLU epilogue", "m": rows, "n": 2 * shp["mlp_dim"],
                                  "k": shp["dim"], "ms": round(ms, 4), "ms_runs": [round(m, 4) for m in runs],
                                  "tflop_per_s": round(flop / (ms * 1e-3) / 1e12, 1), **info}), flush=True)


if __name__ == "__main__":
    main()
