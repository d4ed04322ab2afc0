"""Backbone forward throughput: DINO ViT-S/8, DINOv2 ViT-S/14 / ViT-B/14 / ViT-L/14 and their register variants (4
register tokens), and the torchvision ResNet-18 / ResNet-50 and EfficientNet-B0 feature pyramids, at 448 x 448, B = 32 frames per call,
seeded weights.  `python scripts/bench_backbones.py [--steps 20] [--warmup 3] [--repeats 5] [--batch 32]
[--backbones NAME ...]`.

For each backbone: frames/s from CUDA events around `--steps` back-to-back forward calls (median of `--repeats`
windows after `--warmup` calls), GFLOP/frame from the shapes (below), the achieved TFLOP/s, and the card's name,
power limit and max SM clock read in the same run.  Prints one JSON line per backbone.  Needs an sm_90a GPU; without
one it fails.

GFLOP/frame counts the algorithmic work on the n = grid^2 + 1 + R real tokens (R register tokens; padding rows are not
counted):
patch embed 2 P (3 p^2) D; per block 2 n (3 D^2 + D^2 + 2 D M) for QKV / out-projection / MLP and 4 n^2 D for
Q K^T and P V.  For a ResNet it is 2 Cout Cin k^2 Ho Wo summed over the convs up to the last tap (the whole trunk for
both depths); the row also gives the library's workspace (activations and im2col rows) for the batch, and, in the same
run, the frames/s of the fp32 oracle (oracle/resnet.py) run eagerly on the GPU and of the same ops in bf16,
channels-last, with batch norm folded (cuDNN) as a baseline.  EfficientNet-B0's row is built the same way
(oracle/efficientnet.py); its GFLOP/frame is 2 Cout (Cin / groups) k^2 Ho Wo over every conv (stem, expand, depthwise,
project, head) plus the squeeze-excitations' two small matrix-vector products; the gate multiply and the residual adds
are not counted."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import warnings

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

RESNETS = [("resnet18", 18), ("resnet50", 50)]
BACKBONES = [("dino_vit_s8", "dino", "vit_small", 8), ("dinov2_vit_s14", "dinov2", "vit_small", 14),
             ("dinov2_vit_b14", "dinov2", "vit_base", 14), ("dinov2_reg_vit_s14", "dinov2_reg", "vit_small", 14),
             ("dinov2_reg_vit_b14", "dinov2_reg", "vit_base", 14), ("dinov2_vit_l14", "dinov2", "vit_large", 14),
             ("dinov2_reg_vit_l14", "dinov2_reg", "vit_large", 14)]


def gflop_per_frame(dim, depth, mlp_dim, patch, image_size, registers=0):
    g = image_size // patch
    P, n = g * g, g * g + 1 + registers
    flop = 2 * P * 3 * patch * patch * dim
    flop += depth * (2 * n * (4 * dim * dim + 2 * dim * mlp_dim) + 4 * n * n * dim)
    return flop / 1e9


def resnet_gflop_per_frame(depth, image_size):
    from wild_visual_navigation_b200.feature_extractor.weights import resnet_convs

    flop, side, block, block_stride = 0, image_size // 4, None, 1
    for conv, _, cin, cout, k, stride in resnet_convs(depth):
        if conv == "conv1":
            flop += 2 * cout * cin * k * k * (image_size // 2) ** 2
            continue
        prefix = conv.split(".")[0] + "." + conv.split(".")[1]
        if prefix != block:  # a new block: the previous one's output side is its input side
            side, block, block_stride = side // block_stride, prefix, 1
        block_stride = max(block_stride, stride)
        # ResNet-50's first 1 x 1 conv runs at the block's input side; every other conv at its output side
        out = side if (depth == 50 and conv.endswith("conv1")) else side // block_stride
        flop += 2 * cout * cin * k * k * out * out
    return flop / 1e9


def effnet_gflop_per_frame(image_size):
    from wild_visual_navigation_b200.feature_extractor.weights import efficientnet_b0_blocks

    side = image_size // 2
    flop = 2 * 32 * 3 * 9 * side * side  # the stem
    for _, cin, cexp, cout, k, stride, sq in efficientnet_b0_blocks():
        if cexp != cin:
            flop += 2 * cexp * cin * side * side
        side //= stride
        flop += 2 * cexp * k * k * side * side + 2 * 2 * cexp * sq + 2 * cout * cexp * side * side
    return (flop + 2 * 1280 * 320 * side * side) / 1e9


def time_calls(fn, warmup, repeats, steps, batch):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    rates = []
    for _ in range(repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        rates.append(batch * steps / (e0.elapsed_time(e1) * 1e-3))
    return statistics.median(rates), rates


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
    ap.add_argument("--backbones", nargs="*", default=None, help="names to run (default: all)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_backbones: no CUDA device (this benchmark only runs on the GPU)")
    from wild_visual_navigation_b200.feature_extractor import DinoInterface
    from wild_visual_navigation_b200.feature_extractor.weights import VIT_SHAPES

    info = card()
    S, B = args.image_size, args.batch
    img = torch.rand(B, 3, S, S, generator=torch.Generator().manual_seed(0)).cuda()
    for name, backbone, backbone_type, patch in BACKBONES:
        if args.backbones and name not in args.backbones:
            continue
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")   # seeded weights: timing only
            di = DinoInterface("cuda", backbone=backbone, input_size=S, backbone_type=backbone_type, patch_size=patch,
                               max_batch=B, chunk=B)
        fps, rates = time_calls(lambda: di.inference_tokens(img), args.warmup, args.repeats, args.steps, B)
        shp = VIT_SHAPES[backbone_type]
        gf = gflop_per_frame(shp["dim"], shp["depth"], shp["mlp_dim"], patch, S, di._model.registers)
        print(json.dumps({"backbone": name, "image_size": S, "batch": B, "grid": S // patch, "registers": di._model.registers,
                          "npad": di._model.npad,
                          "frames_per_s": round(fps, 1), "frames_per_s_runs": [round(r, 1) for r in rates],
                          "gflop_per_frame": round(gf, 1), "tflop_per_s": round(fps * gf / 1e3, 1), **info}),
              flush=True)
        del di
        torch.cuda.empty_cache()
    for name, depth in RESNETS:
        if args.backbones and name not in args.backbones:
            continue
        from oracle import resnet as R
        from wild_visual_navigation_b200.feature_extractor import TorchVisionInterface
        from wild_visual_navigation_b200.feature_extractor.weights import fold_resnet_bn, synthetic_resnet_state_dict

        sd = synthetic_resnet_state_dict(depth)
        ti = TorchVisionInterface("cuda", name, S, state_dict=sd, max_batch=B)
        fps, rates = time_calls(lambda: ti.inference_taps(img), args.warmup, args.repeats, args.steps, B)
        gf = resnet_gflop_per_frame(depth, S)
        ws = ti._model.workspace_bytes
        del ti
        torch.cuda.empty_cache()
        # baselines on the same ops: the fp32 oracle eagerly (no TF32), and bf16 channels-last with folded batch norm
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
        sdc = {k: v.cuda() for k, v in sd.items()}
        with torch.no_grad():
            fps_fp32, _ = time_calls(lambda: R.resnet_pyramid(img, sdc, depth), 1, 3, max(1, args.steps // 4), B)
            folded = {}
            for conv, (w, b) in fold_resnet_bn(sd, depth).items():
                folded[conv + ".weight"] = w.cuda().bfloat16().to(memory_format=torch.channels_last)
                folded[conv + ".bias"] = b.cuda().bfloat16()
            img16 = img.bfloat16().to(memory_format=torch.channels_last)
            fps_cudnn, _ = time_calls(lambda: R.resnet_pyramid(img16, folded, depth, folded=True), args.warmup,
                                      args.repeats, args.steps, B)
        del sdc, folded
        torch.cuda.empty_cache()
        stem_col = B * (S // 2) ** 2 * 152 * 2
        print(json.dumps({"backbone": name, "image_size": S, "batch": B, "frames_per_s": round(fps, 1),
                          "frames_per_s_runs": [round(r, 1) for r in rates], "gflop_per_frame": round(gf, 2),
                          "tflop_per_s": round(fps * gf / 1e3, 1), "workspace_gb": round(ws / 1e9, 3),
                          "stem_im2col_gb": round(stem_col / 1e9, 3),
                          "oracle_fp32_eager_frames_per_s": round(fps_fp32, 1),
                          "cudnn_bf16_channels_last_frames_per_s": round(fps_cudnn, 1), **info}), flush=True)
    if not args.backbones or "efficientnet_b0" in args.backbones:
        from oracle import efficientnet as E
        from wild_visual_navigation_b200.feature_extractor import TorchVisionInterface
        from wild_visual_navigation_b200.feature_extractor.weights import (fold_efficientnet_bn,
                                                                           synthetic_efficientnet_b0_state_dict)

        sd = synthetic_efficientnet_b0_state_dict()
        ti = TorchVisionInterface("cuda", "efficientnet_b0", S, state_dict=sd, max_batch=B)
        fps, rates = time_calls(lambda: ti.inference_taps(img), args.warmup, args.repeats, args.steps, B)
        gf = effnet_gflop_per_frame(S)
        ws = ti._model.workspace_bytes
        del ti
        torch.cuda.empty_cache()
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
        sdc = {k: v.cuda() for k, v in sd.items()}
        with torch.no_grad():
            fps_fp32, _ = time_calls(lambda: E.efficientnet_pyramid(img, sdc), 1, 3, max(1, args.steps // 4), B)
            folded = {}
            for m, (w, b) in fold_efficientnet_bn(sd).items():
                w = w.cuda().bfloat16()
                folded[m + ".weight"] = w.to(memory_format=torch.channels_last) if w.dim() == 4 else w
                folded[m + ".bias"] = b.cuda().bfloat16()
            img16 = img.bfloat16().to(memory_format=torch.channels_last)
            fps_cudnn, _ = time_calls(lambda: E.efficientnet_pyramid(img16, folded, folded=True), args.warmup,
                                      args.repeats, args.steps, B)
        del sdc, folded
        torch.cuda.empty_cache()
        print(json.dumps({"backbone": "efficientnet_b0", "image_size": S, "batch": B, "frames_per_s": round(fps, 1),
                          "frames_per_s_runs": [round(r, 1) for r in rates], "gflop_per_frame": round(gf, 2),
                          "tflop_per_s": round(fps * gf / 1e3, 1), "workspace_gb": round(ws / 1e9, 3),
                          "oracle_fp32_eager_frames_per_s": round(fps_fp32, 1),
                          "cudnn_bf16_channels_last_frames_per_s": round(fps_cudnn, 1), **info}), flush=True)


if __name__ == "__main__":
    main()
