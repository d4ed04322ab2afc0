"""Segment-wise maps on the GPU, timed with CUDA events, with the card's name, power limit and SM clocks.  Each figure is
the median over --repeats windows of --steps calls (after --warmup calls), with the spread (min, max) of those windows:

  * HotPathStep.step time per frame, per-pixel against segment-wise (prediction_per_pixel=False), DINO ViT-S/8 + STEGO
    + SimpleMLP at B = 32 / 448 and at B = 1 / 224, eager and replayed from a CUDA graph;
  * wvn_segment_maps alone against the two torch.gather calls it replaces (B = 32, 448 x 448, int64 seg, STEGO's
    smax), in GB/s of the bytes the copy needs (ids read, two maps written);
  * the segment-wise step on ResNet-18 with STEGO / SLIC / grid segmentation (SimpleMLP), and on ResNet-50 and
    EfficientNet-B0 with the LinearRnvp flow, at B = 32 / 448, eager.

Prints one JSON line.  Runs only on a GPU; nothing is written to disk."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import warnings

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return (q.stdout.strip().splitlines() or ["?"])[0]


def timed(fn, warmup, steps, repeats):
    """-> (median, min, max) ms per call over `repeats` windows of `steps` calls."""
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = []
    for _ in range(repeats):
        a.record()
        for _ in range(steps):
            fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b) / steps)
    return statistics.median(ms), min(ms), max(ms)


def _fmt(t, div=1.0):
    return [round(v / div, 4) for v in t]


def _labels(hp, B, seed=0):
    g = torch.Generator().manual_seed(seed)
    n = B * hp.smax
    yv = torch.rand(n, generator=g) < 0.3
    yv[:2] = True
    return torch.where(yv, torch.rand(n, generator=g).clamp(min=0.001), torch.zeros(n)).cuda(), yv.cuda()


def bench_step(hp, B, S, args, replay=True):
    """ms per frame of hp.step (and of the replayed graph) as [median, min, max]."""
    img = torch.rand(B, 3, S, S, generator=torch.Generator().manual_seed(1)).cuda()
    y, yv = _labels(hp, B)
    out = {"eager": _fmt(timed(lambda: hp.step(img, y, yv), args.warmup, args.steps, args.repeats), B)}
    if replay:
        hp.capture(img, y, yv)
        out["replay"] = _fmt(timed(lambda: hp.replay(img), args.warmup, args.steps, args.repeats), B)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    import bench
    from wild_visual_navigation_b200 import HotPathStep, ops
    from wild_visual_navigation_b200.feature_extractor import weights as W

    torch.cuda.set_device(0)
    out = {"card_before": card(), "protocol": f"median [min, max] of {args.repeats} windows of {args.steps} calls"}
    _, sd, hd = bench.make_weights()

    def step(B, S, **kw):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            return HotPathStep("cuda", sd, hd, batch=B, input_size=S, chunk=32, flip_tta=False, run_clustering=True,
                               n_image_clusters=20, **kw)

    # 1. per-pixel vs segment-wise, DINO ViT-S/8 + STEGO + SimpleMLP
    for B, S in ((32, 448), (1, 224)):
        for per_pixel in (True, False):
            hp = step(B, S, prediction_per_pixel=per_pixel)
            key = f"dino_stego_mlp_b{B}_{S}_{'per_pixel' if per_pixel else 'segment_wise'}_ms_per_frame"
            out[key] = bench_step(hp, B, S, args)
            del hp
            torch.cuda.empty_cache()

    # 2. the paint kernel against the two gathers
    B, S, smax = 32, 448, 20
    g = torch.Generator(device="cuda").manual_seed(2)
    seg = torch.randint(0, smax, (B, S, S), generator=g, device="cuda")
    n_rows = torch.full((B,), smax, dtype=torch.int32, device="cuda")
    trav, conf = torch.rand(B, smax, device="cuda"), torch.rand(B, smax, device="cuda")

    def gathers():
        idx = seg.reshape(B, -1).long()
        return trav.gather(1, idx).view_as(seg), conf.gather(1, idx).view_as(seg)

    nbytes = B * S * S * (8 + 4 + 4)
    reps = max(args.steps, 50)
    for name, fn in (("segment_maps", lambda: ops.segment_maps(seg, n_rows, trav, conf)), ("two_gathers", gathers)):
        t = timed(fn, args.warmup, reps, args.repeats)
        out[f"{name}_b{B}_{S}_us"] = _fmt(t, 1e-3)
        out[f"{name}_b{B}_{S}_GBps"] = [round(nbytes / (v * 1e-3) / 1e9, 1) for v in (t[0], t[2], t[1])]

    # 3. torchvision trunks, segment-wise, B = 32 / 448
    trunks = {"resnet18": W.synthetic_resnet_state_dict(18, seed=1), "resnet50": W.synthetic_resnet_state_dict(50, seed=1),
              "efficientnet_b0": W.synthetic_efficientnet_b0_state_dict(seed=1)}
    cases = [("resnet18", "stego", False), ("resnet18", "slic", False), ("resnet18", "grid", False),
             ("resnet50", "stego", True), ("efficientnet_b0", "stego", True)]
    for model_type, seg_type, anomaly in cases:
        hp = step(32, 448, feature_type="torchvision", model_type=model_type, backbone_state_dict=trunks[model_type],
                  segmentation_type=seg_type, prediction_per_pixel=False, anomaly_detection=anomaly)
        learner = "flow" if anomaly else "mlp"
        out[f"{model_type}_{seg_type}_{learner}_b32_448_ms_per_frame"] = bench_step(hp, 32, 448, args, replay=False)
        del hp
        torch.cuda.empty_cache()
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
