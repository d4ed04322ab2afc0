"""The mission graph's supervision event and train() on the device (CUDA events), with the card's name and power limit
printed beside every number:

  * one event into n = 1, 4, 16, 64, 256 in-range nodes at 224^2 and 448^2 (smax 256): ``wvn_mission_propagate`` (one
    launch) against the per-node loop of the existing kernels (``project_and_render`` with the fused fmin into a
    3-channel mask, then ``pool_supervision``), the composition the reference's event maps to;
  * ``TraversabilityEstimator.train()`` sampling 8 of 64 valid nodes from the graph (SimpleMLP, D = 384, smax 256).

Each number is the median of --reps runs of --iters calls, with the run-to-run spread (max / min - 1).
Prints one JSON line.  Usage: python scripts/bench_mission_graph.py [--iters N] [--reps R]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def timed(fn, iters, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    runs = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        b.synchronize()
        runs.append(a.elapsed_time(b) * 1e3 / iters)
    return {"median_us": round(statistics.median(runs), 2), "spread": round(max(runs) / min(runs) - 1, 4)}


def event(n, H, smax, iters, reps):
    from oracle import image_projector as oip
    from wild_visual_navigation_b200 import ops

    dev = "cuda"
    K, poses, fp = oip.synthetic_footprints(n, seed=1, image=H)
    K, poses, pts = K.to(dev), poses.to(dev), fp[0].contiguous().to(dev)
    seg = torch.randint(0, smax, (n, H, H), device=dev, dtype=torch.int32)
    mask = torch.full((n, H, H), float("nan"), device=dev)
    y = torch.zeros(n, smax, device=dev)
    yv = torch.zeros(n, smax, device=dev, dtype=torch.uint8)
    sv = torch.zeros(n, device=dev, dtype=torch.int32)
    slots = torch.arange(n, device=dev, dtype=torch.int32)
    trav = torch.tensor([0.5], device=dev)
    ws = ops.mission_propagate_workspace(n, smax, dev)
    fused = timed(lambda: ops.mission_propagate(slots, None, K, poses, pts, trav, seg, mask, y, yv, sv, ws), iters, reps)
    seg64 = seg.long()
    mask3 = torch.full((n, 3, H, H), float("nan"), device=dev)
    ones = torch.ones(3, device=dev)

    def loop():
        for i in range(n):
            ops.project_and_render(K[i : i + 1], poses[i : i + 1], pts[None], ones, H, H, render=False,
                                   supervision=mask3[i : i + 1], traversability=trav)
            ops.pool_supervision(seg64[i : i + 1], mask3[i : i + 1], smax)

    return {"fused": fused, "per_node_loop": timed(loop, max(1, iters // 4), reps)}


def train(iters, reps):
    from oracle import mission_graph as omg
    from wild_visual_navigation_b200 import TraversabilityEstimator

    te = TraversabilityEstimator(device="cuda", min_samples_for_training=0, mission_graph_capacity=64,
                                 mission_graph_smax=256)
    g = torch.Generator().manual_seed(0)
    seg, nb = omg.segmentation(448, 448, seed=0, cell=32)
    cib = omg.camera_in_base()
    K = torch.tensor([[268.8, 0, 224, 0], [0, 268.8, 224, 0], [0, 0, 1, 0], [0, 0, 0, 1.0]])
    for i in range(64):
        B = omg._pose(0.2 * i, 0.0, 0.0)
        te.add_mission_frames({"seg": seg[None].cuda(), "feat": torch.randn(1, 256, 384, generator=g).cuda(),
                               "n_segments": torch.tensor([nb], dtype=torch.int32).cuda()}, B[None], K, [float(i)],
                              pose_cam_in_base=cib)
    gr = te._mission_graph
    gr.y[:, :nb] = torch.rand(64, nb, generator=g).cuda()
    gr.y_valid[:, :nb] = 1
    gr.slot_valid.fill_(1)
    gr._meta_host = None
    return timed(lambda: te.train(), iters, reps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    out = {"card": card(), "event": {}}
    for H in (224, 448):
        for n in (1, 4, 16, 64, 256):
            out["event"][f"{H}_{n}"] = event(n, H, 256, a.iters, a.reps)
            torch.cuda.empty_cache()
    out["train_from_graph"] = train(a.iters, a.reps)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
