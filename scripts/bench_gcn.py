"""The SimpleGCN learner's padded train step and row inference (CUDA events), with the card's name and power limit:

  * ``GcnTrainer.step_padded`` of ``SimpleGCN(384, True, [256, 128, 1])`` at 128, 1024 and 4096 rows, in frames of
    128 segments with 3.8 directed edges per segment (the density of the reference's assets/graph/graph.pt: 384 edges
    over 100 segments) and 16 % of the rows labelled;
  * ``GcnInference.rows_padded`` (graph build, forward, traversability and confidence) at the same sizes.

Single process, one GPU.  Prints one JSON line.
Usage: python scripts/bench_gcn.py [--iters N]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SEGMENTS, DENSITY = 128, 3.8


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def batch(rows, D=384, seed=0):
    g = torch.Generator().manual_seed(seed)
    G = rows // SEGMENTS
    E = int(DENSITY * SEGMENTS)
    feat = torch.randn(G, SEGMENTS, D, generator=g) * 0.8 + 0.1
    edges = torch.randint(0, SEGMENTS, (G, E, 2), generator=g)
    yv = torch.rand(rows, generator=g) < 0.16
    y = torch.where(yv, torch.rand(rows, generator=g), torch.zeros(rows))
    n_rows = torch.full((G,), SEGMENTS, dtype=torch.int32)
    n_edges = torch.full((G,), E, dtype=torch.int32)
    return [t.cuda() for t in (feat, n_rows, edges, n_edges, y, yv)]


def timed(fn, iters):
    for _ in range(5):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    args = ap.parse_args()
    from wild_visual_navigation_b200 import SimpleGCN, ops

    torch.manual_seed(42)
    model = SimpleGCN(384, True, [256, 128, 1]).cuda()
    tr = ops.GcnTrainer(model, max_rows=4096, max_edges=4096 // SEGMENTS * int(DENSITY * SEGMENTS))
    inf = ops.GcnInference(model, max_rows=4096, max_edges=4096 // SEGMENTS * int(DENSITY * SEGMENTS))
    mean, std = torch.zeros(1, device="cuda"), torch.ones(1, device="cuda")
    out = {"card": card(), "model": "SimpleGCN(384, True, [256, 128, 1])", "segments_per_frame": SEGMENTS,
           "edges_per_segment": DENSITY, "train_step_us": {}, "infer_rows_us": {}}
    for rows in (128, 1024, 4096):
        feat, n_rows, edges, n_edges, y, yv = batch(rows)
        out["train_step_us"][rows] = round(timed(lambda: tr.step_padded(feat, n_rows, edges, n_edges, y, yv),
                                                 args.iters), 1)
        out["infer_rows_us"][rows] = round(timed(lambda: inf.rows_padded(feat, n_rows, edges, n_edges, mean, std, 0.5),
                                                 args.iters), 1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
