"""The three learners on HotPathStep's padded rows (CUDA events), with the card's name and power limit printed beside them:

  * the padded train step (``TraversabilityEstimator.train_on_padded``) of SimpleMLP, DoubleMLP and the LinearRnvp flow
    at HotPathStep's row shape, B = 32 frames x smax padded rows, about 60 % of them live and 16 % of those labelled;
  * ``HotPathStep.step`` in frames/s for each learner at B = 32, 448 x 448, ViT-S/8 (random-init, seeded) with STEGO
    segmentation, eager and through ``capture`` / ``replay``.

Single process, one GPU: the data-parallel exchanges are not measured here.  Prints one JSON line.
Usage: python scripts/bench_learners.py [--iters N]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

LEARNERS = {"SimpleMLP": {}, "DoubleMLP": {"model": "DoubleMLP"}, "LinearRnvp": {"anomaly_detection": True}}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def timed(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters * 1e3   # us per call


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    import bench
    from wild_visual_navigation_b200 import HotPathStep

    torch.cuda.set_device(0)
    B, S = 32, 448
    _, sd, hd = bench.make_weights()
    g = torch.Generator().manual_seed(0)
    imgs = [torch.rand(B, 3, S, S, generator=g).cuda() for _ in range(3)]
    res = {"card": card(), "batch": B, "image": S, "backbone": "ViT-S/8 + STEGO"}
    for name, kw in LEARNERS.items():
        hp = HotPathStep("cuda", sd, hd, batch=B, input_size=S, chunk=32, flip_tta=False, run_clustering=True,
                         n_image_clusters=bench.K_IMAGE_CLUSTERS, **kw)
        n = B * hp.smax
        yv = (torch.rand(n, generator=g) < 0.16).cuda()
        y = torch.where(yv, torch.rand(n, generator=g).clamp(min=0.001).cuda(), torch.zeros(n, device="cuda"))
        # the train step alone, on the padded rows of one real batch
        r = hp.fe.extract_batch(imgs[0])
        feat, n_rows = r["feat"], r["n_segments"]
        us = timed(lambda: hp.te.train_on_padded(feat, n_rows, y, yv), args.iters * 5)
        res[f"{name}_train_step_us"] = round(us, 1)
        res[f"{name}_rows"] = f"{B} x {hp.smax} padded, {int(n_rows.sum())} live"
        # the whole step, eager and replayed
        k = [0]

        def eager():
            hp.step(imgs[k[0] % 3], y, yv)
            k[0] += 1

        res[f"{name}_step_fps"] = round(B / (timed(eager, args.iters) * 1e-6), 1)
        hp.capture(imgs[0], y, yv)

        def replay():
            hp.replay(imgs[k[0] % 3])
            k[0] += 1

        res[f"{name}_replay_fps"] = round(B / (timed(replay, args.iters) * 1e-6), 1)
        del hp
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
