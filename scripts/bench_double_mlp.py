"""DoubleMLP learner timings on the GPU (CUDA events), with the card's name and power limit printed beside them:

  * the train step (csrc/double_mlp_train.cu) at R in {128, 1024, 4096} rows, D = 384, [64, 32, 1];
  * per-pixel maps at B = 32, 448 x 448, from the ViT-S/8's own bf16 tokens (56 x 56 grid): the DoubleMLP [64, 32, 1]
    on the fused head's DoubleMLP instantiation against the SimpleMLP [256, 32, 1] on its fused head, in the same
    process, run alternately (and the DoubleMLP's unfused path from the fp32 tokens, for reference);
  * the ViT-S/8 forward followed by the DoubleMLP map.

Achieved FLOP/s use the dense work the reference's formulation does, computed from the shapes here: per row
2 (D h1 + h1 h2 + h2) for net 0 plus 2 (D h1 + h1 h2 + h2 D) for net 1 (SimpleMLP: 2 (D h1 + h1 h2 + h2 (D + 1))).
Prints one JSON line.  Usage: python scripts/bench_double_mlp.py [--iters N]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def timed(fn, iters, warmup=5):
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


def double_flop(D, h1, h2):
    return 2 * (D * h1 + h1 * h2 + h2) + 2 * (D * h1 + h1 * h2 + h2 * D)


def simple_flop(D, h1, h2):
    return 2 * (D * h1 + h1 * h2 + h2 * (D + 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    from oracle.dino_vit import ViTConfig, synthetic_state_dict
    from wild_visual_navigation_b200 import DoubleMLP, SimpleMLP, ops

    torch.cuda.set_device(0)
    D, h1, h2 = 384, 64, 32
    res = {"card": card(), "shape": f"DoubleMLP({D}, [{h1}, {h2}, 1])"}
    torch.manual_seed(42)
    dm = DoubleMLP(D, [h1, h2, 1]).cuda()
    g = torch.Generator(device="cuda").manual_seed(0)
    tr = ops.DoubleMlpTrainer(dm, max_rows=4096)
    for R in (128, 1024, 4096):
        x = torch.randn(R, D, device="cuda", generator=g)
        yv = torch.rand(R, device="cuda", generator=g) < 0.2
        y = torch.where(yv, torch.rand(R, device="cuda", generator=g), torch.zeros(R, device="cuda"))
        us = timed(lambda: tr.step(x, y, yv), args.iters * 4)
        fl = 3 * R * double_flop(D, h1, h2)   # forward + two backward products per layer
        res[f"train_step_us_R{R}"] = round(us, 2)
        res[f"train_step_gflops_R{R}"] = round(fl / us * 1e-3, 2)

    B, S, grid = 32, 448, 56
    cfg = ViTConfig.from_name("vit_small", 8, S)
    vit = ops.ViTBackbone(S, 8, cfg.dim, cfg.depth, cfg.heads, cfg.mlp_dim, synthetic_state_dict(cfg, seed=3),
                          max_batch=B)
    img = torch.rand(B, 3, S, S, device="cuda", generator=g)
    tokens = vit.forward(img)
    cm, cs = torch.tensor([0.3], device="cuda"), torch.tensor([0.2], device="cuda")
    dh = ops.MlpInference(D, h1, h2, tokens_per_frame=vit.npad, double=True)
    dh.set_params(dm.flat_params)
    torch.manual_seed(42)
    sm = SimpleMLP(D, [256, 32, 1], True).cuda()
    sh = ops.MlpInference(D, 256, 32, tokens_per_frame=vit.npad)
    sh.set_params(sm.flat_params)
    run_d = lambda: dh.pixels_from_vit(vit, B, (S, S), cm, cs, 0.5)       # noqa: E731
    run_s = lambda: sh.pixels_from_vit(vit, B, (S, S), cm, cs, 0.5)       # noqa: E731
    td, ts = [], []
    for _ in range(3):   # alternate the two heads
        td.append(timed(run_d, max(2, args.iters // 5), warmup=2))
        ts.append(timed(run_s, max(2, args.iters // 5), warmup=2))
    td, ts = min(td), min(ts)
    px = B * S * S
    res["double_map_fps"] = round(B / (td * 1e-6), 1)
    res["double_map_tflops"] = round(px * double_flop(D, h1, h2) / (td * 1e-6) * 1e-12, 2)
    res["simple_map_fps"] = round(B / (ts * 1e-6), 1)
    res["simple_map_tflops"] = round(px * simple_flop(D, 256, 32) / (ts * 1e-6) * 1e-12, 2)
    os.environ["WVN_PIXEL_HEAD"] = "unfused"   # read when a handle is created
    du = ops.MlpInference(D, h1, h2, double=True)
    du.set_params(dm.flat_params)
    tu = timed(lambda: du.pixels(tokens, (grid, grid), (S, S), cm, cs, 0.5), max(2, args.iters // 5), warmup=2)
    res["double_map_unfused_fps"] = round(B / (tu * 1e-6), 1)

    def vit_then_map():
        vit.forward(img)
        dh.pixels_from_vit(vit, B, (S, S), cm, cs, 0.5)

    tv = timed(vit_then_map, max(2, args.iters // 5), warmup=2)
    res["vit_plus_double_map_fps"] = round(B / (tv * 1e-6), 1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
