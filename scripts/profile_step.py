"""Where the time of one benchmarked step goes, per kernel and per ViT GEMM role.

    python scripts/profile_step.py --config c3 --out DIR [--steps 3 --warmup 3]

Runs `HotPathStep.step` at bench.py's configuration (same weights, frames and supervision) for a few warmed-up steps
under torch.profiler with CUDA activities, writes the trace to DIR/step_trace.json and prints
  * the card's name, power limit and max SM clock (an nvidia-smi query);
  * per kernel: total time over the profiled steps and launch count;
  * per ViT GEMM role (patch-embed / QKV / proj / fc1 / fc2): measured time per launch next to its compute bound
    (FLOP over 989 TFLOP/s dense BF16) and memory bound (A read + output bytes over 3.35 TB/s HBM3), and the measured
    time over the larger bound.

The role of a GEMM launch comes from its position in the chain.  A block runs LN1, QKV, attention, proj, LN2, fc1,
fc2; proj and fc2 share one kernel instantiation (fp32 residual add, N = D), so the kernel name alone cannot tell them
apart: a residual GEMM that follows the QKV GEMM is proj, one that follows fc1 (bf16 + GELU) is fc2.  The STEGO-head
and pixel-head GEMMs are listed as "other GEMM".  Profiling slows the host; take step times from bench.py instead.
"""
from __future__ import annotations

import argparse
import json
import os
import re
import subprocess
import sys
from collections import OrderedDict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402

PEAK_TFLOPS = 989.0  # H100 SXM data sheet, dense BF16 at 700 W
PEAK_TBPS = 3.35     # H100 SXM data sheet, HBM3

EPI_RESID, EPI_PATCH, EPI_QKV = 2, 3, 4
ACT_GELU = 2
GEMM_RE = re.compile(r"gemm_bf16_kernel<(\d+), ?(\d+), ?(\d+)>")


def gemm_bounds(config, frames_per_launch):
    """role -> (M, N, K, FLOP, HBM bytes) of one launch: A read plus the output (read and written for a residual add)."""
    c = bench.CONFIGS[config]
    grid = c["img"] // bench.PATCH
    npad = (grid * grid + 1 + 127) // 128 * 128
    D, kpe = c["dim"], (3 * bench.PATCH * bench.PATCH + 63) // 64 * 64
    m, mp = frames_per_launch * npad, frames_per_launch * grid * grid
    shapes = OrderedDict([
        ("patch-embed", (mp, D, kpe, mp * kpe * 2 + mp * D * 4)),
        ("QKV", (m, 3 * D, D, m * D * 2 + m * 3 * D * 2)),
        ("proj", (m, D, D, m * D * 2 + 2 * m * D * 4)),
        ("fc1", (m, 4 * D, D, m * D * 2 + m * 4 * D * 2)),
        ("fc2", (m, D, 4 * D, m * 4 * D * 2 + 2 * m * D * 4)),
    ])
    return OrderedDict((r, (M, N, K, 2.0 * M * N * K, b)) for r, (M, N, K, b) in shapes.items())


def label_gemms(kernels):
    """kernels: [(name, dur_us)] in launch order -> role per GEMM launch (None for non-GEMM kernels)."""
    roles, prev = [], None
    for name, _ in kernels:
        m = GEMM_RE.search(name)
        if not m:
            roles.append(None)
            continue
        epi, act = int(m.group(2)), int(m.group(3))
        if epi == EPI_PATCH:
            role = "patch-embed"
        elif epi == EPI_QKV:
            role = "QKV"
        elif epi == EPI_RESID and prev == "QKV":
            role = "proj"
        elif epi == 0 and act == ACT_GELU and prev == "proj":
            role = "fc1"
        elif epi == EPI_RESID and prev == "fc1":
            role = "fc2"
        else:
            role = "other GEMM"
        roles.append(role)
        prev = role
    return roles


def card_header():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[torch.cuda.current_device()] if q else "nvidia-smi: no output"
    except Exception as e:  # noqa: BLE001 — the header is informative only
        return f"nvidia-smi unavailable ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="c3", choices=sorted(bench.CONFIGS))
    ap.add_argument("--out", required=True, help="directory for the trace (step_trace.json) and summary (profile.json)")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--chunk", type=int, default=32, help="frames per ViT activation chunk (bench.py's default)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("profile_step.py needs a CUDA device")

    from torch.profiler import ProfilerActivity, profile

    from wild_visual_navigation_b200 import HotPathStep, _C

    _C.require_device()
    dev = "cuda:0"
    torch.cuda.set_device(0)
    c = bench.CONFIGS[args.config]
    cfg, sd, hd = bench.make_weights(args.config)
    B = c["batch"]
    hp = HotPathStep(dev, sd, hd, batch=B, input_size=c["img"], backbone_type=c["backbone"], patch_size=bench.PATCH,
                     chunk=args.chunk, flip_tta=False, run_clustering=True, n_image_clusters=bench.K_IMAGE_CLUSTERS)
    g = torch.Generator().manual_seed(2)
    yv = (torch.rand(B * hp.smax, generator=g) < 0.16).to(dev)
    y = torch.where(yv, torch.rand(B * hp.smax, generator=g).clamp(min=0.001).to(dev), torch.zeros(B * hp.smax, device=dev))
    imgs = [t.to(dev) for t in bench.synthetic_images(3, B, seed=100, img=c["img"])]
    for k in range(args.warmup):
        hp.step(imgs[k % 3], y, yv)
    torch.cuda.synchronize()

    os.makedirs(args.out, exist_ok=True)
    trace = os.path.join(args.out, "step_trace.json")
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for k in range(args.steps):
            hp.step(imgs[k % 3], y, yv)
        torch.cuda.synchronize()
    prof.export_chrome_trace(trace)
    events = json.load(open(trace))["traceEvents"]
    kern = sorted((e for e in events if e.get("cat") == "kernel"), key=lambda e: e["ts"])
    kernels = [(e["name"], float(e["dur"])) for e in kern]
    roles = label_gemms(kernels)

    print(f"card: {card_header()}")
    print(f"config {args.config}: {c['label']}, B = {B}, {args.steps} profiled steps after {args.warmup} warm-up")
    total_us = sum(d for _, d in kernels)
    per_kernel = OrderedDict()
    for name, d in kernels:
        t = per_kernel.setdefault(name, [0.0, 0])
        t[0] += d
        t[1] += 1
    print(f"\nkernel time per step {total_us / args.steps / 1000:.2f} ms (sum of kernel durations)")
    print(f"{'ms/step':>9} {'share':>6} {'launches':>9}  kernel")
    for name, (d, n) in sorted(per_kernel.items(), key=lambda kv: -kv[1][0]):
        print(f"{d / args.steps / 1000:9.3f} {d / total_us:6.1%} {n:9d}  {name[:150]}")

    bounds = gemm_bounds(args.config, min(args.chunk, B))
    by_role = OrderedDict((r, [0.0, 0]) for r in list(bounds) + ["other GEMM"])
    for (name, d), r in zip(kernels, roles):
        if r is not None:
            by_role[r][0] += d
            by_role[r][1] += 1
    gemm_us = sum(v[0] for v in by_role.values())
    print(f"\nGEMMs: {gemm_us / args.steps / 1000:.2f} ms per step ({gemm_us / total_us:.1%} of kernel time)")
    print(f"{'role':12s} {'M,N,K':>20} {'launches':>9} {'us/launch':>10} {'compute us':>11} {'memory us':>10} "
          f"{'measured/bound':>15}  {'ms/step':>8}")
    summary = {"card": card_header(), "config": args.config, "steps": args.steps,
               "kernel_ms_per_step": total_us / args.steps / 1000, "gemm_ms_per_step": gemm_us / args.steps / 1000,
               "roles": {}}
    for r, (d, n) in by_role.items():
        if n == 0:
            continue
        per = d / n
        line = f"{r:12s} {'':>20} {n:9d} {per:10.1f} {'':>11} {'':>10} {'':>15}  {d / args.steps / 1000:8.3f}"
        entry = {"launches": n, "us_per_launch": per, "ms_per_step": d / args.steps / 1000}
        if r in bounds:
            M, N, K, flop, nbytes = bounds[r]
            tc, tm = flop / (PEAK_TFLOPS * 1e12) * 1e6, nbytes / (PEAK_TBPS * 1e12) * 1e6
            line = (f"{r:12s} {f'{M},{N},{K}':>20} {n:9d} {per:10.1f} {tc:11.1f} {tm:10.1f} {per / max(tc, tm):15.2f}"
                    f"  {d / args.steps / 1000:8.3f}")
            entry.update(compute_bound_us=tc, memory_bound_us=tm, measured_over_bound=per / max(tc, tm),
                         bound="compute" if tc >= tm else "memory")
        summary["roles"][r] = entry
        print(line)
    with open(os.path.join(args.out, "profile.json"), "w") as f:
        json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
