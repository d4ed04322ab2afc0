"""Build-to-build output comparison on seeded inputs.

    WVN_B200_LIB=<lib.so> python scripts/ab_outputs.py write DIR     # once per library build
    python scripts/ab_outputs.py compare DIR_A DIR_B

`write` runs, on fixed seeded inputs, the kernels whose schedules a performance change touches and stores for each
output its SHA-256 plus a strided sample (every 101st element, as float32):
  * ops.attention at the c3 shape (B = 32, 6 heads, 3137 tokens) and the c5 shape (B = 128, 12 heads, 4097 tokens);
  * ops.gemm_bf16 at the four ViT-S GEMM shapes of c3 (M = 32 frames x 3200 rows) with the epilogues they run in the
    backbone: QKV (bf16), attention out-projection (fp32 residual add), fc1 (bf16 + GELU), fc2 (fp32 residual add);
  * DinoInterface tokens of ViT-S/8 @448 at B = 32;
  * the fused per-pixel traversability / confidence maps of a seeded SimpleMLP on those tokens;
  * DinoInterface tokens of ViT-S/16 @448 at B = 8 (the patch-16 loader and patch-embed GEMM).
`compare` reports, per output, whether the two builds agree bit for bit and, where not, the largest difference in
the samples.  Every output here is deterministic for a given build (no atomics race in them), so any difference is
the build's.
"""
import hashlib
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

STRIDE = 101


def _record(out_dir, name, t, index):
    raw = t.detach().contiguous().cpu()
    digest = hashlib.sha256(raw.view(-1).view(torch.uint8).numpy().tobytes()).hexdigest()
    np.save(os.path.join(out_dir, name + ".npy"), raw.reshape(-1)[::STRIDE].float().numpy())
    index[name] = {"sha256": digest, "shape": list(raw.shape), "dtype": str(raw.dtype)}
    print(f"{name:28s} {tuple(raw.shape)} {digest[:16]}", flush=True)


def write(out_dir):
    from wild_visual_navigation_b200 import ops

    os.makedirs(out_dir, exist_ok=True)
    index = {}
    dev = "cuda"

    # ---- attention at the c3 and c5 shapes
    for tag, (B, H, N, std) in {"c3": (32, 6, 3137, 1.8), "c5": (128, 12, 4097, 1.8)}.items():
        g = torch.Generator(device=dev).manual_seed(11)
        npad = (N + 127) // 128 * 128
        q = (torch.randn(B, H, npad, 64, device=dev, generator=g) * std).bfloat16()
        k = (torch.randn(B, H, npad, 64, device=dev, generator=g) * std).bfloat16()
        vt = torch.randn(B, H, 64, npad, device=dev, generator=g).bfloat16()
        _record(out_dir, f"attention_{tag}", ops.attention(q, k, vt, N, 0.125), index)
        del q, k, vt
        torch.cuda.empty_cache()

    # ---- the four ViT-S GEMMs of c3 with their epilogues
    M, D = 32 * 3200, 384
    g = torch.Generator(device=dev).manual_seed(12)
    x = (torch.randn(M, D, device=dev, generator=g)).bfloat16()
    h = (torch.randn(M, 4 * D, device=dev, generator=g) * 0.5).bfloat16()
    for name, (a, n, kind, act) in {
        "gemm_qkv": (x, 3 * D, ops.OUT_BF16, ops.ACT_NONE),
        "gemm_proj_resid": (x, D, ops.OUT_RESID_F32, ops.ACT_NONE),
        "gemm_fc1_gelu": (x, 4 * D, ops.OUT_BF16, ops.ACT_GELU),
        "gemm_fc2_resid": (h, D, ops.OUT_RESID_F32, ops.ACT_NONE),
    }.items():
        w = (torch.randn(n, a.shape[1], device=dev, generator=g) * a.shape[1] ** -0.5).bfloat16()
        bias = torch.randn(n, device=dev, generator=g) * 0.1
        out = None
        if kind == ops.OUT_RESID_F32:
            out = torch.randn(M, n, device=dev, generator=g)
        _record(out_dir, name, ops.gemm_bf16(a, w, bias, out_kind=kind, act=act, out=out), index)
    del x, h
    torch.cuda.empty_cache()

    # ---- DinoInterface tokens (ViT-S/8 @448, B = 32) and the fused per-pixel maps on them
    from oracle.dino_vit import ViTConfig, synthetic_state_dict
    from wild_visual_navigation_b200 import ConfidenceGenerator, SimpleMLP, TraversabilityInference
    from wild_visual_navigation_b200.feature_extractor import DinoInterface

    cfg = ViTConfig.from_name("vit_small", 8, 448)
    sd = synthetic_state_dict(cfg, seed=1)
    di = DinoInterface(dev, input_size=448, backbone_type="vit_small", patch_size=8, state_dict=sd, max_batch=32)
    img = torch.rand(32, 3, 448, 448, generator=torch.Generator().manual_seed(0)).to(dev)
    tokens = di.inference_tokens(img)
    _record(out_dir, "dino_tokens_c3", tokens, index)

    torch.manual_seed(42)
    model = SimpleMLP(384, [256, 32, 1], True).to(dev)
    cg = ConfidenceGenerator(std_factor=0.5, method="latest_measurement").to(dev)
    with torch.no_grad():
        cg.mean[0], cg.std[0] = 0.3, 0.1
    trav, conf = TraversabilityInference(di, model, cg).predict_from_tokens(tokens, 448)
    _record(out_dir, "pixel_trav", trav, index)
    _record(out_dir, "pixel_conf", conf, index)
    del di, tokens
    torch.cuda.empty_cache()

    # ---- the patch-16 loader and patch-embed GEMM (K = 768): DINO ViT-S/16 @448, B = 8
    cfg16 = ViTConfig.from_name("vit_small", 16, 448)
    di16 = DinoInterface(dev, input_size=448, backbone_type="vit_small", patch_size=16,
                         state_dict=synthetic_state_dict(cfg16, seed=1), max_batch=8)
    _record(out_dir, "dino_tokens_s16", di16.inference_tokens(img[:8]), index)
    torch.cuda.synchronize()

    with open(os.path.join(out_dir, "index.json"), "w") as f:
        json.dump(index, f, indent=1)


def compare(dir_a, dir_b):
    ia = json.load(open(os.path.join(dir_a, "index.json")))
    ib = json.load(open(os.path.join(dir_b, "index.json")))
    same = True
    for name in ia:
        if name not in ib:
            print(f"{name:28s} missing in {dir_b}")
            same = False
            continue
        if ia[name]["sha256"] == ib[name]["sha256"]:
            print(f"{name:28s} bit-identical")
            continue
        same = False
        sa, sb = np.load(os.path.join(dir_a, name + ".npy")), np.load(os.path.join(dir_b, name + ".npy"))
        d = np.abs(sa.astype(np.float64) - sb.astype(np.float64))
        print(f"{name:28s} DIFFERENT: sampled max |diff| {d.max():.3e}, {int((d > 0).sum())} of {d.size} samples differ")
    print("ALL BIT-IDENTICAL" if same else "OUTPUTS DIFFER")
    return 0 if same else 1


if __name__ == "__main__":
    if len(sys.argv) == 3 and sys.argv[1] == "write":
        write(sys.argv[2])
    elif len(sys.argv) == 4 and sys.argv[1] == "compare":
        sys.exit(compare(sys.argv[2], sys.argv[3]))
    else:
        sys.exit(__doc__)
