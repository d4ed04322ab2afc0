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
  * the fused per-pixel maps of a seeded DoubleMLP(384, [64, 32, 1]) on the first 8 frames of those tokens, from the
    fp32 tokens (MlpInference.pixels) and from the backbone's own bf16 copy (MlpInference.pixels_from_vit);
  * FlowInference.pixels (traversability and NLL) of a seeded LinearRnvp(384, [200]) on those tokens;
  * DinoInterface tokens of ViT-S/16 @448 at B = 8 (the patch-16 loader and patch-embed GEMM);
  * the taps of seeded ResNet-18, ResNet-50 and EfficientNet-B0 trunks at 448, B = 4;
  * DinoInterface tokens of DINOv2 ViT-S/14-reg and ViT-L/14 @224 at B = 4;
  * StegoInterface (ViT-S/8 @224, B = 4, flip TTA): the flip-averaged head output and the linear / cluster segments;
  * DenseCrf.run on that head output (cluster-probe labels and Q, linear-probe labels) and DenseCrf.workspace_bytes;
  * ops.mlp_forward_f32 of that SimpleMLP at R = 4096 and 65536 rows;
  * MlpInference.rows_padded of that SimpleMLP and of the DoubleMLP (6 groups of 700 rows, partly live);
  * GcnInference.rows_padded of a seeded SimpleGCN(384, True, [256, 128, 1]) on the same rows with seeded edges;
  * FlowInference.rows (z, log_det, logprob) of a seeded LinearRnvp(384, [200]) at R = 4096;
  * after three train steps of each learner (MlpTrainer, DoubleMlpTrainer, GcnTrainer, FlowTrainer) created for
    1024 rows, at R = 1024, 800 and 1500 (the last one replaces the handle by a larger one and copies its generator
    over), per confidence method: the parameters, Adam's moments, the confidence vector, the metrics and the
    generator's mean / std / var / running sums.
`compare` reports, per output, whether the two builds agree bit for bit and, where not, the largest difference in
the samples.  Every output here except the SimpleMLP train record is deterministic for a given build (no atomics race
in them), so any difference there is the build's.  The fused SimpleMLP step adds its per-row and per-tile sums with
atomics, so its record (mlp_train_*) can differ in the last bits between two runs of the same build.
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
    print(f"{name:44s} {tuple(raw.shape)} {digest[:16]}", flush=True)


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

    from wild_visual_navigation_b200 import DoubleMLP

    torch.manual_seed(42)
    double = DoubleMLP(384, [64, 32, 1]).to(dev)
    dmi = ops.MlpInference(384, 64, 32, double=True)
    dmi.set_params(double.flat_params)
    for name, (t, c) in {
        "pixels": dmi.pixels(tokens[:8].contiguous(), (56, 56), (448, 448), cg.mean, cg.std, 0.5),
        "pixels_vit": dmi.pixels_from_vit(di._model, 8, (448, 448), cg.mean, cg.std, 0.5),
    }.items():
        _record(out_dir, f"double_mlp_{name}_trav", t, index)
        _record(out_dir, f"double_mlp_{name}_conf", c, index)

    from wild_visual_navigation_b200 import LinearRnvp

    torch.manual_seed(42)
    flow = LinearRnvp(384, [200], use_permutation=True).to(dev)
    fi = ops.FlowInference(384, 200)
    fi.set_params(flow.flat_params)
    t, nll = fi.pixels(flow, tokens, (56, 56), (448, 448), cg.mean, cg.std, 0.5, want_nll=True)
    _record(out_dir, "flow_pixels_trav", t, index)
    _record(out_dir, "flow_pixels_nll", nll, index)
    del di, tokens, fi
    torch.cuda.empty_cache()

    # ---- the patch-16 loader and patch-embed GEMM (K = 768): DINO ViT-S/16 @448, B = 8
    cfg16 = ViTConfig.from_name("vit_small", 16, 448)
    di16 = DinoInterface(dev, input_size=448, backbone_type="vit_small", patch_size=16,
                         state_dict=synthetic_state_dict(cfg16, seed=1), max_batch=8)
    _record(out_dir, "dino_tokens_s16", di16.inference_tokens(img[:8]), index)
    del di16
    torch.cuda.empty_cache()

    # ---- the convolutional trunks: ResNet-18 / ResNet-50 and EfficientNet-B0 taps @448, B = 4
    from wild_visual_navigation_b200.feature_extractor import weights as W

    for depth in (18, 50):
        rn = ops.ResNetBackbone(448, depth, W.fold_resnet_bn(W.synthetic_resnet_state_dict(depth, seed=1), depth),
                                max_batch=4)
        for i, t in enumerate(rn.forward(img[:4])):
            _record(out_dir, f"resnet{depth}_tap{i + 1}", t, index)
        del rn
    en = ops.EfficientNetBackbone(448, W.fold_efficientnet_bn(W.synthetic_efficientnet_b0_state_dict(seed=1)),
                                  max_batch=4)
    for i, t in enumerate(en.forward(img[:4])):
        _record(out_dir, f"effnet_b0_tap{i + 1}", t, index)
    del en
    torch.cuda.empty_cache()

    # ---- DINOv2 ViT-S/14-reg and ViT-L/14 tokens @224, B = 4
    img224 = torch.rand(4, 3, 224, 224, generator=torch.Generator().manual_seed(1)).to(dev)
    for name, backbone, vit_type in (("dinov2_reg_s14", "dinov2_reg", "vit_small"), ("dinov2_l14", "dinov2", "vit_large")):
        s = W.VIT_SHAPES[vit_type]
        make = W.synthetic_dinov2_reg_state_dict if backbone == "dinov2_reg" else W.synthetic_dinov2_state_dict
        dv = DinoInterface(dev, backbone=backbone, input_size=224, backbone_type=vit_type,
                           state_dict=make(s["dim"], s["depth"], s["mlp_dim"], seed=5), max_batch=4)
        _record(out_dir, f"{name}_tokens", dv.inference_tokens(img224), index)
        del dv
        torch.cuda.empty_cache()

    # ---- the STEGO head with flip TTA (ViT-S/8 @224, B = 4) and its segments
    from wild_visual_navigation_b200.feature_extractor import StegoInterface

    si = StegoInterface(dev, input_size=224, backbone_type="vit_small", patch_size=8, flip_tta=True, max_batch=4,
                        backbone_state_dict=synthetic_state_dict(ViTConfig.from_name("vit_small", 8, 224), seed=6),
                        head_state_dict=W.synthetic_stego_head(384, 90, 32, 27, seed=3))
    linear, cluster = si.inference(img224)
    _record(out_dir, "stego_head_tta", si._head_out, index)
    _record(out_dir, "stego_linear_segments", linear, index)
    _record(out_dir, "stego_cluster_segments", cluster, index)
    _, _, npad, grid, _ = si._geom
    crf = ops.DenseCrf(224, max(si._n_clusters, si._n_classes), chunk=2)
    _record(out_dir, "crf_workspace_bytes", torch.tensor([crf.workspace_bytes], dtype=torch.int64), index)
    labels, q = crf.run(img224, si._head_out, npad, grid, W.HEAD_CLUSTER_COL, si._n_clusters, W.HEAD_CODE_COL,
                        si._code_dim, 2.0, want_q=True)
    _record(out_dir, "crf_cluster_labels", labels, index)
    _record(out_dir, "crf_cluster_q", q, index)
    _record(out_dir, "crf_linear_labels", crf.run(img224, si._head_out, npad, grid, W.HEAD_LINEAR_COL, si._n_classes),
            index)
    del si, crf
    torch.cuda.empty_cache()

    # ---- the fp32 CUDA-core paths: SimpleMLP forward, LinearRnvp row forward and train step
    g = torch.Generator(device=dev).manual_seed(13)
    for R in (4096, 65536):
        x = torch.randn(R, 384, device=dev, generator=g) * 0.5
        _record(out_dir, f"mlp_forward_f32_{R}", ops.mlp_forward_f32(model.flat_params, x, 384, 256, 32), index)

    feat = torch.randn(6, 700, 384, device=dev, generator=g) * 0.5
    n_rows = torch.tensor([700, 0, 1, 350, 699, 128], device=dev, dtype=torch.int32)
    for name, (m, mi) in {"mlp": (model, ops.MlpInference(384, 256, 32)),
                          "double_mlp": (double, ops.MlpInference(384, 64, 32, double=True))}.items():
        mi.set_params(m.flat_params)
        t, c = mi.rows_padded(feat, n_rows, cg.mean, cg.std, 0.5)
        _record(out_dir, f"{name}_rows_padded_trav", t, index)
        _record(out_dir, f"{name}_rows_padded_conf", c, index)

    from wild_visual_navigation_b200 import SimpleGCN

    torch.manual_seed(42)
    gcn = SimpleGCN(384, True, [256, 128, 1]).to(dev)
    edges = torch.randint(0, 700, (6, 2100, 2), device=dev, generator=g)
    n_edges = torch.tensor([2100, 0, 5, 1000, 2100, 300], device=dev, dtype=torch.int32)
    t, c = ops.GcnInference(gcn, max_rows=6 * 700, max_edges=6 * 2100).rows_padded(feat, n_rows, edges, n_edges, cg.mean,
                                                                                   cg.std, 0.5)
    _record(out_dir, "gcn_rows_padded_trav", t, index)
    _record(out_dir, "gcn_rows_padded_conf", c, index)

    x = torch.randn(4096, 384, device=dev, generator=g) * 0.5
    rows = ops.FlowInference(384, 200, max_rows=4096).rows(flow, x)
    for k in ("z", "log_det", "logprob"):
        _record(out_dir, f"flow_rows_{k}", rows[k], index)

    # ---- the four learners' train steps, with a regrowth in the last step
    def learner(kind):
        torch.manual_seed(42)
        if kind == "mlp":
            m = SimpleMLP(384, [256, 32, 1], True).to(dev)
            return m, ops.MlpTrainer(m.flat_params, 384, 256, 32, max_rows=1024)
        if kind == "double_mlp":
            m = DoubleMLP(384, [64, 32, 1]).to(dev)
            return m, ops.DoubleMlpTrainer(m, max_rows=1024)
        if kind == "gcn":
            m = SimpleGCN(384, True, [256, 128, 1]).to(dev)
            return m, ops.GcnTrainer(m, max_rows=1024, max_edges=4096)
        m = LinearRnvp(384, [200], use_permutation=True).to(dev)
        return m, ops.FlowTrainer(m, max_rows=1024)

    for kind in ("mlp", "double_mlp", "gcn", "flow"):
        for method in ("latest_measurement", "running_mean", "kalman_filter", "moving_average"):
            m, tr = learner(kind)
            cg = ConfidenceGenerator(std_factor=0.5, method=method).to(dev)
            tr.cg_mean, tr.cg_std = cg.mean.data, cg.std.data
            kf = getattr(cg, "_kalman_filter", None)
            tr.set_confidence(cg.method_id, cg.var.data, getattr(cg, "running_n", None),
                              getattr(cg, "running_sum", None), getattr(cg, "running_sum_of_squares", None),
                              kf_proc_cov=float(kf.proc_cov.item()) if kf is not None else 0.2,
                              kf_meas_cov=float(kf.meas_cov.item()) if kf is not None else 1.0)
            gs = torch.Generator(device=dev).manual_seed(14)
            for R in (1024, 800, 1500):
                x = torch.randn(R, 384, device=dev, generator=gs) * 0.5
                y = torch.rand(R, device=dev, generator=gs)
                yv = torch.rand(R, device=dev, generator=gs) < 0.4
                if kind == "gcn":
                    ei = torch.randint(0, R, (2, 3 * R), device=dev, generator=gs)
                    conf = tr.step(x, ei, y, yv)
                elif kind == "flow":
                    conf = tr.step(x)   # every row labelled: the whole confidence vector is live
                else:
                    conf = tr.step(x, y, yv)
            assert tr.max_rows > 1024
            out = {"params": m.flat_params, "exp_avg": tr.exp_avg, "exp_avg_sq": tr.exp_avg_sq, "conf": conf,
                   "metrics": tr.metrics, "cg_mean": cg.mean, "cg_std": cg.std, "cg_var": cg.var}
            for k in ("running_n", "running_sum", "running_sum_of_squares"):
                if hasattr(cg, k):
                    out["cg_" + k] = getattr(cg, k)
            for k, t in out.items():
                _record(out_dir, f"{kind}_train_{method}_{k}", t, index)
    torch.cuda.synchronize()

    with open(os.path.join(out_dir, "index.json"), "w") as f:
        json.dump(index, f, indent=1)


def compare(dir_a, dir_b):
    ia = json.load(open(os.path.join(dir_a, "index.json")))
    ib = json.load(open(os.path.join(dir_b, "index.json")))
    same = True
    for name in ia:
        if name not in ib:
            print(f"{name:44s} missing in {dir_b}")
            same = False
            continue
        if ia[name]["sha256"] == ib[name]["sha256"]:
            print(f"{name:44s} bit-identical")
            continue
        same = False
        sa, sb = np.load(os.path.join(dir_a, name + ".npy")), np.load(os.path.join(dir_b, name + ".npy"))
        d = np.abs(sa.astype(np.float64) - sb.astype(np.float64))
        print(f"{name:44s} DIFFERENT: sampled max |diff| {d.max():.3e}, {int((d > 0).sum())} of {d.size} samples differ")
    print("ALL BIT-IDENTICAL" if same else "OUTPUTS DIFFER")
    return 0 if same else 1


if __name__ == "__main__":
    if len(sys.argv) == 3 and sys.argv[1] == "write":
        write(sys.argv[2])
    elif len(sys.argv) == 4 and sys.argv[1] == "compare":
        sys.exit(compare(sys.argv[2], sys.argv[3]))
    else:
        sys.exit(__doc__)
