"""Tensor-level wrappers over the C ABI (include/wvn_b200.h).

Everything here is plumbing: allocate outputs with torch, pass raw pointers + the current stream
to libwvn_b200.so.  The classes in ``feature_extractor/``, ``model/``, ``utils/`` and
``traversability_estimator/`` (the reference's API surface) are built on these.
"""
from __future__ import annotations

import ctypes
import math
from ctypes import byref, c_void_p

import torch
import torch.nn.functional as F

from . import _C
from ._C import EffnetConfig, FlowBuffers, ResnetConfig, TrainConfig, VitConfig, check, lib, ptr, stream

OUT_BF16, OUT_F32, OUT_RESID_F32 = 0, 1, 2
ACT_NONE, ACT_RELU, ACT_GELU, ACT_SILU = 0, 1, 2, 3


# --------------------------------------------------------------------------------------------
# primitives
# --------------------------------------------------------------------------------------------
def gemm_bf16(a, w, bias=None, out_kind=OUT_BF16, act=ACT_NONE, out=None, block_n=0):
    """out = act(a @ w.T + bias).  a: [M,K] bf16, w: [N,K] bf16 with rows round_up(K, 8) apart, bias: [N] f32."""
    M, K = a.shape
    N = w.shape[0]
    assert w.stride(0) == (K + 7) // 8 * 8 and w.stride(1) == 1, "gemm_bf16: w rows must be round_up(K, 8) elements apart"
    if out is None:
        out = torch.empty(M, N, device=a.device, dtype=torch.bfloat16 if out_kind == OUT_BF16 else torch.float32)
    check(lib().wvn_gemm_bf16(ptr(a), a.stride(0), ptr(w), ptr(bias), ptr(out), out.stride(0), M, N, K, out_kind, act,
                              block_n, stream()))
    return out


def attention(q, k, vt, n_valid, scale=0.125):
    """q,k: [B,H,npad,64] bf16; vt: [B,H,64,npad] bf16 -> [B,npad,H*64] bf16."""
    B, H, npad, dh = q.shape
    assert dh == 64
    out = torch.empty(B, npad, H * 64, device=q.device, dtype=torch.bfloat16)
    check(lib().wvn_attention_bf16(ptr(q), ptr(k), ptr(vt), ptr(out), B, H, npad, n_valid, scale, stream()))
    return out


def layernorm(x, gamma, beta, eps=1e-6, *, out=None, out_f32=None, npad=0, n_valid=0, row0=1, reverse=False):
    """LayerNorm of fp32 rows x [rows, dim] -> bf16 rows (``out``, allocated when None).  ``out_f32`` (optional) receives
    the fp32 result of rows [row0, n_valid) of each npad-row frame, compacted (see wvn_layernorm_ex)."""
    rows, dim = x.shape
    if out is None:
        out = torch.empty(rows, dim, device=x.device, dtype=torch.bfloat16)
    check(lib().wvn_layernorm_ex(ptr(x), ptr(gamma), ptr(beta), ptr(out), ptr(out_f32), rows, dim, eps, npad, n_valid,
                                 row0, int(reverse), stream()))
    return out


def image_to_patches(img, image_size, patch, resized_hw=None, batch=None, frame0=0, src_frames=None, flip_from=None,
                     out=None):
    """The ViT patch loader on its own: img (S,3,H,W) fp32 or (S,H,W,3) uint8 -> bf16 patch rows
    [batch * g * g, round_up(3 p^2, 8)] (g = image_size // patch), pad columns left as they are.  Output frame f is
    source frame (frame0 + f) % src_frames, horizontally flipped when frame0 + f >= flip_from (see
    wvn_image_to_patches)."""
    img = img.contiguous()
    u8 = img.dtype == torch.uint8
    S, H, W = (img.shape[0], img.shape[1], img.shape[2]) if u8 else (img.shape[0], img.shape[2], img.shape[3])
    rh, rw = _resized_size(H, W, image_size) if resized_hw is None else resized_hw
    batch = S if batch is None else batch
    src_frames = S if src_frames is None else src_frames
    flip_from = (1 << 30) if flip_from is None else flip_from
    g = image_size // patch
    if out is None:
        out = torch.empty(batch * g * g, (3 * patch * patch + 7) // 8 * 8, device=img.device, dtype=torch.bfloat16)
    check(lib().wvn_image_to_patches(ptr(img), int(u8), batch, H, W, rh, rw, image_size, patch, frame0, src_frames,
                                     flip_from, ptr(out), stream()))
    return out


def init_token_rows(x, cls, pos, reg, n_valid):
    """In place on x [B, npad, D] fp32: CLS row cls + pos[0], register rows reg [R, D] (or None), padding rows 0."""
    B, npad, D = x.shape
    R = 0 if reg is None else reg.shape[0]
    check(lib().wvn_init_token_rows(ptr(x), ptr(cls), ptr(pos), ptr(reg), R, B, npad, n_valid, D, stream()))


def attention_f32_debug(qkv, batch, heads, npad, n_valid, scale=0.125, out=None):
    """fp32 parity-debug attention: qkv [batch * npad, 3 * heads * 64] fp32 -> [batch * npad, heads * 64] bf16."""
    if out is None:
        out = torch.empty(batch * npad, heads * 64, device=qkv.device, dtype=torch.bfloat16)
    check(lib().wvn_attention_f32_debug(ptr(qkv), ptr(out), batch, heads, npad, n_valid, heads * 64, scale, stream()))
    return out


def upsample_dense(tokens, gh, gw, out_h, out_w):
    """tokens [B, gh*gw, D] f32 -> (B, D, out_h, out_w) f32, bilinear align_corners=True."""
    B, P, D = tokens.shape
    out = torch.empty(B, D, out_h, out_w, device=tokens.device, dtype=torch.float32)
    check(lib().wvn_upsample_dense(ptr(tokens), ptr(out), B, D, gh, gw, out_h, out_w, stream()))
    return out


def logits_argmax(logits, col0, classes, batch, npad, gh, gw, out_h, out_w, col0_b=0, classes_b=0):
    """Per-pixel argmax of bilinearly (align_corners=False) upsampled class logits.  With a second
    column range the two segmentations come out of one pass: returns seg or (seg, seg_b)."""
    seg = torch.empty(batch, out_h, out_w, device=logits.device, dtype=torch.int64)
    seg_b = torch.empty_like(seg) if classes_b > 0 else None
    check(lib().wvn_logits_argmax(ptr(logits), logits.stride(0), col0, classes, col0_b, classes_b, batch, npad, gh, gw,
                                  out_h, out_w, ptr(seg), ptr(seg_b), stream()))
    return seg if seg_b is None else (seg, seg_b)


_WS_CACHE = {}


def _workspace(tag, nbytes, device):
    """Scratch that the kernels fully (re)initialise themselves: one buffer per (tag, device), grown on demand, so the
    per-frame calls do not allocate."""
    key = (tag, str(device))
    buf = _WS_CACHE.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty(max(int(nbytes), 1), device=device, dtype=torch.uint8)
        _WS_CACHE[key] = buf
    return buf


def segment_reduce(seg, smax, tokens=None, grid=None, want_centers=True, want_edges=True, max_edges=None):
    """seg: [B,H,W] int64.  Returns dict(feat [B,smax,D] | None, centers [B,smax,2] | None,
    edges [B,max_edges,2] | None, n_edges [B] int32 | None).  Only the first n_edges[b] rows of edges[b] are written
    (n_edges[b] < 0 flags an overflow of max_edges)."""
    B, H, W = seg.shape
    dev = seg.device
    if tokens is not None:
        gh, gw = grid
        D = tokens.shape[-1]
    else:
        gh = gw = 1
        D = 0
    ws_bytes = lib().wvn_segment_workspace_bytes(B, smax, gh, gw)
    ws = _workspace("segment_reduce", ws_bytes, dev)
    feat = torch.empty(B, smax, D, device=dev, dtype=torch.float32) if tokens is not None else None
    centers = torch.empty(B, smax, 2, device=dev, dtype=torch.float32) if want_centers else None
    if want_edges:
        if max_edges is None:
            # STEGO cluster labels are not connected regions: the directed label-pair count can reach smax*(smax-1),
            # so the planar-graph bound only applies to large segment counts (SLIC-like, <= 1024 here: 16 MB worst case)
            max_edges = smax * smax if smax <= 256 else min(smax * smax, 64 * smax)
        edges = torch.empty(B, max_edges, 2, device=dev, dtype=torch.int64)
        n_edges = torch.empty(B, device=dev, dtype=torch.int32)
    else:
        max_edges, edges, n_edges = 0, None, None
    check(lib().wvn_segment_reduce(ptr(seg), B, H, W, smax, ptr(tokens), gh, gw, D, ptr(feat), ptr(centers), ptr(edges),
                                   ptr(n_edges), max_edges, ptr(ws), stream()))
    return {"feat": feat, "centers": centers, "edges": edges, "n_edges": n_edges, "max_edges": max_edges}


def pool_supervision(seg: torch.Tensor, mask: torch.Tensor, smax: int):
    """Per-segment supervision labels (MissionNode.update_supervision_signal, nodes.py:400-440).
    seg (B,H,W) int64; mask (B,C,H,W) or (B,H,W) fp32 with NaN = unlabelled -> y (B,smax) f32, y_valid (B,smax) bool."""
    _C.require_device()
    if mask.dim() == 3:
        mask = mask[:, None]
    B, C, H, W = mask.shape
    assert seg.shape == (B, H, W) and seg.dtype == torch.int64 and mask.dtype == torch.float32
    seg, mask = seg.contiguous(), mask.contiguous()
    y = torch.empty(B, smax, device=seg.device, dtype=torch.float32)
    valid = torch.empty(B, smax, device=seg.device, dtype=torch.uint8)
    ws = torch.empty(B, smax, device=seg.device, dtype=torch.float32)
    check(lib().wvn_supervision_pool(ptr(seg), ptr(mask), B, C, H, W, smax, ptr(y), ptr(valid), ptr(ws), stream()))
    return y, valid.bool()


_slic_luts = {}


def slic_tables():
    """Host lookup tables of the library's 8-bit sRGB -> CIELAB conversion as int32 numpy arrays (g256, m9, f4096)."""
    import ctypes

    import numpy as np

    g, m, f = np.zeros(256, np.int32), np.zeros(9, np.int32), np.zeros(4096, np.int32)
    lib().wvn_slic_tables(g.ctypes.data_as(ctypes.c_void_p), m.ctypes.data_as(ctypes.c_void_p),
                          f.ctypes.data_as(ctypes.c_void_p))
    return g, m, f


def slic_geometry(h, w, num_components):
    """-> (grid interval S, nx, ny); the segmentation has nx * ny clusters."""
    import ctypes

    S, nx, ny = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    check(lib().wvn_slic_geometry(h, w, num_components, ctypes.byref(S), ctypes.byref(nx), ctypes.byref(ny)))
    return S.value, nx.value, ny.value


def slic(img, num_components=100, compactness=10.0, iters=10):
    """SLIC superpixels of img (B,3,H,W) fp32 in [0,1] -> labels (B,H,W) int64 in [0, nx*ny) (see include/wvn_b200.h)."""
    _C.require_device()
    B, C, H, W = img.shape
    assert C == 3 and img.dtype == torch.float32
    img = img.contiguous()
    key = str(img.device)
    if key not in _slic_luts:
        _slic_luts[key] = tuple(torch.from_numpy(t).to(img.device) for t in slic_tables())
    g, m, f = _slic_luts[key]
    ws = _workspace("slic", lib().wvn_slic_workspace_bytes(B, H, W, num_components), img.device)
    labels = torch.empty(B, H, W, device=img.device, dtype=torch.int64)
    check(lib().wvn_slic(ptr(img), B, H, W, num_components, float(compactness), iters, ptr(g), ptr(m), ptr(f), ptr(labels),
                         ptr(ws), stream()))
    return labels


def project_and_render(sK, pose_camera_in_world, points, colors, h, w, render=True, supervision=None, traversability=None):
    """Footprint projection + rasterisation (ImageProjector.project_and_render, image_projector.py:152-197).
    sK (B,4,4) scaled camera matrices, pose (B,4,4), points (B,N,3), colors (B,3) | (3,) | None.
    -> (masks (B,3,h,w) or None, projected (B,N,2), valid (B,N) bool); ``supervision`` (B,3,h,w) is updated in place
    with fmin(supervision, mask * traversability) (traversability_estimator.py:281-284)."""
    _C.require_device()
    B, N = points.shape[0], points.shape[1]
    dev = points.device
    sK, pose, points = sK.float().contiguous(), pose_camera_in_world.float().contiguous(), points.float().contiguous()
    assert sK.shape == (B, 4, 4) and pose.shape == (B, 4, 4) and points.shape == (B, N, 3)
    if colors is not None:
        colors = colors.to(dev, torch.float32).contiguous()
        assert colors.shape in ((3,), (B, 3))
    masks = torch.empty(B, 3, h, w, device=dev, dtype=torch.float32) if render else None
    proj = torch.empty(B, N, 2, device=dev, dtype=torch.float32)
    valid = torch.empty(B, N, device=dev, dtype=torch.uint8)
    if supervision is not None:
        assert supervision.shape == (B, 3, h, w) and supervision.dtype == torch.float32 and supervision.is_contiguous()
    if traversability is not None:
        traversability = traversability.to(dev, torch.float32).reshape(-1)[:1].contiguous()
    check(lib().wvn_project_and_render(ptr(sK), ptr(pose), ptr(points), ptr(colors),
                                       int(colors is not None and colors.dim() == 2), B, N, h, w, ptr(traversability),
                                       ptr(masks), ptr(proj), ptr(valid), ptr(supervision), stream()))
    return masks, proj, valid.bool()


def mission_propagate_workspace(max_slots, smax, device):
    """The zeroed workspace wvn_mission_propagate needs for up to ``max_slots`` list entries (every call leaves it zero)."""
    return torch.zeros(max(int(lib().wvn_mission_propagate_workspace_bytes(max_slots, smax)), 1), device=device,
                       dtype=torch.uint8)


def mission_propagate(slots, restart, K, pose, points, traversability, seg, mask, y, y_valid, slot_valid, workspace):
    """One supervision event into the listed mission-graph slots (see include/wvn_b200.h): slots [n] int32, restart [n]
    uint8 or None, points [N,3] and traversability [1] fp32, all on the device; per slot K / pose [cap,4,4], seg [cap,H,W]
    int32, mask [cap,H,W] fp32 (updated in place), y [cap,smax] fp32, y_valid [cap,smax] uint8, slot_valid [cap] int32 or
    None.  Enqueued on the current stream; nothing is allocated and nothing waits for the device."""
    n, smax = slots.numel(), y.shape[1]
    H, W = mask.shape[1], mask.shape[2]
    assert slots.dtype == torch.int32 and seg.dtype == torch.int32 and mask.dtype == torch.float32
    assert seg.shape == mask.shape and y_valid.shape == y.shape and y_valid.dtype == torch.uint8
    assert workspace.numel() >= lib().wvn_mission_propagate_workspace_bytes(n, smax)
    check(lib().wvn_mission_propagate(ptr(slots), ptr(restart), n, ptr(K), ptr(pose), ptr(points), points.shape[0],
                                      ptr(traversability), ptr(seg), ptr(mask), H, W, smax, ptr(y), ptr(y_valid),
                                      ptr(slot_valid), ptr(workspace), stream()))


def flip_average(head, batch, npad, grid):
    """STEGO flip-TTA merge of the head output [2*batch*npad, C] in place (see include/wvn_b200.h)."""
    assert head.is_contiguous() and head.shape[0] == 2 * batch * npad and head.dtype == torch.float32
    check(lib().wvn_flip_average(ptr(head), batch, npad, grid, head.stride(0), stream()))


def stego_kmeans(head, batch, npad, patches, code_col, code_dim, logit_col, k, iters, centroids_out=None):
    """Per-image k-means of the code columns of the head output ``head`` [batch*npad, ld]; leaves the per-patch
    nearest-centroid scores in columns [logit_col, logit_col + k) (see include/wvn_b200.h)."""
    ws = _workspace("stego_kmeans", lib().wvn_stego_kmeans_workspace_bytes(batch, k, code_dim), head.device)
    check(lib().wvn_stego_kmeans(ptr(head), head.stride(0), batch, npad, patches, code_col, code_dim, logit_col, k, iters,
                                 ptr(centroids_out), ptr(ws), stream()))


def relabel(seg, num_labels):
    """In-place relabel of each frame of seg [B,H,W] to 0..S-1; returns counts [B] int32."""
    B = seg.shape[0]
    scratch = _workspace("relabel", 4 * B * num_labels, seg.device).view(torch.int32)[: B * num_labels]
    counts = torch.empty(B, device=seg.device, dtype=torch.int32)
    check(lib().wvn_segment_relabel(ptr(seg), B, seg[0].numel(), num_labels, ptr(scratch), ptr(counts), stream()))
    return counts


def segment_maps(seg, n_rows, trav, conf=None):
    """Paints per-segment values into per-pixel maps: seg [B, H, W] int64 or int32, n_rows [B] int32 and trav / conf
    [B, smax] fp32 on the device -> (trav_map, conf_map) [B, H, W] fp32 with map[b, p] = v[b, seg[b, p]], NaN where
    the id is outside [0, n_rows[b]).  conf_map is None when conf is.  One kernel, no host synchronisation."""
    assert seg.dtype in (torch.int64, torch.int32), "segment_maps: seg must be int64 or int32"
    assert n_rows.dtype == torch.int32 and trav.dtype == torch.float32 and trav.dim() == 2
    B, smax = trav.shape
    assert seg.shape[0] == B and n_rows.shape == (B,), "segment_maps: seg, n_rows and trav disagree on the batch"
    seg, trav = seg.contiguous(), trav.contiguous()
    tmap = torch.empty(seg.shape, device=seg.device, dtype=torch.float32)
    cmap = None
    if conf is not None:
        assert conf.shape == trav.shape and conf.dtype == torch.float32
        conf = conf.contiguous()
        cmap = torch.empty_like(tmap)
    hw = seg[0].numel() if B > 0 else 0
    check(lib().wvn_segment_maps(ptr(seg), int(seg.dtype == torch.int64), B, hw, ptr(trav), ptr(conf), smax,
                                 ptr(n_rows), ptr(tmap), ptr(cmap), stream()))
    return tmap, cmap


# --------------------------------------------------------------------------------------------
# ViT backbone handle
# --------------------------------------------------------------------------------------------
def interpolate_pos_embed(pos_embed: torch.Tensor, grid: int) -> torch.Tensor:
    """DINO's interpolate_pos_encoding (bicubic, +0.1 trick), done once at weight-load time.  DINOv2's is the same
    formula from its 37 x 37 pre-training grid (the side is read off ``pos_embed``)."""
    n_pre = pos_embed.shape[1] - 1
    if n_pre == grid * grid:
        return pos_embed
    dim = pos_embed.shape[-1]
    side = int(math.sqrt(n_pre))
    w0 = h0 = grid + 0.1
    patch = F.interpolate(pos_embed[:, 1:].reshape(1, side, side, dim).permute(0, 3, 1, 2).float(),
                          scale_factor=(h0 / side, w0 / side), mode="bicubic")
    patch = patch.permute(0, 2, 3, 1).reshape(1, -1, dim)
    return torch.cat((pos_embed[:, :1], patch), dim=1)


def interpolate_pos_embed_antialias(pos_embed: torch.Tensor, grid: int) -> torch.Tensor:
    """The interpolation of the DINOv2 register models (hub ``interpolate_antialias=True, interpolate_offset=0``):
    bicubic with antialias straight to ``size=(grid, grid)``, no +0.1 trick.  The CLS row passes through."""
    n_pre = pos_embed.shape[1] - 1
    if n_pre == grid * grid:
        return pos_embed
    dim = pos_embed.shape[-1]
    side = int(math.sqrt(n_pre))
    patch = F.interpolate(pos_embed[:, 1:].reshape(1, side, side, dim).permute(0, 3, 1, 2).float(),
                          size=(grid, grid), mode="bicubic", antialias=True)
    patch = patch.permute(0, 2, 3, 1).reshape(1, -1, dim)
    return torch.cat((pos_embed[:, :1], patch), dim=1)


def fold_layerscale(sd: dict, depth: int) -> dict:
    """DINOv2's LayerScale ``x += gamma * f(x)`` folded into the layer that ends f, in fp32 before any bf16 cast:
    ``attn.proj`` weight rows and bias times ``ls1.gamma``, ``mlp.fc2`` (``mlp.w3`` of a SwiGLU FFN) weight rows and
    bias times ``ls2.gamma`` (at least fp32; a float64 state dict stays float64).  A state dict without gammas (DINO) is
    returned unchanged."""
    if "blocks.0.ls1.gamma" not in sd:
        return sd
    out = {k: v for k, v in sd.items() if ".ls1.gamma" not in k and ".ls2.gamma" not in k}
    fc2 = "mlp.w3" if "blocks.0.mlp.w3.weight" in sd else "mlp.fc2"
    for i in range(depth):
        b = f"blocks.{i}."
        for ls, layer in (("ls1", "attn.proj"), ("ls2", fc2)):
            w, bias, gamma = sd[b + layer + ".weight"], sd[b + layer + ".bias"], sd[b + ls + ".gamma"]
            dt = torch.promote_types(w.dtype, torch.float32)
            gamma = gamma.to(w.device, dt)
            out[b + layer + ".weight"] = w.to(dt) * gamma[:, None]
            out[b + layer + ".bias"] = bias.to(dt) * gamma
    return out


class ViTBackbone:
    """Owns a ``wvn_vit_t``: DINO / DINOv2 ViT weights (bf16 on device) + L2-sized activation workspaces.  A state dict
    with ``register_tokens`` (1, R, D) (DINOv2 *_reg) gives a handle with R register tokens after CLS, whose position
    embeddings are interpolated by the register models' antialiased form.  A state dict with ``mlp.w12`` / ``mlp.w3``
    (DINOv2 ViT-g/14's SwiGLU FFN, hidden width ``mlp_dim``) gives a handle with that FFN.  Tensors already on the GPU
    are loaded from there, without a copy through host memory."""

    def __init__(self, image_size, patch_size, dim, depth, heads, mlp_dim, state_dict, max_batch=32, chunk=0,
                 head_weights=None, ln_eps=1e-6):
        _C.require_device()
        self.image_size, self.patch_size, self.dim = image_size, patch_size, dim
        self.grid = image_size // patch_size
        self.P = self.grid * self.grid
        self.max_batch = max_batch
        self.head_out = 0 if head_weights is None else int(head_weights["head_a.weight"].shape[0])
        reg = next((v for k, v in state_dict.items() if k.endswith("register_tokens")), None)
        self.registers = 0 if reg is None else int(reg.shape[-2])
        swiglu = any(k.endswith("blocks.0.mlp.w12.weight") for k in state_dict)
        self.ffn = _C.VIT_FFN_SWIGLU if swiglu else _C.VIT_FFN_MLP
        cfg = VitConfig(image_size, patch_size, dim, depth, heads, mlp_dim, max_batch, chunk, ln_eps, self.head_out,
                        self.registers)
        h = c_void_p()
        check(lib().wvn_vit_create_ffn(byref(cfg), self.ffn, byref(h)))
        self._h = h
        self.npad = lib().wvn_vit_npad(h)
        self._load(state_dict, depth)
        if head_weights is not None:
            for k, v in head_weights.items():
                self._set("stego." + k, v)

    def _set(self, name, t):
        t = t.detach().to(dtype=torch.float32, device="cuda" if t.is_cuda else "cpu").contiguous()
        if t.is_cuda:
            torch.cuda.current_stream().synchronize()  # the library reads it on its own stream
        check(lib().wvn_vit_set_weight(self._h, name.encode(), c_void_p(t.data_ptr()), t.numel()))

    def _load(self, sd, depth):
        sd = {k.replace("module.", "").replace("backbone.", ""): v for k, v in sd.items()}
        sd = fold_layerscale(sd, depth)
        self._set("cls_token", sd["cls_token"].reshape(-1))
        interp = interpolate_pos_embed_antialias if self.registers > 0 else interpolate_pos_embed
        self._set("pos_embed", interp(sd["pos_embed"].float().cpu(), self.grid).reshape(-1))
        if self.registers > 0:
            self._set("register_tokens", sd["register_tokens"].reshape(-1))
        self._set("patch_embed.proj.weight", sd["patch_embed.proj.weight"].reshape(self.dim, -1))
        self._set("patch_embed.proj.bias", sd["patch_embed.proj.bias"])
        ffn = (("mlp.w12.weight", "mlp.w12.bias", "mlp.w3.weight", "mlp.w3.bias") if self.ffn == _C.VIT_FFN_SWIGLU else
               ("mlp.fc1.weight", "mlp.fc1.bias", "mlp.fc2.weight", "mlp.fc2.bias"))
        for i in range(depth):
            for leaf in ("norm1.weight", "norm1.bias", "attn.qkv.weight", "attn.qkv.bias", "attn.proj.weight",
                         "attn.proj.bias", "norm2.weight", "norm2.bias") + ffn:
                self._set(f"blocks.{i}.{leaf}", sd[f"blocks.{i}.{leaf}"])
        self._set("norm.weight", sd["norm.weight"])
        self._set("norm.bias", sd["norm.bias"])

    def forward(self, img: torch.Tensor, resized_hw=None, flip_tta: bool = False) -> torch.Tensor:
        """img: (B,3,H,W) f32 CUDA in [0,1], or the camera frames themselves (B,H,W,3) uint8 RGB
        -> final-norm patch tokens (B, P, D) f32.  flip_tta (float input only): (2B, P, D), the second half being the
        pass over the horizontally flipped TRANSFORMED images (STEGO's get_code)."""
        img = img.contiguous()
        if flip_tta:
            B, C, H, W = img.shape
            assert img.dtype == torch.float32
            fn = lib().wvn_vit_forward_tta
        elif img.dtype == torch.uint8:
            B, H, W, C = img.shape
            fn = lib().wvn_vit_forward_u8
        else:
            B, C, H, W = img.shape
            assert img.dtype == torch.float32
            fn = lib().wvn_vit_forward
        assert C == 3
        if resized_hw is None:
            resized_hw = _resized_size(H, W, self.image_size)
        tokens = torch.empty(2 * B if flip_tta else B, self.P, self.dim, device=img.device, dtype=torch.float32)
        check(fn(self._h, ptr(img), B, H, W, resized_hw[0], resized_hw[1], ptr(tokens), stream()))
        self.last_tokens = tokens   # the handle's bf16 copy of exactly these tokens feeds the per-pixel head directly
        return tokens

    def stego_head(self, batch: int) -> torch.Tensor:
        out = torch.empty(batch * self.npad, self.head_out, device="cuda", dtype=torch.float32)
        check(lib().wvn_vit_stego_head(self._h, batch, ptr(out), stream()))
        return out

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                lib().wvn_vit_destroy(self._h)
                self._h = None
        except Exception:
            pass


# --------------------------------------------------------------------------------------------
# ResNet backbone handle and its primitives
# --------------------------------------------------------------------------------------------
# (channels, stride) of the four taps: torchvision_interface.py's return nodes feat1..feat4
RESNET_TAPS = {18: ((64, 4), (128, 8), (256, 16), (512, 32)), 50: ((128, 4), (256, 8), (512, 16), (2048, 32))}


def _ptr_array(tensors):
    return (c_void_p * len(tensors))(*[t.data_ptr() for t in tensors])


def im2col_nhwc(x, k, stride, pad, pitch=None, out=None):
    """x: [B,H,W,C] bf16 NHWC -> rows [B*Ho*Wo, pitch] bf16 in (ky, kx, channel) order; pad columns are left as they are."""
    B, H, W, C = x.shape
    Ho, Wo, K = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1, k * k * C
    pitch = pitch or (K + 7) // 8 * 8
    if out is None:
        out = torch.empty(B * Ho * Wo, pitch, device=x.device, dtype=torch.bfloat16)
    check(lib().wvn_im2col_bf16_nhwc(ptr(x.contiguous()), B, H, W, C, k, stride, pad, ptr(out), pitch, stream()))
    return out


def im2col_image(img, k, stride, pad, pitch=None, out=None):
    """img: [B,3,H,W] fp32 in [0,1] -> ImageNet-normalised, zero-padded rows [B*Ho*Wo, pitch] bf16 (ky, kx, channel)."""
    B, _, H, W = img.shape
    Ho, Wo, K = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1, k * k * 3
    pitch = pitch or (K + 7) // 8 * 8
    if out is None:
        out = torch.empty(B * Ho * Wo, pitch, device=img.device, dtype=torch.bfloat16)
    check(lib().wvn_im2col_image(ptr(img.contiguous()), B, H, W, k, stride, pad, ptr(out), pitch, stream()))
    return out


def maxpool3s2_nhwc(x):
    """3 x 3 / stride 2 / pad 1 max-pool of x [B,H,W,C] bf16 NHWC."""
    B, H, W, C = x.shape
    out = torch.empty(B, (H + 1) // 2, (W + 1) // 2, C, device=x.device, dtype=torch.bfloat16)
    check(lib().wvn_maxpool3s2_bf16_nhwc(ptr(x.contiguous()), B, H, W, C, ptr(out), stream()))
    return out


def segment_pool_pyramid(seg, smax, taps, centers):
    """Multiscale segment pooling (sparsify_features' pyramid branch).  seg [B,H,W] int64, taps: one to five NHWC bf16
    maps [B,h_l,w_l,c_l], each dense or the first c_l channels of a dense [B,h_l,w_l,pitch_l] map, centers [B,smax,2]
    fp32 (col, row) -> feat [B,smax,sum c_l] fp32 (see include/wvn_b200.h, wvn_segment_pool_levels)."""
    B, H, W = seg.shape
    D = sum(t.shape[3] for t in taps)
    out = torch.empty(B, smax, D, device=seg.device, dtype=torch.float32)
    pitch = []
    for t in taps:
        p = t.stride(2)
        assert t.is_cuda and t.dtype == torch.bfloat16 and t.stride(3) == 1 and p >= t.shape[3] and \
            t.stride(1) == t.shape[2] * p and t.stride(0) == t.shape[1] * t.stride(1), "tap must be a dense NHWC map's prefix"
        pitch.append(p)
    ints = ctypes.c_int * len(taps)
    th, tw, tc = ints(*[t.shape[1] for t in taps]), ints(*[t.shape[2] for t in taps]), ints(*[t.shape[3] for t in taps])
    check(lib().wvn_segment_pool_levels(ptr(seg.contiguous()), B, H, W, smax, ptr(centers.contiguous()), len(taps),
                                        _ptr_array(taps), th, tw, tc, ints(*pitch), ptr(out), stream()))
    return out


class ResNetBackbone:
    """Owns a ``wvn_resnet_t``: a torchvision ResNet-18 / ResNet-50 trunk with batch norm folded into its convs (bf16 on
    device) and activation / im2col workspaces sized for ``max_batch``.  ``folded`` maps each conv's name to its
    (weight [out, in, kh, kw], bias [out]) after folding (weights.fold_resnet_bn)."""

    def __init__(self, image_size, depth, folded, max_batch=32):
        _C.require_device()
        self.image_size, self.depth, self.max_batch = image_size, depth, max_batch
        h = c_void_p()
        check(lib().wvn_resnet_create(byref(ResnetConfig(image_size, depth, max_batch)), byref(h)))
        self._h = h
        self.workspace_bytes = lib().wvn_resnet_workspace_bytes(h)
        self.taps = [(c, image_size // s) for c, s in RESNET_TAPS[depth]]
        for name, (w, b) in folded.items():
            w = w.detach().to(dtype=torch.float32, device="cpu").permute(0, 2, 3, 1).contiguous()
            b = b.detach().to(dtype=torch.float32, device="cpu").contiguous()
            check(lib().wvn_resnet_set_weight(h, (name + ".weight").encode(), c_void_p(w.data_ptr()), w.numel()))
            check(lib().wvn_resnet_set_weight(h, (name + ".bias").encode(), c_void_p(b.data_ptr()), b.numel()))

    def forward(self, img: torch.Tensor):
        """img (B,3,S,S) fp32 CUDA in [0,1] -> the four taps, NHWC bf16 [B, S/s_l, S/s_l, c_l]."""
        B = img.shape[0]
        assert img.dtype == torch.float32 and tuple(img.shape[1:]) == (3, self.image_size, self.image_size)
        taps = [torch.empty(B, n, n, c, device=img.device, dtype=torch.bfloat16) for c, n in self.taps]
        check(lib().wvn_resnet_forward(self._h, ptr(img.contiguous()), B, _ptr_array(taps), stream()))
        return taps

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                lib().wvn_resnet_destroy(self._h)
                self._h = None
        except Exception:
            pass


class DenseCrf:
    """Owns a ``wvn_crf_t``: STEGO's dense CRF (oracle/dense_crf.py) for ``size`` x ``size`` frames with up to
    ``max_classes`` labels, refined ``chunk`` frames at a time.  Every workspace is allocated here, for the worst case;
    ``workspace_bytes`` says how much."""

    def __init__(self, size, max_classes, chunk=2, iterations=10):
        _C.require_device()
        self.size, self.max_classes, self.chunk, self.iterations = size, max_classes, chunk, iterations
        h = c_void_p()
        check(lib().wvn_crf_create(size, max_classes, chunk, iterations, byref(h)))
        self._h = h
        self.workspace_bytes = lib().wvn_crf_workspace_bytes(h)

    def _image_args(self, img, resized_hw):
        img = img.contiguous()
        if img.dtype == torch.uint8:
            B, H, W, C = img.shape
        else:
            assert img.dtype == torch.float32
            B, C, H, W = img.shape
        assert C == 3
        rh, rw = resized_hw or _resized_size(H, W, self.size)
        return img, (c_void_p(img.data_ptr()), int(img.dtype == torch.uint8), B, H, W, rh, rw)

    def run(self, img, head, npad, grid, col0, classes, code_col=0, code_dim=0, logit_scale=1.0, resized_hw=None,
            want_q=False):
        """img: the frames the backbone read ((B,3,H,W) fp32 or (B,H,W,3) uint8); head: STEGO head output
        [B*npad, ld] fp32.  -> labels (B, S, S) int64, and with ``want_q`` also Q (B, S*S, classes) fp32."""
        img, args = self._image_args(img, resized_hw)
        B = args[2]
        labels = torch.empty(B, self.size, self.size, device=head.device, dtype=torch.int64)
        q = torch.empty(B, self.size * self.size, classes, device=head.device, dtype=torch.float32) if want_q else None
        check(lib().wvn_crf_run(self._h, *args, ptr(head), head.stride(0), npad, grid, col0, classes, code_col, code_dim,
                                logit_scale, ptr(labels), ptr(q), stream()))
        return (labels, q) if want_q else labels

    def build(self, img, resized_hw=None):
        """Testing: build the two lattices of the frames of ``img`` (at most ``chunk``)."""
        img, args = self._image_args(img, resized_hw)
        check(lib().wvn_crf_build(self._h, *args, stream()))
        self._built = args[2]

    def filter(self, which, values):
        """Testing: values [B*S*S, v] through lattice ``which`` (0 spatial, 1 bilateral) without normalisation."""
        values = values.contiguous()
        out = torch.empty_like(values)
        check(lib().wvn_crf_filter(self._h, which, ptr(values), values.shape[1], ptr(out), stream()))
        return out

    def lattice(self, which):
        """Testing: dict(keys (M,) packed int64 view, counts (M,), offsets (N, d+1), bary (N, d+1)) of lattice ``which``."""
        d = 2 if which == 0 else 5
        n = self._built * self.size * self.size
        dev = "cuda"
        keys = torch.empty(n * (d + 1), device=dev, dtype=torch.int64)
        counts = torch.empty(n * (d + 1), device=dev, dtype=torch.int32)
        offsets = torch.empty(n, d + 1, device=dev, dtype=torch.int32)
        bary = torch.empty(n, d + 1, device=dev, dtype=torch.float32)
        m = torch.empty(1, device=dev, dtype=torch.int32)
        check(lib().wvn_crf_export(self._h, which, ptr(keys), ptr(counts), ptr(offsets), ptr(bary), ptr(m), stream()))
        M = int(m.item())
        return dict(keys=keys[:M], counts=counts[:M], offsets=offsets, bary=bary)

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                lib().wvn_crf_destroy(self._h)
                self._h = None
        except Exception:
            pass


def _resized_size(h, w, size):
    # torchvision Resize(size:int): smaller edge -> size
    if h <= w:
        return size, int(size * w / h)
    return int(size * h / w), size


# --------------------------------------------------------------------------------------------
# traversability MLP: inference handle and trainer
# --------------------------------------------------------------------------------------------
class MlpInference:
    """Per-pixel and per-row traversability / confidence of a SimpleMLP, or with ``double=True`` of a
    DoubleMLP(dim, [h1, h2, 1]) (``set_params`` then takes its flat parameters).  ``fused_shape``: the fused per-pixel
    head takes this shape (SimpleMLP [256, 32, 1], DoubleMLP [64 or 128, 32, 1]), so ``pixels_from_vit`` can run at
    the fused geometries."""

    def __init__(self, dim=384, h1=256, h2=32, chunk_rows=0, tokens_per_frame=0, double=False):
        _C.require_device()
        self.dim, self.h1, self.h2, self.double = dim, h1, h2, double
        self.fused_shape = (h1 in (64, 128) and h2 == 32) if double else (h1 == 256 and h2 == 32)
        h = c_void_p()
        create = lib().wvn_mlp_infer_create_double if double else lib().wvn_mlp_infer_create
        check(create(dim, h1, h2, chunk_rows, byref(h)))
        self._h = h
        if tokens_per_frame > 0:  # all workspaces exist before the first frame arrives
            check(lib().wvn_mlp_infer_reserve(h, tokens_per_frame))

    def set_params(self, flat_params: torch.Tensor):
        assert flat_params.is_cuda and flat_params.dtype == torch.float32
        check(lib().wvn_mlp_infer_set_params(self._h, ptr(flat_params.contiguous()), stream()))

    def pixels(self, tokens, grid, out_hw, cg_mean, cg_std, std_factor):
        B = tokens.shape[0]
        trav = torch.empty(B, out_hw[0], out_hw[1], device=tokens.device, dtype=torch.float32)
        conf = torch.empty_like(trav)
        check(lib().wvn_mlp_infer_pixels(self._h, ptr(tokens), B, grid[0], grid[1], out_hw[0], out_hw[1], ptr(cg_mean),
                                         ptr(cg_std), float(std_factor), ptr(trav), ptr(conf), stream()))
        return trav, conf

    def pixels_from_vit(self, vit: "ViTBackbone", batch, out_hw, cg_mean, cg_std, std_factor):
        """The same maps from the backbone's own bf16 tokens of its last forward (frames [0, batch))."""
        trav = torch.empty(batch, out_hw[0], out_hw[1], device=cg_mean.device, dtype=torch.float32)
        conf = torch.empty_like(trav)
        check(lib().wvn_mlp_infer_pixels_vit(self._h, vit._h, batch, out_hw[0], out_hw[1], ptr(cg_mean), ptr(cg_std),
                                             float(std_factor), ptr(trav), ptr(conf), stream()))
        return trav, conf

    def rows(self, x, cg_mean, cg_std, std_factor):
        R = x.shape[0]
        trav = torch.empty(R, device=x.device, dtype=torch.float32)
        conf = torch.empty_like(trav)
        check(lib().wvn_mlp_infer_rows(self._h, ptr(x.contiguous()), R, ptr(cg_mean), ptr(cg_std), float(std_factor),
                                       ptr(trav), ptr(conf), stream()))
        return trav, conf

    def rows_padded(self, feat, n_rows, cg_mean, cg_std, std_factor):
        """feat [G, S, dim] fp32 with n_rows [G] int32 live rows per group -> (trav [G, S], conf [G, S]); padding rows
        NaN.  A live row's values are bit-identical to ``rows`` on the compacted rows."""
        G, S = _check_padded(feat, n_rows, self.dim)
        trav = torch.empty(G, S, device=feat.device, dtype=torch.float32)
        conf = torch.empty_like(trav)
        check(lib().wvn_mlp_infer_rows_padded(self._h, ptr(feat.contiguous()), G, S, ptr(n_rows), ptr(cg_mean),
                                              ptr(cg_std), float(std_factor), ptr(trav), ptr(conf), stream()))
        return trav, conf

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                lib().wvn_mlp_infer_destroy(self._h)
                self._h = None
        except Exception:
            pass


def mlp_forward_f32(flat_params, x, dim, h1, h2):
    """SimpleMLP.forward in fp32: returns (rows, 1+dim) with column 0 through the sigmoid."""
    R = x.shape[0]
    dev = x.device
    b1 = torch.empty(R, h1, device=dev, dtype=torch.float32)
    b2 = torch.empty(R, h2, device=dev, dtype=torch.float32)
    out = torch.empty(R, 1 + dim, device=dev, dtype=torch.float32)
    check(lib().wvn_mlp_forward_f32(dim, h1, h2, ptr(flat_params), ptr(x.contiguous()), R, ptr(b1), ptr(b2), ptr(out),
                                    stream()))
    return out


def double_mlp_forward_f32(flat_params, x, dim, h1, h2):
    """DoubleMLP.forward in fp32: returns (rows, 1+dim), column 0 = sigmoid(networks[0](x)), then networks[1](x)."""
    R = x.shape[0]
    dev = x.device
    a1 = torch.empty(2, R, h1, device=dev, dtype=torch.float32)
    a2 = torch.empty(2, R, h2, device=dev, dtype=torch.float32)
    out = torch.empty(R, 1 + dim, device=dev, dtype=torch.float32)
    if R == 0:
        return out
    check(lib().wvn_double_mlp_forward_f32(dim, h1, h2, ptr(flat_params), ptr(x.contiguous()), R, ptr(a1), ptr(a2),
                                           ptr(out), stream()))
    return out


def _device_doubles(address, n, device):
    """A float64 tensor over ``n`` doubles of device memory the library owns (no copy)."""
    class _Block:
        __cuda_array_interface__ = {"shape": (n,), "typestr": "<f8", "data": (int(address), False), "version": 2}

    return torch.as_tensor(_Block(), device=device)


class _TrainerHandle:
    """Owns a library trainer handle (``wvn_trainer_t``) with workspaces for ``max_rows`` rows and replaces it by a
    larger one when a call needs more.  Remembers the ConfidenceGenerator binding, so the replacement keeps the generator
    where it was.  Allocates the state every learner's step reads and updates: ``grads`` (``n_grads`` floats),
    Adam's ``exp_avg`` / ``exp_avg_sq`` / ``step_counter``, ``metrics`` (``n_metrics`` floats) and the generator's
    ``cg_mean`` / ``cg_std``.  Subclasses make the handle in ``_new_handle``.

    Data-parallel steps (``process_group``) are run here for every trainer: with an NCCL group the handle gets the
    library's own communicator and the step issues both all-reduces itself, between its kernels; with any other backend
    (gloo in tests) the step runs as phase 1 / all-reduce of the statistics block / phase 2 / all-reduce of the gradient
    / phase 4 through ``torch.distributed`` on the same buffers.  ``stats``: the handle's statistics block (6 sums, the
    extrema, and for some learners a ninth double exchanged with the gradient); ``_grad_exchange()``: the buffers
    summed after phase 2."""

    def __init__(self, device, n_params, cfg, max_rows, process_group, n_metrics=6, n_grads=None):
        self.n_params, self.cfg, self.pg = n_params, cfg, process_group
        self.grads = torch.zeros(n_params if n_grads is None else n_grads, device=device)
        self.exp_avg = torch.zeros(n_params, device=device)
        self.exp_avg_sq = torch.zeros(n_params, device=device)
        self.step_counter = torch.zeros(1, device=device, dtype=torch.int64)
        self.metrics = torch.zeros(n_metrics, device=device)
        self.cg_mean = torch.zeros(1, device=device)
        self.cg_std = torch.ones(1, device=device)
        self._conf = None     # (method id, var, running_n, running_sum, running_sum_of_squares, kf_proc_cov, kf_meas_cov)
        self._h = None
        self._lib_comm = False
        self._create(max_rows)

    def _create(self, max_rows):
        h = self._new_handle(int(max_rows))
        if self._h is not None:
            # both handles' workspaces are alive until the old one is destroyed: peak memory briefly doubles here.
            # The confidence state the old handle kept itself (moving_average's window, var and running sums not bound
            # to caller tensors) moves over, so the generator does not restart
            check(lib().wvn_trainer_copy_confidence(h, self._h, stream()))
            lib().wvn_trainer_destroy(self._h)
        self._h = h
        self.max_rows = int(max_rows)
        self.conf = torch.empty(self.max_rows, device=self.grads.device)
        n = ctypes.c_int()
        self.stats = _device_doubles(lib().wvn_trainer_stats(h, byref(n)), n.value, self.grads.device)
        if self._conf is not None:
            self.set_confidence(*self._conf)
        self._init_comm()

    def _init_comm(self):
        self._lib_comm = False
        if self.pg is None:
            return
        import torch.distributed as dist

        if dist.get_backend(self.pg) == "nccl":
            # the library owns its communicator: rank 0 makes the id, torch.distributed only carries the 128 bytes
            rank, world = dist.get_rank(self.pg), dist.get_world_size(self.pg)
            buf = (ctypes.c_ubyte * 128)()
            if rank == 0:
                check(lib().wvn_comm_unique_id(buf))
            idt = torch.tensor(list(buf), dtype=torch.uint8, device=self.exp_avg.device)
            dist.broadcast(idt, src=dist.get_global_rank(self.pg, 0), group=self.pg)
            raw = (ctypes.c_ubyte * 128)(*idt.cpu().tolist())
            check(lib().wvn_trainer_init_comm(self._h, raw, rank, world))
            self._lib_comm = True

    def _run_phases(self, phase):
        """``phase(mask)`` enqueues those phases of one step on the current stream."""
        if self.pg is None or self._lib_comm:
            phase(7)
            return
        import torch.distributed as dist

        phase(1)
        dist.all_reduce(self.stats[:6], group=self.pg)
        if self._conf is not None and self._conf[0] == 3:   # moving_average normalises by the global extrema
            dist.all_reduce(self.stats[6:7], op=dist.ReduceOp.MIN, group=self.pg)
            dist.all_reduce(self.stats[7:8], op=dist.ReduceOp.MAX, group=self.pg)
        phase(2)
        for t in self._grad_exchange():
            dist.all_reduce(t, group=self.pg)
        phase(4)

    def _reserve(self, rows):
        if rows > self.max_rows:
            self._create(int(rows * 1.5))

    def set_confidence(self, method=0, var=None, running_n=None, running_sum=None, running_sum_of_squares=None,
                       kf_proc_cov=0.2, kf_meas_cov=1.0):
        """ConfidenceGenerator method of the step (0 latest_measurement, 1 running_mean, 2 kalman_filter, 3
        moving_average) and the device tensors holding its state (updated in place by the step; None = private)."""
        self._conf = (int(method), var, running_n, running_sum, running_sum_of_squares, float(kf_proc_cov), float(kf_meas_cov))
        if self._h is not None:
            check(lib().wvn_trainer_set_confidence(self._h, int(method), ptr(var), ptr(running_n), ptr(running_sum),
                                                   ptr(running_sum_of_squares), float(kf_proc_cov), float(kf_meas_cov)))

    def _grad_exchange(self):
        # the gradient, and the ninth double of the statistics block when the learner has one (DoubleMLP, SimpleGCN: the
        # confidence-weighted error sum, kept in fp64)
        return (self.grads, self.stats[8:9]) if self.stats.numel() > 8 else (self.grads,)

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                lib().wvn_trainer_destroy(self._h)
                self._h = None
        except Exception:
            pass


class MlpTrainer(_TrainerHandle):
    """Fused online train step on a flat fp32 parameter buffer (csrc/mlp_train_fused.cu): four kernels, no host
    synchronisation, rows may arrive padded per frame (``step_padded``) exactly as the segment pooling leaves them.

    ``params`` is the tensor that SimpleMLP's layers view into, so the reference's state_dict layout stays intact.
    With ``process_group`` set the step is global-batch exact: the six statistic sums (incl. the row count) and the flat
    gradient are all-reduced between the kernels — by the library's own NCCL communicator when the group's backend is
    NCCL (one rank per GPU), otherwise (e.g. gloo in tests) by ``torch.distributed`` on the same buffers.
    ``legacy=True`` runs round 1's three-phase kernels (csrc/mlp_train.cu), kept for A/B parity tests."""

    def __init__(self, params, dim=384, h1=256, h2=32, max_rows=4096, w_trav=0.03, w_reco=0.5, std_factor=0.5,
                 anomaly_balanced=True, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, process_group=None, legacy=False):
        _C.require_device()
        self.dim, self.h1, self.h2 = dim, h1, h2
        n_params = lib().wvn_mlp_param_count(dim, h1, h2)
        assert params.numel() == n_params and params.is_cuda and params.dtype == torch.float32
        self.params = params
        self.legacy = legacy
        nbytes = lib().wvn_mlp_train_scalars_bytes() if legacy else lib().wvn_mlp_trainer_scalars_bytes()
        self.scalars = torch.zeros((nbytes + 7) // 8, device=params.device, dtype=torch.float64)
        cfg = TrainConfig(w_trav, w_reco, std_factor, int(anomaly_balanced), lr, betas[0], betas[1], eps)
        # the gradient's extra float: the confidence-weighted error sum, exchanged with it
        super().__init__(params.device, n_params, cfg, max_rows, process_group, n_grads=n_params + 1)

    # ---- fused path ---------------------------------------------------------------------------
    def _new_handle(self, max_rows):
        h = c_void_p()
        check(lib().wvn_mlp_trainer_create(self.dim, self.h1, self.h2, max_rows, byref(self.cfg), ptr(self.scalars),
                                           ptr(self.grads), byref(h)))
        return h

    def _create(self, max_rows):
        if self.legacy:
            self._alloc_ws(max_rows)
            return
        super()._create(max_rows)
        self.conf = torch.empty(self.max_rows + 32, device=self.params.device, dtype=torch.float32)

    def set_confidence(self, method=0, *args, **kwargs):
        assert not self.legacy or method == 0, "the round-1 kernels implement latest_measurement only"
        super().set_confidence(method, *args, **kwargs)

    def _run(self, x, groups, rpg, n_rows, y, yv):
        self._reserve(groups * rpg)
        x = x.contiguous()
        y = y.contiguous().float()
        yv = yv.contiguous().to(torch.uint8)
        s = stream()

        def phase(mask):
            check(lib().wvn_mlp_train_step(self._h, ptr(self.params), ptr(self.exp_avg), ptr(self.exp_avg_sq),
                                           ptr(self.step_counter), ptr(x), groups, rpg, ptr(n_rows), ptr(y), ptr(yv),
                                           ptr(self.cg_mean), ptr(self.cg_std), ptr(self.conf), ptr(self.metrics), mask, s))

        self._run_phases(phase)

    def step_padded(self, feat, n_rows, y, y_valid):
        """feat [G, S, D] f32 padded per group, n_rows [G] int32 (device): the first n_rows[g] rows of group g are live.
        y / y_valid are indexed by the compacted row number.  Returns the confidence buffer (compacted order; the live
        prefix has sum(n_rows) entries — no host sync happens here)."""
        assert not self.legacy
        G, S, D = feat.shape
        assert D == self.dim and n_rows.dtype == torch.int32 and y.numel() >= 1
        self._run(feat, G, S, n_rows, y, y_valid)
        return self.conf

    def step(self, x, y, y_valid, n_total=None):
        """x [R,D] f32, y [R] f32, y_valid [R] bool.  Returns the confidence vector [R]; metrics stay
        on the device in ``self.metrics`` (loss_total, loss_trav, loss_reco, loss_trav_conf, mean, std)."""
        if self.legacy:
            return self._step_legacy(x, y, y_valid, n_total)
        R = x.shape[0]
        self._run(x, 1, R, None, y, y_valid)
        return self.conf[:R]

    # ---- round-1 kernels (three phases, ~20 launches) --------------------------------------------
    def _alloc_ws(self, max_rows):
        self.max_rows = max_rows
        nbytes = lib().wvn_mlp_train_workspace_bytes(self.dim, self.h1, self.h2, max_rows)
        self.ws = torch.empty(nbytes // 4, device=self.params.device, dtype=torch.float32)
        self.conf = torch.empty(max_rows, device=self.params.device, dtype=torch.float32)

    def _step_legacy(self, x, y, y_valid, n_total=None):
        R = x.shape[0]
        if R > self.max_rows:
            self._alloc_ws(int(R * 1.5))
        x = x.contiguous()
        y = y.contiguous().float()
        yv = y_valid.contiguous().to(torch.uint8)
        d = (self.dim, self.h1, self.h2)
        s = stream()
        check(lib().wvn_mlp_train_forward_stats(*d, ptr(self.params), ptr(x), ptr(y), ptr(yv), R, self.max_rows,
                                                ptr(self.ws), ptr(self.scalars), s))
        if self.pg is not None:
            import torch.distributed as dist
            dist.all_reduce(self.scalars[:5], group=self.pg)
            if n_total is None:
                nt = torch.tensor([R], device=x.device, dtype=torch.int64)
                dist.all_reduce(nt, group=self.pg)
                n_total = int(nt.item())
        if n_total is None:
            n_total = R
        check(lib().wvn_mlp_train_backward(*d, ptr(self.params), ptr(x), ptr(y), ptr(yv), R, self.max_rows, n_total,
                                           byref(self.cfg), ptr(self.ws), ptr(self.scalars), ptr(self.cg_mean),
                                           ptr(self.cg_std), ptr(self.grads), ptr(self.conf), s))
        if self.pg is not None:
            import torch.distributed as dist
            dist.all_reduce(self.grads, group=self.pg)
        check(lib().wvn_mlp_train_apply(*d, ptr(self.params), ptr(self.grads), ptr(self.exp_avg), ptr(self.exp_avg_sq),
                                        ptr(self.step_counter), n_total, byref(self.cfg), ptr(self.scalars), s))
        check(lib().wvn_mlp_train_read_metrics(ptr(self.scalars), ptr(self.metrics), s))
        return self.conf[:R]


def _check_padded(feat, n_rows, dim):
    G, S, D = feat.shape
    assert D == dim and feat.dtype == torch.float32, "step_padded: feat must be (G, S, dim) float32"
    assert n_rows.dtype == torch.int32 and n_rows.shape == (G,), "step_padded: n_rows must be (G,) int32"
    return G, S


class DoubleMlpTrainer(_TrainerHandle):
    """The online train step of a DoubleMLP on its flat fp32 parameters (csrc/double_mlp_train.cu): forward of both
    networks, TraversabilityLoss with the ConfidenceGenerator update, backward and Adam as one fixed launch sequence
    without host synchronisation, bit-reproducible.  ``exp_avg`` / ``exp_avg_sq`` / ``step_counter`` are
    torch.optim.Adam's state over the 12 parameter tensors, flattened in ``parameters()`` order.  Rows may arrive padded
    per frame (``step_padded``).  With ``process_group`` the step is global-batch exact (see ``_TrainerHandle``): the
    statistic sums, row counts and extrema are all-reduced after the forward, the gradient and the confidence-weighted
    error sum after the backward."""

    def __init__(self, model, max_rows=4096, w_trav=0.03, w_reco=0.5, std_factor=0.5, anomaly_balanced=True, lr=1e-3,
                 betas=(0.9, 0.999), eps=1e-8, process_group=None):
        model.check_supported()
        _C.require_device()
        params = model.flat_params
        self.model = model
        self.dim, (self.h1, self.h2) = model.input_size, model.hidden
        n_params = lib().wvn_double_mlp_param_count(self.dim, self.h1, self.h2)
        assert params.numel() == n_params and params.dtype == torch.float32
        cfg = TrainConfig(w_trav, w_reco, std_factor, int(anomaly_balanced), lr, betas[0], betas[1], eps)
        super().__init__(params.device, n_params, cfg, max_rows, process_group)

    def _new_handle(self, max_rows):
        h = c_void_p()
        check(lib().wvn_double_mlp_trainer_create(self.dim, self.h1, self.h2, max_rows, byref(self.cfg), ptr(self.grads),
                                                  byref(h)))
        return h

    def _run(self, x, groups, rpg, n_rows, y, y_valid):
        self._reserve(groups * rpg)
        x = x.contiguous().float()
        y = y.contiguous().float()
        yv = y_valid.contiguous().to(torch.uint8)
        s = stream()

        def phase(mask):
            check(lib().wvn_double_mlp_train_step_padded(
                self._h, ptr(self.model.flat_params), ptr(self.exp_avg), ptr(self.exp_avg_sq), ptr(self.step_counter),
                ptr(x), groups, rpg, ptr(n_rows), ptr(y), ptr(yv), ptr(self.cg_mean), ptr(self.cg_std), ptr(self.conf),
                ptr(self.metrics), mask, s))

        self._run_phases(phase)

    def step_padded(self, feat, n_rows, y, y_valid):
        """feat [G, S, D] f32 padded per group, n_rows [G] int32 (device): the first n_rows[g] rows of group g are live;
        padding may hold anything.  y / y_valid are indexed by the compacted row number.  Returns the confidence buffer
        (compacted order; the live prefix has sum(n_rows) entries — no host sync happens here)."""
        G, S = _check_padded(feat, n_rows, self.dim)
        self._run(feat, G, S, n_rows, y, y_valid)
        return self.conf

    def step(self, x, y, y_valid, n_total=None):
        """x [R,D] f32, y [R] f32, y_valid [R] bool.  Returns the confidence vector [R]; metrics stay on the device in
        ``self.metrics`` (loss_total, loss_trav, loss_reco, loss_trav_conf, mean, std)."""
        if n_total is not None and n_total != x.shape[0]:
            raise ValueError("DoubleMlpTrainer: the global row count is all-reduced by the step, n_total must be the "
                             "batch's row count")
        R = x.shape[0]
        self._run(x, 1, R, None, y, y_valid)
        return self.conf[:R]


# --------------------------------------------------------------------------------------------
# SimpleGCN learner: graph convolutions over each frame's segment adjacency
# --------------------------------------------------------------------------------------------
def _check_edges(edges, n_edges, groups):
    """edges [G, E, 2] integer (source, target local row ids), n_edges [G] int32 on the device -> (int64 edges, E)."""
    if not torch.is_tensor(edges) or edges.dim() != 3 or edges.shape[0] != groups or edges.shape[2] != 2 \
            or edges.is_floating_point():
        raise ValueError(f"edges must be a ({groups}, E, 2) integer tensor")
    if not torch.is_tensor(n_edges) or n_edges.dtype != torch.int32 or tuple(n_edges.shape) != (groups,):
        raise ValueError(f"n_edges must be a ({groups},) int32 tensor")
    return edges.contiguous().long(), int(edges.shape[1])


def _graph_as_padded(x, edge_index):
    """A batched graph (rows x [N, D], edge_index [2, E]) as one frame of the padded layout, without host sync."""
    if edge_index is None or not torch.is_tensor(edge_index) or edge_index.dim() != 2 or edge_index.shape[0] != 2:
        raise ValueError("SimpleGCN needs the graph's edge_index, a (2, E) integer tensor")
    E = edge_index.shape[1]
    edges = edge_index.to(x.device, torch.int64).t().contiguous().reshape(1, E, 2)
    return edges, torch.full((1,), E, device=x.device, dtype=torch.int32)


def _batch_as_frames(x, edge_index, ptr):
    """A ``Batch.from_data_list`` graph split back into its nodes (``ptr`` [G + 1], host): feat [G, S, D] padded,
    n_rows [G], each node's edges in local ids [G, E, 2] (stably grouped by the source's node) and n_edges [G].  The
    per-frame graph build then scans each node's edges only, and the step is bit-identical to the one-frame form
    (same compacted rows, same in-edge order per row).  Device ops only, no device-to-host copy."""
    _graph_as_padded(x, edge_index)   # argument checks
    ptr = [int(v) for v in ptr]
    G, dev = len(ptr) - 1, x.device
    sizes = [ptr[i + 1] - ptr[i] for i in range(G)]
    S = max(max(sizes), 1)
    idx = torch.tensor([g * S + r for g in range(G) for r in range(sizes[g])], dtype=torch.long)
    feat = torch.zeros(G * S, x.shape[1], device=dev, dtype=torch.float32)
    feat.index_copy_(0, idx.to(dev, non_blocking=True), x.float())
    n_rows = torch.tensor(sizes, dtype=torch.int32).to(dev, non_blocking=True)
    ei = edge_index.to(dev, torch.int64)
    E = ei.shape[1]
    ptr_d = torch.tensor(ptr, dtype=torch.int64).to(dev, non_blocking=True)
    frame = (torch.searchsorted(ptr_d, ei[0].contiguous(), right=True) - 1).clamp(0, G - 1)
    frame, order = torch.sort(frame, stable=True)
    ei = ei[:, order]
    counts = torch.zeros(G, device=dev, dtype=torch.int64).index_add_(0, frame, torch.ones_like(frame))
    pos = torch.arange(E, device=dev) - (torch.cumsum(counts, 0) - counts)[frame]
    edges = torch.full((G, max(E, 1), 2), -1, device=dev, dtype=torch.int64)
    edges[frame, pos] = (ei - ptr_d[frame]).t()
    return feat.view(G, S, -1), n_rows, edges, counts.to(torch.int32)


class GcnTrainer(_TrainerHandle):
    """The online train step of a SimpleGCN on its flat fp32 parameters (csrc/gcn_train.cu): graph build, the three
    graph convolutions, TraversabilityLoss with the ConfidenceGenerator update, backward and Adam as one fixed launch
    sequence without host synchronisation, bit-reproducible.  ``exp_avg`` / ``exp_avg_sq`` / ``step_counter`` are
    torch.optim.Adam's state over the 6 parameter tensors in ``parameters()`` order.  Rows arrive padded per frame with
    each frame's edges (``step_padded``) or as one batched graph (``step``).  With ``process_group`` the step is
    global-batch exact (see ``_TrainerHandle``); no edge crosses frames, so sharding frames loses nothing.
    ``metrics[6]`` is 1 after a step that met a negative edge count (the segment reducer's overflow flag)."""

    def __init__(self, model, max_rows=4096, max_edges=16384, w_trav=0.03, w_reco=0.5, std_factor=0.5,
                 anomaly_balanced=True, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, process_group=None):
        model.check_supported()
        _C.require_device()
        params = model.flat_params
        self.model = model
        self.dim, (self.h1, self.h2) = model.input_size, model.hidden
        n_params = lib().wvn_gcn_param_count(self.dim, self.h1, self.h2)
        assert params.numel() == n_params and params.dtype == torch.float32
        self.max_edges = int(max_edges)
        cfg = TrainConfig(w_trav, w_reco, std_factor, int(anomaly_balanced), lr, betas[0], betas[1], eps)
        super().__init__(params.device, n_params, cfg, max_rows, process_group, n_metrics=7)

    def _new_handle(self, max_rows):
        h = c_void_p()
        check(lib().wvn_gcn_trainer_create(self.dim, self.h1, self.h2, max_rows, self.max_edges, byref(self.cfg),
                                           ptr(self.grads), byref(h)))
        return h

    def _reserve_edges(self, rows, edges):
        if edges > self.max_edges:
            self.max_edges = int(edges * 1.5)
            self._create(max(self.max_rows, int(rows)))
        else:
            self._reserve(rows)

    def _run(self, x, groups, rpg, n_rows, edges, epg, n_edges, y, y_valid):
        self._reserve_edges(groups * rpg, groups * epg)
        x = x.contiguous().float()
        y = y.contiguous().float()
        yv = y_valid.contiguous().to(torch.uint8)
        s = stream()

        def phase(mask):
            check(lib().wvn_gcn_train_step_padded(
                self._h, ptr(self.model.flat_params), ptr(self.exp_avg), ptr(self.exp_avg_sq), ptr(self.step_counter),
                ptr(x), groups, rpg, ptr(n_rows), ptr(edges), epg, ptr(n_edges), ptr(y), ptr(yv), ptr(self.cg_mean),
                ptr(self.cg_std), ptr(self.conf), ptr(self.metrics), mask, s))

        self._run_phases(phase)

    def step_padded(self, feat, n_rows, edges, n_edges, y, y_valid):
        """feat [G, S, D] f32 padded per frame, n_rows [G] int32 (device); edges [G, E, 2] (source, target) local row
        ids with n_edges [G] int32 (device) valid rows.  y / y_valid are indexed by the compacted row number.  Returns
        the confidence buffer (compacted order; the live prefix has sum(n_rows) entries — no host sync happens here)."""
        G, S = _check_padded(feat, n_rows, self.dim)
        edges, E = _check_edges(edges, n_edges, G)
        self._run(feat, G, S, n_rows, edges, E, n_edges, y, y_valid)
        return self.conf

    def step(self, x, edge_index, y, y_valid, ptr=None):
        """x [R, D] f32 with the batched graph edge_index [2, E] (Batch.from_data_list offsets), y [R] f32, y_valid [R]
        bool.  ``ptr`` (host, the batch's node boundaries): each node becomes a frame of its own, so the graph build
        scans each node's edges rather than the whole batch's; the result is the same bit for bit.  Returns the
        confidence vector [R]; metrics stay on the device in ``self.metrics``."""
        R = x.shape[0]
        if ptr is not None and len(ptr) > 2:
            feat, n_rows, edges, n_edges = _batch_as_frames(x, edge_index, ptr)
            self._run(feat, feat.shape[0], feat.shape[1], n_rows, edges, edges.shape[1], n_edges, y, y_valid)
            return self.conf[:R]
        edges, n_edges = _graph_as_padded(x, edge_index)
        self._run(x, 1, R, None, edges, edges.shape[1], n_edges, y, y_valid)
        return self.conf[:R]


class GcnInference:
    """SimpleGCN forward and per-row traversability / confidence on rows with their graph (csrc/gcn_train.cu, the
    trainer's forward kernels on a handle of its own).  Reads the model's flat parameters on every call."""

    def __init__(self, model, max_rows=1024, max_edges=8192):
        model.check_supported()
        _C.require_device()
        self.model = model
        self.dim, (self.h1, self.h2) = model.input_size, model.hidden
        self.cfg = TrainConfig(0.0, 0.0, 0.5, 0, 0.0, 0.9, 0.999, 1e-8)
        self._h = None
        self.max_rows, self.max_edges = 0, 0
        self._create(max_rows, max_edges)

    def _create(self, rows, edges):
        h = c_void_p()
        rows, edges = max(int(rows), self.max_rows), max(int(edges), self.max_edges)
        check(lib().wvn_gcn_trainer_create(self.dim, self.h1, self.h2, rows, edges, byref(self.cfg), None, byref(h)))
        if self._h is not None:
            lib().wvn_trainer_destroy(self._h)
        self._h, self.max_rows, self.max_edges = h, rows, edges

    def _run(self, x, groups, rpg, n_rows, edges, epg, n_edges, cg_mean=None, cg_std=None, std_factor=0.5,
             want_out=False, want_rows=True):
        if groups * rpg > self.max_rows or groups * epg > self.max_edges:
            self._create(max(self.max_rows, int(groups * rpg * 1.5)), max(self.max_edges, int(groups * epg * 1.5)))
        x = x.contiguous().float()
        dev = x.device
        out = torch.empty(groups * rpg, self.dim + 1, device=dev) if want_out else None
        trav = torch.full((2, groups * rpg), float("nan"), device=dev) if want_rows else None
        trav, conf = (trav[0], trav[1]) if want_rows else (None, None)
        check(lib().wvn_gcn_infer_rows(self._h, ptr(self.model.flat_params), ptr(x), groups, rpg, ptr(n_rows), ptr(edges),
                                       epg, ptr(n_edges), ptr(cg_mean), ptr(cg_std), float(std_factor), ptr(out),
                                       ptr(trav), ptr(conf), stream()))
        return out, trav, conf

    def forward_graph(self, x, edge_index):
        """SimpleGCN.forward: x [N, D] with edge_index [2, E] -> (N, 1 + D)."""
        N = x.shape[0]
        edges, n_edges = _graph_as_padded(x, edge_index)
        out, _, _ = self._run(x, 1, N, None, edges, edges.shape[1], n_edges, want_out=True, want_rows=False)
        return out

    def rows(self, x, edge_index, cg_mean, cg_std, std_factor):
        """x [N, D] with its graph edge_index [2, E] -> (trav [N], conf [N]) fp32."""
        N = x.shape[0]
        edges, n_edges = _graph_as_padded(x, edge_index)
        _, trav, conf = self._run(x, 1, N, None, edges, edges.shape[1], n_edges, cg_mean, cg_std, std_factor)
        return trav, conf

    def rows_padded(self, feat, n_rows, edges, n_edges, cg_mean, cg_std, std_factor):
        """feat [G, S, D] with n_rows [G] and the frames' edges [G, E, 2] / n_edges [G] -> (trav [G, S], conf [G, S]),
        padding rows NaN."""
        G, S = _check_padded(feat, n_rows, self.dim)
        edges, E = _check_edges(edges, n_edges, G)
        _, trav, conf = self._run(feat, G, S, n_rows, edges, E, n_edges, cg_mean, cg_std, std_factor)
        return trav.view(G, S), conf.view(G, S)

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                lib().wvn_trainer_destroy(self._h)
                self._h = None
        except Exception:
            pass


# --------------------------------------------------------------------------------------------
# LinearRnvp flow (anomaly-detection learner): fp32 row forward and online train step
# --------------------------------------------------------------------------------------------
def flow_buffers(model):
    """The wvn_flow_buffers of a LinearRnvp: its masks and permutations, read by the kernels on every call."""
    f = model.flows
    for t in (f[0].mask, f[2].mask, f[1].p, f[1].invp, f[3].p, f[3].invp):
        assert t.is_cuda and t.is_contiguous()
    assert f[0].mask.dtype == torch.float32 and f[1].p.dtype == torch.int64
    return FlowBuffers(f[0].mask.data_ptr(), f[2].mask.data_ptr(), f[1].p.data_ptr(), f[1].invp.data_ptr(),
                       f[3].p.data_ptr(), f[3].invp.data_ptr())


class FlowInference:
    """Owns a ``wvn_flow_infer_t`` (forward workspaces only): LinearRnvp.forward on rows in fp32, and the per-pixel
    anomaly map on wgmma (bf16 operands, fp32 accumulation; ``set_params`` re-packs them).  Traversability is
    ``ConfidenceGenerator.inference_without_update`` of the NLL ``-(logprob.sum(1) + log_det)``."""

    def __init__(self, dim=384, hidden=200, max_rows=1024, chunk_pixels=0):
        _C.require_device()
        self.dim, self.hidden, self.chunk_pixels = dim, hidden, chunk_pixels
        self._h = None
        self._params = None
        self._create(max_rows)

    def _create(self, max_rows):
        h = c_void_p()
        check(lib().wvn_flow_infer_create(self.dim, self.hidden, int(max_rows), int(self.chunk_pixels), byref(h)))
        if self._h is not None:
            lib().wvn_flow_infer_destroy(self._h)
        self._h = h
        self.max_rows = int(max_rows)
        if self._params is not None:
            self.set_params(self._params)

    def _reserve(self, rows):
        if rows > self.max_rows:
            self._create(int(rows * 1.5))

    def set_params(self, flat_params):
        """Re-pack the bf16 operands of the per-pixel path (after the parameters changed)."""
        assert flat_params.is_cuda and flat_params.dtype == torch.float32 and flat_params.is_contiguous()
        self._params = flat_params
        check(lib().wvn_flow_infer_set_params(self._h, ptr(flat_params), stream()))

    def rows(self, model, x, want_z=True, want_logprob=True):
        """x (R, D) fp32 -> dict(z (R,D), log_det (R,), logprob (R,D)), the reference's forward outputs."""
        R = x.shape[0]
        self._reserve(R)
        x = x.contiguous().float()
        z = torch.empty(R, self.dim, device=x.device) if want_z else None
        ld = torch.empty(R, device=x.device)
        lp = torch.empty(R, self.dim, device=x.device) if want_logprob else None
        check(lib().wvn_flow_infer_rows(self._h, ptr(model.flat_params), byref(flow_buffers(model)), ptr(x), R, ptr(z),
                                        ptr(ld), ptr(lp), None, None, 0.0, None, stream()))
        return {"z": z, "log_det": ld, "logprob": lp}

    def trav(self, model, x, cg_mean, cg_std, std_factor):
        """x (R, D) fp32 -> the confidence of each row's NLL under the generator (R,) fp32."""
        R = x.shape[0]
        self._reserve(R)
        x = x.contiguous().float()
        out = torch.empty(R, device=x.device)
        check(lib().wvn_flow_infer_rows(self._h, ptr(model.flat_params), byref(flow_buffers(model)), ptr(x), R, None,
                                        None, None, ptr(cg_mean), ptr(cg_std), float(std_factor), ptr(out), stream()))
        return out

    def trav_padded(self, model, feat, n_rows, cg_mean, cg_std, std_factor):
        """feat [G, S, D] fp32 with n_rows [G] int32 live rows per group -> trav [G, S] fp32, NaN on padding rows.
        Allocates nothing in the library once the handle holds G * S rows."""
        G, S = _check_padded(feat, n_rows, self.dim)
        self._reserve(G * S)
        out = torch.empty(G, S, device=feat.device)
        check(lib().wvn_flow_infer_rows_padded(self._h, ptr(model.flat_params), byref(flow_buffers(model)),
                                               ptr(feat.contiguous()), G, S, ptr(n_rows), ptr(cg_mean), ptr(cg_std),
                                               float(std_factor), ptr(out), stream()))
        return out

    def pixels(self, model, tokens, grid, out_hw, cg_mean, cg_std, std_factor, want_nll=False):
        """tokens (B, gh*gw, D) fp32 -> trav (B, H, W) fp32 (and the per-pixel NLL with want_nll).  Uses the operands
        of the last ``set_params``."""
        assert self._params is not None, "FlowInference.pixels: set_params was never called"
        B = tokens.shape[0]
        tokens = tokens.contiguous().float()
        trav = torch.empty(B, out_hw[0], out_hw[1], device=tokens.device)
        nll = torch.empty_like(trav) if want_nll else None
        check(lib().wvn_flow_infer_pixels(self._h, byref(flow_buffers(model)), ptr(tokens), B, grid[0], grid[1],
                                          out_hw[0], out_hw[1], ptr(cg_mean), ptr(cg_std), float(std_factor), ptr(trav),
                                          ptr(nll), stream()))
        return (trav, nll) if want_nll else trav

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                lib().wvn_flow_infer_destroy(self._h)
                self._h = None
        except Exception:
            pass


class FlowTrainer(_TrainerHandle):
    """The anomaly-detection train step on a LinearRnvp's flat fp32 parameters (csrc/flow_train.cu): forward, loss
    ``-mean(logprob.sum(1) + log_det)`` over the labelled rows, ConfidenceGenerator update with the per-row NLL,
    backward and Adam as one fixed launch sequence without host synchronisation.  ``exp_avg`` / ``exp_avg_sq`` /
    ``step_counter`` are torch.optim.Adam's state over the 24 parameter tensors, flattened in ``parameters()`` order.
    Rows may arrive padded per frame (``step_padded``).  With ``process_group`` the step is global-batch exact (see
    ``_TrainerHandle``): the NLL sums, the labelled-row count and the extrema are all-reduced after the forward, the
    gradient after the backward; the loss is the mean over the global labelled count."""

    def __init__(self, model, max_rows=4096, std_factor=0.5, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, process_group=None):
        _C.require_device()
        params = model.flat_params
        assert params.is_cuda and params.dtype == torch.float32
        self.model = model
        self.dim, self.hidden = model.input_size, model.hidden
        cfg = TrainConfig(0.0, 0.0, float(std_factor), 0, float(lr), betas[0], betas[1], float(eps))
        super().__init__(params.device, lib().wvn_flow_param_count(self.dim, self.hidden), cfg, max_rows, process_group)

    def _new_handle(self, max_rows):
        h = c_void_p()
        check(lib().wvn_flow_trainer_create(self.dim, self.hidden, max_rows, byref(self.cfg), ptr(self.grads),
                                            byref(h)))
        return h

    def _run(self, x, groups, rpg, n_rows, y_valid):
        self._reserve(groups * rpg)
        x = x.contiguous().float()
        yv = None if y_valid is None else y_valid.contiguous().to(torch.uint8)
        s = stream()

        def phase(mask):
            check(lib().wvn_flow_train_step_padded(
                self._h, ptr(self.model.flat_params), ptr(self.exp_avg), ptr(self.exp_avg_sq), ptr(self.step_counter),
                byref(flow_buffers(self.model)), ptr(x), groups, rpg, ptr(n_rows), ptr(yv), ptr(self.cg_mean),
                ptr(self.cg_std), ptr(self.conf), ptr(self.metrics), mask, s))

        self._run_phases(phase)

    def step_padded(self, feat, n_rows, y, y_valid):
        """feat [G, S, D] f32 padded per group, n_rows [G] int32 (device); y_valid (compacted numbering) selects the rows
        the flow learns from; ``y`` is ignored (AnomalyLoss uses no labels).  Returns the confidence buffer: the selected
        rows' confidences in order (the live prefix has metrics[3] entries — no host sync happens here)."""
        G, S = _check_padded(feat, n_rows, self.dim)
        self._run(feat, G, S, n_rows, y_valid)
        return self.conf

    def step(self, x, y_valid=None, phase_mask=7):
        """x (R, D) fp32; y_valid (R,) bool or None (every row).  Returns the confidence of the labelled rows in
        order (a view of length R whose first n entries are live; n is metrics[3]).  phase_mask (single process only):
        1 = forward + statistics + generator update, 2 = backward, 4 = Adam."""
        R = x.shape[0]
        if self.pg is not None:
            assert phase_mask == 7, "FlowTrainer.step: a data-parallel step runs whole"
            self._run(x, 1, R, None, y_valid)
            return self.conf[:R]
        self._reserve(R)
        x = x.contiguous().float()
        yv = None if y_valid is None else y_valid.contiguous().to(torch.uint8)
        check(lib().wvn_flow_train_step(self._h, ptr(self.model.flat_params), ptr(self.exp_avg), ptr(self.exp_avg_sq),
                                        ptr(self.step_counter), byref(flow_buffers(self.model)), ptr(x), R, ptr(yv),
                                        ptr(self.cg_mean), ptr(self.cg_std), ptr(self.conf), ptr(self.metrics),
                                        int(phase_mask), stream()))
        return self.conf[:R]


# --------------------------------------------------------------------------------------------
# EfficientNet-B0 backbone handle and its primitives
# --------------------------------------------------------------------------------------------
# (channels, stride) of the five taps: features.{2,3,4,6}.0.block.0 (expand convs) and features.8 (the head)
EFFNET_B0_TAPS = ((96, 2), (144, 4), (240, 8), (672, 16), (1280, 32))


def channel_pitch(c):
    """Channel pitch of the EfficientNet path's NHWC maps: c rounded up to 64, the GEMM's narrowest tile."""
    return (c + 63) // 64 * 64


def depthwise_silu(x, weight, bias, stride, out=None, partial=None):
    """x [B,H,W,P] bf16 NHWC (P % 8 == 0), weight [k,k,P] fp32, bias [P] fp32 -> (out [B,Ho,Wo,P] bf16 =
    bf16(SiLU(depthwise conv + bias)), partial [B, nblk, P] fp32 pool sums of the rounded outputs)."""
    B, H, W, P = x.shape
    k = weight.shape[0]
    pad = (k - 1) // 2
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    if out is None:
        out = torch.empty(B, Ho, Wo, P, device=x.device, dtype=torch.bfloat16)
    if partial is None:
        partial = torch.empty(B, lib().wvn_depthwise_pool_blocks(Ho, Wo), P, device=x.device, dtype=torch.float32)
    check(lib().wvn_depthwise_silu_bf16_nhwc(ptr(x.contiguous()), B, H, W, P, k, stride, ptr(weight.contiguous()),
                                             ptr(bias.contiguous()), ptr(out), ptr(partial), stream()))
    return out, partial


def se_gates(partial, hw, channels, fc1_w, fc1_b, fc2_w, fc2_b):
    """partial [B, nblk, P] (depthwise_silu's) -> gates [B, P] fp32 = sigmoid(fc2(SiLU(fc1(sum / hw)))), 0 past
    ``channels``; fc1_w [sq, P], fc2_w [P, sq]."""
    B, nblk, P = partial.shape
    gates = torch.empty(B, P, device=partial.device, dtype=torch.float32)
    check(lib().wvn_se_gates(ptr(partial.contiguous()), B, nblk, hw, channels, P, ptr(fc1_w.contiguous()),
                             ptr(fc1_b.contiguous()), fc1_w.shape[0], ptr(fc2_w.contiguous()), ptr(fc2_b.contiguous()),
                             ptr(gates), stream()))
    return gates


def channel_scale(x, gates):
    """In place: x [B,H,W,P] bf16 *= gates [B,P] per channel, rounded to bf16."""
    B, H, W, P = x.shape
    assert x.is_contiguous()
    check(lib().wvn_channel_scale_bf16_nhwc(ptr(x), B, H * W, P, ptr(gates.contiguous()), stream()))
    return x


def _pad_to(t, shape):
    out = torch.zeros(shape, dtype=torch.float32)
    out[tuple(slice(0, n) for n in t.shape)] = t
    return out


class EfficientNetBackbone:
    """Owns a ``wvn_effnet_t``: a torchvision EfficientNet-B0 trunk with batch norm folded in (GEMM weights bf16,
    depthwise and squeeze-excitation weights fp32, on device) and workspaces sized for ``max_batch``.  ``folded`` is
    weights.fold_efficientnet_bn's dict; this class zero-pads each tensor to the handle's channel pitches."""

    def __init__(self, image_size, folded, max_batch=32):
        _C.require_device()
        self.image_size, self.max_batch = image_size, max_batch
        h = c_void_p()
        check(lib().wvn_effnet_create(byref(EffnetConfig(image_size, max_batch)), byref(h)))
        self._h = h
        self.workspace_bytes = lib().wvn_effnet_workspace_bytes(h)
        # (channels, side, pitch) of each tap
        self.taps = [(c, image_size // s, channel_pitch(c)) for c, s in EFFNET_B0_TAPS]
        for name, (w, b) in folded.items():
            w = w.detach().to(dtype=torch.float32, device="cpu")
            b = b.detach().to(dtype=torch.float32, device="cpu")
            if name.endswith(".fc1"):
                w = _pad_to(w, (w.shape[0], channel_pitch(w.shape[1])))
            elif name.endswith(".fc2"):
                w, b = _pad_to(w, (channel_pitch(w.shape[0]), w.shape[1])), _pad_to(b, (channel_pitch(b.shape[0]),))
            elif w.shape[1] == 1 and w.shape[2] > 1:  # depthwise [c, 1, k, k] -> [k, k, P(c)]
                w = _pad_to(w[:, 0].permute(1, 2, 0), (w.shape[2], w.shape[3], channel_pitch(w.shape[0])))
                b = _pad_to(b, (channel_pitch(b.shape[0]),))
            elif name == "features.0":  # the stem: [out, (ky, kx, in)], rows padded
                w = _pad_to(w.permute(0, 2, 3, 1).reshape(w.shape[0], -1), (channel_pitch(w.shape[0]), 27))
                b = _pad_to(b, (channel_pitch(b.shape[0]),))
            else:  # 1 x 1 conv [out, in, 1, 1] -> [P(out), P(in)]
                w = _pad_to(w[:, :, 0, 0], (channel_pitch(w.shape[0]), channel_pitch(w.shape[1])))
                b = _pad_to(b, (channel_pitch(b.shape[0]),))
            w, b = w.contiguous(), b.contiguous()
            check(lib().wvn_effnet_set_weight(h, (name + ".weight").encode(), c_void_p(w.data_ptr()), w.numel()))
            check(lib().wvn_effnet_set_weight(h, (name + ".bias").encode(), c_void_p(b.data_ptr()), b.numel()))

    def forward(self, img: torch.Tensor):
        """img (B,3,S,S) fp32 CUDA in [0,1] -> the five taps, NHWC bf16 [B, S/s_l, S/s_l, c_l]: views of the first c_l
        channels of maps at the handle's channel pitch (whose pad channels are zero)."""
        B = img.shape[0]
        assert img.dtype == torch.float32 and tuple(img.shape[1:]) == (3, self.image_size, self.image_size)
        bufs = [torch.empty(B, n, n, p, device=img.device, dtype=torch.bfloat16) for _, n, p in self.taps]
        check(lib().wvn_effnet_forward(self._h, ptr(img.contiguous()), B, _ptr_array(bufs), stream()))
        return [t[..., :c] for t, (c, _, _) in zip(bufs, self.taps)]

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                lib().wvn_effnet_destroy(self._h)
                self._h = None
        except Exception:
            pass
