"""GPU parity of the footprint projection + rasterisation (csrc/footprint_kernels.cu, ImageProjector) against the golden
written by the reference's own ImageProjector class and against the oracle (oracle/image_projector.py) at the bench
image size; then the whole label path footprint -> supervision masks -> per-segment labels.

Bar: the rasterised masks are integer work (which pixels are inside) — identical NaN pattern and identical values,
except that a pixel whose centre lies within float rounding of a polygon edge may fall on the other side, because the
projected vertices differ in the last bits (the reference inverts the pose by LU in fp32 and multiplies with an
unspecified summation order; the kernel uses a cofactor inverse in fp64 and FMAs): projected points <= 2e-5 relative
(+ 1e-4 px), at most 1e-4 of the pixels of a mask may differ and only next to an edge.
"""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu


def _compare_masks(got, want, max_frac=1e-4, check_border=True):
    assert got.shape == want.shape
    diff = (got.isnan() != want.isnan()) | (torch.nan_to_num(got) != torch.nan_to_num(want))
    frac = diff.float().mean().item()
    if frac > 0 and check_border:   # a differing pixel must touch the boundary of the reference's fill
        inside = ~want.isnan().all(1, keepdim=True)
        f = inside.float()
        border = torch.nn.functional.max_pool2d(f, 3, 1, 1) != -torch.nn.functional.max_pool2d(-f, 3, 1, 1)
        assert not (diff.any(1, keepdim=True) & ~border).any(), "mask differs away from a polygon edge"
    assert frac <= max_frac, f"{frac:.2e} of the mask pixels differ"
    return frac


def _close_points(got, want):
    assert torch.equal(got.isnan(), want.isnan())
    g, w = torch.nan_to_num(got), torch.nan_to_num(want)
    assert ((g - w).abs() <= 2e-5 * w.abs() + 1e-4).all(), (g - w).abs().max().item()


def test_image_projector_matches_reference_golden(golden_dir):
    from wild_visual_navigation_b200.image_projector import ImageProjector

    g = torch.load(os.path.join(golden_dir, "image_projector.pt"))
    B = g["K"].shape[0]
    fp = g["polygon"][None].repeat(B, 1, 1).cuda()
    for tag in ("square", "rect", "native"):
        w = g[tag]
        im = ImageProjector(g["K"].cuda(), torch.tensor(g["h"]), torch.tensor(g["w"]), **w["kw"])
        assert torch.equal(im.camera.intrinsics.cpu(), w["sK"])
        assert torch.equal(im.scaled_camera_matrix.cpu(), w["sK"][:3, :3])
        masks, overlay, proj, valid = im.project_and_render(g["poses"].cuda(), fp, w["colors"].cuda())
        assert overlay is None
        _close_points(proj.cpu(), w["projected"])
        assert torch.equal(valid.cpu(), w["valid"])
        _compare_masks(masks.cpu(), w["masks"], max_frac=2e-3)   # tiny masks: one edge pixel is already 1e-3
        assert torch.equal(im.resize_image(g["img"].cuda()).cpu(), w["resized"])
        p2, v2, vz = im.project(g["poses"].cuda(), fp)
        assert torch.equal(torch.nan_to_num(p2), torch.nan_to_num(proj)) and torch.equal(v2, valid)
        assert torch.equal(vz.cpu(), ~w["projected"][..., 0].isnan())


@pytest.mark.parametrize("batch,colors", [(32, "ones"), (5, "batched"), (1, "zero_channel")])
def test_project_and_render_vs_oracle_448(batch, colors):
    from oracle import image_projector as oip
    from wild_visual_navigation_b200.image_projector import ImageProjector

    K, poses, fp = oip.synthetic_footprints(batch, seed=batch)
    col = {"ones": torch.ones(3), "batched": torch.rand(batch, 3, generator=torch.Generator().manual_seed(1)) + 0.1,
           "zero_channel": torch.tensor([0.0, 1.0, 0.0])}[colors]
    sK, H, W = oip.scaled_camera_matrix(K, 1080, 1440, 448)
    want, wproj, wvalid = oip.project_and_render(sK, H, W, poses, fp, col)
    im = ImageProjector(K.cuda(), 1080, 1440, new_h=448)
    masks, _, proj, valid = im.project_and_render(poses.cuda(), fp.cuda(), col.cuda())
    _close_points(proj.cpu(), wproj)
    assert torch.equal(valid.cpu(), wvalid)
    frac = _compare_masks(masks.cpu(), want)
    drawn = (~want.isnan()).any(1).flatten(1).any(1).sum().item()
    print(f"B={batch} colors={colors}: {drawn} of {batch} cameras see the footprint; differing pixels {frac:.1e}")
    assert drawn >= max(1, batch // 2)
    # the image overlay (visualisation branch of project_and_render)
    img = torch.rand(batch, 3, 448, 448, generator=torch.Generator().manual_seed(2))
    _, overlay, _, _ = im.project_and_render(poses.cuda(), fp.cuda(), col.cuda(), img.cuda())
    want_overlay = oip.draw_convex_polygon(img.clone(), wproj, col)
    same = ((overlay.cpu() - want_overlay).abs() <= 1e-6).float().mean().item()   # img + (col - img) rounds, col does not
    assert same >= 1 - 1e-4


def test_fused_supervision_update_and_label_pooling():
    """traversability_estimator.py:261-289 as the CUDA path runs it: several footprints rendered into the mission nodes'
    supervision masks (fmin with mask * traversability, in place, no temporaries), then the per-segment labels
    (update_supervision_signal) from those masks — against the oracle chain."""
    from oracle import image_projector as oip
    from oracle import wvn_path
    from wild_visual_navigation_b200 import ops
    from wild_visual_navigation_b200.image_projector import ImageProjector

    B, S = 8, 448
    K, poses, fp = oip.synthetic_footprints(B, seed=11)
    sK, H, W = oip.scaled_camera_matrix(K, S, S)
    im = ImageProjector(K.cuda(), S, S)
    sup_ref = torch.full((B, 3, S, S), float("nan"))
    sup = sup_ref.clone().cuda()
    color = torch.ones(3)
    g = torch.Generator().manual_seed(4)
    for step in range(4):    # the robot advances: the footprint moves forward, each with its own traversability
        pts = fp + torch.tensor([0.35 * step, 0.05 * step, 0.0])
        trav = torch.rand(1, generator=g) * 0.9 + 0.05
        masks, _, _ = oip.project_and_render(sK, H, W, poses, pts, color)
        sup_ref = oip.update_supervision_masks(sup_ref, masks, trav)
        im.update_supervision_masks(sup, poses.cuda(), pts.cuda(), color.cuda(), trav.cuda())
    _compare_masks(sup.cpu(), sup_ref, max_frac=4e-4, check_border=False)   # four overlapping outlines
    labelled = (~sup_ref.isnan()).float().mean().item()
    assert labelled > 0.01
    # per-segment labels from the masks: 7x7 grid segments
    seg = (torch.arange(S)[:, None] // 64 * 7 + torch.arange(S)[None, :] // 64).expand(B, S, S).contiguous()
    y, yv = ops.pool_supervision(seg.cuda(), sup, 49)
    for b in range(B):
        y_ref, yv_ref = wvn_path.update_supervision_signal(sup.cpu()[b], seg[b])
        assert torch.equal(yv[b].cpu(), yv_ref) and (y[b].cpu() - y_ref).abs().max() <= 1e-5   # fp32 means over 4096-pixel cells, other summation order
