"""TEST INFRASTRUCTURE ONLY (see oracle/__init__.py) — CPU/torch restatement of the footprint projection + rasterisation
that produces the supervision masks (SURVEY.md §8f rank 3, second half).

Follows wild_visual_navigation/image_projector/image_projector.py:
  ImageProjector.__init__ :17-86 (scaled camera matrix), check_validity :103-124, project :126-150,
  project_and_render :152-197, and its use in TraversabilityEstimator.add_supervision_node
  (traversability_estimator/traversability_estimator.py:261-284: mask * traversability, fmin into the nodes' masks).

The three kornia routines it calls are NOT in the reference repository (setup.py:11 ``kornia>=0.6.5``, unpinned, not installed
here) -> [EXTERNAL-RECALLED], restated from kornia's published source, parity unpinned against kornia itself:
  kornia.geometry.linalg.transform_points, kornia.geometry.camera.pinhole.PinholeCamera.project
  (both end in convert_points_from_homogeneous: scale = 1 / (z + 1e-8) where |z| > 1e-8, else 1),
  kornia.utils.draw.draw_convex_polygon / _get_convex_edges (scan-line fill between the left-most and right-most
  active edge of every image row).
``make_polygon_from_points`` follows wild_visual_navigation/utils/meshes.py:156-165 (pinned by tests/test_oracle.py
against the reference's own function, which is torch-only).
"""
from __future__ import annotations

import torch

EPS_H = 1e-8


def convert_points_from_homogeneous(p: torch.Tensor) -> torch.Tensor:
    z = p[..., -1:]
    scale = torch.where(z.abs() > EPS_H, 1.0 / (z + EPS_H), torch.ones_like(z))
    return scale * p[..., :-1]


def transform_points(T: torch.Tensor, pts: torch.Tensor) -> torch.Tensor:
    """T (B,4,4), pts (B,N,3) -> (B,N,3)."""
    ph = torch.cat([pts, torch.ones_like(pts[..., :1])], dim=-1)
    return convert_points_from_homogeneous(torch.bmm(ph, T.transpose(1, 2)))


def scaled_camera_matrix(K: torch.Tensor, h: int, w: int, new_h: int | None = None, new_w: int | None = None):
    """image_projector.py:44-75.  Returns (sK (B,4,4), H, W) of the rendered masks."""
    new_h = int(h) if new_h is None else new_h
    sy = new_h / h
    sx = (new_w / w) if new_w is not None else sy
    sK = K.clone()
    if new_w is None or new_w == new_h:
        sK[:, 0, 0] = K[:, 1, 1] * sy
        sK[:, 0, 2] = K[:, 1, 2] * sy
        sK[:, 1, 1] = K[:, 1, 1] * sy
        sK[:, 1, 2] = K[:, 1, 2] * sy
    else:
        sK[:, 0, 0] = K[:, 0, 0] * sx
        sK[:, 0, 2] = K[:, 0, 2] * sx
        sK[:, 1, 1] = K[:, 1, 1] * sy
        sK[:, 1, 2] = K[:, 1, 2] * sy
    return sK, new_h, (new_w if new_w is not None else new_h)


def project(sK: torch.Tensor, H: int, W: int, pose_camera_in_world: torch.Tensor, points_W: torch.Tensor):
    """image_projector.py:126-150 -> (projected (B,N,2), valid (B,N), valid_z (B,N))."""
    T_CW = pose_camera_in_world.inverse()
    pts_C = transform_points(T_CW, points_W)
    proj = convert_points_from_homogeneous(transform_points(sK, pts_C))      # PinholeCamera.project, extrinsics = I
    valid_z = pts_C[..., 2] >= 0
    valid = valid_z & (proj[..., 0] >= 0) & (proj[..., 0] <= W) & (proj[..., 1] >= 0) & (proj[..., 1] <= H)
    return proj, valid, valid_z


def convex_edges(polygon: torch.Tensor, h: int, w: int):
    """kornia.utils.draw._get_convex_edges: per image row the [x_left, x_right] span of the polygon."""
    if not torch.allclose(polygon[..., -1, :], polygon[..., 0, :]):
        polygon = torch.cat((polygon, polygon[..., :1, :]), dim=-2)
    x_start, y_start = polygon[..., :-1, 0], polygon[..., :-1, 1]
    x_end, y_end = polygon[..., 1:, 0], polygon[..., 1:, 1]
    ys = torch.arange(h, device=polygon.device, dtype=polygon.dtype)
    dx = ((x_end - x_start) / (y_end - y_start + 1e-12)).clamp(-w, w)
    xs = (ys[..., :, None] - y_start[..., None, :]) * dx[..., None, :] + x_start[..., None, :]
    valid = (y_start[..., None, :] <= ys[..., :, None]) & (ys[..., :, None] <= y_end[..., None, :])
    valid |= (y_start[..., None, :] >= ys[..., :, None]) & (ys[..., :, None] >= y_end[..., None, :])
    x_left = torch.where(valid, xs, torch.full_like(xs, w)).min(dim=-1).values
    x_right = torch.where(valid, xs, torch.full_like(xs, -1)).max(dim=-1).values
    return x_left, x_right


def draw_convex_polygon(images: torch.Tensor, polygons: torch.Tensor, colors: torch.Tensor) -> torch.Tensor:
    """kornia.utils.draw.draw_convex_polygon: images (B,C,H,W), polygons (B,N,2) as (x, y), colors (B,C) or (C,)."""
    B, C, H, W = images.shape
    if colors.dim() == 1:
        colors = colors.expand(B, C)
    x_left, x_right = convex_edges(polygons, H, W)
    ws = torch.arange(W, device=images.device, dtype=polygons.dtype)[None, None, :]
    fill = (ws >= x_left[..., :, None]) & (ws <= x_right[..., :, None])                # (B,H,W)
    return images + fill[:, None] * (colors[..., None, None] - images)


def project_and_render(sK, H, W, pose_camera_in_world, points, colors):
    """image_projector.py:152-197 without the optional overlay image -> (masks (B,3,H,W) NaN outside, projected, valid)."""
    proj, valid, valid_z = project(sK, H, W, pose_camera_in_world, points)
    proj = proj.clone()
    proj[~valid_z, :] = float("nan")
    masks = draw_convex_polygon(torch.zeros(sK.shape[0], 3, H, W, dtype=torch.float32, device=sK.device), proj, colors)
    masks[masks == 0.0] = float("nan")
    return masks, proj, valid


def update_supervision_masks(supervision_masks, masks, traversability):
    """traversability_estimator.py:282-284."""
    return torch.fmin(supervision_masks, masks * traversability)


def make_polygon_from_points(points: torch.Tensor, grid_size: int = 10) -> torch.Tensor:
    """utils/meshes.py:156-165: every edge of the (sorted) corner list sampled at grid_size points."""
    n = points.shape[0]
    w = torch.linspace(0, 1, steps=grid_size, device=points.device)
    out = [torch.lerp(points[i], points[(i + 1) % n], wi)[None] for i in range(n) for wi in w]
    return torch.cat(out, dim=0)


def synthetic_footprints(batch: int, seed: int = 0, image: int = 448):
    """A robot driving forward under ``batch`` cameras that look down at the ground ahead of it: (K (B,4,4),
    pose_camera_in_world (B,4,4), footprint (B,N,3)); some cameras see the footprint only partly or from behind."""
    g = torch.Generator().manual_seed(seed)
    f = 0.75 * image
    K = torch.tensor([[f, 0, image / 2, 0], [0, f, image / 2, 0], [0, 0, 1, 0], [0, 0, 0, 1.0]]).repeat(batch, 1, 1)
    poses = torch.eye(4).repeat(batch, 1, 1)
    for b in range(batch):
        pitch = 0.3 + 0.5 * torch.rand(1, generator=g).item()        # camera z axis pitched down towards the ground
        yaw = (torch.rand(1, generator=g).item() - 0.5) * 0.8
        cp, sp, cy, sy = torch.cos(torch.tensor(pitch)), torch.sin(torch.tensor(pitch)), torch.cos(torch.tensor(yaw)), torch.sin(torch.tensor(yaw))
        # camera axes in world: z forward-down, x right, y down
        z = torch.stack([cp * cy, cp * sy, -sp])
        x = torch.stack([sy, -cy, torch.tensor(0.0)])
        y = torch.linalg.cross(z, x)
        poses[b, :3, 0], poses[b, :3, 1], poses[b, :3, 2] = x, y, z
        poses[b, :3, 3] = torch.tensor([-0.6 - 1.5 * torch.rand(1, generator=g).item(), 0.6 * (torch.rand(1, generator=g).item() - 0.5),
                                        0.5 + 0.5 * torch.rand(1, generator=g).item()])
        if b % 7 == 6:  # a camera that has driven past the footprint: part of it is behind the image plane
            poses[b, 0, 3] = 0.9
    corners = torch.tensor([[0.4, 0.3, 0.0], [0.4, -0.3, 0.0], [1.3, -0.35, 0.0], [1.3, 0.25, 0.0]])
    fp = make_polygon_from_points(corners)[None].repeat(batch, 1, 1)
    return K, poses, fp
