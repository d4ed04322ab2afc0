"""ORACLE (test infrastructure only) — CPU/PyTorch fp32 restatement of the in-repo half of the
WVN hot path.  Never imported by the product package.

Each function cites the reference code it follows (paths relative to the reference repo).
PARITY STATUS: pinned against the reference itself — ``tests/golden/make_golden.py`` path-imports
the reference's own ``SimpleMLP`` / ``TraversabilityLoss`` / ``ConfidenceGenerator`` /
``SegmentExtractor`` / ``DinoInterface.inference`` wrapper code from the reference repository and
stores their outputs as fixtures; ``tests/test_oracle.py`` checks this file against them
(plus the shipped known-answer ``assets/graph/{seg,center}.pt`` for the segment stage).
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from .dino_vit import ViTConfig, vit_feature_map

IMAGENET_MEAN = (0.485, 0.456, 0.406)
IMAGENET_STD = (0.229, 0.224, 0.225)


# ------------------------------------------------------------------------------------------
# transform + DinoInterface.inference          (feature_extractor/dino_interface.py:52-59, 70-92)
# ------------------------------------------------------------------------------------------
def resized_size(in_h: int, in_w: int, size: int) -> tuple[int, int]:
    """torchvision ``Resize(size:int)``: smaller edge -> size, aspect preserved (long = int(size*long/short))."""
    if in_h <= in_w:
        return size, int(size * in_w / in_h)
    return int(size * in_h / in_w), size


def wvn_transform(img: torch.Tensor, input_size: int) -> torch.Tensor:
    """``T.Compose([Resize(input_size, NEAREST), CenterCrop(input_size), Normalize(...)])``."""
    B, C, H, W = img.shape
    rh, rw = resized_size(H, W, input_size)
    if (rh, rw) != (H, W):
        img = F.interpolate(img, size=(rh, rw), mode="nearest")
    top = int(round((rh - input_size) / 2.0))
    left = int(round((rw - input_size) / 2.0))
    img = img[:, :, top : top + input_size, left : left + input_size]
    mean = torch.tensor(IMAGENET_MEAN, dtype=img.dtype, device=img.device).view(1, 3, 1, 1)
    std = torch.tensor(IMAGENET_STD, dtype=img.dtype, device=img.device).view(1, 3, 1, 1)
    return (img - mean) / std


def ros_image_to_float(img_u8_hwc: torch.Tensor) -> torch.Tensor:
    """``ros_image_to_torch`` (wild_visual_navigation_ros/.../ros_converter.py:113-126): torchvision ``ToTensor`` on
    the decoded rgb8 frame — (B,H,W,3) uint8 -> (B,3,H,W) float32 = value / 255."""
    return img_u8_hwc.permute(0, 3, 1, 2).to(torch.float32).div(255)


def resize_image(img: torch.Tensor, new_h: int) -> torch.Tensor:
    """``ImageProjector.resize_image`` for the square configuration (image_projector.py:55-59,199-200):
    ``T.Compose([T.Resize(new_h, NEAREST), T.CenterCrop(new_h)])`` on a (B,3,H,W) tensor."""
    B, C, H, W = img.shape
    if isinstance(new_h, (tuple, list)):   # T.Resize([new_h, new_w], NEAREST): the non-square configuration, no crop
        return F.interpolate(img, size=tuple(new_h), mode="nearest")
    rh, rw = resized_size(H, W, new_h)
    if (rh, rw) != (H, W):
        img = F.interpolate(img, size=(rh, rw), mode="nearest")
    top = int(round((rh - new_h) / 2.0))
    left = int(round((rw - new_h) / 2.0))
    return img[:, :, top : top + new_h, left : left + new_h]


@torch.no_grad()
def dino_inference(img: torch.Tensor, sd: dict, cfg: ViTConfig) -> torch.Tensor:
    """``DinoInterface.inference``: transform -> backbone -> bilinear(align_corners=True) to (H, H).

    Quirk kept: the output is (H, H) even if W != H (dino_interface.py:87-88)."""
    feats = vit_feature_map(wvn_transform(img, cfg.image_size), sd, cfg)
    H = img.shape[2]
    return F.interpolate(feats, (H, H), mode="bilinear", align_corners=True)


# ------------------------------------------------------------------------------------------
# Supervision label pooling                  (traversability_estimator/nodes.py:400-440)
# ------------------------------------------------------------------------------------------
@torch.no_grad()
def update_supervision_signal(supervision_mask: torch.Tensor, feature_segments: torch.Tensor):
    """``MissionNode.update_supervision_signal``: mask (C,H,W) with NaN = unlabelled, segments (H,W) long ->
    (supervision_signal (S,), supervision_signal_valid (S,)), S = segments.max() + 1.  Same arithmetic as the
    reference (nanmean over channels, per-segment sum / count of the non-NaN pixels, nan_to_num(0), > 0) without
    its (H, W, S) expansion."""
    signal = supervision_mask.nanmean(axis=0)
    S = int(feature_segments.max()) + 1
    ok = ~torch.isnan(signal)
    ids = feature_segments[ok]
    cnt = torch.zeros(S, dtype=signal.dtype, device=signal.device).index_add_(0, ids, torch.ones_like(signal[ok]))
    tot = torch.zeros(S, dtype=signal.dtype, device=signal.device).index_add_(0, ids, signal[ok])
    mean = (tot / cnt).nan_to_num(0)
    return mean, mean > 0


# ------------------------------------------------------------------------------------------
# SegmentExtractor                              (feature_extractor/segment_extractor.py:40-92)
# ------------------------------------------------------------------------------------------
@torch.no_grad()
def adjacency_list(seg: torch.Tensor) -> torch.Tensor:
    """seg: (1,1,H,W) long.  Directed pairs (left/top id, right/bottom id) of 4-neighbour segment
    boundaries, unique, ordered by key = left + right*(max+1) — what the reference's four shifted
    difference filters + float64 ``torch.unique`` produce."""
    s = seg[0, 0]
    div = int(s.max()) + 1
    hl, hr = s[:, :-1], s[:, 1:]
    vt, vb = s[:-1, :], s[1:, :]
    mh, mv = hl != hr, vt != vb
    left = torch.cat([hl[mh], vt[mv]])
    right = torch.cat([hr[mh], vb[mv]])
    key = torch.unique(left + right * div)
    return torch.stack([key % div, key // div], dim=1)


@torch.no_grad()
def centers(seg: torch.Tensor) -> torch.Tensor:
    """Per-segment centroid in (x=col, y=row) order (segment_extractor.py:83-89)."""
    s = seg[0, 0]
    n = int(s.max()) + 1
    out = []
    for i in range(n):
        ys, xs = torch.where(s == i)
        out.append(torch.stack([xs.float().mean(), ys.float().mean()]))
    return torch.stack(out)


# ------------------------------------------------------------------------------------------
# FeatureExtractor.sparsify_features default branch     (feature_extractor.py:389-396)
# ------------------------------------------------------------------------------------------
@torch.no_grad()
def sparsify_features(dense: torch.Tensor, seg: torch.Tensor) -> torch.Tensor:
    feats = []
    for i in range(int(seg.max()) + 1):
        x, y = torch.where(seg == i)
        feats.append(dense[0, :, x, y].mean(dim=1))
    return torch.stack(feats, dim=1).T


def relabel(seg: torch.Tensor) -> torch.Tensor:
    """``for i, k in enumerate(seg.unique()): seg[seg == k] = i`` (feature_extractor.py:245-246)."""
    out = seg.clone()
    for i, k in enumerate(seg.unique()):
        out[seg == k] = i
    return out


# ------------------------------------------------------------------------------------------
# SimpleMLP                                      (model/simple_mlp.py:10-39)
# ------------------------------------------------------------------------------------------
def mlp_init(dim: int = 384, hidden=(256, 32), seed: int = 42) -> dict:
    """``torch.manual_seed(42); SimpleMLP(D, [256, 32, 1], reconstruction=True)`` — same module
    construction order as the reference, so the same seeded init (traversability_estimator.py:78-80)."""
    torch.manual_seed(seed)
    sizes = list(hidden) + [1 + dim]
    layers, inp = [], dim
    for hs in sizes[:-1]:
        layers.append(torch.nn.Linear(inp, hs))
        layers.append(torch.nn.ReLU())
        inp = hs
    layers.append(torch.nn.Linear(inp, sizes[-1]))
    seq = torch.nn.Sequential(*layers)
    return {f"layers.{k}": v.detach().clone() for k, v in seq.state_dict().items()}


def mlp_forward(x: torch.Tensor, sd: dict) -> torch.Tensor:
    h = F.relu(F.linear(x, sd["layers.0.weight"], sd["layers.0.bias"]))
    h = F.relu(F.linear(h, sd["layers.2.weight"], sd["layers.2.bias"]))
    out = F.linear(h, sd["layers.4.weight"], sd["layers.4.bias"])
    return torch.cat([torch.sigmoid(out[:, :1]), out[:, 1:]], dim=1)  # x[:, :1] = sigmoid(x[:, :1])


# ------------------------------------------------------------------------------------------
# ConfidenceGenerator                           (utils/confidence_generator.py:78-82, 182-193)
# ------------------------------------------------------------------------------------------
def confidence_inference(x: torch.Tensor, mean: torch.Tensor, std: torch.Tensor, std_factor: float) -> torch.Tensor:
    shifted = mean + std * std_factor
    lo = torch.maximum(shifted - std, torch.zeros_like(std))
    hi = shifted + std
    xc = torch.clip(x, lo, hi)
    return (1 - ((xc - lo) / (hi - lo))).float()


class ConfidenceState:
    """``ConfidenceGenerator`` (utils/confidence_generator.py:13-212) as a plain state machine: ``update(x, x_positive)``
    for the four methods — latest_measurement :78-82, running_mean :94-115, moving_average :117-129 (window 5),
    kalman_filter :131-145 with ``KalmanFilter`` (utils/kalman_filter.py:78-111; D = 1, proc_model 1, proc_cov 0.2,
    meas_model 1, meas_cov 1, no outlier rejection) — with the reference's dtypes (float32 state, float64 running sums)."""

    def __init__(self, std_factor: float, method: str = "latest_measurement"):
        assert method in ("latest_measurement", "running_mean", "moving_average", "kalman_filter")
        self.std_factor, self.method = std_factor, method
        self.mean, self.var, self.std = torch.zeros(1), torch.ones(1, 1), torch.ones(1)
        self.running = torch.zeros(3, dtype=torch.float64)      # n, sum, sum of squares
        self.window = []                                        # the deque(maxlen=5) of x_positive tensors
        self.kf_proc_cov, self.kf_meas_cov = 0.2, 1.0

    def update(self, x: torch.Tensor, xp: torch.Tensor) -> torch.Tensor:
        x, xp = x.detach(), xp.detach()
        if self.mean.device != x.device:   # the state follows the data (the GPU-eager leg of bench.py runs on cuda)
            self.mean, self.var, self.std = self.mean.to(x.device), self.var.to(x.device), self.std.to(x.device)
            self.running = self.running.to(x.device)
        m = self.method
        if m == "latest_measurement":
            self.mean[0], self.std[0] = xp.mean(), xp.std()
            return confidence_inference(x, self.mean, self.std, self.std_factor)
        if m == "running_mean":
            self.running += torch.stack([torch.tensor(float(xp.numel()), dtype=torch.float64, device=x.device), xp.sum().double(),
                                         (xp ** 2).sum().double()])
            self.mean[0] = self.running[1] / self.running[0]
            self.var[0] = self.running[2:3] / self.running[0] - self.mean ** 2     # float64 - float32 -> float64 -> float32
            self.std[0] = torch.sqrt(self.var)[0, 0]
            return confidence_inference(x, self.mean, self.std, self.std_factor)
        if m == "moving_average":
            self.window = (self.window + [xp])[-5:]
            w = torch.cat(self.window, dim=0)
            self.mean[0], self.std[0] = w.mean(), w.std()
            xc = torch.clip(x, self.mean - 2 * self.std, self.mean + 2 * self.std)
            return ((xc - xc.min()) / (xc.max() - xc.min())).float()
        # kalman_filter
        if xp.shape[0] != 0:
            meas = xp.mean()
            state, cov = self.mean.clone(), self.var.clone() + self.kf_proc_cov        # prediction with F = 1
            innovation = meas - state
            gain = cov / (cov + self.kf_meas_cov)
            self.mean[0] = (state + (gain @ innovation))[0]
            self.var[0, 0] = ((1.0 - gain) @ cov)[0, 0]
        self.std[0] = torch.sqrt(self.var)[0, 0]
        conf = torch.exp(-(((x - self.mean) / (self.std * self.std_factor)) ** 2) * 0.5)
        conf[x < self.mean] = 1.0
        return conf.float()


# ------------------------------------------------------------------------------------------
# TraversabilityLoss.forward                     (utils/loss.py:93-160), anomaly_balanced, MSE
# ------------------------------------------------------------------------------------------
def traversability_loss(res, x, y, y_valid, w_trav=0.03, w_reco=0.5, std_factor=0.5, anomaly_balanced=True, cg=None):
    """Returns (loss, aux) with aux holding loss_reco, loss_trav, loss_trav_confidence, confidence,
    and the updated generator (mean, std).  ``cg``: a ConfidenceState carried across steps (default: a fresh
    'latest_measurement' generator, which has no memory)."""
    D = x.shape[1]
    loss_reco = F.mse_loss(res[:, -D:], x, reduction="none").mean(dim=1)
    with torch.no_grad():
        if cg is None:
            cg = ConfidenceState(std_factor)
        conf = cg.update(loss_reco, loss_reco[y_valid])
        mean, std = cg.mean.clone(), cg.std.clone()
    raw = F.mse_loss(res[:, :-D].squeeze(), y, reduction="none")
    labeled = raw[y_valid]
    unlabeled_w = raw[~y_valid] * (1 - conf)[~y_valid]
    if anomaly_balanced:
        l_trav = (unlabeled_w.sum() + labeled.sum()) / y.shape[0]
    else:
        l_trav = raw.mean()
    l_reco = loss_reco[y_valid].mean()
    loss = w_trav * l_trav + w_reco * l_reco
    aux = {
        "loss_reco": l_reco,
        "loss_trav": raw.mean(),
        "loss_trav_confidence": l_trav,
        "confidence": conf,
        "mean": mean,
        "std": std,
    }
    return loss, aux


def train_step(sd: dict, opt_state: dict, x, y, y_valid, lr=1e-3, **loss_kw):
    """One ``TraversabilityEstimator.train()`` body (traversability_estimator.py:464-477) using
    torch autograd + ``torch.optim.Adam`` on copies of ``sd``.  Returns (new_sd, new_opt_state, metrics)."""
    params = {k: v.detach().clone().requires_grad_(True) for k, v in sd.items()}
    opt = torch.optim.Adam(list(params.values()), lr=lr)
    if opt_state:
        opt.load_state_dict(opt_state)
    res = mlp_forward(x, params)
    loss, aux = traversability_loss(res, x, y, y_valid, **loss_kw)
    opt.zero_grad()
    loss.backward()
    grads = {k: v.grad.detach().clone() for k, v in params.items()}
    opt.step()
    new_sd = {k: v.detach().clone() for k, v in params.items()}
    metrics = {
        "loss_total": loss.item(),
        "loss_trav": aux["loss_trav"].item(),
        "loss_reco": aux["loss_reco"].item(),
        "loss_trav_confidence": aux["loss_trav_confidence"].item(),
        "mean": aux["mean"].item(),
        "std": aux["std"].item(),
        "confidence": aux["confidence"].detach(),
        "grads": grads,
    }
    return new_sd, opt.state_dict(), metrics


# ------------------------------------------------------------------------------------------
# per-pixel inference          (wild_visual_navigation_ros/scripts/wvn_feature_extractor_node.py:319-370)
# ------------------------------------------------------------------------------------------
@torch.no_grad()
def pixel_inference(dense: torch.Tensor, mlp_sd: dict, mean, std, std_factor: float):
    """dense: (1, D, H, W) -> (trav (H,W), conf (H,W))."""
    _, D, H, W = dense.shape
    x = dense[0].permute(1, 2, 0).reshape(-1, D)
    pred = mlp_forward(x, mlp_sd)
    trav = pred.reshape(H, W, -1)[:, :, 0]
    loss_reco = F.mse_loss(pred[:, 1:], x, reduction="none").mean(dim=1)
    conf = confidence_inference(loss_reco, mean, std, std_factor).reshape(H, W)
    return trav, conf


def synthetic_supervision(n_rows: int, seed: int = 2, p_valid: float = 0.16):
    """y_valid ~ Bernoulli(0.16), y = y_valid * U(0.001, 1] (SURVEY.md §8d; mirrors assets/graph/graph.pt
    statistics and the clamp(min=0.001) of supervision_generator.py:127)."""
    g = torch.Generator().manual_seed(seed)
    y_valid = torch.rand(n_rows, generator=g) < p_valid
    if y_valid.sum() < 2:
        y_valid[:2] = True
    y = torch.where(y_valid, torch.rand(n_rows, generator=g).clamp(min=0.001), torch.zeros(n_rows))
    return y, y_valid
