"""CPU tests of the segment-wise inference mode's arithmetic (oracle/segment_wise.py): the node's per-pixel evaluation of
``feat[seg.reshape(-1)]`` equals one evaluation per segment painted through ``seg``, in float64, for the SimpleMLP and
LinearRnvp goldens the reference's own modules made (tests/golden/make_golden.py, make_golden_rnvp.py)."""
import os

import pytest
import torch

from oracle import linear_rnvp as orn
from oracle import segment_wise as sw
from oracle import wvn_path


def _d(sd):
    return {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}


def _seg(n_segments, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    seg = torch.randint(0, n_segments, (h, w), generator=g)
    seg.view(-1)[:n_segments] = torch.arange(n_segments)   # every segment has a pixel
    return seg


def _same(a, b):
    return a.shape == b.shape and bool(((a - b).abs() <= 1e-12).all())


@pytest.fixture(scope="module")
def mlp_golden(golden_dir):
    return torch.load(os.path.join(golden_dir, "mlp_train.pt"))


@pytest.fixture(scope="module")
def flow_golden(golden_dir):
    return torch.load(os.path.join(golden_dir, "linear_rnvp.pt"), weights_only=False)["train"][("latest_measurement",
                                                                                               "odds")]


def _final_sd(g):
    """The model after the golden's training steps: the one whose prediction on xq the golden holds."""
    return _d(g["steps"][-1]["state_dict"])


def test_simple_mlp_rows_match_the_reference_prediction(mlp_golden):
    sd = _final_sd(mlp_golden)
    pred = wvn_path.mlp_forward(mlp_golden["xq"].double(), sd)
    assert (pred - mlp_golden["pred"].double()).abs().max().item() <= 1e-6


@pytest.mark.parametrize("hw", [(24, 24), (17, 31)])
def test_simple_mlp_segment_wise_equals_per_pixel(mlp_golden, hw):
    sd = _final_sd(mlp_golden)
    feat = mlp_golden["xq"].double()                       # 10 pooled rows
    seg = _seg(feat.shape[0], *hw, seed=hw[1])
    lr = ((wvn_path.mlp_forward(feat, sd)[:, 1:] - feat) ** 2).mean(1)
    mean, std = lr.mean().reshape(1) - 0.5 * lr.std(), lr.std().reshape(1)   # puts the rows inside the interval
    head = sw.mlp_head(sd, mean, std, 0.5)
    t_node, c_node = sw.node_maps(feat, seg, head)
    t_seg, c_seg = sw.segment_maps(feat, seg, head)
    assert t_node.dtype == torch.float64 and c_node.dtype == torch.float64
    assert _same(t_node, t_seg) and _same(c_node, c_seg)
    # the painted traversability is the reference's own prediction of the row
    assert (t_seg - mlp_golden["pred"].double()[:, 0][seg]).abs().max().item() <= 1e-6
    assert c_seg.std().item() > 0
    # negative control: another segmentation paints other rows
    t_other, _ = sw.segment_maps(feat, (seg + 1) % feat.shape[0], head)
    assert not _same(t_node, t_other)


def test_linear_rnvp_rows_match_the_reference_forward(flow_golden):
    sd = _d(flow_golden["init"])
    st = flow_golden["steps"][0]
    r = orn.forward(sd, st["x"].double())
    assert (r["log_det"] - st["log_det"].double()).abs().max().item() <= 1e-5
    assert (r["logprob"] - st["logprob"].double()).abs().max().item() <= 1e-5


@pytest.mark.parametrize("hw", [(24, 24), (13, 40)])
def test_linear_rnvp_segment_wise_equals_per_pixel(flow_golden, hw):
    sd = _d(flow_golden["init"])
    feat = flow_golden["steps"][0]["x"].double()            # 24 pooled rows
    seg = _seg(feat.shape[0], *hw, seed=hw[0])
    n = orn.nll(sd, feat)
    mean, std = n.mean().reshape(1) - 0.5 * n.std(), n.std().reshape(1)   # puts the rows inside the interval
    head = sw.flow_head(sd, mean, std, 0.5)
    t_node, c_node = sw.node_maps(feat, seg, head)
    t_seg, c_seg = sw.segment_maps(feat, seg, head)
    assert c_node is None and c_seg is None
    assert _same(t_node, t_seg)
    assert 0.05 < t_seg.mean().item() < 0.95
    t_other, _ = sw.segment_maps(feat, (seg + 1) % feat.shape[0], head)
    assert not _same(t_node, t_other)
