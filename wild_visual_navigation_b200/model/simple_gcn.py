"""SimpleGCN (reference: wild_visual_navigation/model/simple_gcn.py).

A stack of graph convolutions over the segment adjacency, ReLU between them, sigmoid on the first
``hidden_sizes[-1]`` output columns; with ``reconstruction`` the last layer also reconstructs the input, so the output
has SimpleMLP's ``(N, 1 + D)`` layout and ``TraversabilityLoss`` and the confidence generator apply unchanged.

Upstream imports ``GCNConv`` from torch_geometric (the import is commented out there, so upstream construction raises
``NameError``).  ``GCNConv`` below is the parameter container of torch_geometric 2.x's ``GCNConv(in, out)`` with its
defaults: ``bias`` [out] and ``lin.weight`` [out, in] in that ``state_dict`` order, glorot-uniform weight (drawn twice,
as torch_geometric's ``Linear.__init__`` and then ``GCNConv.reset_parameters`` do) and zero bias.  The arithmetic is
the CUDA kernels' (csrc/gcn_train.cu), which compute ``D^-1/2 (A + I) D^-1/2 X W^T + b`` with A directed as the edges
give it and D the in-degree plus one.  All parameters are views into one flat fp32 buffer (``flat_params``) in
``parameters()`` order, which is also torch.optim.Adam's state order.
"""
from __future__ import annotations

import math

import torch

from .simple_mlp import _flatten_parameters

MAX_DIM, MAX_HIDDEN = 1024, 512


class _Linear(torch.nn.Module):
    def __init__(self, in_channels: int, out_channels: int):
        super().__init__()
        self.weight = torch.nn.Parameter(torch.empty(out_channels, in_channels))
        self.reset_parameters()

    def reset_parameters(self):
        a = math.sqrt(6.0 / (self.weight.size(-2) + self.weight.size(-1)))
        with torch.no_grad():
            self.weight.uniform_(-a, a)


class GCNConv(torch.nn.Module):
    """The parameters of ``torch_geometric.nn.GCNConv(in_channels, out_channels)`` (defaults); see the module doc."""

    def __init__(self, in_channels: int, out_channels: int):
        super().__init__()
        self.in_channels, self.out_channels = in_channels, out_channels
        self.lin = _Linear(in_channels, out_channels)
        self.bias = torch.nn.Parameter(torch.empty(out_channels))
        self.reset_parameters()

    def reset_parameters(self):
        self.lin.reset_parameters()
        with torch.no_grad():
            self.bias.zero_()


class SimpleGCN(torch.nn.Module):
    """``SimpleGCN(input_size, reconstruction, hidden_sizes)`` with the reference's signature; the caller's
    ``hidden_sizes`` is left alone.  The kernels take ``hidden_sizes == [h1, h2, 1]`` with ``reconstruction=True``,
    1 <= D <= 1024 and 1 <= h1, h2 <= 512; any other shape can be built, but ``shape_error`` names what is missing and
    the trainer / inference handles raise ``ValueError``.  ``forward(data)`` needs ``data.edge_index``."""

    def __init__(self, input_size: int, reconstruction: bool, hidden_sizes=[64, 32, 1]):
        super().__init__()
        self.input_size = input_size
        self.reconstruction = reconstruction
        self.nr_sigmoid_layers = hidden_sizes[-1]
        layers, inp = [], input_size
        for j, h in enumerate(hidden_sizes):
            if reconstruction and j == len(hidden_sizes) - 1:
                h = h + input_size
            layers.append(GCNConv(inp, h))
            inp = h
        self.layers = torch.nn.ModuleList(layers)
        self.output_features = inp
        self.hidden = [int(h) for h in hidden_sizes[:-1]]
        self.flat_params = None
        self._infer = None
        self._flatten()

    def _flatten(self):
        _flatten_parameters(self, list(self.layers.parameters()))

    def _apply(self, fn, *args, **kwargs):
        super()._apply(fn, *args, **kwargs)
        self._flatten()  # .to(device) re-allocates: rebuild the flat buffer and the views
        return self

    def shape_error(self):
        """None when the CUDA kernels take this shape, else why they do not."""
        D = self.input_size
        if not self.reconstruction:
            return "SimpleGCN: the kernels need reconstruction=True (the loss reads the reconstruction columns)"
        if len(self.hidden) != 2 or self.nr_sigmoid_layers != 1:
            return f"SimpleGCN: the kernels take hidden_sizes [h1, h2, 1], got {self.hidden + [self.nr_sigmoid_layers]}"
        h1, h2 = self.hidden
        if not (1 <= D <= MAX_DIM and 1 <= h1 <= MAX_HIDDEN and 1 <= h2 <= MAX_HIDDEN):
            return (f"SimpleGCN({D}, [{h1}, {h2}, 1]) is outside the kernels' range (1 <= D <= {MAX_DIM}, "
                    f"1 <= h1, h2 <= {MAX_HIDDEN})")
        return None

    def check_supported(self):
        err = self.shape_error()
        if err is not None:
            raise ValueError(err)
        if self.flat_params is None or not self.flat_params.is_cuda:
            raise ValueError("SimpleGCN: the parameters must be on a CUDA device (no CPU fallback)")

    @torch.no_grad()
    def forward(self, data) -> torch.Tensor:
        """Returns (N, 1 + D) fp32 from the fp32 CUDA kernels: column 0 through the sigmoid, then the reconstruction,
        on the graph ``data.edge_index`` (2, E) over the rows ``data.x``."""
        self.check_supported()
        if getattr(data, "edge_index", None) is None:
            raise ValueError("SimpleGCN.forward: data has no edge_index")
        from .. import ops

        if self._infer is None:
            self._infer = ops.GcnInference(self)
        return self._infer.forward_graph(data.x, data.edge_index)
