"""SimpleMLP and DoubleMLP (reference: wild_visual_navigation/model/simple_mlp.py:10-67).

``D -> 256 -> 32 -> (1 + D)`` with ReLU, sigmoid on column 0, reconstruction head on the rest.
The module structure (``layers.{0,2,4}.{weight,bias}``), the seeded init and the quirk of
mutating the caller's ``hidden_sizes`` list are kept; all parameters are views into one flat
fp32 buffer (``flat_params``) in state-dict order so the fused CUDA train step / inference
kernels work on the very storage that ``state_dict()`` exposes.
"""
from __future__ import annotations

import torch

from .. import ops


def _flatten_parameters(module, ps):
    """Makes the parameters ``ps`` views into one flat fp32 buffer ``module.flat_params``, in that order."""
    if module.flat_params is not None and ps and ps[0].device == module.flat_params.device:
        off, same = 0, True
        for p in ps:  # already views of the flat buffer (a second .to(same device) must not move the storage the
            same &= p.data_ptr() == module.flat_params.data_ptr() + 4 * off  # CUDA trainer / inference handles hold)
            off += p.numel()
        if same:
            return
    flat = torch.cat([p.detach().reshape(-1) for p in ps]).contiguous()
    off = 0
    for p in ps:
        n = p.numel()
        p.data = flat[off : off + n].view_as(p)
        off += n
    module.flat_params = flat


class SimpleMLP(torch.nn.Module):
    def __init__(self, input_size: int = 64, hidden_sizes=[255], reconstruction: bool = False):
        super().__init__()
        layers = []
        self.nr_sigmoid_layers = hidden_sizes[-1]
        self.input_size = input_size
        if reconstruction:
            hidden_sizes[-1] = hidden_sizes[-1] + input_size  # mutates the caller's list, as upstream
        inp = input_size
        for hs in hidden_sizes[:-1]:
            layers.append(torch.nn.Linear(inp, hs))
            layers.append(torch.nn.ReLU())
            inp = hs
        layers.append(torch.nn.Linear(inp, hidden_sizes[-1]))
        self.layers = torch.nn.Sequential(*layers)
        self.output_features = hidden_sizes[-1]
        self.hidden = [int(h) for h in hidden_sizes[:-1]]
        self.reconstruction = reconstruction
        self.flat_params = None
        self._flatten()

    # ---- flat storage ---------------------------------------------------------------------
    def _flatten(self):
        _flatten_parameters(self, list(self.layers.parameters()))

    def _apply(self, fn, *args, **kwargs):
        super()._apply(fn, *args, **kwargs)
        self._flatten()  # .to(device) re-allocates: rebuild the flat buffer and the views
        return self

    def fused_ok(self) -> bool:
        return (self.reconstruction and len(self.hidden) == 2 and self.nr_sigmoid_layers == 1
                and self.flat_params is not None and self.flat_params.is_cuda)

    # ---- forward --------------------------------------------------------------------------
    @torch.no_grad()
    def forward(self, data) -> torch.Tensor:
        """Returns (M, 1 + D) fp32: column 0 through the sigmoid (fp32 CUDA-core kernels).
        The per-pixel node path does not go through here — see ``TraversabilityInference``."""
        if not self.fused_ok():
            raise RuntimeError("SimpleMLP.forward: only the hot-path shape (2 hidden layers, reconstruction, "
                               "1 sigmoid output, parameters on a CUDA device) is implemented; no CPU fallback")
        x = data.x
        return ops.mlp_forward_f32(self.flat_params, x.float(), self.input_size, self.hidden[0], self.hidden[1])


class DoubleMLP(torch.nn.Module):
    """DoubleMLP (reference: wild_visual_navigation/model/simple_mlp.py:42-67).

    Two networks read the same features: ``networks[0]`` is ``D -> h1 -> h2 -> 1`` through a sigmoid (traversability),
    ``networks[1]`` is ``D -> h1 -> h2 -> D`` (reconstruction); the output ``cat([sigmoid(net0(x)), net1(x)], 1)`` has
    SimpleMLP's ``(N, 1 + D)`` layout, so the loss, the confidence and the per-pixel heads read it unchanged.  The
    reconstruction error (the confidence signal) shares no hidden features with the traversability head.

    The module tree (``networks.{0,1}.{0,2,4}.{weight,bias}``), the seeded init and ``output_features`` are the
    reference's; unlike SimpleMLP it leaves the caller's ``hidden_sizes`` alone.  All 12 parameters are views into one
    flat fp32 buffer (``flat_params``) in ``parameters()`` order, which the CUDA train step and inference handles
    work on.  The kernels take two hidden layers and one sigmoid output (``hidden_sizes == [h1, h2, 1]``) with
    1 <= D <= 1024, 4 <= h1 <= 256, h1 % 4 == 0 and 1 <= h2 <= 32; any other shape can be built, but ``shape_error``
    names what is missing and the trainer / inference handles raise ``ValueError``."""

    def __init__(self, input_size: int = 64, hidden_sizes=[255]):
        super().__init__()
        self.nr_sigmoid_layers = hidden_sizes[-1]
        self.input_size = input_size
        networks = []
        for last in [hidden_sizes[-1], input_size]:
            layers, inp = [], input_size
            for hs in hidden_sizes[:-1]:
                layers.append(torch.nn.Linear(inp, hs))
                layers.append(torch.nn.ReLU())
                inp = hs
            layers.append(torch.nn.Linear(inp, last))
            networks.append(torch.nn.Sequential(*layers))
        self.networks = torch.nn.ModuleList(networks)
        self.output_features = hidden_sizes[-1] + input_size
        self.hidden = [int(h) for h in hidden_sizes[:-1]]
        self.flat_params = None
        self._flatten()

    def _flatten(self):
        _flatten_parameters(self, list(self.networks.parameters()))

    def _apply(self, fn, *args, **kwargs):
        super()._apply(fn, *args, **kwargs)
        self._flatten()  # .to(device) re-allocates: rebuild the flat buffer and the views
        return self

    def shape_error(self):
        """None when the CUDA kernels take this shape, else why they do not."""
        D = self.input_size
        if len(self.hidden) != 2 or self.nr_sigmoid_layers != 1:
            return (f"DoubleMLP: the kernels take hidden_sizes [h1, h2, 1], got {self.hidden + [self.nr_sigmoid_layers]}")
        h1, h2 = self.hidden
        if not (1 <= D <= 1024 and 4 <= h1 <= 256 and h1 % 4 == 0 and 1 <= h2 <= 32):
            return (f"DoubleMLP({D}, [{h1}, {h2}, 1]) is outside the kernels' range (1 <= D <= 1024, 4 <= h1 <= 256 and "
                    "a multiple of 4, 1 <= h2 <= 32)")
        return None

    def check_supported(self):
        err = self.shape_error()
        if err is not None:
            raise ValueError(err)
        if self.flat_params is None or not self.flat_params.is_cuda:
            raise ValueError("DoubleMLP: the parameters must be on a CUDA device (no CPU fallback)")

    @torch.no_grad()
    def forward(self, data) -> torch.Tensor:
        """Returns (M, 1 + D) fp32 from fp32 CUDA-core kernels: column 0 is sigmoid(networks[0](x)), columns 1..D are
        networks[1](x)."""
        self.check_supported()
        return ops.double_mlp_forward_f32(self.flat_params, data.x.float(), self.input_size, self.hidden[0],
                                          self.hidden[1])
