"""LinearRnvp (reference: wild_visual_navigation/model/linear_rnvp.py:216-296), the anomaly-detection learner.

A RealNVP flow: ``flows`` = [coupling 0, permutation 1, coupling 2, permutation 3].  Every coupling holds a ``mask``
buffer and two nets ``s`` and ``t`` (``Linear(D,h) ReLU Linear(h,h) ReLU Linear(h,D)``, ``t`` a deep copy of ``s``);
every permutation holds ``p`` and ``invp``.  The module tree, the state-dict names / shapes / order (buffers included)
and the seeded init (the same ``nn.Linear`` and ``randperm`` calls in the same order) are the reference's.  All
parameters are views into one flat fp32 buffer (``flat_params``) in ``parameters()`` order, so the CUDA kernels
(csrc/flow_train.cu) and ``torch.optim.Adam``-format checkpoints see the very storage ``state_dict()`` exposes.

Supported is what the configuration can express and the kernels honour: a one-element ``coupling_topology`` [h] with
8 <= h <= 512 and h a multiple of 8, 2 <= input_size <= 4096, ``mask_type`` "odds" or "half", ``use_permutation=True``,
``flow_n=2``.  Everything else raises ``ValueError`` at construction.  The inverse flow (``backward`` / ``sample``) has no
caller in WVN and is not implemented.
"""
from __future__ import annotations

import copy

import torch
from torch import nn

from .. import ops


class LinearCouplingLayer(nn.Module):
    """The reference's coupling layer (linear_rnvp.py:67-152) without conditioning: parameters and mask only; the
    arithmetic runs in the flow kernels."""

    def __init__(self, input_size: int, mask: torch.Tensor, hidden: int):
        super().__init__()
        self.register_buffer("mask", mask)
        self.dim = input_size
        # Linear(D, h), then the topology loop's Linear(topology[-1], h) (linear_rnvp.py:96-104), then Linear(h, D)
        self.s = nn.Sequential(nn.Linear(input_size, hidden), nn.ReLU(), nn.Linear(hidden, hidden), nn.ReLU(),
                               nn.Linear(hidden, input_size))
        self.t = copy.deepcopy(self.s)


class Permutation(nn.Module):
    """linear_rnvp.py:155-174: ``p = randperm(in_ch)``, ``invp = argsort(p)``."""

    def __init__(self, in_ch: int):
        super().__init__()
        self.in_ch = in_ch
        self.register_buffer("p", torch.randperm(in_ch))
        self.register_buffer("invp", torch.argsort(self.p))


class LinearRnvp(nn.Module):
    def __init__(self, input_size, coupling_topology, flow_n=2, use_permutation=False, batch_norm=False,
                 mask_type="odds", conditioning_size=None, single_function=False, **kwargs):
        super().__init__()
        if conditioning_size:
            raise ValueError("LinearRnvp: conditioning (conditioning_size > 0) is not supported")
        if single_function:
            raise ValueError("LinearRnvp: single_function=True is not supported")
        if batch_norm:
            raise ValueError("LinearRnvp: batch_norm=True is not supported")
        if not use_permutation:
            raise ValueError("LinearRnvp: only use_permutation=True (the configured value) is supported")
        if flow_n != 2:
            raise ValueError(f"LinearRnvp: flow_n={flow_n}; only 2 (the reference's default) is supported")
        if coupling_topology is None or len(coupling_topology) != 1:
            raise ValueError(f"LinearRnvp: coupling_topology must have exactly one width, got {coupling_topology!r}")
        hidden = int(coupling_topology[0])
        if not (8 <= hidden <= 512 and hidden % 8 == 0):
            raise ValueError(f"LinearRnvp: hidden width {hidden} outside the kernels' range (8..512, multiple of 8)")
        input_size = int(input_size)
        if not 2 <= input_size <= 4096:
            raise ValueError(f"LinearRnvp: input_size {input_size} outside the kernels' range (2..4096)")
        if mask_type == "odds":
            mask = torch.arange(0, input_size).float() % 2
        elif mask_type == "half":
            mask = torch.zeros(input_size)
            mask[: input_size // 2] = 1
        else:
            raise ValueError(f"LinearRnvp: mask_type {mask_type!r} (odds, half)")
        self.input_size = input_size
        self.hidden = hidden
        self.mask_type = mask_type
        self.register_buffer("prior_mean", torch.zeros(input_size))
        self.register_buffer("prior_var", torch.ones(input_size))
        blocks = []
        for _ in range(flow_n):
            blocks.append(LinearCouplingLayer(input_size, mask, hidden))   # both couplings hold the same mask (:252-265)
            blocks.append(Permutation(input_size))
        self.flows = nn.Sequential(*blocks)
        self.flat_params = None
        self._rows = None
        self._flatten()

    # ---- flat storage (as SimpleMLP) ---------------------------------------------------------
    def _flatten(self):
        ps = list(self.parameters())
        if self.flat_params is not None and ps[0].device == self.flat_params.device:
            off, same = 0, True
            for p in ps:
                same &= p.data_ptr() == self.flat_params.data_ptr() + 4 * off
                off += p.numel()
            if same:
                return
        flat = torch.cat([p.detach().reshape(-1) for p in ps]).contiguous()
        off = 0
        for p in ps:
            n = p.numel()
            p.data = flat[off : off + n].view_as(p)
            off += n
        self.flat_params = flat

    def _apply(self, fn, *args, **kwargs):
        super()._apply(fn, *args, **kwargs)
        self._flatten()
        self._rows = None
        return self

    def load_state_dict(self, state_dict, strict: bool = True, assign: bool = False):
        for key, want in (("prior_mean", 0.0), ("prior_var", 1.0)):
            v = state_dict.get(key)
            if v is not None and not bool(torch.all(v == want)):
                raise ValueError(f"LinearRnvp: {key} must be all {want} (the kernels assume the N(0, 1) prior)")
        if assign:
            raise ValueError("LinearRnvp: assign=True would detach the parameters from flat_params")
        return super().load_state_dict(state_dict, strict=strict)

    # ---- forward --------------------------------------------------------------------------------
    @property
    def prior(self):
        return torch.distributions.Normal(self.prior_mean, self.prior_var)   # prior_var is the scale, as upstream

    def _row_handle(self, rows):
        if self.flat_params is None or not self.flat_params.is_cuda:
            raise RuntimeError("LinearRnvp.forward: parameters must be on a CUDA device; there is no CPU fallback")
        if self._rows is None:   # forward workspaces only
            self._rows = ops.FlowInference(self.input_size, self.hidden, max(int(rows), 64))
        return self._rows

    @torch.no_grad()
    def forward(self, data):
        """The reference's ``{"z", "log_det", "logprob"}`` for ``data.x`` (R, D), from the fp32 row kernels."""
        x = data.x
        return self._row_handle(x.shape[0]).rows(self, x)

    @torch.no_grad()
    def nll_confidence(self, x, confidence_generator):
        """Per-row traversability in anomaly mode: ``inference_without_update`` of -(logprob.sum(1) + log_det)."""
        cg = confidence_generator
        return self._row_handle(x.shape[0]).trav(self, x, cg.mean.data, cg.std.data, cg.std_factor)

    def backward(self, u, y=None, return_step=False):
        raise NotImplementedError("LinearRnvp.backward (the inverse flow) has no caller in WVN and is not implemented")

    def sample(self, samples=1, y=None, return_step=False, return_logdet=False):
        raise NotImplementedError("LinearRnvp.sample (the inverse flow) has no caller in WVN and is not implemented")
