"""Plugin surface of a scene representation (what slam/models/base_model.py:22-70 and the
`_target` / `setup()` convention of slam/configs/base_config.py:28-37 define), re-declared
py3.12-safe: the reference's dataclass-instance defaults do not import on python >= 3.11
(SURVEY.md section 0.4).

A Model owns the map parameters and launches the fused CUDA step; the Algorithm (algorithm.py)
drives it through exactly four calls: ``forward(input)``, ``get_loss_dict(...)``,
``get_param_groups()`` and -- CUDA-path additions -- the two switches below."""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Any, Dict, List, Type, Union

import torch
from torch import nn
from torch.nn import Parameter

Outputs = Dict[str, Union[torch.Tensor, List]]


def upstream_scale(g_losses: torch.Tensor, n_live: int = None) -> torch.Tensor:
    """Device scalar that the in-kernel gradients are multiplied with in ``backward``.

    The fused steps compute d(sum of the weighted loss terms)/d(parameters) during forward.
    Autograd's upstream gradient ``g_losses`` (one entry per loss term) is 1 under the plugin
    contract ``loss = reduce(add, loss_dict.values()); loss.backward()``
    (slam/algorithms/base_algorithm.py:263-266); a caller that scales the TOTAL loss
    (``(c * loss).backward()``, gradient-accumulation scaling) sends c for every term and gets
    c * gradient.  Unequal per-term scales cannot be honoured from the summed gradient: the
    scalar becomes NaN so the mistake is loud (Co-SLAM's ``strict_loss_grad`` re-runs the
    fused pass with the per-term scales instead).  ``n_live``: only the first n_live terms
    entered the in-kernel gradient (NICE / Point-SLAM leave the colour term out of some
    stages; its upstream gradient is then 0 and is ignored).  No host synchronisation."""
    g = g_losses.detach().reshape(-1).float()
    if n_live is not None:
        g = g[:n_live]
    same = (g == g[0]).all()
    return torch.where(same, g[0], torch.full_like(g[0], float('nan')))


def scale_grads(grads, s):
    """In-place ``t *= s`` for every tensor in a (nested) list; None passes through."""
    out = []
    for t in grads:
        if t is None:
            out.append(None)
        elif isinstance(t, (list, tuple)):
            out.append(scale_grads(t, s))
        else:
            out.append(t.mul_(s.to(t.dtype)))
    return out


class FusedStep(torch.autograd.Function):
    """``(losses, *outputs) = FusedStep.apply(launch, n_live, *inputs)``: autograd bridge of a
    fused step, which computes its gradients during forward.

    ``inputs`` are the tensors autograd may differentiate.  ``launch(needs)`` receives their
    ``needs_input_grad`` flags and returns ``(losses, outputs, grads)``: ``outputs`` is a tuple
    of non-differentiable tensors, ``grads`` a list aligned with ``inputs`` (None where no
    gradient exists), or None for a forward-only launch.  backward hands ``grads`` out scaled
    by ``upstream_scale(g_losses, n_live)``."""
    @staticmethod
    def forward(ctx, launch, n_live, *inputs):
        losses, outputs, grads = launch(ctx.needs_input_grad[2:])
        ctx.grads, ctx.n_live = grads, n_live
        ctx.mark_non_differentiable(*outputs)
        return (losses, *outputs)

    @staticmethod
    def backward(ctx, g_losses, *_):
        if ctx.grads is None:
            raise RuntimeError('backward through a forward-only fused pass')
        return (None, None, *scale_grads(ctx.grads, upstream_scale(g_losses, ctx.n_live)))


@dataclass
class InstantiateConfig:
    """A config knows the class it configures: ``cfg.setup(**kw)`` builds ``_target(cfg, **kw)``."""
    _target: Type = None

    def setup(self, **kwargs) -> Any:
        if self._target is None:
            raise TypeError(f'{type(self).__name__} has no _target')
        return self._target(self, **kwargs)


@dataclass
class ModelConfig(InstantiateConfig):
    _target: Type = field(default_factory=lambda: Model)


class Model(nn.Module):
    config: ModelConfig
    # tracking optimises the pose only: subclasses skip map / decoder gradients when set
    freeze_map_grads: bool = False
    # dp.MappingDataParallel when mapping rays are sharded over ranks
    dp = None

    def __init__(self, config: ModelConfig, camera, bounding_box=None, **kwargs) -> None:
        super().__init__()
        self.config, self.camera, self.bounding_box, self.kwargs = config, camera, bounding_box, kwargs
        self.populate_modules()

    def populate_modules(self):
        """Subclasses create their parameters here (and call super() first)."""
        self.device_indicator_param = nn.Parameter(torch.empty(0))

    @property
    def device(self) -> torch.device:
        return self.device_indicator_param.device

    def forward(self, input) -> Outputs:
        return self.get_outputs(input)

    def map_inputs(self, *tensors) -> List[torch.Tensor]:
        """Map / decoder tensors as they enter a fused step: detached while
        ``freeze_map_grads`` is set, so the step computes pose gradients only."""
        return [t.detach() for t in tensors] if self.freeze_map_grads else list(tensors)

    # ---- the contract every representation implements -------------------------------
    def get_outputs(self, input) -> Outputs:
        raise NotImplementedError

    def get_loss_dict(self, outputs, inputs, is_mapping, stage=None) -> Dict[str, torch.Tensor]:
        raise NotImplementedError

    def get_param_groups(self) -> Dict[str, List[Parameter]]:
        raise NotImplementedError
