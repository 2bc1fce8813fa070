"""Per-parameter-group Adam set (mirror of slam/engine/optimizers.py): group
names are the contract between Model.get_param_groups() and the config."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Any, Dict, List, Optional, Tuple, Type

import torch
from torch.nn.parameter import Parameter

from . import _cabi


def adam_desc(param, grad, exp_avg, exp_avg_sq, lr, betas, eps, weight_decay,
              bias_corrections=(1.0, 1.0), dyn=None, row_mask=None):
    """XrdAdamTensor of one device fp32 tensor.  `dyn`, a device pointer to {lr, bias_correction1,
    bias_correction2}, overrides those host values; rows whose `row_mask` entry is 0 are kept."""
    a = _cabi.XrdAdamTensor(
        param=param.data_ptr(), grad=grad.data_ptr(), exp_avg=exp_avg.data_ptr(),
        exp_avg_sq=exp_avg_sq.data_ptr(), n=param.numel(), lr=lr, beta1=betas[0],
        beta2=betas[1], eps=eps, weight_decay=weight_decay,
        bias_correction1=bias_corrections[0], bias_correction2=bias_corrections[1], dyn=dyn)
    if row_mask is not None:
        a.row_mask, a.row_len = row_mask.data_ptr(), param.numel() // row_mask.numel()
    return a


def init_adam_state(state, p):
    """Fill an empty `state` with torch.optim.Adam's `step`, `exp_avg` and `exp_avg_sq`."""
    if not state:
        state['step'] = torch.tensor(0.0)
        state['exp_avg'] = torch.zeros_like(p)
        state['exp_avg_sq'] = torch.zeros_like(p)
    return state


class FusedAdam(torch.optim.Optimizer):
    """torch.optim.Adam (amsgrad=False) for device-resident fp32 parameters: every tensor of
    the group is updated by ONE launch of csrc/adam.cu (xrd_adam_step) instead of torch's
    ~10 foreach launches.  A parameter may carry `_xrd_row_mask` (uint8, one entry per row):
    rows whose mask is 0 are left untouched (NICE-SLAM frustum feature selection without the
    reference's compact-copy / scatter-back round trip).  State keys are torch's (`step`, `exp_avg`, `exp_avg_sq`) so
    optimizer checkpoints interchange with torch.optim.Adam."""
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0):
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))

    @torch.no_grad()
    def step(self, closure=None):
        loss = closure() if closure is not None else None
        descs, grads, dev = [], [], None
        for group in self.param_groups:
            b1, b2 = group['betas']
            for p in group['params']:
                if p.grad is None:
                    continue
                if not p.is_cuda or p.dtype != torch.float32 or not p.is_contiguous():
                    raise RuntimeError('FusedAdam needs contiguous fp32 CUDA parameters')
                st = init_adam_state(self.state[p], p)
                st['step'] += 1
                t = float(st['step'])
                g = p.grad if p.grad.is_contiguous() else p.grad.contiguous()
                grads.append(g)  # a contiguous copy must outlive the launch
                mask = getattr(p, '_xrd_row_mask', None)  # frustum feature selection (NICE-SLAM)
                if mask is not None:
                    assert mask.is_cuda and mask.dtype == torch.uint8 and mask.is_contiguous() and \
                        p.numel() % mask.numel() == 0
                descs.append(adam_desc(p, g, st['exp_avg'], st['exp_avg_sq'], float(group['lr']),
                                       (b1, b2), group['eps'], group['weight_decay'],
                                       (1.0 - b1**t, 1.0 - b2**t), row_mask=mask))
                dev = p.device
        if not descs:
            return loss
        arr = (_cabi.XrdAdamTensor * len(descs))(*descs)
        _cabi.launch_on(dev, 'xrd_adam_step', arr, len(descs), 0)
        return loss


@dataclass
class OptimizerConfig:
    _target: Type = torch.optim.Adam
    lr: float = 0.0005
    eps: float = 1e-08
    betas: Tuple[float, float] = (0.9, 0.999)
    max_norm: Optional[float] = None
    accum_step: Optional[int] = None

    def setup(self, params) -> torch.optim.Optimizer:
        kwargs = {k: v for k, v in vars(self).items()
                  if k not in ('_target', 'max_norm', 'accum_step')}
        params = list(params)
        target = self._target
        if target is torch.optim.Adam and params and all(
                torch.is_tensor(p) and p.is_cuda and p.dtype == torch.float32 for p in params):
            target = FusedAdam  # same update rule, one launch per group
        return target(params, **kwargs)


@dataclass
class AdamOptimizerConfig(OptimizerConfig):
    _target: Type = torch.optim.Adam
    weight_decay: float = 0


class Optimizers:
    def __init__(self, config: Dict[str, Any] = None,
                 param_groups: Dict[str, List[Parameter]] = None,
                 optimizers: Dict[str, Any] = None) -> None:
        self.config = config
        self.schedulers = {}
        if optimizers:
            self.optimizers = optimizers
            self.parameters = {}
            return
        self.optimizers, self.parameters = {}, {}
        for name, params in param_groups.items():
            if name not in config:
                raise RuntimeError(
                    f"Optimizer config for '{name}' not found; provided: "
                    f'{list(config.keys())}')
            oc = config[name]['optimizer']
            self.optimizers[name] = oc.setup(params=params)
            self.parameters[name] = params
            sched = config[name].get('scheduler')
            if sched:
                self.schedulers[name] = sched.setup().get_scheduler(
                    optimizer=self.optimizers[name], lr_init=oc.lr)

    def __add__(self, other: 'Optimizers') -> 'Optimizers':
        """Co-SLAM: pose optimizers + the persistent model optimizers."""
        return Optimizers(config={**self.config, **other.config},
                          optimizers={**self.optimizers, **other.optimizers})

    def zero_grad_all(self) -> None:
        for name, opt in self.optimizers.items():
            if self.config[name]['optimizer'].accum_step is None:
                opt.zero_grad(set_to_none=True)

    def optimizer_step_all(self, step: int) -> None:
        for name, opt in self.optimizers.items():
            oc = self.config[name]['optimizer']
            if oc.max_norm is not None and name in self.parameters:
                torch.nn.utils.clip_grad_norm_(self.parameters[name], oc.max_norm)
            if oc.accum_step is None:
                opt.step()
            elif (step + 1) % oc.accum_step == 0:
                opt.step()
                opt.zero_grad(set_to_none=True)

    def scheduler_step_all(self) -> None:
        for sched in self.schedulers.values():
            sched.step()

    def load_optimizers(self, loaded_state: Dict[str, Any]) -> None:
        for k, v in loaded_state.items():
            self.optimizers[k].load_state_dict(v)
