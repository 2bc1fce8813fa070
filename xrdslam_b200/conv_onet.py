"""NICE-SLAM model behind the reference's ``Model`` plugin surface, H100-native.

Host-side mirror of slam/models/conv_onet.py (reference @ f0366f20): same class / config
field names, same ``forward / get_loss_dict / get_param_groups`` signatures, same
parameter-group names (``decoder``, ``grid_middle``, ``grid_fine``, ``grid_color``) and the
decoder state_dict keys of slam/model_components/decoder_nice.py (``embedder._B``,
``fc_c.i``, ``pts_linears.i``, ``output_linear``).  The render / loss / backward run in
``xrd_nice_step`` (csrc/nice.cu) through the C-ABI; no PyTorch fallback exists.

Feature grids are stored CHANNEL-LAST ``[Z,Y,X,32]`` (one voxel = one 128-byte line);
``grid_c[key]`` exposes the reference layout ``[1,32,Z,Y,X]`` as a permuted view.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from pathlib import Path
from typing import Dict, List, Optional, Type, Union

import numpy as np
import torch
from torch import nn
from torch.nn import Parameter

from . import _cabi
from ._cabi import (XrdNiceCfg, XrdNiceCoarseCfg, XrdNiceCoarseDecoder, XrdNiceDecoder,
                    XrdNiceDecoderGrads, XrdNiceGrads, XrdNiceGrid, XrdNiceOut, XrdRays, ptr)
from .base_model import FusedStep, Model, ModelConfig

MAX_SAMPLES = 128  # samples per ray of the CUDA renderer (pass 2 with importance sampling)
STAGES = {'middle': 0, 'fine': 1, 'color': 2}  # 'coarse' has its own entry (xrd_nice_coarse_step)
GRIDS = ('grid_middle', 'grid_fine', 'grid_color')  # indexed by STAGES


@dataclass
class ConvOnetConfig(ModelConfig):
    """slam/models/conv_onet.py:18-63 (field names and defaults kept)."""
    _target: Type = field(default_factory=lambda: ConvOnet)
    coarse: bool = False  # model default (conv_onet.py:23); the nice-slam run config sets True
    occupancy: bool = True
    pretrained_decoders_coarse: Optional[Path] = None
    pretrained_decoders_middle_fine: Optional[Path] = None
    data_dim: int = 3
    model_c_dim: int = 32
    model_pos_embedding_method: str = 'fourier'
    model_coarse_bound_enlarge: int = 2
    grid_len_coarse: float = 2
    grid_len_middle: float = 0.32
    grid_len_fine: float = 0.16
    grid_len_color: float = 0.16
    grid_bound_divisible: float = 0.32
    rendering_n_samples: int = 32
    rendering_n_surface: int = 16
    rendering_n_importance: int = 0
    rendering_lindisp: bool = False
    rendering_perturb: float = 0.0
    seed: int = 0  # Philox seed of the in-kernel draws when no noise / importance_u is passed
    points_batch_size: int = 500000
    tracking_w_color_loss: float = 0.5
    mapping_w_color_loss: float = 0.2
    tracking_handle_dynamic: bool = True
    tracking_use_color_in_tracking: bool = True
    mapping_fix_fine: bool = True
    mapping_fix_color: bool = False
    mapping_frustum_feature_selection: bool = True


class _Embedder(nn.Module):
    def __init__(self, gen=None):
        super().__init__()
        self._B = nn.Parameter(torch.randn((3, 93), generator=gen) * 25)


class _DenseLayer(nn.Linear):
    """decoder_nice.py:76-91: xavier_uniform with the activation's gain, zero bias."""
    def __init__(self, in_dim, out_dim, activation='relu'):
        self.activation = activation
        super().__init__(in_dim, out_dim)

    def reset_parameters(self) -> None:
        nn.init.xavier_uniform_(self.weight,
                                gain=nn.init.calculate_gain(self.activation))
        if self.bias is not None:
            nn.init.zeros_(self.bias)


class MLP(nn.Module):
    """Parameter container of decoder_nice.py:101-234 (hidden 32, 5 blocks, skip at 2)."""
    def __init__(self, name, c_dim, color, hidden_size=32):
        super().__init__()
        self.name, self.c_dim, self.color = name, c_dim, color
        self.fc_c = nn.ModuleList([nn.Linear(c_dim, hidden_size) for _ in range(5)])
        self.embedder = _Embedder()
        dims = [93, hidden_size, hidden_size, hidden_size + 93, hidden_size]
        self.pts_linears = nn.ModuleList([_DenseLayer(d, hidden_size) for d in dims])
        self.output_linear = _DenseLayer(hidden_size, 4 if color else 1, 'linear')

    def tensors(self):
        t = [self.embedder._B]
        for i in range(5):
            t += [self.pts_linears[i].weight, self.pts_linears[i].bias]
        for i in range(5):
            t += [self.fc_c[i].weight, self.fc_c[i].bias]
        return t + [self.output_linear.weight, self.output_linear.bias]


class MLP_no_xyz(nn.Module):
    """Parameter container of decoder_nice.py:237-320 (the coarse decoder): 5 blocks of width
    32 on the grid feature alone, the feature re-concatenated after block 2."""
    def __init__(self, name, c_dim, hidden_size=32):
        super().__init__()
        self.name, self.c_dim = name, c_dim
        dims = [hidden_size, hidden_size, hidden_size, hidden_size + c_dim, hidden_size]
        self.pts_linears = nn.ModuleList([_DenseLayer(d, hidden_size) for d in dims])
        self.output_linear = _DenseLayer(hidden_size, 1, 'linear')


class NICE(nn.Module):
    """decoder_nice.py:323-384."""
    def __init__(self, c_dim=32, coarse=False):
        super().__init__()
        if coarse:
            self.coarse_decoder = MLP_no_xyz('coarse', c_dim)
        self.middle_decoder = MLP('middle', c_dim, False)
        self.fine_decoder = MLP('fine', 2 * c_dim, False)
        self.color_decoder = MLP('color', c_dim, True)


def _dec_struct(tensors, c_dim, n_out, cls=XrdNiceDecoder):
    d = cls()
    d.B = ptr(tensors[0])
    for i in range(5):
        d.pts_w[i] = ptr(tensors[1 + 2 * i])
        d.pts_b[i] = ptr(tensors[2 + 2 * i])
        d.fcc_w[i] = ptr(tensors[11 + 2 * i])
        d.fcc_b[i] = ptr(tensors[12 + 2 * i])
    d.out_w = ptr(tensors[21])
    d.out_b = ptr(tensors[22])
    if cls is XrdNiceDecoder:
        d.c_dim, d.n_out = c_dim, n_out
    return d


class ConvOnet(Model):
    """Model class (slam/models/conv_onet.py:66-524)."""

    config: ConvOnetConfig

    def __init__(self, config: ConvOnetConfig, camera, bounding_box, **kwargs) -> None:
        super().__init__(config=config, camera=camera, bounding_box=bounding_box, **kwargs)

    def populate_modules(self):
        super().populate_modules()
        cfg = self.config
        if cfg.rendering_lindisp:
            # conv_onet.py:462-468: near = 0.01 * gt_depth is 0 on rays without depth, and
            # 1 / near * (1 - t) at t = 1 is inf * 0 = NaN in their depth, uncertainty and rgb
            raise NotImplementedError(
                'rendering_lindisp: the reference samples in disparity from near = 0.01 * depth, '
                'which is 0 on rays without depth and makes their depth, uncertainty and rgb NaN '
                '(1 / near * (1 - t) = inf * 0 at t = 1)')
        if not cfg.occupancy:
            raise NotImplementedError('occupancy=False: the CUDA path composites occupancies')
        if cfg.rendering_n_importance < 0:
            raise ValueError(f'rendering_n_importance = {cfg.rendering_n_importance} < 0')
        # pass 2 takes every sample; the coarse stage's n_samples + N is never more
        total = cfg.rendering_n_samples + cfg.rendering_n_surface + cfg.rendering_n_importance
        if total > MAX_SAMPLES:
            raise ValueError(f'rendering_n_samples + rendering_n_surface + rendering_n_importance '
                             f'= {total}: the renderer takes at most {MAX_SAMPLES} samples per ray')
        self.bounding_box = torch.as_tensor(np.asarray(self.bounding_box),
                                            dtype=torch.float64).clone()
        self.decoder = NICE(cfg.model_c_dim, coarse=cfg.coarse)
        self.load_bound()
        self.load_pretrain()
        self.grid_init()
        self.grid_opti_mask = {}
        self.dp = None  # xrdslam_b200.dp.MappingDataParallel when mapping rays are sharded
        self.register_buffer('_t_uniform', torch.linspace(0., 1., steps=cfg.rendering_n_samples),
                             persistent=False)
        self.register_buffer('_t_surface', torch.linspace(0., 1., steps=cfg.rendering_n_surface),
                             persistent=False)
        n = max(cfg.rendering_n_importance, 1)  # sample_pdf's det draw (utils.py:50-54)
        self.register_buffer('_t_importance', torch.linspace(0. + 0.5 / n, 1. - 0.5 / n, steps=n),
                             persistent=False)
        self._step_count = 0

    def load_bound(self):
        """conv_onet.py:324-337 with its dtype chain (int32 * python float -> float32, Q2)."""
        bd = self.config.grid_bound_divisible
        self.bounding_box[:, 1] = (((self.bounding_box[:, 1] - self.bounding_box[:, 0]) /
                                    bd).int() + 1) * bd + self.bounding_box[:, 0]

    def load_pretrain(self):
        """conv_onet.py:293-322: the frozen decoders come from the pretrained ConvONet
        checkpoints -- ckpt['model'] keys 'decoder.*' -> coarse decoder, 'decoder.coarse.*' ->
        MIDDLE decoder, 'decoder.fine.*' -> fine decoder (encoder keys dropped).  A path that
        is set must load; without a path the decoders keep their seeded xavier init (the
        reference checkpoints are Git-LFS objects that do not ship with the repository:
        synthetic benchmarks and parity tests run that way) and a warning says so, because
        NICE-SLAM never trains the middle / fine / coarse decoders."""
        cfg = self.config

        def load(path):
            ckpt = torch.load(path, map_location='cpu', weights_only=False)
            if not isinstance(ckpt, dict) or 'model' not in ckpt:
                raise RuntimeError(f'{path}: not a ConvONet checkpoint (no "model" entry)')
            return ckpt['model']
        missing = []
        if cfg.coarse:
            if cfg.pretrained_decoders_coarse is not None:
                sd = {k[8:]: v for k, v in load(cfg.pretrained_decoders_coarse).items()
                      if 'decoder' in k and 'encoder' not in k}
                self.decoder.coarse_decoder.load_state_dict(sd)
            else:
                missing.append('coarse')
        if cfg.pretrained_decoders_middle_fine is not None:
            mid, fine = {}, {}
            for k, v in load(cfg.pretrained_decoders_middle_fine).items():
                if 'decoder' in k and 'encoder' not in k:
                    if 'coarse' in k:
                        mid[k[8 + 7:]] = v
                    elif 'fine' in k:
                        fine[k[8 + 5:]] = v
            self.decoder.middle_decoder.load_state_dict(mid)
            self.decoder.fine_decoder.load_state_dict(fine)
        else:
            missing += ['middle', 'fine']
        if missing:
            import warnings
            warnings.warn('ConvOnet: no pretrained checkpoint for the frozen ' + '/'.join(missing) +
                          ' decoder(s) (pretrained_decoders_*): they stay randomly initialised',
                          RuntimeWarning, stacklevel=3)

    def grid_init(self):
        """conv_onet.py:254-291 + feature_grid_nice.py (shapes), channel-last storage."""
        cfg = self.config
        xyz_len = self.bounding_box[:, 1] - self.bounding_box[:, 0]
        self.grids = nn.ParameterDict()
        levels = [('grid_middle', xyz_len, cfg.grid_len_middle, 0.01),
                  ('grid_fine', xyz_len, cfg.grid_len_fine, 0.0001),
                  ('grid_color', xyz_len, cfg.grid_len_color, 0.01)]
        if cfg.coarse:  # conv_onet.py:256-275: the coarse grid spans the enlarged extent
            levels.insert(0, ('grid_coarse', xyz_len * cfg.model_coarse_bound_enlarge,
                              cfg.grid_len_coarse, 0.01))
        for key, ext, gl, std in levels:
            s = list(map(int, (ext / gl).tolist()))  # (X, Y, Z) counts
            val = torch.zeros([s[2], s[1], s[0], cfg.model_c_dim]).normal_(mean=0, std=std)
            self.grids[key] = nn.Parameter(val)

    @property
    def grid_c(self):
        """Reference layout views [1, C, Z, Y, X]."""
        return {k: v.permute(3, 0, 1, 2).unsqueeze(0) for k, v in self.grids.items()}

    def set_grid(self, key, val_ref_layout):
        with torch.no_grad():
            self.grids[key].copy_(val_ref_layout.squeeze(0).permute(1, 2, 3, 0))

    # ------------------------------------------------------------- C-ABI ---
    def _level_structs(self):
        """(XrdNiceGrid[3], XrdNiceDecoder[3], keep) of the middle / fine / colour levels;
        ``keep`` holds the detached tensors the structs point into, for the caller to keep
        alive until its launch."""
        grids, decs, keep = (XrdNiceGrid * 3)(), (XrdNiceDecoder * 3)(), []
        dmods = (self.decoder.middle_decoder, self.decoder.fine_decoder,
                 self.decoder.color_decoder)
        for i, (k, m) in enumerate(zip(GRIDS, dmods)):
            g = self.grids[k].detach()
            t = [x.detach() for x in m.tensors()]
            keep += [g, t]
            grids[i] = XrdNiceGrid(ptr(g), g.shape[2], g.shape[1], g.shape[0])
            decs[i] = _dec_struct(t, m.c_dim, 4 if m.color else 1)
        return grids, decs, keep

    def _out_struct(self, o):
        """XrdNiceOut over the output dict of a launch (sample depths go to the test hook
        ``_z_capture`` when it is set)."""
        return XrdNiceOut(ptr(o['rgb']), ptr(o['depth']), ptr(o['uncertainty']),
                          ptr(getattr(self, '_z_capture', None)), None, ptr(o['losses']))

    def _sampling(self, c, R, S0, noise, importance_u, dev, keep):
        """Fill the sampling fields of a step struct (rendering_perturb / rendering_n_importance,
        conv_onet.py:470-506): explicit uniforms `noise` [R, n_samples] and `importance_u`
        [R, N] when given, else draws from a seed that advances every launch (and differs per
        rank under data-parallel mapping).  -> samples per ray of the last pass."""
        cfg = self.config
        N = cfg.rendering_n_importance
        c.n_importance, c.perturb = N, float(cfg.rendering_perturb)
        self._step_count += 1
        rank = self.dp.rank if self.dp is not None else 0
        c.seed = ((cfg.seed << 32) + self._step_count + (rank << 24)) & ((1 << 64) - 1)
        f32 = dict(dtype=torch.float32, device=dev)
        if noise is not None and cfg.rendering_perturb > 0:
            noise = noise.detach().to(**f32).contiguous()
            if tuple(noise.shape) != (R, cfg.rendering_n_samples):
                raise ValueError(f'noise: shape {tuple(noise.shape)}, expected '
                                 f'({R}, {cfg.rendering_n_samples})')
            keep.append(noise)
            c.perturb_u = ptr(noise)
        if N > 0:
            if importance_u is not None:
                importance_u = importance_u.detach().to(**f32).contiguous()
                if tuple(importance_u.shape) != (R, N):
                    raise ValueError(f'importance_u: shape {tuple(importance_u.shape)}, '
                                     f'expected ({R}, {N})')
                keep.append(importance_u)
                c.importance_u = ptr(importance_u)
            c.t_importance = ptr(self._t_importance)
        return S0 + max(N, 0)

    def _launch(self, stage, is_mapping, rays_o, rays_d, target_s, target_d, with_grads,
                need_rays=False, need_grid=(False, False, False), need_col=False, noise=None,
                importance_u=None):
        cfg = self.config
        dev = self.grids['grid_middle'].device
        _cabi.require_cuda(dev, 'model')
        f32 = dict(dtype=torch.float32, device=dev)
        f64 = dict(dtype=torch.float64, device=dev)
        rays_o = rays_o.detach().to(**f32).contiguous()
        rays_d = rays_d.detach().to(**f32).contiguous()
        R = rays_o.shape[0]
        td = target_d.detach().to(**f32).reshape(-1).contiguous()
        ts = target_s.detach().to(**f32).contiguous() if target_s is not None else None
        o = dict(rgb=torch.empty(R, 3, **f32), depth=torch.empty(R, **f64),
                 uncertainty=torch.empty(R, **f64), losses=torch.zeros(2, **f32))
        rays = XrdRays(R, ptr(rays_o), ptr(rays_d), ptr(ts), ptr(td))
        grids, decs, keep = self._level_structs()
        c = XrdNiceCfg()
        c.stage = STAGES[stage]
        c.is_mapping = int(is_mapping)
        c.n_samples, c.n_surface = cfg.rendering_n_samples, cfg.rendering_n_surface
        for d in range(3):
            c.bound_min[d] = float(self.bounding_box[d, 0])
            c.bound_max[d] = float(self.bounding_box[d, 1])
        c.w_color = cfg.mapping_w_color_loss if is_mapping else cfg.tracking_w_color_loss
        c.handle_dynamic = int(cfg.tracking_handle_dynamic)
        c.use_color_in_tracking = int(cfg.tracking_use_color_in_tracking)
        c.t_uniform, c.t_surface = ptr(self._t_uniform), ptr(self._t_surface)
        maxd = None
        if self.dp is not None and self.dp.world > 1 and is_mapping and with_grads:
            maxd = self.dp.all_reduce_max(td.max().reshape(1))  # batch-global (Q9), no host sync
        c.max_depth_global = ptr(maxd)
        S = self._sampling(c, R, cfg.rendering_n_samples + cfg.rendering_n_surface, noise,
                           importance_u, dev, keep)
        out = self._out_struct(o)
        g = None
        gs = None
        if with_grads:
            if ts is None:
                raise RuntimeError('gradients need target_s')
            dgrid = [torch.zeros_like(self.grids[k]) if (need_grid[i] and i <= c.stage) else None
                     for i, k in enumerate(GRIDS)]
            dcol = None
            if need_col and c.stage == 2:
                dcol = [torch.zeros_like(t) for t in self.decoder.color_decoder.tensors()]
            g = dict(d_grid=dgrid, d_color=dcol if dcol is not None else [None] * 23,
                     d_rays_o=torch.empty(R, 3, **f32) if need_rays else None,
                     d_rays_d=torch.empty(R, 3, **f32) if need_rays else None)
            gs = XrdNiceGrads()
            for i in range(3):
                gs.d_grid[i] = ptr(dgrid[i])
            if dcol is not None:
                dg = _dec_struct(dcol, 0, 0, XrdNiceDecoderGrads)
                keep.append(dg)
                gs.d_color = C.pointer(dg)
            gs.d_rays_o, gs.d_rays_d = ptr(g['d_rays_o']), ptr(g['d_rays_d'])
        ws, nb = _cabi.workspace(dev, 'nice', R, S, int(with_grads))
        _cabi.launch_on(dev, 'xrd_nice_step', C.byref(rays), grids, decs, C.byref(c), C.byref(out),
                        C.byref(gs) if gs is not None else None, ptr(ws), nb)
        return o, g

    def _launch_coarse(self, rays_o, rays_d, target_d, with_grads, need_rays=False,
                       need_grid=False, noise=None, importance_u=None):
        """Stage 'coarse' through xrd_nice_coarse_step (csrc/nice.cu)."""
        cfg = self.config
        if not cfg.coarse:
            raise RuntimeError("stage 'coarse' needs ConvOnetConfig(coarse=True)")
        grid = self.grids['grid_coarse']
        dev = grid.device
        _cabi.require_cuda(dev, 'model')
        f32 = dict(dtype=torch.float32, device=dev)
        f64 = dict(dtype=torch.float64, device=dev)
        rays_o = rays_o.detach().to(**f32).contiguous()
        rays_d = rays_d.detach().to(**f32).contiguous()
        R, S = rays_o.shape[0], cfg.rendering_n_samples
        td = target_d.detach().to(**f32).reshape(-1).contiguous() if target_d is not None else None
        o = dict(rgb=torch.zeros(R, 3, **f32), depth=torch.empty(R, **f64),
                 uncertainty=torch.empty(R, **f64), losses=torch.zeros(2, **f32))
        rays = XrdRays(R, ptr(rays_o), ptr(rays_d), None, ptr(td))
        g = grid.detach()
        gs = XrdNiceGrid(ptr(g), g.shape[2], g.shape[1], g.shape[0])
        d = self.decoder.coarse_decoder
        keep = [t.detach() for l in d.pts_linears for t in (l.weight, l.bias)] + \
            [d.output_linear.weight.detach(), d.output_linear.bias.detach()]
        dec = XrdNiceCoarseDecoder()
        for i in range(5):
            dec.pts_w[i], dec.pts_b[i] = ptr(keep[2 * i]), ptr(keep[2 * i + 1])
        dec.out_w, dec.out_b = ptr(keep[10]), ptr(keep[11])
        c = XrdNiceCoarseCfg()
        c.n_samples = S
        e = cfg.model_coarse_bound_enlarge
        for k in range(3):
            c.bound_min[k] = float(self.bounding_box[k, 0])
            c.bound_max[k] = float(self.bounding_box[k, 1])
            c.coarse_bound_min[k] = float(self.bounding_box[k, 0] * e)
            c.coarse_bound_max[k] = float(self.bounding_box[k, 1] * e)
        c.t_uniform = ptr(self._t_uniform)
        S = self._sampling(c, R, S, noise, importance_u, dev, keep)
        out = self._out_struct(o)
        gr = None
        if with_grads:
            if td is None:
                raise RuntimeError('gradients need target_d')
            gr = dict(d_grid=torch.zeros_like(grid) if need_grid else None,
                      d_rays_o=torch.empty(R, 3, **f32) if need_rays else None,
                      d_rays_d=torch.empty(R, 3, **f32) if need_rays else None)
        ws, nb = _cabi.workspace(dev, 'nice_coarse', R, S, int(with_grads))
        _cabi.launch_on(dev, 'xrd_nice_coarse_step', C.byref(rays), C.byref(gs), C.byref(dec),
                        C.byref(c), C.byref(out), ptr(gr['d_grid']) if gr else None,
                        ptr(gr['d_rays_o']) if gr else None, ptr(gr['d_rays_d']) if gr else None,
                        int(with_grads), ptr(ws), nb)
        return o, gr

    # --------------------------------------------------------- Model API ---
    def get_outputs(self, input) -> Dict[str, Union[torch.Tensor, List]]:
        """conv_onet.py:132-143."""
        stage = input['stage']
        rays_o, rays_d = input['rays_o'], input['rays_d']
        target_d, target_s = input['target_d'], input.get('target_s')
        # explicit uniforms of the jitter [R, n_samples] and of sample_pdf [R, N] (parity tests)
        smp = dict(noise=input.get('noise'), importance_u=input.get('importance_u'))
        fused = torch.is_grad_enabled() and target_s is not None and 'is_mapping' in input
        if not fused:
            # conv_onet.py:137-138: the coarse level renders without depth guidance; the
            # target depth only enters the (mapping) loss
            o, _ = self._launch_coarse(rays_o, rays_d, target_d, False, **smp) \
                if stage == 'coarse' else \
                self._launch(stage, True, rays_o, rays_d, target_s, target_d, False, **smp)
            o.pop('losses')
            return o
        if stage == 'coarse':
            maps, n_live = [self.grids['grid_coarse']], 1

            def launch(needs):
                need_rays, need_grid = needs[0] or needs[1], needs[2]
                o, g = self._launch_coarse(rays_o, rays_d, target_d, need_rays or need_grid,
                                           need_rays, need_grid, **smp)
                grads = None if g is None else [g['d_rays_o'], g['d_rays_d'], g['d_grid']]
                return o['losses'], (o['rgb'], o['depth'], o['uncertainty']), grads
        else:
            is_mapping, cfg = input['is_mapping'], self.config
            maps = [self.grids[k] for k in GRIDS] + self.decoder.color_decoder.tensors()
            # the colour term is live exactly when get_loss_dict returns it
            n_live = 2 if ((not is_mapping and cfg.tracking_use_color_in_tracking) or
                           (is_mapping and stage == 'color')) else 1

            def launch(needs):
                need_rays, need_grid, need_col = needs[0] or needs[1], needs[2:5], any(needs[5:])
                o, g = self._launch(stage, is_mapping, rays_o, rays_d, target_s, target_d,
                                    need_rays or any(need_grid) or need_col, need_rays,
                                    need_grid, need_col, **smp)
                grads = None if g is None else \
                    [g['d_rays_o'], g['d_rays_d'], *g['d_grid'], *g['d_color']]
                return o['losses'], (o['rgb'], o['depth'], o['uncertainty']), grads
        losses, rgb, depth, unc = FusedStep.apply(launch, n_live, rays_o, rays_d,
                                                  *self.map_inputs(*maps))
        return {'rgb': rgb, 'depth': depth, 'uncertainty': unc, '_losses': losses}

    # ---- mesher-facing queries (conv_onet.py:213-240) -----------------------------------
    def _query(self, pi, stage):
        dev = self.grids['grid_middle'].device
        _cabi.require_cuda(dev, 'model')
        pts = pi.detach().reshape(-1, 3).to(device=dev, dtype=torch.float32).contiguous()
        P = pts.shape[0]
        grids, decs, keep = self._level_structs()
        bmin = (C.c_double * 3)(*[float(self.bounding_box[d, 0]) for d in range(3)])
        bmax = (C.c_double * 3)(*[float(self.bounding_box[d, 1]) for d in range(3)])
        raw = torch.empty(P, 4, dtype=torch.float32, device=dev)
        ws, nb = _cabi.workspace(dev, 'nice_query', P)
        _cabi.launch_on(dev, 'xrd_nice_query', ptr(pts), P, grids, decs, bmin, bmax, STAGES[stage],
                        ptr(raw), ptr(ws), nb)
        return raw

    def query_fn(self, pi):
        """conv_onet.py:213-230: NICE.forward(stage='fine') at points [N,3] -> raw [N,4]
        (zeros, occupancy logit middle + fine)."""
        return self._query(pi, 'fine')

    def color_func(self, pi):
        """conv_onet.py:232-239: stage 'color' -> raw [N,4] (rgb, occupancy logit)."""
        return self._query(pi, 'color')

    def get_loss_dict(self, outputs, inputs, is_mapping, stage=None) -> Dict[str, torch.Tensor]:
        """conv_onet.py:145-185: terms come from the fused pass (forward needs
        ``input['is_mapping']`` -- the Algorithm sets it -- to pick the loss form)."""
        if '_losses' not in outputs:
            raise RuntimeError('get_loss_dict needs a forward() run with grad enabled, '
                               "target_s and input['is_mapping']")
        if bool(inputs['is_mapping']) != bool(is_mapping):
            raise RuntimeError("input['is_mapping'] disagrees with get_loss_dict(is_mapping)")
        ls = outputs['_losses']
        d = {'depth_loss': ls[0]}
        cfg = self.config
        if (not is_mapping and cfg.tracking_use_color_in_tracking) or \
                (is_mapping and (stage or inputs['stage']) == 'color'):
            d['rgb_loss'] = ls[1]
        return d

    # ---- frustum feature selection (conv_onet.py:94-130, rows N2 / N3) -------------------
    def pre_precessing(self, cur_frame):
        """Voxel masks of the current frustum (utils.py:298-375), one uint8 per voxel of the
        channel-last grids.  The reference then optimises a compacted copy of the masked
        voxels and scatters it back into the full 43 MB grid every iteration
        (grid_processing / post_processing); here the full grid stays the parameter and the
        Adam kernel skips the rows outside the mask -- same values, no scatter."""
        if not self.config.mapping_frustum_feature_selection:
            return
        from .keyframe_selection import frustum_mask
        dev = self.device
        bb = self.bounding_box
        c2w = cur_frame.get_pose().detach()
        for key, g in self.grids.items():
            if key == 'grid_coarse':
                continue  # utils.py:323-325: the coarse grid is optimised whole
            Z, Y, X = g.shape[:3]
            zs = torch.linspace(float(bb[2][0]), float(bb[2][1]), Z)
            ys = torch.linspace(float(bb[1][0]), float(bb[1][1]), Y)
            xs = torch.linspace(float(bb[0][0]), float(bb[0][1]), X)
            gz, gy, gx = torch.meshgrid(zs, ys, xs, indexing='ij')  # [Z,Y,X] storage order
            pts = torch.stack([gx, gy, gz], -1).reshape(-1, 3).to(dev)
            m = frustum_mask(self.camera, c2w, pts, cur_frame.depth, edge=0, near_cam=0.5)
            self.grid_opti_mask[key] = m.reshape(Z, Y, X).to(torch.uint8).contiguous()

    def grid_processing(self, coarse=False):
        """No-op: see pre_precessing (the reference re-scatters val[mask] = val_grad here)."""

    def post_processing(self, coarse=False):
        """No-op: the full grid is the parameter; nothing to write back."""

    def get_param_groups(self) -> Dict[str, List[Parameter]]:
        """conv_onet.py:187-211; with frustum selection the grids carry a row mask that the
        fused Adam honours (optimizers.FusedAdam)."""
        groups = {}
        dec = []
        if not self.config.mapping_fix_fine:
            raise NotImplementedError('mapping_fix_fine=False')
        if not self.config.mapping_fix_color:
            dec += list(self.decoder.color_decoder.parameters())
        if dec:
            groups['decoder'] = dec
        for key in self.grids:  # conv_onet.py:197-211: every grid of grid_c, coarse included
            p = self.grids[key]
            # get_mask_from_c2w returns an all-ones mask for 'grid_coarse' (utils.py:323-325)
            p._xrd_row_mask = self.grid_opti_mask.get(key) \
                if (self.config.mapping_frustum_feature_selection and key != 'grid_coarse') else None
            groups[key] = [p]
        return groups
