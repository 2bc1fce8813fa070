"""Co-SLAM model behind the reference's ``Model`` plugin surface, H100-native.

Host-side mirror of slam/models/joint_encoding.py (reference @ f0366f20): same
class name, same config fields, same ``forward / get_outputs / get_loss_dict /
get_param_groups / smoothness / query_sdf / query_color / query_fn / color_func``
signatures, same parameter-group names (``decoder``, ``embed_fn``, and
``embed_fn_color`` with ``oneGrid=False``) and the same state_dict keys
(``embed_fn.params``, ``embed_fn_color.params``, ``decoder.sdf_net.model.{0,2}.weight``,
``decoder.color_net.model.{0,2}.weight``).

Nothing is computed in PyTorch: ``forward`` enqueues the fused sm_90a kernels of
``xrd_coslam_step`` through the C-ABI (forward + loss + full backward in one
launch when targets are present and grad is enabled) and ``get_loss_dict``
hands the already-computed loss terms back, wired into autograd so that
``loss.backward()`` (slam/algorithms/base_algorithm.py:266) delivers the
in-kernel gradients to the hash table, the four weight matrices and -- through
``rays_o / rays_d`` -- to the pose.  No CPU / PyTorch fallback exists.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import Dict, List, Type, Union

import numpy as np
import torch
from torch import nn
from torch.nn import Parameter

from . import _cabi
from ._cabi import (XrdCoslamCfg, XrdCoslamGrads, XrdCoslamImportance, XrdCoslamMlp,
                    XrdCoslamOut, XrdHashGrid, XrdRays, ptr)
from .base_model import Model, ModelConfig, scale_grads, upstream_scale


@dataclass
class JointEncodingConfig(ModelConfig):
    """slam/models/joint_encoding.py:17-66 (field names and defaults kept)."""
    _target: Type = field(default_factory=lambda: JointEncoding)
    voxel_sdf: float = 0.02
    voxel_color: float = 0.08
    enc: str = 'HashGrid'
    pos_enc: str = 'OneBlob'
    pos_nbins: int = 16
    hashsize: int = 16
    oneGrid: bool = True
    geo_feat_dim: int = 15
    hidden_dim: int = 32
    num_layers: int = 2
    num_layers_color: int = 2
    hidden_dim_color: int = 32
    tcnn_network: bool = False
    tcnn_encoding: bool = True
    trainging_rgb_weight: float = 5.0
    trainging_depth_weight: float = 0.1
    trainging_sdf_weight: float = 1000
    trainging_fs_weight: float = 10
    trainging_smooth_weight: float = 0.000001
    trainging_smooth_pts: int = 32
    trainging_smooth_vox: float = 0.1
    trainging_smooth_margin: float = 0.05
    training_n_samples: int = 256
    training_n_sample_d: int = 32
    training_range_d: float = 0.1
    training_n_range_d: int = 11
    training_n_importance: int = 0
    training_perturb: int = 1
    training_white_bkgd: bool = False
    training_trunc: float = 0.1
    training_rgb_missing: float = 0.05
    data_sc_factor: int = 1
    data_translation: int = 0
    cam_near: float = 0.0
    cam_far: float = 5.0
    cam_depth_trunc: float = 100.0
    mesh_render_color: bool = False
    # --- CUDA path knobs (not in the reference) ---
    seed: int = 0  # Philox seed for in-kernel jitter when no noise is passed
    strict_loss_grad: bool = False  # verify upstream d(total)/d(term) == 1
    rays_per_tile: int = 0   # 0 automatic, -1 tile kernel (k_fused), -2 grouped kernel (k_fused_g)
    # decoder GEMMs on tensor cores: 0 = 3xTF32 everywhere (fp32-level parity),
    # 1 = 3xTF32 forward + TF32 backward, 2 = TF32 everywhere
    precision: int = 0


class HashGridParams(nn.Module):
    """Stands in for ``tcnn.Encoding('HashGrid', dtype=float)``: owns the flat
    fp32 ``params`` tensor in tcnn's layout (encodings_coslam.py:39-53)."""
    def __init__(self, n_levels, log2_hashmap_size, base_resolution,
                 per_level_scale, seed=1337):
        super().__init__()
        g = XrdHashGrid()
        _cabi.call('xrd_hashgrid_layout', C.byref(g), n_levels, log2_hashmap_size,
                   base_resolution, float(np.float32(per_level_scale)))
        self.layout = g
        self.n_levels = n_levels
        self.n_output_dims = 2 * n_levels
        gen = torch.Generator().manual_seed(seed)
        p = (torch.rand(int(g.n_entries) * 2, generator=gen) * 2 - 1) * 1e-4
        self.params = nn.Parameter(p.float())


class _Seq(nn.Module):
    """nn.Sequential-shaped holder so state_dict keys equal the reference's
    (decoder_coslam.py:40-56, :94-111: Linear, ReLU, Linear; bias=False)."""
    def __init__(self, d_in, d_hidden, d_out):
        super().__init__()
        self.model = nn.Sequential(nn.Linear(d_in, d_hidden, bias=False),
                                   nn.ReLU(inplace=True),
                                   nn.Linear(d_hidden, d_out, bias=False))


class ColorSDFNet_v2(nn.Module):
    """Parameter container of decoder_coslam.py:139-163 (no forward: the MLP runs
    inside the fused kernel)."""
    def __init__(self, config, input_ch, input_ch_pos):
        super().__init__()
        self.color_net = _Seq(input_ch_pos + config.geo_feat_dim,
                              config.hidden_dim_color, 3)
        self.sdf_net = _Seq(input_ch + input_ch_pos, config.hidden_dim,
                            1 + config.geo_feat_dim)


class ColorSDFNet(nn.Module):
    """Parameter container of decoder_coslam.py:113-136 (colour grid + SDF grid): the
    colour branch reads [oneblob48, colour_hash32, geo15]."""
    def __init__(self, config, input_ch, input_ch_color, input_ch_pos):
        super().__init__()
        self.color_net = _Seq(input_ch_pos + input_ch_color + config.geo_feat_dim,
                              config.hidden_dim_color, 3)
        self.sdf_net = _Seq(input_ch + input_ch_pos, config.hidden_dim,
                            1 + config.geo_feat_dim)


# render_rays outputs (joint_encoding.py:317-341); the second tuple only with
# training_n_importance > 0 (the coarse pass's maps and the spread of the fine samples)
OUT_KEYS = ('rgb', 'depth', 'disp_map', 'acc_map', 'depth_var', 'z_vals', 'raw')
IMPORTANCE_KEYS = ('rgb0', 'disp0', 'acc0', 'depth0', 'depth_var0', 'z_std')
# samples per ray the fused kernels march at most (xrd_coslam_step); a gradient pass with a
# colour grid (oneGrid=False) at most 224
MAX_SAMPLES, MAX_SAMPLES_COLOR_GRID = 256, 224


class _CoslamStep(torch.autograd.Function):
    """losses[4] = fused(rays, table, weights[, colour table]); backward hands out the
    gradients the kernel already produced."""
    @staticmethod
    def forward(ctx, rays_o, rays_d, table, w0, w1, wc0, wc1, model, target_s,
                target_d, noise, table_c=None, importance_u=None):
        need = any(ctx.needs_input_grad[:7]) or ctx.needs_input_grad[11]
        need_rays = ctx.needs_input_grad[0] or ctx.needs_input_grad[1]
        # tracking: only the pose is optimised -> skip scatter / weight-gradient tiles
        map_grads = (any(ctx.needs_input_grad[2:7]) or ctx.needs_input_grad[11]) and not (
            model.freeze_map_grads and need_rays)
        outs, grads = model._launch(rays_o, rays_d, table, w0, w1, wc0, wc1,
                                    target_s, target_d, noise, with_grads=need,
                                    need_ray_grads=need_rays,
                                    map_grads=map_grads, table_c=table_c,
                                    importance_u=importance_u)
        ctx.grads = grads
        ctx.model = model
        ctx.strict = model.config.strict_loss_grad
        ctx.inputs = (rays_o, rays_d, table, w0, w1, wc0, wc1, target_s,
                      target_d, noise, model._last_seed, table_c, importance_u)
        ret = (outs['losses'],) + tuple(outs[k] for k in model._out_keys())
        ctx.mark_non_differentiable(*ret[1:])
        return ret

    @staticmethod
    def backward(ctx, g_losses, *_):
        grads = ctx.grads
        if grads is None:
            raise RuntimeError('backward through a forward-only Co-SLAM pass')
        if ctx.strict:
            g = g_losses.detach().float().cpu()
            if not bool(torch.all(g == 1.0)):
                # non-unit upstream gradient: re-run the fused pass with the
                # per-term scales (the kernel is linear in them)
                (rays_o, rays_d, table, w0, w1, wc0, wc1, ts, td, noise,
                 seed, table_c, importance_u) = ctx.inputs
                _, grads = ctx.model._launch(
                    rays_o, rays_d, table, w0, w1, wc0, wc1, ts, td, noise,
                    with_grads=True, need_ray_grads=True,
                    loss_scale=[float(v) for v in g], seed=seed, table_c=table_c,
                    importance_u=importance_u)
        else:
            # sync-free: total-loss scaling is honoured, unequal per-term scales poison
            # the gradients with NaN (base_model.upstream_scale)
            s = upstream_scale(g_losses)
            keys = ('d_rays_o', 'd_rays_d', 'd_table', 'd_w_sdf0', 'd_w_sdf1', 'd_w_col0',
                    'd_w_col1', 'd_table_color')
            grads = dict(zip(keys, scale_grads([grads[k] for k in keys], s)))
        return (grads['d_rays_o'], grads['d_rays_d'], grads['d_table'],
                grads['d_w_sdf0'], grads['d_w_sdf1'], grads['d_w_col0'],
                grads['d_w_col1'], None, None, None, None, grads['d_table_color'], None)


class CoarseToFine:
    """A step with training_n_importance = N > 0 (joint_encoding.py:301-341): the coarse pass
    over S samples per ray (its rgb and depth terms alone count), xrd_coslam_importance, the fine
    pass over the S + N merged samples, which takes the coarse pass's terms and ray gradients in.
    Owns both passes' outputs, the importance buffers, the fine counts and the coarse ray
    gradients.  ws, ws_fine: (buffer, bytes); grads(d_rays_o, d_rays_d, loss_scale) -> the
    caller's XrdCoslamGrads (None: forward only); d_rays: the caller's ray-gradient buffers;
    structs: the step's (XrdRays, XrdHashGrid, XrdCoslamMlp)."""

    def __init__(self, model, R, S, dev, ws, ws_fine, grads=None, d_rays=(None, None),
                 loss_scale=(1.0,) * 4):
        self.model, self.R, self.S, self.N = model, R, S, model.config.training_n_importance
        self.dev, self.ws, self.ws_fine, self.grads, self.d_rays = dev, ws, ws_fine, grads, d_rays
        self.loss_scale = list(loss_scale)
        self.coarse, self._coarse = model._outputs(R, S, dev)
        self.imp, _ = model._importance_struct(R, S, dev, self.coarse['z_vals'], self.coarse['raw'])
        self.fine, self._fine = model._outputs(R, S + self.N, dev, z_vals=self.imp['z_vals'])
        self.counts = torch.zeros(4, dtype=torch.int32, device=dev)
        self.d_rays_c = [d if d is None else torch.zeros_like(d) for d in d_rays]

    def run(self, stream, structs, cfg, td, noise=None, u=None, reduce=None):
        """coarse_pass(), reduce(counts) (the all-reduce of a sharded batch), fine_pass()."""
        self.coarse_pass(stream, structs, cfg, td, noise, u)
        if reduce is not None:
            reduce(self.counts)
        self.fine_pass(stream, structs)

    def coarse_pass(self, stream, structs, cfg, td, noise=None, u=None):
        """The coarse pass (XrdCoslamCfg `cfg`), then the importance step: uniforms u [R,N], else
        drawn from cfg's seed; with the depth targets td it counts the fine pass's normalisers."""
        self._cfg, self._counts = cfg, self.counts if td is not None else None
        self._step(stream, structs, cfg, noise, self._coarse, self.loss_scale[:2] + [0.0, 0.0],
                   self.d_rays_c, self.ws)
        _, q = self.model._importance_struct(self.R, self.S, self.dev, self.coarse['z_vals'],
                                             self.coarse['raw'], td, u, seed=cfg.seed,
                                             counts=self._counts, bufs=self.imp)
        q.seed_dev = cfg.seed_dev
        _cabi.launch('xrd_coslam_importance', C.byref(q), stream=stream)

    def fine_pass(self, stream, structs):
        """The fine pass, then the coarse pass's rgb and depth terms and ray gradients added in."""
        c = XrdCoslamCfg.from_buffer_copy(self._cfg)
        c.n_samples, c.phase, c.n_importance = self.S + self.N, 2, self.N
        c.counts_out, c.counts_global = None, ptr(self._counts)
        self._step(stream, structs, c, None, self._fine, self.loss_scale, self.d_rays, self.ws_fine)
        if self.grads is not None:
            self.fine['losses'][:2] += self.coarse['losses'][:2]
        for d, d_c in zip(self.d_rays, self.d_rays_c):
            if d is not None:
                d += d_c

    def _step(self, stream, structs, cfg, noise, out, loss_scale, d_rays, ws):
        gs = self.grads(*d_rays, loss_scale) if self.grads else None
        rays, grid, mlp = structs
        _cabi.launch('xrd_coslam_step', C.byref(rays), C.byref(grid), C.byref(mlp), C.byref(cfg),
                     ptr(noise), C.byref(out), None if gs is None else C.byref(gs), ptr(ws[0]),
                     ws[1], stream=stream)


class JointEncoding(Model):
    """Model class (slam/models/joint_encoding.py:69-531)."""

    config: JointEncodingConfig

    def __init__(self, config: JointEncodingConfig, camera, bounding_box,
                 **kwargs) -> None:
        super().__init__(config=config, camera=camera,
                         bounding_box=bounding_box, **kwargs)

    # ------------------------------------------------------------- set-up ---
    def populate_modules(self):
        super().populate_modules()
        cfg = self.config
        if cfg.tcnn_network:
            raise NotImplementedError(
                'CUDA path covers tcnn_network=False (the reference default, '
                'input_config.py:253-254)')
        N = cfg.training_n_importance
        if N < 0:
            raise ValueError(f'training_n_importance must be >= 0, got {N}')
        if N:
            # the fine pass of every training step marches the depth-guided samples plus N
            limit = MAX_SAMPLES if cfg.oneGrid else MAX_SAMPLES_COLOR_GRID
            S = cfg.training_n_sample_d + cfg.training_n_range_d + N
            if S > limit:
                raise ValueError(
                    f'training_n_importance={N}: the fine pass would march training_n_sample_d + '
                    f'training_n_range_d + training_n_importance = {S} samples per ray; the '
                    f'fused kernels take at most {limit}'
                    + ('' if cfg.oneGrid else ' with a colour grid (oneGrid=False)'))
        if not cfg.tcnn_encoding:
            raise NotImplementedError('tcnn_encoding=True is the co-slam '
                                      'default (input_config.py:254)')
        if (cfg.hidden_dim, cfg.hidden_dim_color, cfg.geo_feat_dim,
                cfg.pos_nbins, cfg.num_layers, cfg.num_layers_color) != (
                    32, 32, 15, 16, 2, 2):
            raise NotImplementedError('decoder shape fixed to the reference '
                                      'default 80-32-16 / 63-32-3 (95-32-3 with oneGrid=False)')
        self.bounding_box = torch.as_tensor(np.asarray(self.bounding_box),
                                            dtype=torch.float64)
        self.get_resolution()
        self.get_encoding()
        self.get_decoder()
        n = cfg.training_n_range_d
        ls = torch.linspace
        self.register_buffer('_lin_uniform',
                             ls(cfg.cam_near, cfg.cam_far,
                                cfg.training_n_sample_d), persistent=False)
        self.register_buffer('_lin_range',
                             ls(-cfg.training_range_d, cfg.training_range_d,
                                steps=n), persistent=False)
        self.register_buffer('_lin_nodepth',
                             ls(cfg.cam_near, cfg.cam_far, steps=n),
                             persistent=False)
        self.register_buffer('_lin_full',
                             ls(cfg.cam_near, cfg.cam_far,
                                cfg.training_n_samples), persistent=False)
        # sample_pdf's det draw (utils.py:50-54), used when training_perturb == 0
        N = cfg.training_n_importance
        self.register_buffer('_lin_u', ls(0. + 0.5 / N, 1. - 0.5 / N, steps=N) if N else None,
                             persistent=False)
        self._step_count = 0
        # set by the Algorithm around tracking (only pose params have optimizers
        # there, base_algorithm.py:168-181): the fused pass then produces d rays only
        self.freeze_map_grads = False
        self.dp = None  # xrdslam_b200.dp.MappingDataParallel when mapping rays are sharded

    def get_resolution(self):
        """joint_encoding.py:199-210."""
        dim_max = (self.bounding_box[:, 1] - self.bounding_box[:, 0]).max()
        if self.config.voxel_sdf > 10:
            self.resolution_sdf = self.config.voxel_sdf
        else:
            self.resolution_sdf = int(dim_max / self.config.voxel_sdf)
        if self.config.voxel_color > 10:
            self.resolution_color = self.config.voxel_color
        else:
            self.resolution_color = int(dim_max / self.config.voxel_color)

    def get_encoding(self):
        """joint_encoding.py:212-234 + encodings_coslam.py:39-53,66-75."""
        n_levels, base = 16, 16
        per_level_scale = np.exp2(
            np.log2(self.resolution_sdf / base) / (n_levels - 1))
        self.embed_fn = HashGridParams(n_levels, self.config.hashsize, base,
                                       per_level_scale)
        self.input_ch = self.embed_fn.n_output_dims
        self.input_ch_pos = 3 * self.config.pos_nbins  # OneBlob, no params
        if not self.config.oneGrid:
            # the colour grid: the same HashGrid config at resolution_color
            pls_color = np.exp2(np.log2(self.resolution_color / base) / (n_levels - 1))
            self.embed_fn_color = HashGridParams(n_levels, self.config.hashsize, base,
                                                 pls_color, seed=1338)
            self.input_ch_color = self.embed_fn_color.n_output_dims

    def get_decoder(self):
        if not self.config.oneGrid:
            self.decoder = ColorSDFNet(self.config, input_ch=self.input_ch,
                                       input_ch_color=self.input_ch_color,
                                       input_ch_pos=self.input_ch_pos)
        else:
            self.decoder = ColorSDFNet_v2(self.config, input_ch=self.input_ch,
                                          input_ch_pos=self.input_ch_pos)

    # ------------------------------------------------------ C-ABI plumbing ---
    def _grid_struct(self, table, enc=None):
        """XrdHashGrid of `table` in the layout of `enc` (default: embed_fn)."""
        g = XrdHashGrid()
        C.memmove(C.byref(g), C.byref((enc or self.embed_fn).layout), C.sizeof(g))
        bb = self.bounding_box
        for d in range(3):
            g.bbox_min[d] = float(bb[d, 0])
            g.bbox_max[d] = float(bb[d, 1])
        g.table = ptr(table)
        return g

    def _weights(self):
        d = self.decoder
        return (d.sdf_net.model[0].weight, d.sdf_net.model[2].weight,
                d.color_net.model[0].weight, d.color_net.model[2].weight)

    def _n_samples(self, with_depth=True):
        cfg = self.config
        return (cfg.training_n_sample_d +
                cfg.training_n_range_d) if with_depth else cfg.training_n_samples

    def _mlp_struct(self, weights, table_c=None):
        """XrdCoslamMlp of the four weights; with oneGrid=False also the colour grid
        (`table_c`, default embed_fn_color.params)."""
        m = XrdCoslamMlp(*(ptr(w.detach()) for w in weights))
        if not self.config.oneGrid:
            tc = self.embed_fn_color.params if table_c is None else table_c
            m.grid_color = C.pointer(self._grid_struct(tc.detach(), self.embed_fn_color))
        return m

    def _out_keys(self):
        return OUT_KEYS + (IMPORTANCE_KEYS if self.config.training_n_importance else ())

    def _cfg_struct(self, S, seed=0, seed_dev=None, phase=0, n_rays_global=0,
                    counts_global=None, counts_out=None, n_importance=0):
        """XrdCoslamCfg for S samples per ray; seed_dev and the counts are device tensors.
        n_importance: a fine pass (phase 2) over the z_vals of _importance_struct."""
        cfg = self.config
        return XrdCoslamCfg(
            n_samples=S, n_sample_d=cfg.training_n_sample_d, n_range_d=cfg.training_n_range_d,
            perturb=int(cfg.training_perturb > 0),
            trunc=cfg.training_trunc * cfg.data_sc_factor, depth_trunc=cfg.cam_depth_trunc,
            w_rgb=cfg.trainging_rgb_weight, w_depth=cfg.trainging_depth_weight,
            w_sdf=cfg.trainging_sdf_weight, w_fs=cfg.trainging_fs_weight,
            lin_uniform=ptr(self._lin_uniform), lin_range=ptr(self._lin_range),
            lin_nodepth=ptr(self._lin_nodepth), lin_full=ptr(self._lin_full),
            seed=seed, rays_per_tile=cfg.rays_per_tile, precision=cfg.precision, phase=phase,
            n_rays_global=n_rays_global, counts_global=ptr(counts_global),
            counts_out=ptr(counts_out), seed_dev=ptr(seed_dev), n_importance=n_importance)

    def _importance_struct(self, R, S, dev, z_vals, raw, target_d=None, u=None, seed=0,
                           seed_dev=None, counts=None, bufs=None):
        """-> (buffers z_vals [R,S+N], z_samples [R,N], z_std [R], XrdCoslamImportance) of the
        hierarchical sampling after a coarse pass of S samples per ray (its z_vals, raw);
        counts: DEVICE int32 [4] receiving the fine pass's loss-normaliser counts; bufs: the
        buffers of an earlier call to write again."""
        cfg = self.config
        N = cfg.training_n_importance
        f32 = dict(dtype=torch.float32, device=dev)
        b = bufs or dict(z_vals=torch.empty(R, S + N, **f32), z_samples=torch.empty(R, N, **f32),
                         z_std=torch.empty(R, **f32))
        q = XrdCoslamImportance(
            n_rays=R, n_samples=S, n_importance=N, det=int(cfg.training_perturb == 0),
            trunc=cfg.training_trunc * cfg.data_sc_factor, depth_trunc=cfg.cam_depth_trunc,
            z_vals=ptr(z_vals), raw=ptr(raw), target_d=ptr(target_d), u=ptr(u),
            lin_u=ptr(self._lin_u), seed=seed, seed_dev=ptr(seed_dev), z_fine=ptr(b['z_vals']),
            z_samples=ptr(b['z_samples']), z_std=ptr(b['z_std']), counts_out=ptr(counts))
        return b, q

    def _check_fine_samples(self, S):
        """Raise ValueError naming the limit when the fine pass after a coarse pass of S samples
        per ray is longer than the fused kernels take (a render without depth:
        training_n_samples + N)."""
        N = self.config.training_n_importance
        if S + N > MAX_SAMPLES:
            raise ValueError(
                f'Co-SLAM importance sampling: the fine pass would march {S + N} samples per ray '
                f'({S} + training_n_importance = {N}); the fused kernels take at most '
                f'{MAX_SAMPLES} (a render without a depth target marches training_n_samples in '
                f'its coarse pass)')

    def _outputs(self, R, S, dev, z_vals=None):
        """-> (buffers, XrdCoslamOut) of one pass over R rays of S samples (z_vals: a given
        [R,S] buffer instead of a new one)."""
        f32 = dict(dtype=torch.float32, device=dev)
        o = dict(rgb=torch.empty(R, 3, **f32), depth=torch.empty(R, **f32),
                 disp_map=torch.empty(R, **f32), acc_map=torch.empty(R, **f32),
                 depth_var=torch.empty(R, **f32),
                 z_vals=torch.empty(R, S, **f32) if z_vals is None else z_vals,
                 raw=torch.empty(R, S, 4, **f32),
                 losses=torch.zeros(4, **f32))
        out = XrdCoslamOut(rgb=ptr(o['rgb']), depth=ptr(o['depth']), disp=ptr(o['disp_map']),
                           acc=ptr(o['acc_map']), depth_var=ptr(o['depth_var']),
                           z_vals=ptr(o['z_vals']), raw=ptr(o['raw']), losses=ptr(o['losses']))
        return o, out

    def _next_seed(self, rank=0):
        """Philox seed of the next pass, distinct per rank when mapping rays are sharded."""
        self._step_count += 1
        return (self.config.seed << 32) + self._step_count + (rank << 24)

    def _launch(self, rays_o, rays_d, table, w0, w1, wc0, wc1, target_s,
                target_d, noise, with_grads, need_ray_grads=True,
                loss_scale=None, seed=None, map_grads=True, table_c=None, importance_u=None):
        """table_c: the colour grid's table (oneGrid=False; default embed_fn_color.params).
        With training_n_importance = N > 0 (joint_encoding.py:301-341): the coarse pass, whose
        rgb and depth terms alone enter the losses and gradients, then xrd_coslam_importance
        (importance_u [R,N]: its uniforms, else drawn from `seed`), then the fine pass over the
        merged samples; the table and weight gradients of both passes add up in g, the ray
        gradients are summed."""
        cfg = self.config
        if not cfg.oneGrid and table_c is None:
            table_c = self.embed_fn_color.params
        dev = table.device
        _cabi.require_cuda(dev, 'model')
        f32 = dict(dtype=torch.float32, device=dev)
        rays_o = rays_o.detach().to(**f32).contiguous()
        rays_d = rays_d.detach().to(**f32).contiguous()
        R = rays_o.shape[0]
        has_d = target_d is not None
        S = self._n_samples(has_d)
        if has_d and cfg.training_n_sample_d <= 0:
            raise NotImplementedError('training_n_sample_d must be > 0')
        td = target_d.detach().to(**f32).reshape(-1).contiguous() if has_d \
            else None
        ts = target_s.detach().to(**f32).contiguous() \
            if target_s is not None else None
        if noise is not None:
            noise = noise.detach().to(**f32).contiguous()
            assert noise.shape == (R, S)
        N = cfg.training_n_importance
        if N:
            self._check_fine_samples(S)  # before any launch
        if importance_u is not None:
            importance_u = importance_u.detach().to(**f32).contiguous()
            assert importance_u.shape == (R, N)
        rays = XrdRays(R, ptr(rays_o), ptr(rays_d), ptr(ts), ptr(td))
        grid = self._grid_struct(table.detach())
        mlp = self._mlp_struct((w0, w1, wc0, wc1), table_c)
        if seed is None:
            seed = self._next_seed()
        # sharding applies to mapping only (tracking is per-frame sequential, single GPU)
        dp = self.dp if (self.dp is not None and self.dp.world > 1 and with_grads
                         and map_grads) else None
        c = self._cfg_struct(S, seed=seed)
        g = grads = None
        if with_grads:
            if not has_d or ts is None:
                raise RuntimeError('gradients need target_s and target_d')
            z = torch.zeros_like
            g = dict(d_table=z(table, **f32) if map_grads else None,
                     d_w_sdf0=z(w0) if map_grads else None,
                     d_w_sdf1=z(w1) if map_grads else None,
                     d_w_col0=z(wc0) if map_grads else None,
                     d_w_col1=z(wc1) if map_grads else None,
                     d_rays_o=torch.empty(R, 3, **f32) if need_ray_grads else None,
                     d_rays_d=torch.empty(R, 3, **f32) if need_ray_grads else None,
                     d_table_color=z(table_c, **f32) if (map_grads and table_c is not None)
                     else None)
            grads = lambda d_o, d_d, sc: self._grads_struct(dict(g, d_rays_o=d_o, d_rays_d=d_d), sc)
        sc = list(loss_scale or [1.0, 1.0, 1.0, 1.0])
        ws = _cabi.workspace(dev, 'coslam', R, S)
        c2f = CoarseToFine(self, R, S, dev, ws, _cabi.workspace(dev, 'coslam', R, S + N), grads,
                           (g['d_rays_o'], g['d_rays_d']) if g else (None, None), sc) if N else None
        o, out = (c2f.coarse, c2f._coarse) if N else self._outputs(R, S, dev)

        def step(gs):
            _cabi.launch_on(dev, 'xrd_coslam_step', C.byref(rays), C.byref(grid), C.byref(mlp),
                            C.byref(c), ptr(noise), C.byref(out), gs, ptr(ws[0]), ws[1])
        if dp is not None:
            # sharded mapping: the loss normalisers are batch-global (SURVEY Q9):
            # sample -> all-reduce the three counters -> render with the global counts
            counts = torch.zeros(4, dtype=torch.int32, device=dev)
            c.phase, c.counts_out = 1, ptr(counts)
            step(None)
            dp.all_reduce_sum(counts)
            c.phase, c.counts_global = 2, ptr(counts)
            c.n_rays_global = R * dp.world  # equal shards
        self._last_seed = seed
        if not N:
            step(C.byref(self._grads_struct(g, sc)) if g is not None else None)
            return o, g
        # importance sampling -> the fine pass over S + N samples (phase 2, its own counts)
        with torch.cuda.device(dev):
            c2f.run(torch.cuda.current_stream(dev).cuda_stream, (rays, grid, mlp), c, td, noise,
                    importance_u, dp.all_reduce_sum if dp is not None else None)
        return dict(c2f.fine, rgb0=o['rgb'], disp0=o['disp_map'], acc0=o['acc_map'],
                    depth0=o['depth'], depth_var0=o['depth_var'], z_std=c2f.imp['z_std']), g

    @staticmethod
    def _grads_struct(g, scale):
        """XrdCoslamGrads of the gradient buffers g with per-term loss scales `scale`."""
        return XrdCoslamGrads(ptr(g['d_table']), ptr(g['d_w_sdf0']), ptr(g['d_w_sdf1']),
                              ptr(g['d_w_col0']), ptr(g['d_w_col1']), ptr(g['d_rays_o']),
                              ptr(g['d_rays_d']), (C.c_float * 4)(*scale),
                              ptr(g['d_table_color']))

    def _launch_smooth(self, table, rand6, need_grad, weight=1.0):
        cfg = self.config
        dev = table.device
        grid = self._grid_struct(table.detach())
        loss = torch.zeros(1, dtype=torch.float32, device=dev)
        d_table = torch.zeros_like(table) if need_grad else None
        r = (C.c_float * 6)(*[float(v) for v in rand6])
        ws, nb = _cabi.workspace(dev, 'coslam_smoothness', cfg.trainging_smooth_pts)
        _cabi.launch_on(dev, 'xrd_coslam_smoothness', C.byref(grid), cfg.trainging_smooth_pts,
                        cfg.trainging_smooth_vox, cfg.trainging_smooth_margin, weight, r,
                        ptr(loss), ptr(d_table), 1.0, ptr(ws), nb)
        return loss[0], d_table

    # --------------------------------------------------------- Model API ---
    def get_outputs(self, input) -> Dict[str, Union[torch.Tensor, List]]:
        """joint_encoding.py:158-163.  Extra optional key ``noise`` [R,S]
        replaces torch.rand(z_vals.shape) (:292) for parity runs, and with
        training_n_importance = N > 0 ``importance_u`` [R,N] replaces sample_pdf's
        torch.rand (utils.py:56) / linspace."""
        return self.render_rays(input['rays_o'], input['rays_d'],
                                target_d=input.get('target_d'),
                                target_s=input.get('target_s'),
                                noise=input.get('noise'),
                                importance_u=input.get('importance_u'))

    def render_rays(self, rays_o, rays_d, target_d=None, target_s=None,
                    noise=None, importance_u=None):
        table = self.embed_fn.params
        w0, w1, wc0, wc1 = self._weights()
        fused = (torch.is_grad_enabled() and target_d is not None
                 and target_s is not None)
        table_c = None if self.config.oneGrid else self.embed_fn_color.params
        if fused:
            losses, *outs = _CoslamStep.apply(rays_o, rays_d, table, w0, w1, wc0, wc1,
                                              self, target_s, target_d, noise, table_c,
                                              importance_u)
            ret = dict(zip(self._out_keys(), outs))
            ret['_losses'] = losses
            return ret
        o, _ = self._launch(rays_o, rays_d, table, w0, w1, wc0, wc1, target_s,
                            target_d, noise, with_grads=False, table_c=table_c,
                            importance_u=importance_u)
        o.pop('losses')
        return o

    def get_loss_dict(self, outputs, inputs, is_mapping,
                      stage=None) -> Dict[str, torch.Tensor]:
        """joint_encoding.py:94-147 -- the four terms were produced (already
        weighted) by the fused kernel during forward()."""
        if '_losses' not in outputs:
            raise RuntimeError('get_loss_dict needs outputs of a forward() '
                               'run with grad enabled and targets present')
        ls = outputs['_losses']
        loss_dict = {
            'rgb_loss': ls[0],
            'depth_loss': ls[1],
            'sdf_loss': ls[2],
            'fs_loss': ls[3],
        }
        if is_mapping and not inputs['first']:
            # weight folded into the kernel (loss and gradient), :140-145
            loss_dict['smooth_loss'] = self.smoothness(
                self.config.trainging_smooth_pts,
                self.config.trainging_smooth_vox,
                self.config.trainging_smooth_margin,
                rand=inputs.get('smooth_rand'),
                weight=self.config.trainging_smooth_weight)
        return loss_dict

    def get_param_groups(self) -> Dict[str, List[Parameter]]:
        groups = {
            'decoder': list(self.decoder.parameters()),
            'embed_fn': list(self.embed_fn.parameters()),
        }
        if not self.config.oneGrid:
            groups['embed_fn_color'] = list(self.embed_fn_color.parameters())
        return groups

    def smoothness(self, sample_points=256, voxel_size=0.1, margin=0.05,
                   rand=None, weight=None):
        """joint_encoding.py:165-197.  ``rand`` = [torch.rand(3), torch.rand(3)]
        (the two CPU draws of :176 / :179) -- drawn here when not given."""
        cfg = self.config
        if (sample_points, voxel_size, margin) != (cfg.trainging_smooth_pts,
                                                   cfg.trainging_smooth_vox,
                                                   cfg.trainging_smooth_margin):
            raise NotImplementedError
        if rand is None:
            rand = torch.cat([torch.rand(3), torch.rand((1, 1, 1, 3)).reshape(3)])
        rand6 = torch.as_tensor(rand, dtype=torch.float32).reshape(6).tolist()
        return _SmoothFn.apply(self.embed_fn.params, self, rand6, weight)

    # ---- mesher-facing queries (joint_encoding.py:408-481) ----------------
    def _query(self, pts, normalised, want_raw=True, want_geo=False, want_feat=False):
        """xrd_coslam_query on [..., 3] points -> dict of flat [P, k] tensors (inference)."""
        table = self.embed_fn.params
        dev = table.device
        _cabi.require_cuda(dev, 'model')
        flat = pts.detach().reshape(-1, 3).to(device=dev, dtype=torch.float32).contiguous()
        P = flat.shape[0]
        f32 = dict(dtype=torch.float32, device=dev)
        raw = torch.empty(P, 4, **f32) if want_raw else None
        geo = torch.empty(P, 15, **f32) if want_geo else None
        feat = torch.empty(P, 32, **f32) if want_feat else None
        grid = self._grid_struct(table.detach())
        mlp = self._mlp_struct(self._weights())
        _cabi.launch_on(dev, 'xrd_coslam_query', C.byref(grid), C.byref(mlp), ptr(flat), P,
                        int(normalised), ptr(raw), ptr(geo), ptr(feat))
        return dict(raw=raw, geo=geo, feat=feat)

    def query_fn(self, pi):
        """:409-416: SDF at world points [N,3] -> [N,1]."""
        return self._query(pi, False)['raw'][:, 3:4]

    def color_func(self, pi):
        """:419-425: colour at world points [N,3] -> [N,1,3]."""
        return torch.sigmoid(self._query(pi, False)['raw'][:, None, :3])

    def query_sdf(self, query_points, return_geo=False, embed=False):
        """:427-456, points already normalised to the unit cube."""
        shp = list(query_points.shape[:-1])
        if embed:
            return self._query(query_points, True, False, False, True)['feat'].reshape(shp + [32])
        o = self._query(query_points, True, True, return_geo)
        sdf = o['raw'][:, 3].reshape(shp)
        if not return_geo:
            return sdf
        return sdf, o['geo'].reshape(shp + [15])

    def query_color_sdf(self, query_points):
        """:463-481 -> raw [..., 4] (rgb logits ++ sdf) at normalised points."""
        return self._query(query_points, True)['raw'].reshape(list(query_points.shape[:-1]) + [4])

    def query_color(self, query_points):
        """:458-461."""
        return torch.sigmoid(self.query_color_sdf(query_points)[..., :3])

    def run_network(self, inputs):
        """:483-507: raw [..., 4] at WORLD points (normalised inside, float64 like the
        reference's bounding-box arithmetic)."""
        return self._query(inputs, False)['raw'].reshape(list(inputs.shape[:-1]) + [4])


class _SmoothFn(torch.autograd.Function):
    """weight=None: plain TV loss, exact upstream scaling in backward.
    weight=w: loss and gradient come out of the kernel already multiplied by w
    and backward assumes the unit upstream gradient of the plugin contract
    (loss = reduce(add, loss_dict.values()); loss.backward(), coslam.py:242)
    unless config.strict_loss_grad."""
    @staticmethod
    def forward(ctx, table, model, rand6, weight):
        loss, d_table = model._launch_smooth(
            table, rand6, ctx.needs_input_grad[0],
            1.0 if weight is None else float(weight))
        ctx.d_table = d_table
        ctx.exact = weight is None or model.config.strict_loss_grad
        return loss

    @staticmethod
    def backward(ctx, g):
        d = ctx.d_table  # linear in the upstream gradient: exact for any g, no host sync
        return (d * g if d is not None else None), None, None, None
