"""Point-SLAM model behind the reference's ``Model`` plugin surface, H100-native.

Host-side mirror of slam/models/conv_onet_pointslam.py (class ConvOnet2, same config fields,
``forward / get_loss_dict / get_param_groups`` signatures, groups ``decoder``, ``geometry``,
``color``).  Both stages run in csrc/pointslam.cu through the C-ABI: 'geometry' (kNN feature
interpolation + 5x32 Fourier MLP + normalised occupancy compositing + losses + backward)
and 'color' (adds the per-neighbour MLP, the 128-wide softplus colour trunk, colour
compositing / loss and their backward).  There is no PyTorch fallback on the product path."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from pathlib import Path
from typing import Dict, List, Optional, Type, Union

import torch
from torch import nn
from torch.nn import Parameter

from . import _cabi
from ._cabi import (XrdNiceDecoder, XrdPointCfg, XrdPointColorDecoder,
                    XrdPointColorDecoderGrads, XrdPointFeats, XrdPointGrads, XrdPointOut,
                    XrdRays, ptr)
from .base_model import FusedStep, Model, ModelConfig
from .conv_onet import MLP as _GeoMLP
from .conv_onet import _dec_struct
from .neural_point_cloud import NeuralPointCloud


@dataclass
class ConvOnet2Config(ModelConfig):
    """slam/models/conv_onet_pointslam.py:18-72 (field names and defaults kept)."""
    _target: Type = field(default_factory=lambda: ConvOnet2)
    use_dynamic_radius: bool = True
    points_batch_size: int = 50000
    cuda_id: int = 0
    pretrained_decoders_middle_fine: Optional[Path] = None
    model_c_dim: int = 32
    model_pos_embedding_method: str = 'fourier'
    model_use_view_direction: bool = False
    model_encode_rel_pos_in_col: bool = True
    model_encode_exposure: bool = False
    model_encode_viewd: bool = True
    model_exposure_dim: int = 8
    pointcloud_nn_weighting: str = 'distance'
    pointcloud_nn_num: int = 8
    pointcloud_min_nn_num: int = 2
    pointcloud_radius_add: float = 0.04
    pointcloud_radius_min: float = 0.02
    pointcloud_radius_query: float = 0.08
    pointcloud_fix_interval_when_add_along_ray: bool = False
    pointcloud_n_add: int = 3
    rendering_n_surface: int = 5
    rendering_sample_near_pcl: bool = False
    rendering_near_end_surface: float = 0.98
    rendering_near_end: float = 0.3
    rendering_far_end_surface: float = 1.02
    rendering_sigmoid_coef_mapper: float = 0.1
    tracking_w_color_loss: float = 0.5
    mapping_w_color_loss: float = 0.1
    tracking_handle_dynamic: bool = True
    tracking_use_color_in_tracking: bool = True
    mapping_fix_color_decoder: bool = False
    mapping_fix_geo_decoder: bool = True
    mapping_pixels_based_on_color_grad: int = 1000


class _Embedder(nn.Module):
    def __init__(self, mapping_size, scale, learnable):
        super().__init__()
        B = torch.randn(3, mapping_size) * scale
        if learnable:
            self._B = nn.Parameter(B)
        else:  # a plain attribute in the reference (not in its state_dict): keep it that way
            self.register_buffer('_B', B, persistent=False)


class _ColNeighbor(nn.Module):
    def __init__(self, c_dim, emb, hidden):
        super().__init__()
        self.linear1 = nn.Linear(c_dim + emb, hidden)
        self.linear2 = nn.Linear(hidden, c_dim)
        nn.init.xavier_uniform_(self.linear1.weight)
        nn.init.xavier_uniform_(self.linear2.weight)


class MLPColor(nn.Module):
    """Parameter container with the reference MLP_color's state_dict keys
    (decoder_pointslam.py:313-404): fc_c.i, embedder_rel_pos._B, mlp_col_neighbor.linear{1,2},
    pts_linears.i, output_linear."""
    def __init__(self, c_dim=32, hidden=128):
        super().__init__()
        self.fc_c = nn.ModuleList([nn.Linear(c_dim, hidden) for _ in range(5)])
        self.embedder = _Embedder(20, 32, False)
        self.embedder_rel_pos = _Embedder(10, 32, True)
        self.mlp_col_neighbor = _ColNeighbor(c_dim, 20, hidden)
        dims = [40, hidden, hidden, hidden + 40, hidden]
        self.pts_linears = nn.ModuleList([nn.Linear(d, hidden) for d in dims])
        self.output_linear = nn.Linear(hidden, 3)
        g = nn.init.calculate_gain('relu')
        for lin in self.pts_linears:
            nn.init.xavier_uniform_(lin.weight, gain=g)
            nn.init.zeros_(lin.bias)
        nn.init.xavier_uniform_(self.output_linear.weight)
        nn.init.zeros_(self.output_linear.bias)

    def tensors(self):
        """Learnable tensors in the field order of XrdPointColorDecoderGrads."""
        n = self.mlp_col_neighbor
        return ([self.embedder_rel_pos._B, n.linear1.weight, n.linear1.bias, n.linear2.weight,
                 n.linear2.bias] + [l.weight for l in self.pts_linears] +
                [l.bias for l in self.pts_linears] + [l.weight for l in self.fc_c] +
                [l.bias for l in self.fc_c] + [self.output_linear.weight, self.output_linear.bias])


def _color_struct(cls, tensors, B=None):
    """tensors in MLPColor.tensors() order -> XrdPointColorDecoder / ...Grads."""
    st = cls()
    it = iter(tensors)
    if B is not None:
        st.B = ptr(B)
    st.B_rel = ptr(next(it))
    st.nb_w1, st.nb_b1, st.nb_w2, st.nb_b2 = (ptr(next(it)) for _ in range(4))
    for name in ('w', 'b', 'wc', 'bc'):
        arr = getattr(st, name)
        for i in range(5):
            arr[i] = ptr(next(it))
    st.wo, st.bo = ptr(next(it)), ptr(next(it))
    return st


class POINT(nn.Module):
    """Parameter container of decoder_pointslam.py:545-594: geometry decoder (the 5x32 Fourier
    MLP with fc_c, same tensor layout as the NICE decoders) + colour decoder."""
    def __init__(self, c_dim=32):
        super().__init__()
        self.geo_decoder = _GeoMLP('geometry', c_dim, False)
        self.color_decoder = MLPColor(c_dim)


class ConvOnet2(Model):
    config: ConvOnet2Config

    def __init__(self, config: ConvOnet2Config, camera, **kwargs) -> None:
        super().__init__(config=config, camera=camera, bounding_box=None, **kwargs)

    def populate_modules(self):
        super().populate_modules()
        cfg = self.config
        if not cfg.use_dynamic_radius or cfg.pointcloud_nn_weighting != 'distance' or \
                cfg.model_encode_exposure:
            raise NotImplementedError('CUDA path covers the reference point-slam config')
        self.decoder = POINT(cfg.model_c_dim)
        self.load_pretrain()
        self.neural_point_cloud = None
        self.register_buffer('_t_surface', torch.linspace(0.0, 1.0, steps=cfg.rendering_n_surface),
                             persistent=False)

    def load_pretrain(self):
        """conv_onet_pointslam.py:228-246: the (frozen) geometry decoder takes the
        'decoder.coarse.*' entries of the pretrained ConvONet middle_fine checkpoint,
        strict=False (the checkpoint has no colour-only members).  A path that is set must
        load; without one the decoder keeps its seeded init and a warning says so (the
        reference checkpoints are Git-LFS objects that do not ship with the repository)."""
        path = self.config.pretrained_decoders_middle_fine
        if path is None:
            import warnings
            warnings.warn('ConvOnet2: no pretrained checkpoint for the frozen geometry decoder '
                          '(pretrained_decoders_middle_fine): it stays randomly initialised',
                          RuntimeWarning, stacklevel=3)
            return
        ckpt = torch.load(path, map_location='cpu', weights_only=False)
        if not isinstance(ckpt, dict) or 'model' not in ckpt:
            raise RuntimeError(f'{path}: not a ConvONet checkpoint (no "model" entry)')
        middle = {}
        for k, v in ckpt['model'].items():
            if 'decoder' in k and 'encoder' not in k and 'coarse' in k:
                middle[k[8 + 7:]] = v
        res = self.decoder.geo_decoder.load_state_dict(middle, strict=False)
        if len(res.missing_keys) == len(self.decoder.geo_decoder.state_dict()):
            raise RuntimeError(f'{path}: no decoder.coarse.* entries for the geometry decoder')

    def model_update(self, device=None):
        """conv_onet_pointslam.py:98-128: create the point cloud lazily."""
        if self.neural_point_cloud is None:
            cfg = self.config
            self.neural_point_cloud = NeuralPointCloud(
                c_dim=cfg.model_c_dim, nn_num=cfg.pointcloud_nn_num,
                radius_add=cfg.pointcloud_radius_add, radius_min=cfg.pointcloud_radius_min,
                radius_query=cfg.pointcloud_radius_query, n_add=cfg.pointcloud_n_add,
                near_end_surface=cfg.rendering_near_end_surface,
                far_end_surface=cfg.rendering_far_end_surface,
                device=device or self._t_surface.device)
        return self.neural_point_cloud

    def _launch(self, stage, is_mapping, rays_o, rays_d, target_s, target_d, radius, rand_feat,
                with_grads, need_rays=False, need_feats=False, rand_feat_color=None,
                need_col_feats=False, need_cdec=False):
        if stage not in ('geometry', 'color'):
            raise ValueError(stage)
        cfg = self.config
        color = stage == 'color'
        npc = self.neural_point_cloud
        dev = npc.device
        _cabi.require_cuda(dev, 'the neural point cloud')
        f32 = dict(dtype=torch.float32, device=dev)
        rays_o = rays_o.detach().to(**f32).contiguous()
        rays_d = rays_d.detach().to(**f32).contiguous()
        R, S = rays_o.shape[0], cfg.rendering_n_surface
        ts = target_s.detach().to(**f32).contiguous() if target_s is not None else None
        radius = radius.detach().to(**f32).reshape(-1).contiguous()
        if target_d is not None:
            td = target_d.detach().to(**f32).reshape(-1).contiguous()
            # far = min(5 * mean(d), max(1.2 * d)) (conv_onet_pointslam.py:340-342), batch-global
            far = torch.minimum(5 * td.mean(), torch.max(td * 1.2)).reshape(1).float().contiguous()
        else:  # no depth at all: every ray is rendered over 10 m (conv_onet_pointslam.py:350-354)
            td = torch.zeros(R, **f32)
            far = torch.full((1,), 10.0, **f32)
        zn = nm = None
        if cfg.rendering_sample_near_pcl:
            zn, nm = npc.near_pcl_samples(rays_o, rays_d, td, far, cfg.rendering_near_end, S)
        o = dict(rgb=torch.empty(R, 3, **f32), depth=torch.empty(R, **f32),
                 uncertainty=torch.empty(R, **f32),
                 valid_ray_mask=torch.empty(R, dtype=torch.uint8, device=dev),
                 losses=torch.zeros(2, **f32))
        rays = XrdRays(R, ptr(rays_o), ptr(rays_d), ptr(ts), ptr(td))
        ix = npc.index_struct()
        feats = XrdPointFeats(ptr(npc.geo_feats.detach()), ptr(npc.frustum_mask),
                              ptr(npc.col_feats.detach()) if color else None)
        dec = _dec_struct([t.detach() for t in self.decoder.geo_decoder.tensors()], 32, 1)
        cd = self.decoder.color_decoder
        cparams = [t.detach() for t in cd.tensors()]
        cdec = _color_struct(XrdPointColorDecoder, cparams, cd.embedder._B) if color else None
        rf = rand_feat.detach().to(**f32).contiguous() if rand_feat is not None else None
        rfc = rand_feat_color.detach().to(**f32).contiguous() \
            if rand_feat_color is not None else None
        c = XrdPointCfg(int(color), int(is_mapping), S, cfg.rendering_near_end_surface,
                        cfg.rendering_far_end_surface, cfg.rendering_near_end,
                        cfg.rendering_sigmoid_coef_mapper, cfg.pointcloud_min_nn_num,
                        cfg.mapping_w_color_loss if is_mapping else cfg.tracking_w_color_loss,
                        int(cfg.tracking_handle_dynamic), int(cfg.tracking_use_color_in_tracking),
                        ptr(self._t_surface), ptr(far), ptr(radius), ptr(rf), ptr(rfc),
                        ptr(zn), ptr(nm))
        zc = getattr(self, '_z_capture', None)
        out = XrdPointOut(ptr(o['rgb']), ptr(o['depth']), ptr(o['uncertainty']),
                          ptr(o['valid_ray_mask']), ptr(zc), ptr(o['losses']))
        g, gs = None, None
        if with_grads:
            if ts is None:
                ts = torch.zeros(R, 3, **f32)
                rays.target_s = ptr(ts)
            g = dict(d_geo_feats=torch.zeros_like(npc.geo_feats) if need_feats else None,
                     d_col_feats=torch.zeros_like(npc.col_feats) if need_col_feats else None,
                     d_rays_o=torch.empty(R, 3, **f32) if need_rays else None,
                     d_rays_d=torch.empty(R, 3, **f32) if need_rays else None,
                     d_cdec=[torch.zeros_like(t) for t in cparams] if need_cdec else None)
            cg = _color_struct(XrdPointColorDecoderGrads, g['d_cdec']) if need_cdec else None
            gs = XrdPointGrads(ptr(g['d_geo_feats']), ptr(g['d_rays_o']), ptr(g['d_rays_d']),
                               ptr(g['d_col_feats']), C.pointer(cg) if cg is not None else None)
        ws, nb = _cabi.workspace(dev, 'pointslam', R, S, int(color), int(with_grads))
        _cabi.launch_on(dev, 'xrd_pointslam_step', C.byref(rays), C.byref(ix), C.byref(feats),
                        C.byref(dec), C.byref(cdec) if cdec is not None else None, C.byref(c),
                        C.byref(out), C.byref(gs) if gs is not None else None, ptr(ws), nb)
        o['valid_ray_mask'] = o['valid_ray_mask'].bool()
        return o, g

    def get_outputs(self, input) -> Dict[str, Union[torch.Tensor, List]]:
        """conv_onet_pointslam.py:130-142.  Optional ``rand_feat`` / ``rand_feat_color`` [32]
        replace the random features of samples with too few neighbours (Q6)."""
        stage = input['stage']
        rays_o, rays_d = input['rays_o'], input['rays_d']
        td, ts = input['target_d'], input.get('target_s')
        radius = input['batch_dynamic_r']
        npc = self.neural_point_cloud
        fused = torch.is_grad_enabled() and 'is_mapping' in input
        if fused:
            is_mapping, color = input['is_mapping'], stage == 'color'
            maps = [npc.geo_feats, npc.col_feats, *self.decoder.color_decoder.tensors()]
            # the colour term enters the in-kernel gradient only in stage 'color' (get_loss_dict
            # lists ls[1] in geometry-stage tracking too, where it is identically 0)
            n_live = 2 if (color and (is_mapping or self.config.tracking_use_color_in_tracking)) \
                else 1

            def launch(needs):
                o, g = self._launch(
                    stage, is_mapping, rays_o, rays_d, ts, td, radius, input.get('rand_feat'),
                    True, need_rays=needs[0] or needs[1], need_feats=needs[2],
                    rand_feat_color=input.get('rand_feat_color'),
                    need_col_feats=color and needs[3], need_cdec=color and any(needs[4:]))
                dc = g['d_cdec'] if g['d_cdec'] is not None else [None] * len(needs[4:])
                grads = [g['d_rays_o'], g['d_rays_d'], g['d_geo_feats'], g['d_col_feats'], *dc]
                return (o['losses'], (o['rgb'], o['depth'], o['uncertainty'], o['valid_ray_mask']),
                        grads)
            losses, rgb, depth, unc, valid = FusedStep.apply(launch, n_live, rays_o, rays_d,
                                                             *self.map_inputs(*maps))
            return {'rgb': rgb, 'depth': depth, 'uncertainty': unc, 'valid_ray_mask': valid,
                    'stage': stage, '_losses': losses}
        o, _ = self._launch(stage, True, rays_o, rays_d, ts, td, radius, input.get('rand_feat'),
                            False, rand_feat_color=input.get('rand_feat_color'))
        o.pop('losses')
        o['stage'] = stage
        return o

    def get_loss_dict(self, outputs, inputs, is_mapping, stage=None) -> Dict[str, torch.Tensor]:
        """conv_onet_pointslam.py:144-195 (terms produced, already weighted, by the kernel)."""
        ls = outputs['_losses']
        d = {'geo_loss': ls[0]}
        if (is_mapping and outputs['stage'] == 'color') or \
                (not is_mapping and self.config.tracking_use_color_in_tracking):
            d['rgb_loss'] = ls[1]
        return d

    def get_param_groups(self) -> Dict[str, List[Parameter]]:
        """conv_onet_pointslam.py:197-210."""
        groups = {}
        if not self.config.mapping_fix_geo_decoder:
            raise NotImplementedError('geometry decoder is fixed (reference default)')
        groups['decoder'] = [] if self.config.mapping_fix_color_decoder else \
            list(self.decoder.color_decoder.parameters())
        npc = self.neural_point_cloud
        groups['geometry'] = [npc.geo_feats]
        groups['color'] = [npc.col_feats]
        return groups
