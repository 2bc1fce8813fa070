"""The SLAM run over an RGB-D sequence (slam/pipeline/{xrdslam,tracker,mapper}.py) in one process.

The reference runs the tracker and the mapper as two processes around a Manager-proxied
Algorithm, but the tracker blocks on every map frame until the mapper is done with it
(tracker.py:149-155), so the work happens in exactly this sequential order:

  per frame   [relative pose] -> predict_current_pose -> Frame -> do_tracking -> set_pose (once
              initialised) -> add_framepose -> check_mapframe -> (map frames) do_mapping,
              update_framepose, add_keyframe every keyframe_every-th frame -> finish_frame
  at the end  eval_re_render (PSNR / MS-SSIM / depth L1) -> final_mesh.ply + final_mesh_rec.ply
              -> eval.tar  (save_re_render_frames, tracker.py:343-420)

The output directory is what `python -m xrdslam_b200.eval --output_dir DIR` reads.  The
visualiser, the debug images / point clouds and the open3d ground-truth mesh are not part of
this package: enable_vis, save_debug_result and save_gt_mesh raise NotImplementedError."""
from __future__ import annotations

import dataclasses
import os
import time
from dataclasses import dataclass, field
from pathlib import Path
from typing import Any, Optional

import numpy as np
import torch


@dataclass
class TrackerConfig:
    """slam/pipeline/tracker.py:20-30 (same names and defaults)."""
    render_freq: int = 1
    map_every: int = 1
    lazy_start: int = -1  # frames with fid <= lazy_start are all mapped
    use_relative_pose: bool = False
    save_debug_result: bool = False
    save_gt_mesh: bool = False
    save_re_render_result: bool = True
    init_pose_offset: int = 0


@dataclass
class MapperConfig:
    """slam/pipeline/mapper.py:10-13."""
    keyframe_every: int = 5


@dataclass
class XRDSLAMConfig:
    """slam/pipeline/xrdslam.py:20-36 without the visualiser (enable_vis must stay False)."""
    data: Optional[Path] = None
    data_type: Optional[str] = 'replica'
    out_dir: Path = Path('outputs')
    algorithm_name: Optional[str] = None
    tracker: TrackerConfig = field(default_factory=TrackerConfig)
    mapper: MapperConfig = field(default_factory=MapperConfig)
    algorithm: Any = None
    enable_vis: bool = False
    device: str = 'cuda:0'
    # synchronise the device at phase boundaries so run()['timing'] splits the wall time into
    # ingest, tracking, mapping and the final pass (off: the phases overlap as they can)
    profile: bool = False


# slam/configs/input_config.py: the tracker / mapper values, the scalar algorithm values and the
# literal values of the nested model / mesher configs of the four presets (44-60, 158-175,
# 205-215, 300-311).  Values equal to the package's defaults are listed too, so the preset states
# the reference's configuration.  `pretrained` lists the reference's decoder checkpoints: they
# are not shipped, so they are not carried (make_config / the CLI take them as paths; without
# them the frozen decoders stay randomly initialised, with a RuntimeWarning).  The optimizer
# dicts are not restated here.  `preset_differences` lists every value that differs from the
# package's defaults:
#   nice-slam   model.points_batch_size 100000 (package default 500000)
#   point-slam  model.points_batch_size 500000 (package default 50000)
# and the not-carried values: nice-slam model.pretrained_decoders_coarse / _middle_fine,
# point-slam model.pretrained_decoders_middle_fine and model.cuda_id (the device comes from
# XRDSLAMConfig.device).  The package's model configs keep points_batch_size for the names'
# sake; no code reads it (the mesher's own points_batch_size sets the query chunks).
PRESETS = {
    'nice-slam': dict(
        algorithm='nice_slam.NiceSLAMConfig',
        tracker=dict(map_every=5, render_freq=50, use_relative_pose=False,
                     save_debug_result=False),
        mapper=dict(keyframe_every=50),
        algorithm_values=dict(
            coarse=True, tracking_n_iters=10, mapping_n_iters=60, mapping_first_n_iters=1500,
            mapping_window_size=5, tracking_sample=200, mapping_sample=1000,
            min_sample_pixels=200, ray_batch_size=100000, tracking_Wedge=100,
            tracking_Hedge=100,
            mapping_bound=[[-5.5, 5.9], [-6.7, 5.4], [-4.7, 5.3]],
            marching_cubes_bound=[[-5.5, 5.9], [-6.7, 5.4], [-4.7, 5.3]],
            mapping_middle_iter_ratio=0.4, mapping_fine_iter_ratio=0.6, mapping_lr_factor=1.0,
            mapping_lr_first_factor=5.0),
        mesher_values=dict(resolution=256, points_batch_size=30000),
        model_values=dict(points_batch_size=100000, mapping_frustum_feature_selection=True),
        pretrained=dict(pretrained_decoders_coarse='pretrained/nice_slam/coarse.pt',
                        pretrained_decoders_middle_fine='pretrained/nice_slam/middle_fine.pt')),
    'vox-fusion': dict(
        algorithm='voxfusion.VoxFusionConfig',
        tracker=dict(map_every=1, render_freq=50, use_relative_pose=True,
                     save_debug_result=False, init_pose_offset=10),
        mapper=dict(keyframe_every=50),
        algorithm_values=dict(
            keyframe_selection_method='random', tracking_n_iters=30, mapping_n_iters=15,
            mapping_first_n_iters=30, mapping_window_size=5, mapping_sample=1024,
            tracking_sample=1024, ray_batch_size=3000),
        mesher_values={}, model_values={}, pretrained={}),
    'co-slam': dict(
        algorithm='coslam.CoSLAMConfig',
        tracker=dict(map_every=5, render_freq=50, use_relative_pose=False,
                     save_debug_result=False),
        mapper=dict(keyframe_every=5),
        algorithm_values=dict(
            separate_LR=True, retain_graph=True, rot_rep='axis_angle', tracking_n_iters=10,
            mapping_n_iters=10, mapping_first_n_iters=200, keyframe_selection_method='all',
            mapping_sample=2048, tracking_sample=1024, min_sample_pixels=100,
            ray_batch_size=30000, tracking_Wedge=20, tracking_Hedge=20,
            mapping_bound=[[-3, 3], [-4, 2.5], [-2, 2.5]],
            marching_cubes_bound=[[-2.2, 2.6], [-3.4, 2.1], [-1.4, 2.0]]),
        mesher_values=dict(resolution=256, points_batch_size=30000),
        model_values=dict(cam_depth_trunc=100.0, tcnn_encoding=True), pretrained={}),
    'point-slam': dict(
        algorithm='point_slam.PointSLAMConfig',
        tracker=dict(map_every=5, lazy_start=20, render_freq=50, use_relative_pose=False,
                     save_debug_result=False),
        mapper=dict(keyframe_every=20),
        algorithm_values=dict(
            separate_LR=True, tracking_n_iters=40, mapping_n_iters=300,
            mapping_first_n_iters=1500, mapping_window_size=12, tracking_sample=1500,
            mapping_sample=5000, min_sample_pixels=40, ray_batch_size=3000,
            tracking_Wedge=100, tracking_Hedge=100, mapping_BA=False,
            mapping_frustum_feature_selection=True,
            mapping_pixels_based_on_color_grad=1000),
        mesher_values={}, model_values=dict(points_batch_size=500000),
        not_carried=dict(cuda_id=0),
        pretrained=dict(pretrained_decoders_middle_fine='pretrained/point_slam/middle_fine.pt')),
}


def algorithm_config_class(method):
    import importlib
    mod, cls = PRESETS[method]['algorithm'].split('.')
    return getattr(importlib.import_module('.' + mod, __package__), cls)


def preset_differences(method):
    """The preset's values against the package's defaults: {'algorithm' | 'model' | 'mesher':
    {field: (reference value, package default)}} for the carried values that differ (a field
    the package's config lacks shows its default as the string 'missing'), and 'not_carried':
    {field: reference value} for the checkpoints and the values the package has no use for."""
    p = PRESETS[method]
    default = algorithm_config_class(method)()
    out = {'algorithm': {}, 'model': {}, 'mesher': {}}
    for section, cfg in (('algorithm', default), ('model', getattr(default, 'model', None)),
                         ('mesher', getattr(default, 'mesher', None))):
        names = {f.name for f in dataclasses.fields(cfg)} if cfg is not None else set()
        for k, v in p.get(section + '_values', {}).items():
            if k not in names:
                out[section][k] = (v, 'missing')
            elif getattr(cfg, k) != v:
                out[section][k] = (v, getattr(cfg, k))
    out['not_carried'] = {**p.get('pretrained', {}), **p.get('not_carried', {})}
    return out


OVERRIDE_SECTIONS = ('model', 'mesher', 'tracker', 'mapper')


def split_overrides(method, overrides):
    """Sort config overrides by the config they reach: -> {'algorithm' | 'model' | 'mesher' |
    'tracker' | 'mapper': {field: value}}.  A plain name is a field of the method's algorithm
    config; 'model.', 'mesher.', 'tracker.' and 'mapper.' prefixes name a field of the nested
    model / mesher config or of TrackerConfig / MapperConfig.  An unknown name raises ValueError
    listing the fields it could have been."""
    default = algorithm_config_class(method)()
    fields = {'algorithm': default, 'model': getattr(default, 'model', None),
              'mesher': getattr(default, 'mesher', None), 'tracker': TrackerConfig(),
              'mapper': MapperConfig()}
    fields = {k: set() if c is None else {f.name for f in dataclasses.fields(c)}
              for k, c in fields.items()}
    out = {k: {} for k in fields}
    for key, value in overrides.items():
        section, _, name = key.rpartition('.')
        section = section or 'algorithm'
        if section not in fields or (section == 'algorithm' and '.' in key):
            raise ValueError(f'{key!r}: a field of the algorithm config, or one prefixed with '
                             f'{", ".join(s + "." for s in OVERRIDE_SECTIONS)}')
        if name not in fields[section]:
            raise ValueError(f'{method} has no {section} config field {name!r}; its fields: '
                             f'{sorted(fields[section])}')
        out[section][name] = value
    return out


def make_config(method, data=None, data_type='replica', out_dir='outputs', device='cuda:0',
                pretrained_decoders_coarse=None, pretrained_decoders_middle_fine=None,
                **overrides):
    """XRDSLAMConfig of a preset: the reference's tracker and mapper values, and the package's
    algorithm config with the reference preset's algorithm, model and mesher values and then
    `overrides` applied (`split_overrides`: a plain name sets an algorithm-config field,
    'model.x', 'mesher.x', 'tracker.x' and 'mapper.x' the nested ones, e.g.
    make_config('co-slam', **{'mesher.resolution': 128})).  The pretrained_decoders_* paths
    (NICE-SLAM: coarse and middle_fine; Point-SLAM: middle_fine) go to the model config."""
    if method not in PRESETS:
        raise ValueError(f'unknown method {method!r}; one of {sorted(PRESETS)}')
    p = PRESETS[method]
    cls = algorithm_config_class(method)
    sets = split_overrides(method, overrides)
    algo = cls(**{**p['algorithm_values'], **sets['algorithm']})
    model_values = dict(p['model_values'])
    for name, path in (('pretrained_decoders_coarse', pretrained_decoders_coarse),
                       ('pretrained_decoders_middle_fine', pretrained_decoders_middle_fine)):
        if path is not None:
            if name not in p['pretrained']:
                raise ValueError(f'{method} has no {name}')
            model_values[name] = Path(path)
    model_values.update(sets['model'])
    mesher_values = {**p['mesher_values'], **sets['mesher']}
    if model_values:
        algo.model = dataclasses.replace(algo.model, **model_values)
    if mesher_values:
        algo.mesher = dataclasses.replace(algo.mesher, **mesher_values)
    return XRDSLAMConfig(data=data, data_type=data_type, out_dir=Path(out_dir),
                         algorithm_name=method,
                         tracker=TrackerConfig(**{**p['tracker'], **sets['tracker']}),
                         mapper=MapperConfig(**{**p['mapper'], **sets['mapper']}),
                         algorithm=algo, device=device)


def relative_pose(idx, gt_c2w_np, state, init_pose_offset):
    """tracker.py:76-88: frame 0 becomes the identity moved by init_pose_offset, later frames
    first_new @ inv(first_old) @ c2w.  `state` carries (first_pose_old, first_pose_new)."""
    if idx == 0:
        state['old'] = gt_c2w_np
        new = np.eye(4)
        new[:3, 3] += init_pose_offset
        state['new'] = new
        return new
    delta = np.linalg.inv(state['old']) @ gt_c2w_np
    return state['new'] @ delta


def predict_current_pose(frame_id, gt_c2w_np, estimate_c2w_list):
    """tracker.py:185-199: constant-velocity motion model on the estimated poses."""
    if frame_id < 1:
        return gt_c2w_np
    elif frame_id == 1:
        return estimate_c2w_list[frame_id - 1].detach().cpu().numpy()
    c2w_est_prev_prev = estimate_c2w_list[frame_id - 2].detach().cpu().numpy()
    c2w_est_prev = estimate_c2w_list[frame_id - 1].detach().cpu().numpy()
    delta = c2w_est_prev @ np.linalg.inv(c2w_est_prev_prev)
    return delta @ c2w_est_prev


def check_mapframe(tracker_cfg, frame, n_frames):
    """tracker.py:171-183: is `frame` a map frame?  Sets frame.is_final_frame on map frames."""
    map_every = 1 if frame.fid <= tracker_cfg.lazy_start else tracker_cfg.map_every
    if map_every != -1 and (frame.fid % map_every == 0 or frame.fid == n_frames - 1):
        frame.is_final_frame = frame.fid == n_frames - 1
        return True
    return False


class XRDSLAM:
    """`XRDSLAM(config).run()`: the whole run.  `dataset` and `algorithm` may be given instead
    of being built from config.data / config.algorithm."""

    def __init__(self, config: XRDSLAMConfig, dataset=None, algorithm=None) -> None:
        t = config.tracker
        for name, on in (('enable_vis', config.enable_vis),
                         ('tracker.save_debug_result', t.save_debug_result),
                         ('tracker.save_gt_mesh', t.save_gt_mesh)):
            if on:
                raise NotImplementedError(
                    f'{name}=True: the visualiser, debug images / point clouds and the '
                    'ground-truth mesh are not part of this package')
        self.config = config
        if dataset is None:
            from .datasets import get_dataset
            dataset = get_dataset(config.data, config.data_type, config.device)
        self.dataset = dataset
        self.camera = dataset.get_camera()
        if algorithm is None:
            algorithm = config.algorithm.setup(camera=self.camera, device=config.device)
        self.algorithm = algorithm

    def _sync(self):
        if self.config.profile and torch.cuda.is_available():
            torch.cuda.synchronize()

    def run(self):
        """-> {'n_frames', 'render': eval_re_render's result or None, 'final_mesh': paths or
        None, 'eval_tar': path or None, 'timing': seconds per phase}."""
        from .frame import Frame
        cfg, tcfg = self.config, self.config.tracker
        algo, ds = self.algorithm, self.dataset
        n = len(ds)
        rel_state = {}
        timing = dict(ingest=0.0, tracking=0.0, mapping=0.0, final=0.0)
        last_idx = None
        clock = time.perf_counter
        it = iter(ds)
        while True:
            t0 = clock()
            try:
                idx, rgb, depth, c2w = next(it)
            except StopIteration:
                break
            idx = int(idx)
            gt_c2w_np = c2w.cpu().numpy()
            gt_c2w_ori = torch.from_numpy(gt_c2w_np)
            if tcfg.use_relative_pose:
                gt_c2w_np = relative_pose(idx, gt_c2w_np, rel_state, tcfg.init_pose_offset)
            gt_c2w = torch.from_numpy(gt_c2w_np)
            rgb_np = rgb.cpu().numpy()
            depth_np = None if depth is None else depth.cpu().numpy()
            self._sync()
            t1 = clock()
            timing['ingest'] += t1 - t0
            init_pose = predict_current_pose(idx, gt_c2w_np, algo.get_estimate_c2w_list())
            frame = Frame(fid=idx, rgb=rgb_np, depth=depth_np, gt_pose=gt_c2w_np,
                          init_pose=init_pose, separate_LR=algo.is_separate_LR(),
                          rot_rep=algo.get_rot_rep())
            algo.seed_frame_tensors(frame, rgb=rgb, depth=depth)
            candidate_c2w = algo.do_tracking(frame)
            if algo.is_initialized():
                frame.set_pose(candidate_c2w, separate_LR=algo.is_separate_LR(),
                               rot_rep=algo.get_rot_rep())
            algo.add_framepose(frame.get_pose().detach(), gt_c2w, gt_c2w_ori)
            self._sync()
            t2 = clock()
            timing['tracking'] += t2 - t1
            if check_mapframe(tcfg, frame, n):
                algo.do_mapping(frame)
                algo.update_framepose(frame.fid, frame.get_pose().detach())
                if frame.fid % cfg.mapper.keyframe_every == 0:
                    algo.add_keyframe(frame)
            algo.finish_frame(frame)
            self._sync()
            timing['mapping'] += clock() - t2
            last_idx = idx
        res = {'n_frames': n, 'render': None, 'final_mesh': None, 'eval_tar': None}
        t0 = clock()
        if tcfg.save_re_render_result and last_idx is not None:
            out_dir = str(cfg.out_dir)
            os.makedirs(out_dir, exist_ok=True)
            res['render'] = algo.eval_re_render(ds, render_freq=tcfg.render_freq)
            res['final_mesh'] = algo.save_final_mesh(out_dir, ds)
            res['eval_tar'] = algo.save_eval(out_dir, last_idx)
        algo.set_finished()
        self._sync()
        timing['final'] = clock() - t0
        res['timing'] = timing
        return res
