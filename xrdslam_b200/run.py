"""`ds-run` for this package: one SLAM run over a dataset folder.

    python -m xrdslam_b200.run co-slam --data DIR --data_type tumrgbd --out_dir OUT \
        [--device cuda:0] [--set FIELD=VALUE ...]

Methods: co-slam, nice-slam, vox-fusion, point-slam (the reference's presets, see
pipeline.PRESETS).  Data types: replica (the default), tumrgbd, scannet, 7scenes, azure and
cofusion (datasets.dataset_dict; each folder holds the devices.yaml with the camera).  OUT then
holds eval.tar, final_mesh.ply and final_mesh_rec.ply, which
`python -m xrdslam_b200.eval --output_dir OUT --gt_mesh MESH` scores.

The presets carry Replica office0's bounds; another scene needs its own, e.g.
    --set 'mapping_bound=[[-3,3],[-3,3],[-1,3]]' --set 'marching_cubes_bound=[[-3,3],[-3,3],[-1,3]]'
`--set` may be repeated.  A plain FIELD is a field of the method's algorithm config; 'model.',
'mesher.', 'tracker.' and 'mapper.' prefixes reach the nested configs (e.g. --set
mesher.resolution=128, --set tracker.map_every=2).  VALUE is read with ast.literal_eval; a value
that is not a Python literal is taken as a string (--set keyframe_selection_method=all).  An
unknown FIELD is an error before the run starts.

NICE-SLAM and Point-SLAM freeze pretrained decoders; the checkpoints are not shipped, so pass them
with --pretrained_decoders_coarse / --pretrained_decoders_middle_fine (without them the decoders
stay randomly initialised and a RuntimeWarning says so)."""
from __future__ import annotations

import argparse
import ast
import json


def parse_set(items):
    """['FIELD=VALUE', ...] -> {FIELD: value}; a later FIELD wins."""
    out = {}
    for item in items or ():
        field, sep, text = item.partition('=')
        field = field.strip()
        if not sep or not field:
            raise ValueError(f'--set {item!r}: expected FIELD=VALUE')
        try:
            value = ast.literal_eval(text.strip())
        except (ValueError, SyntaxError):
            value = text.strip()
        out[field] = value
    return out


def parser():
    from .datasets import dataset_dict
    from .pipeline import PRESETS
    ap = argparse.ArgumentParser(prog='python -m xrdslam_b200.run', description=__doc__,
                                 formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('method', choices=sorted(PRESETS))
    ap.add_argument('--data', required=True)
    ap.add_argument('--data_type', '--data-type', default='replica', choices=sorted(dataset_dict))
    ap.add_argument('--out_dir', '--out-dir', default='outputs')
    ap.add_argument('--device', default='cuda:0')
    ap.add_argument('--set', dest='overrides', action='append', default=[],
                    metavar='FIELD=VALUE',
                    help='override a config field (repeatable): FIELD, model.FIELD, '
                         'mesher.FIELD, tracker.FIELD or mapper.FIELD')
    ap.add_argument('--pretrained_decoders_coarse', default=None,
                    help="NICE-SLAM's coarse decoder checkpoint (the reference's "
                         'pretrained/nice_slam/coarse.pt)')
    ap.add_argument('--pretrained_decoders_middle_fine', default=None,
                    help="NICE-SLAM's or Point-SLAM's middle / fine decoder checkpoint (the "
                         "reference's pretrained/{nice_slam,point_slam}/middle_fine.pt)")
    return ap


def main(argv=None):
    from .pipeline import XRDSLAM, make_config
    ap = parser()
    args = ap.parse_args(argv)
    try:
        overrides = parse_set(args.overrides)
        cfg = make_config(args.method, data=args.data, data_type=args.data_type,
                          out_dir=args.out_dir, device=args.device,
                          pretrained_decoders_coarse=args.pretrained_decoders_coarse,
                          pretrained_decoders_middle_fine=args.pretrained_decoders_middle_fine,
                          **overrides)
    except (ValueError, TypeError) as e:
        ap.error(str(e))
    res = XRDSLAM(cfg).run()
    render = res['render'] or {}
    summary = {k: render.get(k) for k in ('avg_psnr', 'avg_ssim', 'avg_lpips', 'avg_depth_l1')}
    print(json.dumps({'method': args.method, 'n_frames': res['n_frames'],
                      'eval_tar': res['eval_tar'], 'timing_s': res['timing'], **summary}))
    return res


if __name__ == '__main__':
    main()
