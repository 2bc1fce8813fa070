"""`ds-run` for this package: one SLAM run over a dataset folder.

    python -m xrdslam_b200.run co-slam --data DIR --data_type replica --out_dir OUT \
        [--device cuda:0]

Methods: co-slam, nice-slam, vox-fusion, point-slam (the reference's presets, see
pipeline.PRESETS).  OUT then holds eval.tar, final_mesh.ply and final_mesh_rec.ply, which
`python -m xrdslam_b200.eval --output_dir OUT --gt_mesh MESH` scores.  NICE-SLAM and Point-SLAM
freeze pretrained decoders; the checkpoints are not shipped, so pass them with
--pretrained_decoders_coarse / --pretrained_decoders_middle_fine (without them the decoders stay
randomly initialised and a RuntimeWarning says so)."""
from __future__ import annotations

import argparse
import json


def main(argv=None):
    from .pipeline import PRESETS, XRDSLAM, make_config
    ap = argparse.ArgumentParser(prog='python -m xrdslam_b200.run', description=__doc__,
                                 formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('method', choices=sorted(PRESETS))
    ap.add_argument('--data', required=True)
    ap.add_argument('--data_type', '--data-type', default='replica', choices=['replica'])
    ap.add_argument('--out_dir', '--out-dir', default='outputs')
    ap.add_argument('--device', default='cuda:0')
    ap.add_argument('--pretrained_decoders_coarse', default=None,
                    help="NICE-SLAM's coarse decoder checkpoint (the reference's "
                         'pretrained/nice_slam/coarse.pt)')
    ap.add_argument('--pretrained_decoders_middle_fine', default=None,
                    help="NICE-SLAM's or Point-SLAM's middle / fine decoder checkpoint (the "
                         "reference's pretrained/{nice_slam,point_slam}/middle_fine.pt)")
    args = ap.parse_args(argv)
    cfg = make_config(args.method, data=args.data, data_type=args.data_type,
                      out_dir=args.out_dir, device=args.device,
                      pretrained_decoders_coarse=args.pretrained_decoders_coarse,
                      pretrained_decoders_middle_fine=args.pretrained_decoders_middle_fine)
    res = XRDSLAM(cfg).run()
    render = res['render'] or {}
    summary = {k: render.get(k) for k in ('avg_psnr', 'avg_ssim', 'avg_lpips', 'avg_depth_l1')}
    print(json.dumps({'method': args.method, 'n_frames': res['n_frames'],
                      'eval_tar': res['eval_tar'], 'timing_s': res['timing'], **summary}))
    return res


if __name__ == '__main__':
    main()
