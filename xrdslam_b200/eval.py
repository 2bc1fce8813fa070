"""ds-eval (scripts/eval.py, reference @ f0366f20): the trajectory's ATE from eval.tar, the
3D reconstruction metrics of final_mesh_rec.ply against a ground-truth mesh and, with
eval_2d_metric, the 2D depth L1 (calc_2d_metric), which reads <gt>_pc_unseen.npy beside the mesh.

    python -m xrdslam_b200.eval --output_dir <run dir> --gt_mesh <gt.ply> [--eval_2d_metric true]

eval_2d_metric defaults to False here; the reference's default is True.  A run that asks for
it fails before any other work when the unseen point cloud is missing."""
from __future__ import annotations

import argparse
import os
from dataclasses import dataclass
from pathlib import Path
from typing import Optional

import numpy as np

from .io_formats import ate_rmse, load_eval_tar


class MissingUnseenPointCloud(FileNotFoundError, NotImplementedError):
    """The depth-L1 metric's <gt>_pc_unseen.npy does not exist.  A FileNotFoundError, as the
    reference's np.load raises, and a NotImplementedError: without it the metric cannot run."""


@dataclass
class EvalMatrics:
    """Evaluate trajectory accuracy and 3D reconstruction quality."""

    output_dir: Path
    gt_mesh: Optional[str] = 'None'

    eval_traj: bool = True
    eval_recon: bool = True
    correct_scale: bool = False

    distance_thresh: float = 0.01
    eval_2d_metric: bool = False
    seed: int = 0
    device: str = 'cuda:0'

    def trajectory(self):
        """scripts/eval.py:39-54: -> (ATE dict with rot / trans, 4x4 transform) or None."""
        eval_pose_tar = f'{self.output_dir}/eval.tar'
        if not os.path.exists(eval_pose_tar):
            print('traj file: ', eval_pose_tar, ' is not exist!')
            return None
        est, gt_ori, N = load_eval_tar(eval_pose_tar)
        traj_result = ate_rmse(gt_ori, est, N, correct_scale=self.correct_scale)
        transform_matrix = np.eye(4)
        transform_matrix[:3, :3] = traj_result['rot']
        transform_matrix[:3, 3] = np.asarray(traj_result['trans']).reshape(-1)
        return traj_result, transform_matrix

    def main(self):
        """-> the merged metric dict (also printed), or None when an input is missing."""
        if self.eval_2d_metric and self.eval_recon and self.gt_mesh is not None and \
                os.path.exists(str(self.gt_mesh)):
            from .eval_recon import unseen_file
            unseen = unseen_file(self.gt_mesh)
            if not os.path.exists(unseen):
                raise MissingUnseenPointCloud(
                    2, f'eval_2d_metric: the depth renderer draws only views that do not see '
                    f'the unseen region, and its point cloud {unseen} does not exist', unseen)
        eval_mesh = f'{self.output_dir}/final_mesh_rec.ply'
        transform_matrix = None
        self.traj_result = None
        if self.eval_traj:
            t = self.trajectory()
            if t is None:
                return None
            self.traj_result, transform_matrix = t
            print(self.traj_result)
        if not self.eval_recon:
            return self.traj_result
        if self.gt_mesh is None or not os.path.exists(str(self.gt_mesh)):
            print('gt_mesh file: ', self.gt_mesh, ' is not exist!')
            return None
        from .eval_recon import calc_3d_metric, calc_3d_metric_New
        result_3d = calc_3d_metric(eval_mesh, str(self.gt_mesh), transform_matrix=transform_matrix,
                                   seed=self.seed, device=self.device)
        result_3d_more = calc_3d_metric_New(eval_mesh, str(self.gt_mesh),
                                            distance_thresh=self.distance_thresh,
                                            transform_matrix=transform_matrix,
                                            seed=self.seed + 2, device=self.device)
        result = result_3d | result_3d_more
        if self.eval_2d_metric:
            from .eval_recon import calc_2d_metric
            result_2d = calc_2d_metric(eval_mesh, str(self.gt_mesh),
                                       transform_matrix=transform_matrix, n_imgs=1000,
                                       seed=self.seed, device=self.device)
            result = result_2d | result
        print(result)
        return result


def entrypoint(argv=None):
    p = argparse.ArgumentParser(description=EvalMatrics.__doc__)
    p.add_argument('--output_dir', type=Path, required=True)
    p.add_argument('--gt_mesh', type=str, default='None')
    for name in ('eval_traj', 'eval_recon', 'correct_scale', 'eval_2d_metric'):
        default = EvalMatrics.__dataclass_fields__[name].default
        p.add_argument(f'--{name}', type=lambda s: s.lower() in ('1', 'true', 'yes'),
                       default=default)
    p.add_argument('--distance_thresh', type=float, default=0.01)
    p.add_argument('--seed', type=int, default=0)
    p.add_argument('--device', type=str, default='cuda:0')
    return EvalMatrics(**vars(p.parse_args(argv))).main()


if __name__ == '__main__':
    entrypoint()
