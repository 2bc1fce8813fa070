"""NICE-SLAM with stratified jitter and importance sampling end to end: a short run on the
synthetic Replica folder of test_pipeline_gpu.py (reduced iteration counts) and ds-eval on what
it writes; then data-parallel mapping with the uniforms sliced from the global batch (two GPUs,
skipped below)."""
import math
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from test_pipeline_gpu import N_FRAMES, REDUCED, gt_mesh, replica_folder  # noqa: F401

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.mark.gpu
def test_short_run_with_importance(cuda_dev, replica_folder, gt_mesh, tmp_path):  # noqa: F811
    import warnings

    from xrdslam_b200.eval import EvalMatrics
    from xrdslam_b200.pipeline import XRDSLAM, make_config
    torch.manual_seed(0)
    np.random.seed(0)
    out = tmp_path / 'out'
    cfg = make_config('nice-slam', data=replica_folder, out_dir=str(out), device=str(cuda_dev),
                      **REDUCED['nice-slam'], **{'model.rendering_n_importance': 16,
                                                 'model.rendering_perturb': 1.0})
    cfg.tracker.render_freq = 5
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', UserWarning)
        res = XRDSLAM(cfg).run()
    assert res['n_frames'] == N_FRAMES
    for name in ('eval.tar', 'final_mesh.ply', 'final_mesh_rec.ply'):
        assert os.path.exists(out / name), name
    ev = EvalMatrics(output_dir=out, gt_mesh=gt_mesh, device=str(cuda_dev))
    m = ev.main()
    ate = float(ev.traj_result['rmse'])
    acc, comp = float(m['accuracy']), float(m['completion'])
    print(f'nice-slam N=16 perturb=1: ATE {ate:.5f}, accuracy {acc:.4f}, completion {comp:.4f}, '
          f'psnr {res["render"]["avg_psnr"]:.3f}')
    assert math.isfinite(ate) and math.isfinite(acc) and math.isfinite(comp)
    assert math.isfinite(float(res['render']['avg_psnr']))


def _worker(rank, world, port, ret):
    sys.path.insert(0, HERE)
    sys.path.insert(0, os.path.dirname(HERE))
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device('cuda', rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=dev)
    from helpers import rel_err
    from test_nice_gpu import nice_pair, rays
    from test_nice_importance_gpu import configure, draws
    from xrdslam_b200.dp import MappingDataParallel
    torch.manual_seed(0)
    _, nm = nice_pair(dev)
    configure(nm, 16, 1.0)
    R = 256
    ro, rd, ts, td = rays(R, 17)
    noise, u = draws(R, 32, 16, 1.0, 5)
    full = dict(rays_o=ro.to(dev), rays_d=rd.to(dev), target_s=ts.to(dev), target_d=td.to(dev),
                noise=noise.to(dev), importance_u=u.to(dev), stage='color', is_mapping=True)
    params = [nm.grids[k] for k in ('grid_middle', 'grid_fine', 'grid_color')] + \
        list(nm.decoder.color_decoder.parameters())
    ld = nm.get_loss_dict(nm(full), full, True, 'color')
    sum(ld.values()).backward()
    ref = [p.grad.clone() for p in params]
    ref_loss = torch.stack([ld['depth_loss'].detach(), ld['rgb_loss'].detach()])
    for p in params:
        p.grad = None
    dp = MappingDataParallel(params)
    nm.dp = dp
    sl = dp.shard(R)
    part = {k: (v[sl] if torch.is_tensor(v) else v) for k, v in full.items()}
    ld = nm.get_loss_dict(nm(part), part, True, 'color')
    sum(ld.values()).backward()
    loss = torch.stack([ld['depth_loss'].detach(), ld['rgb_loss'].detach()])
    dp.all_reduce_grads(extra=[loss])
    ret[rank] = dict(grad=max(rel_err(p.grad, g) for p, g in zip(params, ref)),
                     loss=float((loss - ref_loss).abs().max() / ref_loss.abs().max()))
    dist.destroy_process_group()


@pytest.mark.gpu
def test_sharded_mapping_with_importance_equals_single_gpu():
    """Rays and their explicit uniforms sharded over 2 ranks == the whole batch on one GPU, to
    test_dp_gpu.py's gates (pass 1 and sample_pdf are per ray; max depth is already global)."""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs')
    world = 2
    ret = mp.Manager().dict()
    port = 29500 + (os.getpid() % 2000) + 7
    mp.spawn(_worker, args=(world, port, ret), nprocs=world, join=True)
    for r in range(world):
        assert ret[r]['grad'] < 1e-4 and ret[r]['loss'] < 1e-5, dict(ret)
