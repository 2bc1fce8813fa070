"""Generate tests/golden/pointslam_near_pcl.npz: Point-SLAM's rendering_sample_near_pcl as the
REFERENCE's own code computes it (NeuralPointCloud.sample_near_pcl and render_batch_ray with the
option on), run on CPU through oracle/ref_harness.py with the exact-kNN stand-in for faiss.

    python tests/golden/make_golden_near_pcl.py

The model, cloud and decoders are those of pointslam_geo_step.npz (make_golden.py:pointslam).
Only runs where the reference is available.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

from helpers import load_golden_pointslam  # noqa: E402
from oracle import ref_harness  # noqa: E402


def reference_model(g):
    """The reference ConvOnet2 with the option on, holding the golden cloud and decoders."""
    torch.manual_seed(0)
    ref = ref_harness.ref_conv_onet2(rendering_sample_near_pcl=True)
    rd0 = torch.from_numpy(g['add_rays_d'])
    R0 = rd0.shape[0]
    e = torch.zeros(0)
    ref.model_update(dict(batch_rays_o=torch.zeros(R0, 3), batch_rays_d=rd0,
                          batch_gt_depth=torch.from_numpy(g['add_depth']),
                          batch_gt_color=torch.zeros(R0, 3),
                          batch_dynamic_r=torch.full((R0,), 0.04),
                          batch_rays_o_grad=torch.zeros(0, 3), batch_rays_d_grad=torch.zeros(0, 3),
                          batch_gt_depth_grad=e, batch_gt_color_grad=torch.zeros(0, 3),
                          batch_dynamic_r_grad=e))
    npc = ref.neural_point_cloud
    assert np.array_equal(np.asarray(npc._cloud_pos, np.float32), g['cloud_pos'])
    t = lambda k: torch.from_numpy(g[k])
    gd, cd = ref.decoder.geo_decoder, ref.decoder.color_decoder
    own = gd.state_dict().keys()
    gd.load_state_dict({k[4:]: t(k) for k in g if k.startswith('dec.') and k[4:] in own},
                       strict=False)
    cd.load_state_dict({k[5:]: t(k) for k in g if k.startswith('cdec.') and
                        k != 'cdec.embedder._B'}, strict=False)
    with torch.no_grad():
        gd.embedder._B.copy_(t('dec.embedder._B'))
        cd.embedder._B.copy_(t('cdec.embedder._B'))
        npc.geo_feats.copy_(t('geo_feats'))
        npc.col_feats.copy_(t('col_feats'))
    return ref


def march_rays(g):
    """Rays from the origin towards cloud points, with hit patterns chosen by moving the
    target point along the ray: the march depth of point 0 .. 24 is 0.3 + k (far - 0.3) / 24."""
    pos = torch.from_numpy(g['cloud_pos'])
    gen = torch.Generator().manual_seed(5)
    idx = torch.randint(0, pos.shape[0], (48,), generator=gen)
    d = torch.nn.functional.normalize(pos[idx], dim=-1)
    d[40:] = -d[40:]  # looking away from the cloud: no hit
    return torch.zeros_like(d), d


def main():
    assert ref_harness.available(), 'needs the reference'
    g = load_golden_pointslam()
    ref = reference_model(g)
    npc = ref.neural_point_cloud
    blob = {}
    # ---- the sampler alone: the golden's rays and the march rays, two far values
    ro_m, rd_m = march_rays(g)
    ro = torch.cat([torch.from_numpy(g['rays_o']), ro_m])
    rd = torch.cat([torch.from_numpy(g['rays_d']), rd_m])
    blob['s.rays_o'], blob['s.rays_d'] = ro.numpy(), rd.numpy()
    for i, far in enumerate((2.4, 3.1)):
        far_t = torch.tensor(far, dtype=torch.float32)
        z, invalid = npc.sample_near_pcl(ro.clone(), rd.clone(), 0.3, far_t, 5)
        blob[f's{i}.far'] = far_t.numpy()
        blob[f's{i}.z'], blob[f's{i}.invalid'] = z.numpy(), invalid.numpy()
    # ---- render_batch_ray with the option on, both stages, mapping and tracking
    captured = []
    orig = npc.sample_near_pcl

    def capture(*a, **k):
        z, inv = orig(*a, **k)
        captured.append((z.clone(), inv.clone()))
        return z, inv
    npc.sample_near_pcl = capture
    rays_o = torch.from_numpy(g['rays_o']).clone()
    rays_d = torch.from_numpy(g['rays_d']).clone()
    td = torch.from_numpy(g['target_d']).clone().reshape(-1, 1)
    td[2::4] = 0  # about a third of the rays without depth
    radius = torch.from_numpy(g['radius'])
    target_s = torch.from_numpy(g['target_s'])
    blob['r.target_d'] = td.numpy()
    cd = ref.decoder.color_decoder
    for stage in ('geometry', 'color'):
        for tag, is_mapping in (('map', True), ('trk', False)):
            key = f'{stage[0]}{tag}'
            ro_ = rays_o.clone().requires_grad_(True)
            rd_ = rays_d.clone().requires_grad_(True)
            for t in [npc.geo_feats, npc.col_feats] + list(cd.parameters()):
                t.grad = None
            inp = dict(rays_o=ro_, rays_d=rd_, target_d=td,
                       target_s=target_s if stage == 'color' else torch.zeros_like(target_s),
                       stage=stage, batch_dynamic_r=radius)
            torch.manual_seed(777)
            captured.clear()
            out = ref(inp)
            ld = ref.get_loss_dict(out, inp, is_mapping)
            loss = sum(ld.values()) if stage == 'color' else ld['geo_loss']
            loss.backward()
            nz = (td.reshape(-1) > 0).numpy()
            zc, invc = captured[0]
            blob[key + '.z_zero'], blob[key + '.invalid_zero'] = zc.numpy(), invc.numpy()
            blob[key + '.zero_rays'] = np.flatnonzero(~nz)
            for k in ('depth', 'uncertainty', 'rgb'):
                blob[f'{key}.{k}'] = out[k].detach().numpy()
            blob[key + '.valid'] = out['valid_ray_mask'].numpy()
            blob[key + '.losses'] = np.array([float(v.detach()) for v in ld.values()], np.float32)
            blob[key + '.d_geo_feats'] = npc.geo_feats.grad.numpy().copy()
            blob[key + '.d_rays_o'] = ro_.grad.numpy().copy()
            blob[key + '.d_rays_d'] = rd_.grad.numpy().copy()
            if stage == 'color':
                blob[key + '.d_col_feats'] = npc.col_feats.grad.numpy().copy()
    # ---- render without depth (far = 10)
    with torch.no_grad():
        torch.manual_seed(777)
        captured.clear()
        out = ref.render_batch_ray(rays_d, rays_o, 'color', gt_depth=None,
                                   dynamic_r_query=radius)
    blob['nodepth.z'], blob['nodepth.invalid'] = captured[0][0].numpy(), captured[0][1].numpy()
    for k in ('depth', 'rgb'):
        blob['nodepth.' + k] = out[k].numpy()
    blob['nodepth.valid'] = out['valid_ray_mask'].numpy()
    np.savez_compressed(os.path.join(HERE, 'pointslam_near_pcl.npz'), **blob)
    print('wrote pointslam_near_pcl.npz', {k: v.shape for k, v in blob.items()})


if __name__ == '__main__':
    main()
