"""Record tests/golden/reference_live.npz: what the reference's OWN code returns on the inputs
of the tests that compare this package (and its oracles) with it -- Co-SLAM's JointEncoding,
NICE-SLAM's ConvOnet (stages coarse, middle, fine, color), the host front-end, optimisers,
keyframe selection and pixel-gradient sampler, Vox-Fusion's SparseVoxel and the compiled
svo.Octree.

Needs the reference checkout (oracle/ref_harness.py) and oracle/_ref/svo.so built by
oracle/build_ref.py; runs on the CPU.  Where a comparison used parameters initialised by the
reference, the oracle's seeded parameters are copied into the reference here instead, so the
tests can rebuild them without it.  Exact-equality outputs too large to store are kept as
SHA-256 digests (tests/helpers.py:digest).

    python tests/golden/make_golden_live.py [OUT.npz]
"""
import os
import sys
from types import SimpleNamespace

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import test_oracle_cpu as TO  # noqa: E402
import test_voxfusion_cpu as TV  # noqa: E402
from helpers import BOUND, REFERENCE_LIVE, digest  # noqa: E402
from oracle import ref_harness  # noqa: E402


def np_(t):
    return t.detach().cpu().numpy() if torch.is_tensor(t) else np.asarray(t)


def svo():
    torch.classes.load_library(os.path.join(ROOT, 'oracle', '_ref', 'svo.so'))
    o = torch.classes.svo.Octree()
    o.init(256, 16, 0.2)
    v0, _, _ = o.get_centres_and_children()
    assert int(v0.shape[0]) == 1, 'svo node ids are process-global: run this first'
    out = {}
    for it, pts in enumerate(TV.octree_batches()):
        o.insert(pts)
        v, c, f = o.get_centres_and_children()
        out.update({f'{it}.n': np.int64(v.shape[0]), f'{it}.voxels': digest(v),
                    f'{it}.children': digest(c), f'{it}.features': digest(f)})
    return out


def coslam():
    ora, (rays_o, rays_d, ts, td) = TO.coslam_live_case()
    ref = ref_harness.ref_joint_encoding(torch.from_numpy(BOUND))
    with torch.no_grad():
        ref.embed_fn.params.copy_(ora.embed_fn.params)
        ref.decoder.sdf_net.model[0].weight.copy_(ora.sdf0.weight)
        ref.decoder.sdf_net.model[2].weight.copy_(ora.sdf1.weight)
        ref.decoder.color_net.model[0].weight.copy_(ora.col0.weight)
        ref.decoder.color_net.model[2].weight.copy_(ora.col1.weight)
    torch.manual_seed(9)
    inp = dict(rays_o=rays_o, rays_d=rays_d, target_s=ts, target_d=td, first=False)
    out_r = ref(inp)
    ld_r = ref.get_loss_dict(out_r, inp, True, 0)
    out = {k: digest(out_r[k]) if k in TO.COSLAM_DIGEST_KEYS else np_(out_r[k])
           for k in TO.COSLAM_OUT_KEYS}
    out.update({'loss.' + k: np_(v) for k, v in ld_r.items()})
    torch.manual_seed(4)
    o2 = ref(dict(rays_o=rays_o, rays_d=rays_d, target_s=None, target_d=None))
    out['render.rgb'], out['render.depth'] = np_(o2['rgb']), np_(o2['depth'])
    return out


def nice_coarse():
    ora, bound, (rays_o, rays_d, ts, td) = TO.nice_coarse_case()
    ref = ref_harness.ref_conv_onet(bound, coarse=True)
    ref_harness.copy_nice_oracle_to_ref(ora, ref)
    ref.grid_c['grid_coarse'].requires_grad_(True)
    inp = dict(rays_o=rays_o, rays_d=rays_d, target_s=ts, target_d=td, stage='coarse')
    with ref_harness.cuda_calls_are_noops():
        out_r = ref(inp)
    ld_r = ref.get_loss_dict(out_r, inp, True, 'coarse')
    assert set(ld_r) == {'depth_loss'}
    ld_r['depth_loss'].backward()
    return {'depth': np_(out_r['depth']), 'uncertainty': np_(out_r['uncertainty']),
            'loss.depth_loss': np_(ld_r['depth_loss']),
            'grid_coarse.grad': np_(ref.grid_c['grid_coarse'].grad),
            'grid_coarse.shape': np.array(ref.grid_c['grid_coarse'].shape),
            'coarse_bound': np_(ref.decoder.coarse_decoder.bound)}


def nice():
    ora, bound, (rays_o, rays_d, ts, td) = TO.nice_live_case()
    ref = ref_harness.ref_conv_onet(bound)
    ref_harness.copy_nice_oracle_to_ref(ora, ref)
    out = {'bounding_box': np_(ref.bounding_box)}
    for stage in ('color', 'middle', 'fine'):
        inp = dict(rays_o=rays_o, rays_d=rays_d, target_s=ts, target_d=td, stage=stage)
        with ref_harness.cuda_calls_are_noops():
            out_r = ref(inp)
        keys = ('rgb', 'depth', 'uncertainty') if stage == 'color' else ('depth', 'uncertainty')
        out.update({f'{stage}.{k}': np_(out_r[k]) for k in keys})
        for m in (True, False):
            ld_r = ref.get_loss_dict(out_r, inp, m, stage)
            out.update({f'{stage}.{m}.loss.{k}': np_(v) for k, v in ld_r.items()})
    ref2 = ref_harness.ref_conv_onet(np.array([[-5.5, 5.9], [-6.7, 5.4], [-4.7, 5.3]]))
    out['office0.grid_middle.shape'] = np.array(ref2.grid_c['grid_middle'].shape)
    out['office0.grid_fine.shape'] = np.array(ref2.grid_c['grid_fine'].shape)
    return out


def frontend():
    import slam.common.common as rc
    import slam.utils.utils as ru
    from slam.common.camera import Camera as RCam
    from xrdslam_b200.synthetic import make_sequence
    cam, poses, fr = make_sequence(1, width=160, height=120)
    rcam = RCam(cam.fx, cam.fy, cam.cx, cam.cy, cam.width, cam.height)
    c2w = torch.from_numpy(poses[0])
    rgb, depth = fr[0]
    out = {}
    for i, kw in enumerate(TO.FRONTEND_SAMPLE_KW):
        torch.manual_seed(5)
        a = rc.get_samples(rcam, 333, c2w, depth, rgb, device='cpu', **kw)
        out[f'samples.{i}.n'] = np.int64(len(a))
        out.update({f'samples.{i}.{j}': digest(x) for j, x in enumerate(a)})
    rays = rc.get_rays(rcam, c2w, 'cpu')
    out['rays.n'] = np.int64(len(rays))
    out.update({f'rays.{j}': digest(x) for j, x in enumerate(rays)})
    out['camera_rays'] = digest(torch.as_tensor(ru.get_camera_rays(120, 160, cam.fx, cam.fy,
                                                                   cam.cx, cam.cy)))
    return out


def optimizers():
    import slam.engine.optimizers as ro
    return {k: np_(v) for k, v in TO.run_optimizers(ro).items()}


def keyframes():
    import slam.common.common as rc
    from slam.common.camera import Camera as RCam
    cam, frames = TO.keyframe_case()
    rcam = RCam(cam.fx, cam.fy, cam.cx, cam.cy, cam.width, cam.height)
    out = {}
    for k in (2, 4, 8):
        torch.manual_seed(3)
        np.random.seed(3)
        a = rc.keyframe_selection_overlap(rcam, frames[0], frames[1:], k, device='cpu')
        out[f'k{k}'] = np.array([f.fid for f in a], np.int64)
    return out


def pixel_grad():
    from scipy import ndimage
    import slam.common.common as rc
    from slam.common.camera import Camera as RCam
    import xrdslam_b200.common as mc
    from xrdslam_b200.synthetic import make_sequence
    hs = np.array([[1, 2, 1], [0, 0, 0], [-1, -2, -1]], dtype=np.float64) / 4.0
    rc.rgb2gray = mc.rgb2gray_np
    rc.filters = SimpleNamespace(sobel_h=lambda im: ndimage.convolve(im, hs, mode='reflect'),
                                 sobel_v=lambda im: ndimage.convolve(im, hs.T, mode='reflect'))
    cam, poses, fr = make_sequence(1, width=160, height=120)
    rcam = RCam(cam.fx, cam.fy, cam.cx, cam.cy, cam.width, cam.height)
    c2w = torch.from_numpy(poses[0])
    rgb, depth = fr[0]
    np.random.seed(3)
    out = {'uv': np.asarray(rc.get_sample_uv_with_grad(5, 115, 7, 150, 40, rgb))}
    for i, kw in enumerate(TO.PIXEL_GRAD_KW):
        np.random.seed(11)
        ra = rc.get_samples_with_pixel_grad(rcam, 60, c2w, depth, rgb, device='cpu', **kw)
        assert len(ra) == 6
        out.update({f'samples.{i}.{j}': digest(x) for j, x in enumerate(ra)})
    return out


def vox_oracle():
    ora, marched, (ro, rd, ts, td) = TV.vox_oracle_case()
    inter, hits, samples = marched
    R = ro.shape[0]
    ms = {'voxel_vertex_idx': ora.vertex_idx, 'voxel_center_xyz': ora.centres,
          'voxel_structure': ora.children}
    full_inter = {k: torch.zeros((R,) + v.shape[1:], dtype=v.dtype) for k, v in inter.items()}
    for k in full_inter:
        full_inter[k][hits] = inter[k]
    ref, sv = ref_harness.ref_sparse_voxel_cpu(ms, ora.embeddings.detach(),
                                               (full_inter, hits, samples))
    od = ora.decoder
    with torch.no_grad():
        rd_ = ref.decoder
        for dst, src in ((rd_.pts_linears[0], od.pts_linears[0]), (rd_.pts_linears[1], od.pts_linears[1]),
                         (rd_.sdf_out, od.sdf_out), (rd_.color_out[0], od.color_out[0]),
                         (rd_.color_out[2], od.color_out[2])):
            dst.weight.copy_(src.weight)
            dst.bias.copy_(src.bias)
    with ref_harness.cuda_calls_are_noops():
        out_r = ref.render_rays(ro.unsqueeze(0), rd.unsqueeze(0), target_d=td.unsqueeze(0))
    ld_r = ref.get_loss_dict(out_r, {'target_d': td, 'target_s': ts}, True)
    sum(ld_r.values()).backward()
    ge = ref.embeddings.grad
    rows = torch.nonzero(ge.abs().sum(1) > 0).reshape(-1)
    out = {k: np_(out_r[k]) for k in ('ray_mask', 'depth', 'rgb', 'sdf')}
    out.update({'loss.' + k: np_(v) for k, v in ld_r.items()})
    out.update({'emb_grad.rows': np_(rows), 'emb_grad.values': np_(ge[rows]),
                'sdf_out.weight.grad': np_(ref.decoder.sdf_out.weight.grad)})
    return out


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 else REFERENCE_LIVE
    ref_harness.install()
    store = {}
    for name, fn in (('svo', svo), ('coslam', coslam), ('nice_coarse', nice_coarse),
                     ('nice', nice), ('frontend', frontend), ('optimizers', optimizers),
                     ('keyframes', keyframes), ('pixel_grad', pixel_grad),
                     ('vox_oracle', vox_oracle)):
        for k, v in fn().items():
            store[f'{name}/{k}'] = np.asarray(v)
    np.savez_compressed(out_path, **store)
    print('wrote', out_path, len(store), 'arrays', os.path.getsize(out_path), 'bytes')


if __name__ == '__main__':
    main()
