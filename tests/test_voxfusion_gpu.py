"""Vox-Fusion GPU parity: (1) the raw intersection / sampling kernels bit-for-bit against the
reference's OWN `grid` CUDA extension, (2) the full march + render step against
oracle/voxfusion.py.

The reference extension is not part of this repository.  Its outputs on the inputs these tests
build were recorded once (tests/golden/make_golden_vox_grid.py runs the extension compiled from
the reference sources) as SHA-256 digests in tests/golden/vox_grid_digests.json.  Here the
package's own kernels stand in for `grid`, and every call checks that they return exactly the
reference's bits; the oracle is then fed those verified bits, as it used to be fed the
extension's."""
import ctypes as C
import hashlib
import json
import os

import numpy as np
import pytest
import torch

from helpers import max_abs, rel_err

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DIGESTS = os.path.join(ROOT, 'tests', 'golden', 'vox_grid_digests.json')
OFFSET = 25.6  # voxels_each_dim / 2 * voxel_size: keeps coordinates inside [0, 256) voxels


def digest(*ts):
    """SHA-256 over dtype, shape and bytes of each tensor."""
    h = hashlib.sha256()
    for t in ts:
        a = t.detach().cpu().contiguous().numpy()
        h.update(f'{a.dtype}{a.shape}'.encode())
        h.update(a.tobytes())
    return h.hexdigest()


def call_digests(name, args, outs):
    """(inputs, outputs) digests of one `grid` call; tmin / tmax only where a voxel was hit."""
    tensors = [a for a in args if torch.is_tensor(a)]
    if name == 'svo_intersect':
        inds, tmin, tmax = outs
        hit = inds >= 0
        outs = (inds, tmin[hit], tmax[hit])
    return digest(*tensors), digest(*outs)


class OwnGrid:
    """The reference extension's two entry points on the package's kernels, same signatures
    and layouts (voxel_helpers_voxfusion.py:237-255, 399-481)."""

    def __init__(self, model):
        self.model = model

    def svo_intersect(self, ro, rd, cen, ch, vs, n_max):
        from xrdslam_b200 import _cabi
        dev = ro.device
        R = ro.shape[1]
        ro, rd = ro[0].contiguous(), rd[0].contiguous()
        cen = cen[0].to(dev, torch.float32).contiguous()
        ch = ch[0].to(dev, torch.int32).contiguous()
        ms = self.model.map_states
        assert cen.shape[0] == ms['voxel_center_xyz'].shape[0]
        emb = self.model.embeddings.detach()
        mp = _cabi.XrdVoxMap(cen.shape[0], cen.data_ptr(), ch.data_ptr(),
                             ms['voxel_vertex_idx'].data_ptr(), emb.data_ptr(), emb.shape[0])
        idx = torch.empty(R, n_max, dtype=torch.int32, device=dev)
        lo = torch.empty(R, n_max, device=dev)
        hi = torch.empty(R, n_max, device=dev)
        rays = _cabi.XrdRays(R, ro.data_ptr(), rd.data_ptr(), None, None)
        _cabi.check('xrd_voxfusion_intersect_raw', _cabi.lib().xrd_voxfusion_intersect_raw(
            C.byref(rays), C.byref(mp), vs, n_max, idx.data_ptr(), lo.data_ptr(), hi.data_ptr(),
            None))
        return idx[None], lo[None], hi[None]

    def inverse_cdf_sampling(self, pi, mn, mx, noise, pr, stp, fixed):
        from xrdslam_b200 import _cabi
        assert fixed == -1
        G, K, P = pi.shape
        ms, dev = noise.shape[-1], pi.device
        s_idx = torch.empty(G, K, ms, dtype=torch.int32, device=dev)
        s_depth = torch.empty(G, K, ms, device=dev)
        s_dist = torch.empty(G, K, ms, device=dev)
        d = lambda t: t.contiguous().data_ptr()
        _cabi.check('xrd_voxfusion_sample_raw', _cabi.lib().xrd_voxfusion_sample_raw(
            G * K, P, ms, K, d(pi.to(torch.int32)), d(mn), d(mx), d(noise), d(pr), d(stp),
            s_idx.data_ptr(), s_depth.data_ptr(), s_dist.data_ptr(), None))
        return s_idx, s_depth, s_dist


class CheckedGrid:
    """Wraps a `grid` implementation; call i of test `key` must see the inputs the reference
    saw and return the reference's exact outputs."""

    def __init__(self, key, impl):
        with open(DIGESTS) as f:
            self.expect = json.load(f)[key]
        self.key, self.impl, self.n = key, impl, 0

    def _call(self, name, *args):
        outs = getattr(self.impl, name)(*args)
        torch.cuda.synchronize()
        d_in, d_out = call_digests(name, args, outs)
        e = self.expect[self.n]
        self.n += 1
        assert e['fn'] == name, (self.key, self.n, e['fn'], name)
        assert d_in == e['inputs'], f'{self.key} call {self.n}: inputs differ from the recorded ones'
        assert d_out == e['outputs'], f'{self.key} call {self.n}: {name} differs from the reference'
        return outs

    def svo_intersect(self, *args):
        return self._call('svo_intersect', *args)

    def inverse_cdf_sampling(self, *args):
        return self._call('inverse_cdf_sampling', *args)


def ref_grid(key, model):
    return CheckedGrid(key, OwnGrid(model))


def scene(device, n_frames=2, R=700, seed=0):
    """Model with a map built from synthetic depth frames + a ray batch from the last pose."""
    from xrdslam_b200.sparse_voxel import SparseVoxelConfig
    from xrdslam_b200.synthetic import make_sequence
    cam, poses, frames = make_sequence(n_frames, width=160, height=120, offset=(OFFSET,) * 3)
    torch.manual_seed(seed)
    model = SparseVoxelConfig().setup(camera=cam).to(device)
    H, W = cam.height, cam.width
    j, i = torch.meshgrid(torch.arange(H, dtype=torch.float32),
                          torch.arange(W, dtype=torch.float32), indexing='ij')
    dirs = torch.stack([(i - cam.cx) / cam.fx, -(j - cam.cy) / cam.fy, -torch.ones_like(i)], -1)
    for (rgb, depth), c2w in zip(frames, poses):
        c2w = torch.from_numpy(c2w)
        d = torch.from_numpy(depth)
        pts = (dirs * d[..., None])[d > 0].reshape(-1, 3)
        pts = pts @ c2w[:3, :3].T + c2w[:3, 3]
        model.insert_points(pts)
    g = torch.Generator().manual_seed(seed)
    pix = torch.randint(0, H * W, (R,), generator=g)
    c2w = torch.from_numpy(poses[-1])
    rays_d = (dirs.reshape(-1, 3)[pix] @ c2w[:3, :3].T).contiguous()
    rays_o = c2w[:3, 3].expand(R, 3).contiguous()
    # a few rays that miss everything
    rays_d[:5] = torch.tensor([0.0, 0.0, 1.0])
    rays_o[:5] = torch.tensor([1.0, 1.0, 1.0])
    td = torch.from_numpy(frames[-1][1]).reshape(-1, 1)[pix].contiguous()
    ts = torch.from_numpy(frames[-1][0]).reshape(-1, 3)[pix].contiguous()
    return model, rays_o, rays_d, ts, td


def test_intersect_kernel_bit_exact_vs_reference_grid(cuda_dev):
    from xrdslam_b200 import _cabi
    model, rays_o, rays_d, _, _ = scene(cuda_dev)
    grid = ref_grid('intersect', model)
    ms = model.map_states
    ro, rd = rays_o.to(cuda_dev), rays_d.to(cuda_dev)
    R = ro.shape[0]
    # reference call exactly as voxel_helpers_voxfusion.py:237-255 would issue it with G = 1
    inds, tmin, tmax = grid.svo_intersect(ro[None].contiguous(), rd[None].contiguous(),
                                          ms['voxel_center_xyz'][None].contiguous(),
                                          ms['voxel_structure'][None].contiguous(), 0.2, 50)
    idx = torch.empty(R, 50, dtype=torch.int32, device=cuda_dev)
    lo = torch.empty(R, 50, device=cuda_dev)
    hi = torch.empty(R, 50, device=cuda_dev)
    rays = _cabi.XrdRays(R, ro.data_ptr(), rd.data_ptr(), None, None)
    mp = model._map_struct(model.embeddings.detach())
    st = _cabi.lib().xrd_voxfusion_intersect_raw(C.byref(rays), C.byref(mp), 0.2, 50,
                                                 idx.data_ptr(), lo.data_ptr(), hi.data_ptr(), None)
    _cabi.check('xrd_voxfusion_intersect_raw', st)
    torch.cuda.synchronize()
    assert torch.equal(idx, inds[0])  # node ids, visiting order: bit-exact
    m = idx >= 0
    assert m.sum() > R  # plenty of hits
    assert torch.equal(lo[m], tmin[0][m]) and torch.equal(hi[m], tmax[0][m])  # t values bit-exact


def test_sampling_kernel_bit_exact_vs_reference_grid(cuda_dev):
    from oracle.voxfusion import ray_intersect
    from xrdslam_b200 import _cabi
    model, rays_o, rays_d, _, _ = scene(cuda_dev, R=900)
    grid = ref_grid('sampling', model)
    ms = model.map_states
    dev = cuda_dev

    def gpu_intersect(ro, rd, cen, ch, vs, n_max):
        i, a, b = grid.svo_intersect(ro[None].to(dev).contiguous(), rd[None].to(dev).contiguous(),
                                     cen[None].contiguous(), ch[None].contiguous(), vs, n_max)
        return i[0].cpu(), a[0].cpu(), b[0].cpu()
    inter, hits = ray_intersect(rays_o, rays_d, ms['voxel_center_xyz'], ms['voxel_structure'],
                                0.2, intersect_fn=gpu_intersect)
    inter = {k: v[hits].to(dev) for k, v in inter.items()}
    # ray_sample + InverseCDFRaySampling.forward (voxel_helpers_voxfusion.py:399-481,690-714)
    dists = (inter['max_depth'] - inter['min_depth']).masked_fill(
        inter['intersected_voxel_idx'].eq(-1), 0)
    probs = dists / dists.sum(dim=-1, keepdim=True)
    steps = dists.sum(-1) / 0.01
    pts_idx = inter['intersected_voxel_idx']
    G, N, P = 200, pts_idx.size(0), pts_idx.size(1)
    Hh = int(np.ceil(N / G)) * G
    pad = lambda t: torch.cat([t, t[:1].expand(Hh - N, *t.shape[1:])], 0) if Hh > N else t
    pi, mn, mx, pr, stp = map(pad, (pts_idx, inter['min_depth'], inter['max_depth'], probs, steps))
    K = Hh // G
    max_steps = int(steps.ceil().long().max()) + P
    gen = torch.Generator(device='cpu').manual_seed(3)
    noise = torch.rand(G, K, max_steps, generator=gen).clamp(min=0.001, max=0.999).to(dev)
    r_idx, r_depth, r_dist = grid.inverse_cdf_sampling(
        pi.reshape(G, K, P).contiguous(), mn.reshape(G, K, P).contiguous(),
        mx.reshape(G, K, P).contiguous(), noise.contiguous(), pr.reshape(G, K, P).contiguous(),
        stp.reshape(G, K).contiguous(), -1)
    s_idx = torch.empty(Hh, max_steps, dtype=torch.int32, device=dev)
    s_depth = torch.empty(Hh, max_steps, device=dev)
    s_dist = torch.empty(Hh, max_steps, device=dev)
    st = _cabi.lib().xrd_voxfusion_sample_raw(
        Hh, P, max_steps, K, pi.contiguous().data_ptr(), mn.contiguous().data_ptr(),
        mx.contiguous().data_ptr(), noise.reshape(Hh, max_steps).data_ptr(),
        pr.contiguous().data_ptr(), stp.contiguous().data_ptr(), s_idx.data_ptr(),
        s_depth.data_ptr(), s_dist.data_ptr(), None)
    _cabi.check('xrd_voxfusion_sample_raw', st)
    torch.cuda.synchronize()
    assert torch.equal(s_idx, r_idx.reshape(Hh, -1))      # voxel of every sample: bit-exact
    assert torch.equal(s_depth, r_depth.reshape(Hh, -1))  # mid-point depths: bit-exact
    assert torch.equal(s_dist, r_dist.reshape(Hh, -1))


@pytest.mark.parametrize('need_pose', [True, False])
def test_full_step_vs_oracle(cuda_dev, need_pose):
    from oracle.voxfusion import VoxOracle
    model, rays_o, rays_d, ts, td = scene(cuda_dev, R=300, seed=2)
    dev = cuda_dev
    ora = VoxOracle()
    with torch.no_grad():
        g = torch.Generator().manual_seed(9)
        model.embeddings.copy_(torch.randn(model.embeddings.shape, generator=g) * 0.3)
        ora.embeddings.copy_(model.embeddings.cpu())
        ora.decoder.load_state_dict(model.decoder.state_dict())
    voxels, children, features = model.export_octree()
    ora.set_map(voxels, children, features)
    # noise by hit rank (the reference draws a [G, K, max_steps] tensor)
    gen = torch.Generator().manual_seed(5)
    noise_rank = torch.rand(rays_o.shape[0], model.config.max_samples_per_ray,
                            generator=gen).clamp(0.001, 0.999)

    def noise_fn(shape):
        G, K, ms = shape
        out = torch.full((G * K, ms), 0.5)
        n = min(G * K, noise_rank.shape[0])
        out[:n] = noise_rank[:n, :ms]
        return out.reshape(G, K, ms)
    ro_o = rays_o.clone().requires_grad_(True)
    rd_o = rays_d.clone().requires_grad_(True)
    marched = ora.march(ro_o.detach(), rd_o.detach(), noise_fn)
    out_o, ld_o = ora.render(ro_o, rd_o, ts, td, marched)
    sum(ld_o.values()).backward()
    hits = marched[1]
    rank = torch.cumsum(hits.long(), 0) - 1
    noise = torch.full((rays_o.shape[0], model.config.max_samples_per_ray), 0.5)
    noise[hits] = noise_rank[rank[hits]]
    ro = rays_o.to(dev).requires_grad_(need_pose)
    rd = rays_d.to(dev).requires_grad_(need_pose)
    inp = dict(rays_o=ro, rays_d=rd, target_s=ts.to(dev), target_d=td.to(dev), noise=noise.to(dev))
    out = model(inp)
    ld = model.get_loss_dict(out, inp, True, 0)
    sum(ld.values()).backward()
    torch.cuda.synchronize()
    m = model.last_march
    assert m['overflow'] == 0
    assert torch.equal(out['ray_mask'].cpu(), hits)
    # sample structure: voxel ids exact, depths to a few ulp (true division vs __fdividef)
    smp = marched[2]
    S = smp['sampled_point_voxel_idx'].shape[1]
    assert m['s_max'] == S and m['n_hit_rays'] == int(hits.sum())
    got_idx = m['smp_idx'].cpu()[hits][:, :S]
    assert (got_idx != smp['sampled_point_voxel_idx']).float().mean() < 2e-3
    same = got_idx == smp['sampled_point_voxel_idx']
    dd = (m['smp_depth'].cpu()[hits][:, :S] - smp['sampled_point_depth']).abs()
    assert float(dd[same].max()) < 1e-5
    assert max_abs(out['depth'], out_o['depth']) < 2e-4
    assert max_abs(out['rgb'], out_o['rgb']) < 2e-4
    for k in ld_o:
        a, b = float(ld[k].detach()), float(ld_o[k].detach())
        assert abs(a - b) <= 5e-4 * max(abs(b), 1e-6), (k, a, b)
    assert rel_err(model.embeddings.grad, ora.embeddings.grad) < 5e-3
    sd_o = dict(ora.decoder.named_parameters())
    for n, p in model.decoder.named_parameters():
        assert rel_err(p.grad, sd_o[n].grad) < 5e-3, n
    if need_pose:
        assert rel_err(ro.grad, ro_o.grad) < 5e-3
        assert rel_err(rd.grad, rd_o.grad) < 5e-3


def test_no_hit_returns_none(cuda_dev):
    model, rays_o, rays_d, ts, td = scene(cuda_dev, R=64)
    dev = cuda_dev
    ro = torch.ones(16, 3, device=dev)
    rd = torch.tensor([[0.0, 0.0, 1.0]], device=dev).expand(16, 3).contiguous()
    out = model(dict(rays_o=ro, rays_d=rd, target_s=ts[:16].to(dev), target_d=td[:16].to(dev)))
    assert out is None  # reference: render_rays prints "no hit" and returns None


def _march_through_reference_grid(grid, ora, rays_o, rays_d, noise_fn, dev):
    """VoxOracle.march with BOTH native stages (svo_intersect + inverse_cdf_sampling) returning
    the reference extension's own bits, glued exactly as voxel_helpers_voxfusion.py:237-255,
    399-481 glue them.  The CPU restatement divides exactly where the reference kernels use
    __fdividef; chained through these stages the oracle sees the reference's own bits."""
    from oracle.voxfusion import MAX_DEPTH, ray_intersect

    def gpu_intersect(ro, rd, cen, ch, vs, n_max):
        i, a, b = grid.svo_intersect(ro[None].to(dev).contiguous(), rd[None].to(dev).contiguous(),
                                     cen[None].to(dev).contiguous(), ch[None].to(dev).contiguous(),
                                     vs, n_max)
        return i[0].cpu(), a[0].cpu(), b[0].cpu()
    inter, hits = ray_intersect(rays_o, rays_d, ora.centres, ora.children, ora.voxel_size,
                                intersect_fn=gpu_intersect)
    inter = {k: v[hits] for k, v in inter.items()}
    dists = (inter['max_depth'] - inter['min_depth']).masked_fill(
        inter['intersected_voxel_idx'].eq(-1), 0)
    probs = dists / dists.sum(dim=-1, keepdim=True)
    steps = dists.sum(-1) / ora.step_size
    pts_idx = inter['intersected_voxel_idx']
    G, N, P = 200, pts_idx.size(0), pts_idx.size(1)
    Hh = int(np.ceil(N / G)) * G
    pad = lambda t: torch.cat([t, t[:1].expand(Hh - N, *t.shape[1:])], 0) if Hh > N else t
    pi, mn, mx, pr, stp = map(pad, (pts_idx, inter['min_depth'], inter['max_depth'], probs, steps))
    K = Hh // G
    max_steps = int(steps.ceil().long().max()) + P
    noise = noise_fn((G, K, max_steps))
    d = lambda t: t.to(dev).contiguous()
    r_idx, r_depth, r_dist = grid.inverse_cdf_sampling(
        d(pi.reshape(G, K, P)), d(mn.reshape(G, K, P)), d(mx.reshape(G, K, P)), d(noise),
        d(pr.reshape(G, K, P)), d(stp.reshape(G, K)), -1)
    s_idx = r_idx.reshape(Hh, -1)[:N].cpu()
    s_depth = r_depth.reshape(Hh, -1)[:N].cpu()
    s_dist = r_dist.reshape(Hh, -1)[:N].cpu()
    max_len = int(s_idx.ne(-1).sum(-1).max())
    s_idx, s_depth, s_dist = s_idx[:, :max_len], s_depth[:, :max_len], s_dist[:, :max_len]
    s_dist = s_dist.clamp(min=0.0)
    s_depth = s_depth.masked_fill(s_idx.eq(-1), MAX_DEPTH)
    s_dist = s_dist.masked_fill(s_idx.eq(-1), 0.0)
    samples = {'sampled_point_depth': s_depth, 'sampled_point_distance': s_dist,
               'sampled_point_voxel_idx': s_idx, 'probs': probs, 'steps': steps, 'K': K}
    return inter, hits, samples


@pytest.mark.parametrize('R', [300, 5 * 1024])
def test_full_step_vs_oracle_chained_through_reference_grid(cuda_dev, R):
    """Full step (march + sample + decode + composite + loss + backward) with the oracle fed
    the reference extension's own intersections / samples: sample->voxel ids and depths
    BIT-EXACT, gradients rel-l2 <= 5e-4.  R = 5 x 1024 is the default mapping batch
    (5 keyframes x 1024 rays, slam/configs/input_config.py vox-fusion entry)."""
    from oracle.voxfusion import VoxOracle
    model, rays_o, rays_d, ts, td = scene(cuda_dev, R=R, seed=4)
    grid = ref_grid(f'chained_{R}', model)
    dev = cuda_dev
    ora = VoxOracle()
    with torch.no_grad():
        g = torch.Generator().manual_seed(9)
        model.embeddings.copy_(torch.randn(model.embeddings.shape, generator=g) * 0.3)
        ora.embeddings.copy_(model.embeddings.cpu())
        ora.decoder.load_state_dict(model.decoder.state_dict())
    voxels, children, features = model.export_octree()
    ora.set_map(voxels, children, features)
    gen = torch.Generator().manual_seed(5)
    noise_rank = torch.rand(rays_o.shape[0], model.config.max_samples_per_ray,
                            generator=gen).clamp(0.001, 0.999)

    def noise_fn(shape):
        G, K, ms = shape
        out = torch.full((G * K, ms), 0.5)
        n = min(G * K, noise_rank.shape[0])
        out[:n] = noise_rank[:n, :ms]
        return out.reshape(G, K, ms)
    ro_o = rays_o.clone().requires_grad_(True)
    rd_o = rays_d.clone().requires_grad_(True)
    marched = _march_through_reference_grid(grid, ora, ro_o.detach(), rd_o.detach(), noise_fn, dev)
    out_o, ld_o = ora.render(ro_o, rd_o, ts, td, marched)
    sum(ld_o.values()).backward()
    hits = marched[1]
    rank = torch.cumsum(hits.long(), 0) - 1
    noise = torch.full((rays_o.shape[0], model.config.max_samples_per_ray), 0.5)
    noise[hits] = noise_rank[rank[hits]]
    ro = rays_o.to(dev).requires_grad_(True)
    rd = rays_d.to(dev).requires_grad_(True)
    inp = dict(rays_o=ro, rays_d=rd, target_s=ts.to(dev), target_d=td.to(dev), noise=noise.to(dev))
    out = model(inp)
    ld = model.get_loss_dict(out, inp, True, 0)
    sum(ld.values()).backward()
    torch.cuda.synchronize()
    m = model.last_march
    assert m['overflow'] == 0
    assert torch.equal(out['ray_mask'].cpu(), hits)
    smp = marched[2]
    S = smp['sampled_point_voxel_idx'].shape[1]
    assert m['s_max'] == S and m['n_hit_rays'] == int(hits.sum())
    got_idx = m['smp_idx'].cpu()[hits][:, :S]
    assert torch.equal(got_idx, smp['sampled_point_voxel_idx'])               # bit-exact
    valid = got_idx >= 0
    assert torch.equal(m['smp_depth'].cpu()[hits][:, :S][valid],
                       smp['sampled_point_depth'][valid])                     # bit-exact
    assert max_abs(out['depth'], out_o['depth']) < 5e-5
    assert max_abs(out['rgb'], out_o['rgb']) < 5e-5
    for k in ld_o:
        a, b = float(ld[k].detach()), float(ld_o[k].detach())
        assert abs(a - b) <= 1e-4 * max(abs(b), 1e-6), (k, a, b)
    TOL = 5e-4
    assert rel_err(model.embeddings.grad, ora.embeddings.grad) < TOL
    sd_o = dict(ora.decoder.named_parameters())
    for n, p in model.decoder.named_parameters():
        assert rel_err(p.grad, sd_o[n].grad) < TOL, n
    assert rel_err(ro.grad, ro_o.grad) < TOL
    assert rel_err(rd.grad, rd_o.grad) < TOL


def test_device_octree_on_gpu_equals_host_octree(cuda_dev):
    """The map grown on the device (default) == the map grown by the host C++ octree: same
    node count, centres, structure and vertex tables after two frames."""
    from xrdslam_b200.sparse_voxel import SparseVoxelConfig
    from xrdslam_b200.synthetic import make_sequence
    cam, poses, frames = make_sequence(2, width=160, height=120, offset=(OFFSET,) * 3)
    H, W = cam.height, cam.width
    j, i = torch.meshgrid(torch.arange(H, dtype=torch.float32),
                          torch.arange(W, dtype=torch.float32), indexing='ij')
    dirs = torch.stack([(i - cam.cx) / cam.fx, -(j - cam.cy) / cam.fy, -torch.ones_like(i)], -1)
    models = [SparseVoxelConfig(device_octree=flag).setup(camera=cam).to(cuda_dev)
              for flag in (True, False)]
    for (rgb, depth), c2w in zip(frames, poses):
        c2w = torch.from_numpy(c2w)
        d = torch.from_numpy(depth)
        pts = (dirs * d[..., None])[d > 0].reshape(-1, 3)
        pts = (pts @ c2w[:3, :3].T + c2w[:3, 3]).to(cuda_dev)
        for m in models:
            m.insert_points(pts)
    a, b = models[0].map_states, models[1].map_states
    assert models[0]._dev_svo is not None and models[1]._dev_svo is None
    for k in ('voxel_vertex_idx', 'voxel_center_xyz', 'voxel_structure'):
        assert a[k].shape == b[k].shape and torch.equal(a[k], b[k]), k
    for x, y in zip(models[0].export_octree(), models[1].export_octree()):
        assert torch.equal(x, y)
