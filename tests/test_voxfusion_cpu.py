"""CPU tests for the Vox-Fusion map structure: this package's octree (csrc/octree.cpp) against
the reference's own svo.Octree compiled from its sources, and oracle/voxfusion.py against the
reference's SparseVoxel.  The reference's outputs on these inputs were recorded by
tests/golden/make_golden_live.py (tests/golden/reference_live.npz)."""
import os

import numpy as np
import torch

from helpers import digest, reference_live

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def octree_batches():
    """4 insert calls of integer voxel coordinates: grid corners and duplicates in the first."""
    g = torch.Generator().manual_seed(4)
    out = []
    for it in range(4):
        pts = (torch.rand(2500, 3, generator=g) * 25 + 30 + 7 * it).int().contiguous()
        if it == 0:
            pts[0] = torch.tensor([0, 0, 0])
            pts[1] = torch.tensor([254, 254, 254])
            pts[2] = pts[3]  # duplicates
        out.append(pts)
    return out


def test_octree_bit_exact_vs_reference_svo():
    """After every insert: node count, centres / sizes, children and corner tables identical to
    the reference's svo.Octree (as the first tree of a process, whose node ids start at 0)."""
    from xrdslam_b200 import _cabi
    lib = _cabi.lib()
    ref = reference_live('svo')
    t = lib.xrd_octree_create(256)
    try:
        for it, pts in enumerate(octree_batches()):
            n = lib.xrd_octree_insert(t, pts.data_ptr(), pts.shape[0])
            assert n == int(ref[f'{it}.n']) == lib.xrd_octree_num_nodes(t)
            mv = torch.empty(n, 4)
            mc = torch.empty(n, 8)
            mf = torch.empty(n, 8, dtype=torch.int32)
            assert lib.xrd_octree_export(t, mv.data_ptr(), mc.data_ptr(), mf.data_ptr()) == n
            assert digest(mv) == str(ref[f'{it}.voxels'])
            assert digest(mc) == str(ref[f'{it}.children'])
            assert digest(mf) == str(ref[f'{it}.features'])
    finally:
        lib.xrd_octree_destroy(t)


def test_model_map_states_match_reference_formulas():
    from xrdslam_b200.camera import Camera
    from xrdslam_b200.sparse_voxel import SparseVoxelConfig
    m = SparseVoxelConfig().setup(camera=Camera(320, 320, 319.5, 239.5, 640, 480))
    g = torch.Generator().manual_seed(0)
    pts = torch.rand(800, 3, generator=g) * 3 + 24.1
    m.insert_points(pts)
    ms = m.map_states
    N = ms['voxel_center_xyz'].shape[0]
    assert ms['voxel_structure'].shape == (N, 9) and ms['voxel_vertex_idx'].shape == (N, 8)
    leaf = ms['voxel_structure'][:, 8] == 1
    surf = leaf & (ms['voxel_vertex_idx'][:, 0] >= 0)
    # every inserted point lies inside a SURFACE leaf: centre = (floor(p/0.2) + 0.5) * 0.2
    want = {tuple(v) for v in torch.div(pts, 0.2, rounding_mode='floor').int().tolist()}
    have = {tuple(v) for v in torch.round(ms['voxel_center_xyz'][surf] / 0.2 - 0.5).int().tolist()}
    assert want <= have and len(have) == len(want)
    assert int(ms['voxel_vertex_idx'].max()) < m.config.num_embeddings


def vox_oracle_case():
    """Oracle on a wall of voxels at z ~ 12.0 m (offset world) built by this package's octree,
    96 rays from above (some missing the map), marched and sampled by the oracle."""
    from oracle.voxfusion import VoxOracle
    from xrdslam_b200.camera import Camera
    from xrdslam_b200.sparse_voxel import SparseVoxelConfig
    torch.manual_seed(5)  # decoder initialisation
    g = torch.Generator().manual_seed(3)
    xy = torch.rand(3000, 2, generator=g) * 2.0 + 11.0
    pts = torch.cat([xy, torch.full((3000, 1), 12.05) + torch.rand(3000, 1, generator=g) * 0.3], 1)
    builder = SparseVoxelConfig().setup(camera=Camera(320, 320, 319.5, 239.5, 640, 480))
    builder.insert_points(pts)
    voxels, children, features = builder.export_octree()
    ora = VoxOracle(seed=5)
    ora.set_map(voxels, children, features)
    with torch.no_grad():
        ora.embeddings.mul_(30.0)
    R = 96
    ro = torch.cat([torch.rand(R, 2, generator=g) * 1.6 + 11.2, torch.full((R, 1), 10.5)], 1)
    rd = torch.nn.functional.normalize(
        torch.cat([torch.randn(R, 2, generator=g) * 0.15, torch.ones(R, 1)], 1), dim=-1)
    rd[::13] = torch.tensor([0.0, 0.0, -1.0])  # rays that miss the map
    marched = ora.march(ro, rd, lambda shape: torch.rand(shape, generator=g))
    td = torch.full((R, 1), 1.62) + torch.rand(R, 1, generator=g) * 0.2
    td[5::11] = 0
    ts = torch.rand(R, 3, generator=g)
    return ora, marched, (ro, rd, ts, td)


def test_vox_oracle_torch_part_matches_reference_python():
    """oracle/voxfusion.py's features / decoder / sdf2weights / losses against the reference's
    own SparseVoxel.render_rays + get_loss_dict on the same map, embeddings, decoder and samples
    (its two CUDA ops fed the oracle's intersections and samples, which the GPU tests pin
    bit-for-bit against the reference's compiled kernels)."""
    ref = reference_live('vox_oracle')
    ora, marched, (ro, rd, ts, td) = vox_oracle_case()
    assert marched is not None
    inter, hits, samples = marched
    assert hits.any() and not hits.all()
    out_o, ld_o = ora.render(ro, rd, ts, td, marched)
    assert np.array_equal(out_o['ray_mask'].numpy(), ref['ray_mask'])
    for k in ('depth', 'rgb', 'sdf'):
        assert np.abs(out_o[k].detach().numpy() - ref[k]).max() < 1e-6, k
    losses = {k[5:] for k in ref if k.startswith('loss.')}
    assert losses == set(ld_o)
    for k in losses:
        r = float(ref['loss.' + k])
        assert abs(float(ld_o[k]) - r) <= 1e-5 * max(1e-3, abs(r)), k
    # gradients of the summed loss w.r.t. embeddings and decoder
    sum(ld_o.values()).backward()
    ge_r = np.zeros(tuple(ora.embeddings.shape), np.float32)
    ge_r[ref['emb_grad.rows']] = ref['emb_grad.values']
    ge_o = ora.embeddings.grad.numpy()
    assert np.abs(ge_o - ge_r).max() <= 1e-5 * np.abs(ge_r).max()
    gw_r = ref['sdf_out.weight.grad']
    assert np.abs(ora.decoder.sdf_out.weight.grad.numpy() - gw_r).max() <= 1e-5 * np.abs(gw_r).max()


def test_device_octree_equals_host_octree_numbering():
    """octree_device.DeviceOctree (data-parallel build: unique / sort / searchsorted) produces
    the SAME node ids, codes, child tables and corner-leaf tables as the host C++ octree (which
    is bit-exact against the reference's compiled svo.Octree, test above) -- over duplicate
    voxels, two successive insert calls, coordinates at the grid edge (wrap quirk) and an
    empty second call.  Runs on the host here; the same tensor program runs on the GPU."""
    from xrdslam_b200 import _cabi
    from xrdslam_b200.octree_device import DeviceOctree
    lib = _cabi.lib()

    def host(vlist):
        t = lib.xrd_octree_create(256)
        for v in vlist:
            v = v.int().contiguous()
            lib.xrd_octree_insert(t, v.data_ptr(), v.shape[0])
        N = lib.xrd_octree_num_nodes(t)
        vo, ch, fe = torch.empty(N, 4), torch.empty(N, 8), torch.empty(N, 8, dtype=torch.int32)
        lib.xrd_octree_export(t, vo.data_ptr(), ch.data_ptr(), fe.data_ptr())
        lib.xrd_octree_destroy(t)
        return vo, ch, fe
    g = torch.Generator().manual_seed(0)
    for trial, (n1, n2) in enumerate([(50, 30), (2000, 1500), (1, 1), (5000, 5000), (300, 0)]):
        base = torch.randint(100, 150, (max(n1 // 4, 1), 3), generator=g)
        v1 = base[torch.randint(0, base.shape[0], (n1,), generator=g)] + \
            torch.randint(-2, 3, (n1, 3), generator=g)
        v2 = base[torch.randint(0, base.shape[0], (max(n2, 1),), generator=g)][:n2] + \
            torch.randint(-6, 7, (n2, 3), generator=g)
        if trial == 3:
            v1[:5] = torch.tensor([[255, 255, 255], [0, 0, 0], [255, 0, 128], [254, 255, 3],
                                   [128, 128, 128]])
        ref = host([v1, v2] if n2 else [v1])
        t = DeviceOctree(256)
        t.insert(v1)
        t.insert(v2)
        got = t.export()
        assert t.num_nodes() == ref[0].shape[0]
        for a, b in zip(ref, got):
            assert a.dtype == b.dtype and torch.equal(a, b), trial
