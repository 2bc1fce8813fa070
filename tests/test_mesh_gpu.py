"""Mesh extraction on the device: CUDA marching cubes bit-for-bit against the numpy
restatement (oracle/marching_cubes.py), the Vox-Fusion lattice / point queries against the
float64 restatement (oracle/vox_mesh.py), and get_mesh end to end for Co-SLAM, NICE-SLAM and
Vox-Fusion (device volume vs oracle queries; device mesh == oracle marching cubes run on the
DEVICE volume, so that near-zero cells cannot flip between two separately computed volumes)."""
import numpy as np
import pytest
import torch

from helpers import BOUND, coslam_pair, max_abs
from oracle import marching_cubes as omc
from oracle import vox_mesh

pytestmark = pytest.mark.gpu
f32 = np.float32


def _smooth(shape, seed, quantise=False):
    rng = np.random.default_rng(seed)
    axes = [np.linspace(-1, 1, k) for k in shape]
    X, Y, Z = np.meshgrid(*axes, indexing='ij')
    f = np.full(X.shape, 0.3)
    for _ in range(10):
        c = rng.uniform(-0.9, 0.9, 3)
        s = rng.uniform(0.1, 0.4)
        f -= rng.uniform(0.2, 1.0) * np.exp(-((X - c[0]) ** 2 + (Y - c[1]) ** 2 + (Z - c[2]) ** 2) / s ** 2)
    if quantise:
        f = np.round(f * 8) / 8
    return f.astype(f32)


def _mc_both(vals, level, spacing, shift=(0, 0, 0), scale=(1, 1, 1), origin=None, dev=None):
    from xrdslam_b200.mesher import marching_cubes
    o = None if origin is None else torch.from_numpy(origin).to(dev)
    v, f = marching_cubes(torch.from_numpy(vals).to(dev), level, spacing, shift, scale, o)
    torch.cuda.synchronize()
    ov, of = omc.marching_cubes(vals, level, spacing, shift, scale, origin)
    return v.cpu().numpy(), f.cpu().numpy(), ov, of


def _assert_bits(v, f, ov, of):
    assert v.shape == ov.shape and f.shape == of.shape
    assert np.array_equal(v.view(np.uint32), ov.view(np.uint32))
    assert np.array_equal(f, of)


def test_mc_noncubic_volume_bit_exact(cuda_dev):
    vals = _smooth((37, 29, 45), 0)[None]
    v, f, ov, of = _mc_both(vals, 0.0, (0.1, 0.07, 0.13), (-1.5, 2.25, 0.3), dev=cuda_dev)
    assert f.shape[0] > 1000
    _assert_bits(v, f, ov, of)
    # a level other than 0
    _assert_bits(*_mc_both(vals, -0.2, (1, 1, 1), dev=cuda_dev))


def test_mc_batch_of_small_volumes_bit_exact(cuda_dev):
    rng = np.random.default_rng(1)
    B, r = 300, 8
    vals = (rng.standard_normal((B, r, r, r)) * 0.3 + rng.uniform(-0.4, 0.4, (B, 1, 1, 1))).astype(f32)
    vals[:10] = np.abs(vals[:10]) + 0.1  # volumes without a crossing in the batch
    origin = rng.uniform(-3, 3, (B, 3)).astype(f32)
    s = 1.0 / (r - 1)
    v, f, ov, of = _mc_both(vals, 0.0, (s, s, s), (-0.5,) * 3, (0.2,) * 3, origin, dev=cuda_dev)
    assert f.shape[0] > 10000
    _assert_bits(v, f, ov, of)


def test_mc_values_exactly_at_level(cuda_dev):
    vals = _smooth((24, 31, 19), 2, quantise=True)[None]
    assert (vals == 0).sum() > 100
    v, f, ov, of = _mc_both(vals, 0.0, (0.5, 0.25, 0.125), dev=cuda_dev)
    _assert_bits(v, f, ov, of)


def test_mc_no_crossing(cuda_dev):
    for val in (1.0, -1.0, 0.0):
        v, f, ov, of = _mc_both(np.full((3, 6, 7, 5), val, f32), 0.0, (1, 1, 1), dev=cuda_dev)
        assert v.shape == (0, 3) and f.shape == (0, 3)


# ---- Vox-Fusion queries --------------------------------------------------------------------
def _vox_algo(dev, seed=0, emb_std=1.0):
    """VoxFusion with a map grown from synthetic 160x120 frames; embeddings spread so the sdf
    varies inside voxels and the sdf bias centred on the lattice values (a surface exists)."""
    from xrdslam_b200.synthetic import make_sequence
    from xrdslam_b200.voxfusion import VoxFusionConfig
    OFFSET = 25.6
    cam, poses, frames = make_sequence(2, width=160, height=120, offset=(OFFSET,) * 3)
    torch.manual_seed(seed)
    algo = VoxFusionConfig().setup(camera=cam, device=dev)
    model = algo.model
    H, W = cam.height, cam.width
    j, i = torch.meshgrid(torch.arange(H, dtype=torch.float32),
                          torch.arange(W, dtype=torch.float32), indexing='ij')
    dirs = torch.stack([(i - cam.cx) / cam.fx, -(j - cam.cy) / cam.fy, -torch.ones_like(i)], -1)
    for (rgb, depth), c2w in zip(frames, poses):
        c2w = torch.from_numpy(c2w)
        d = torch.from_numpy(depth)
        pts = (dirs * d[..., None])[d > 0].reshape(-1, 3)
        model.insert_points((pts @ c2w[:3, :3].T + c2w[:3, 3]).to(dev))
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        model.embeddings.copy_(torch.randn(model.embeddings.shape, generator=g) * emb_std)
        ids, _, _ = algo.surface_voxels()
        med = model.get_scores(ids, 4).median()
        model.decoder.sdf_out.bias[0] -= med
    return algo


def _map_cpu(model):
    ms = model.map_states
    return (ms['voxel_center_xyz'].cpu(), ms['voxel_vertex_idx'].cpu(),
            model.embeddings.detach().cpu())


def test_vox_lattice_and_point_queries_vs_oracle(cuda_dev):
    algo = _vox_algo(cuda_dev)
    model = algo.model
    ids, voxels, centres = algo.surface_voxels()
    assert ids.numel() > 50
    cen, vidx, emb = _map_cpu(model)
    vs = model.config.voxel_size
    for res in (8, 5):
        sdf = model.get_scores(ids, res)
        ref = vox_mesh.get_scores(_cpu_decoder(model), ids.cpu(), cen, vidx, emb, vs, res)
        assert sdf.shape == (ids.numel(), res, res, res)
        assert max_abs(sdf, ref) < 2e-5
        assert (sdf < 0).any() and (sdf > 0).any()
    # point mode: random points in random surface voxels (including their faces)
    g = torch.Generator().manual_seed(3)
    P = 20000
    pick = ids.cpu()[torch.randint(0, ids.numel(), (P,), generator=g)]
    xyz = cen[pick] + (torch.rand(P, 3, generator=g) - 0.5) * vs
    xyz[:100] = cen[pick[:100]] + 0.5 * vs
    rgb = model.eval_points(xyz.to(cuda_dev), pick.to(cuda_dev))
    ref = vox_mesh.eval_points(_cpu_decoder(model), xyz, pick, cen, vidx, emb, vs)
    assert rgb.shape == (P, 3) and max_abs(rgb, ref) < 2e-5


def _cpu_decoder(model):
    from oracle.voxfusion import VoxDecoder
    d = VoxDecoder()
    d.load_state_dict({k: v.detach().cpu() for k, v in model.decoder.state_dict().items()})
    return d


def test_voxfusion_extract_mesh_end_to_end(cuda_dev, tmp_path):
    from xrdslam_b200 import io_formats
    algo = _vox_algo(cuda_dev, seed=4)
    model = algo.model
    vs = model.config.voxel_size
    mesh = algo.get_mesh()
    assert mesh is not None and mesh.faces.shape[0] > 100
    ids, voxels, centres = algo.surface_voxels()
    sdf = model.get_scores(ids, 8)
    cen, vidx, emb = _map_cpu(model)
    assert max_abs(sdf, vox_mesh.get_scores(_cpu_decoder(model), ids.cpu(), cen, vidx, emb, vs, 8)) < 2e-5
    # the device mesh == the oracle's marching cubes on the device volume
    s = 1.0 / 7
    ov, of = omc.marching_cubes(sdf.cpu().numpy(), 0.0, (s, s, s), (-0.5,) * 3, (vs,) * 3,
                                centres.cpu().numpy())
    _assert_bits(mesh.vertices, mesh.faces, ov, of)
    # colours: the reference's O(V N) vertex -> voxel compare + float64 eval_points
    vox_cpu = voxels.cpu()
    hit = torch.cat([vox_mesh.vertex_voxels(torch.from_numpy(ov[i:i + 4096]), vox_cpu, vs)
                     for i in range(0, ov.shape[0], 4096)])
    assert (hit >= 0).float().mean() > 0.5
    col = torch.zeros(ov.shape[0], 3, dtype=torch.float64)
    m = hit >= 0
    col[m] = vox_mesh.eval_points(_cpu_decoder(model), torch.from_numpy(ov)[m],
                                  ids.cpu()[hit[m]], cen, vidx, emb, vs)
    ref_u8 = (col.clamp(0, 1) * 255).to(torch.uint8).numpy().astype(int)
    diff = np.abs(mesh.vertex_colors.astype(int) - ref_u8)
    assert diff.max() <= 1 and (diff == 0).mean() > 0.99
    assert np.array_equal(mesh.vertex_colors[~m.numpy()], np.zeros(((~m).sum().item(), 3), np.uint8))
    p = mesh.export(str(tmp_path / 'final_mesh.ply'))
    v2, f2, c2 = io_formats.read_ply(p)
    assert np.array_equal(v2, mesh.vertices) and np.array_equal(f2, mesh.faces)
    assert np.array_equal(c2, mesh.vertex_colors)


# ---- Mesher: Co-SLAM and NICE-SLAM ---------------------------------------------------------
def _check_mesher_run(algo, ora_raw, tol, tmp_path):
    """algo.get_mesh() against: oracle queries of the lattice (volume), oracle marching cubes
    of the device volume (mesh), oracle colours at the vertices, PLY round trip."""
    from xrdslam_b200 import io_formats
    mesh = algo.get_mesh()
    assert mesh is not None and mesh.faces.shape[0] > 100
    mesher = algo.mesher
    vol, xyz = mesher.query_volume(algo.model.query_fn, algo.device)
    n = vol.numel()
    pts = mesher.grid_points(xyz, 0, n, 'cpu')
    bb = mesher.bounding_box
    inside = ((pts[:, 0] < bb[0][1]) & (pts[:, 0] > bb[0][0]) & (pts[:, 1] < bb[1][1]) &
              (pts[:, 1] > bb[1][0]) & (pts[:, 2] < bb[2][1]) & (pts[:, 2] > bb[2][0]))
    assert 0 < int(inside.sum()) < n
    ref = torch.full((n,), 100.0, dtype=torch.float64)
    ref[inside] = ora_raw(pts[inside])[:, 3].double()
    assert max_abs(vol.reshape(-1), ref) < tol
    sp = [a[2] - a[1] for a in xyz]
    ov, of = omc.marching_cubes(vol.cpu().numpy(), mesher.config.level_set, sp, [a[0] for a in xyz])
    _assert_bits(mesh.vertices, mesh.faces, ov, of)
    vt = torch.from_numpy(ov)
    vin = ((vt[:, 0] < bb[0][1]) & (vt[:, 0] > bb[0][0]) & (vt[:, 1] < bb[1][1]) &
           (vt[:, 1] > bb[1][0]) & (vt[:, 2] < bb[2][1]) & (vt[:, 2] > bb[2][0]))
    col = torch.full((vt.shape[0], 3), 100.0, dtype=torch.float64)
    col[vin] = ora_raw(vt[vin], colour=True)[:, :3].double()
    ref_u8 = (col.clamp(0, 1) * 255).to(torch.uint8).numpy().astype(int)
    diff = np.abs(mesh.vertex_colors.astype(int) - ref_u8)
    assert diff.max() <= 1 and (diff == 0).mean() > 0.99
    p = mesh.export(str(tmp_path / 'final_mesh.ply'))
    v2, f2, c2 = io_formats.read_ply(p)
    assert np.array_equal(v2, mesh.vertices) and np.array_equal(f2, mesh.faces)
    assert np.array_equal(c2, mesh.vertex_colors)


def test_coslam_get_mesh_end_to_end(cuda_dev, tmp_path):
    from xrdslam_b200.coslam import CoSLAMConfig
    from xrdslam_b200.mesher import MesherConfig
    from xrdslam_b200.synthetic import make_camera
    ora, model = coslam_pair(cuda_dev)
    cfg = CoSLAMConfig(mapping_bound=BOUND.tolist(),
                       marching_cubes_bound=[[-3.3, 3.1], [-4.1, 2.8], [-2.4, 2.2]],
                       mesher=MesherConfig(resolution=40, points_batch_size=7000))
    algo = cfg.setup(camera=make_camera(160, 120), device=cuda_dev)
    algo.model = model
    bb = torch.as_tensor(BOUND, dtype=torch.float64)

    def ora_raw(p, colour=False):
        xn = (p.double() - bb[:, 0]) / (bb[:, 1] - bb[:, 0])
        with torch.no_grad():
            r = ora.query_color_sdf(xn)
        return torch.cat([torch.sigmoid(r[:, :3]), r[:, 3:]], 1) if colour else r
    _check_mesher_run(algo, ora_raw, 2e-5, tmp_path)


def test_nice_get_mesh_end_to_end(cuda_dev, tmp_path):
    from test_nice_gpu import BOUND as NICE_BOUND
    from test_nice_gpu import nice_pair
    from xrdslam_b200.mesher import MesherConfig
    from xrdslam_b200.nice_slam import NiceSLAMConfig
    from xrdslam_b200.synthetic import make_camera
    ora, model = nice_pair(cuda_dev)
    cfg = NiceSLAMConfig(mapping_bound=NICE_BOUND.tolist(),
                         marching_cubes_bound=[[-2.3, 2.1], [-1.9, 2.4], [-2.2, 1.8]],
                         mesher=MesherConfig(resolution=40, points_batch_size=9000))
    algo = cfg.setup(camera=make_camera(160, 120), device=cuda_dev)
    algo.model = model

    def ora_raw(p, colour=False):
        with torch.no_grad():
            return ora.decode(p.float(), 'color' if colour else 'fine')
    _check_mesher_run(algo, ora_raw, 2e-4, tmp_path)
