"""Every C-ABI entry point that takes a workspace rejects one byte less than its
xrd_*_workspace_bytes with XRD_E_WORKSPACE before it launches anything, for several shapes and
both gradient settings.  This is what catches a workspace size and a workspace carve that
disagree.  It runs on the GPU because cub's temp-storage queries need a device."""
import ctypes as C

import pytest
import torch

from xrdslam_b200 import _cabi

pytestmark = pytest.mark.gpu
E_WORKSPACE = -3


@pytest.fixture
def env(cuda_dev):
    # every data pointer aims into one zeroed buffer: a call that launched would change it
    buf = torch.zeros(1 << 20, dtype=torch.float32, device=cuda_dev)
    yield _cabi.lib(), buf.data_ptr(), torch.cuda.current_stream().cuda_stream
    torch.cuda.synchronize()
    assert not buf.any()


def _filled(cls, p, **kw):
    """cls with every pointer field set to p (pointer arrays too), then the keyword fields."""
    s = cls()
    for name, t in cls._fields_:
        if t is C.c_void_p:
            setattr(s, name, p)
        elif issubclass(t, C.Array) and t._type_ is C.c_void_p:
            getattr(s, name)[:] = [p] * t._length_
    for k, v in kw.items():
        setattr(s, k, v)
    return s


def _ref(s):
    return C.byref(s) if s is not None else None


@pytest.mark.parametrize('shape', [(1, 5, 6, 7), (4, 17, 9, 33)])
def test_mesh_mc(env, shape):
    lib, p, s = env
    nb = lib.xrd_mesh_mc_workspace_bytes(*shape)
    affine = _filled(_cabi.XrdMeshAffine, p)
    assert lib.xrd_mesh_mc_count(p, *shape, 0.0, p, p, nb - 1, s) == E_WORKSPACE
    assert lib.xrd_mesh_mc_emit(p, *shape, 0.0, C.byref(affine), p, p, p, nb - 1, s) == E_WORKSPACE


@pytest.mark.parametrize('V,F', [(10, 7), (1000, 3000)])
def test_cull(env, V, F):
    lib, p, s = env
    nb = lib.xrd_cull_workspace_bytes(V, F)
    assert lib.xrd_cull_count(p, V, p, F, p, p, nb - 1, s) == E_WORKSPACE
    assert lib.xrd_cull_emit(p, p, 3, V, p, F, p, p, p, p, nb - 1, s) == E_WORKSPACE


def _tsdf_params():
    return _cabi.XrdTsdfParams(voxel_length=0.04, sdf_trunc=0.12, depth_trunc=3.0, fx=500.0,
                               fy=500.0, cx=320.0, cy=240.0, stride=4)


@pytest.mark.parametrize('K,H,W', [(1, 48, 64), (4, 480, 640)])
def test_tsdf_alloc(env, K, H, W):
    lib, p, s = env
    P = _tsdf_params()
    nb = lib.xrd_tsdf_alloc_workspace_bytes(K, H, W, P.stride)
    assert lib.xrd_tsdf_alloc_count(p, p, K, H, W, C.byref(P), p, p, nb - 1, s) == E_WORKSPACE
    assert lib.xrd_tsdf_alloc_emit(K, H, W, C.byref(P), 10, p, p, p, nb - 1, s) == E_WORKSPACE


@pytest.mark.parametrize('n_blocks', [1, 37])
def test_tsdf_mc(env, n_blocks):
    lib, p, s = env
    P = _tsdf_params()
    nb = lib.xrd_tsdf_mc_workspace_bytes(n_blocks)
    assert lib.xrd_tsdf_mc_count(p, n_blocks, p, p, p, p, nb - 1, s) == E_WORKSPACE
    assert lib.xrd_tsdf_mc_emit(p, n_blocks, p, p, C.byref(P), p, p, p, p, nb - 1,
                                s) == E_WORKSPACE


@pytest.mark.parametrize('n', [1, 100000])
def test_eval_surface_and_reductions(env, n):
    lib, p, s = env
    nb = lib.xrd_eval_surface_workspace_bytes(n)
    assert lib.xrd_eval_surface_prepare(p, 3, p, n, p, p, p, p, nb - 1, s) == E_WORKSPACE
    nb = lib.xrd_eval_reduce_workspace_bytes(n)
    assert lib.xrd_eval_dist_stats(p, n, 0.05, p, p, nb - 1, s) == E_WORKSPACE
    assert lib.xrd_eval_icp_stats(p, p, p, p, n, p, p, nb - 1, s) == E_WORKSPACE


@pytest.mark.parametrize('n', [100, 50000])
def test_nn_build(env, n):
    lib, p, s = env
    I = _cabi.XrdNnIndex()
    lo, hi = (C.c_double * 3)(0, 0, 0), (C.c_double * 3)(2, 3, 1)
    _cabi.check('xrd_nn_layout', lib.xrd_nn_layout(n, lo, hi, C.byref(I)))
    I.cell_ptr = I.occ = I.sorted = p
    nb = lib.xrd_nn_build_workspace_bytes(C.byref(I))
    assert lib.xrd_nn_build(p, C.byref(I), p, nb - 1, s) == E_WORKSPACE


@pytest.mark.parametrize('with_grads', [0, 1])
@pytest.mark.parametrize('R', [64, 4096])
def test_coslam_step(env, R, with_grads):
    lib, p, s = env
    S = 43
    rays = _filled(_cabi.XrdRays, p, n_rays=R)
    grid = _filled(_cabi.XrdHashGrid, p)
    mlp = _filled(_cabi.XrdCoslamMlp, p)
    cfg = _filled(_cabi.XrdCoslamCfg, p, n_samples=S, n_sample_d=32, n_range_d=11)
    out = _filled(_cabi.XrdCoslamOut, p)
    grads = _filled(_cabi.XrdCoslamGrads, p) if with_grads else None
    nb = lib.xrd_coslam_workspace_bytes(R, S)
    assert lib.xrd_coslam_step(C.byref(rays), C.byref(grid), C.byref(mlp), C.byref(cfg), p,
                               C.byref(out), _ref(grads), p, nb - 1, s) == E_WORKSPACE


@pytest.mark.parametrize('with_grads', [0, 1])
@pytest.mark.parametrize('sample_points', [3, 32])
def test_coslam_smoothness(env, sample_points, with_grads):
    lib, p, s = env
    grid = _filled(_cabi.XrdHashGrid, p)
    d_table = p if with_grads else None
    nb = lib.xrd_coslam_smoothness_workspace_bytes(sample_points)
    rand = C.cast(p, _cabi.fp)
    assert lib.xrd_coslam_smoothness(C.byref(grid), sample_points, 0.1, 0.1, 1.0, rand, p,
                                     d_table, 1.0, p, nb - 1, s) == E_WORKSPACE
    assert lib.xrd_coslam_smoothness_dev(C.byref(grid), sample_points, 0.1, 0.1, 1.0, p, p,
                                         d_table, 1.0, p, nb - 1, s) == E_WORKSPACE


def _nice_decoders(p):
    return (_cabi.XrdNiceDecoder * 3)(*[_filled(_cabi.XrdNiceDecoder, p, c_dim=c, n_out=o)
                                        for c, o in ((32, 1), (64, 1), (32, 4))])


@pytest.mark.parametrize('with_grads', [0, 1])
@pytest.mark.parametrize('R,stage', [(200, 0), (1000, 2)])
def test_nice_step(env, R, stage, with_grads):
    lib, p, s = env
    rays = _filled(_cabi.XrdRays, p, n_rays=R)
    grids = (_cabi.XrdNiceGrid * 3)(*[_filled(_cabi.XrdNiceGrid, p, nx=4, ny=5, nz=6)] * 3)
    cfg = _filled(_cabi.XrdNiceCfg, p, stage=stage, is_mapping=1, n_samples=32, n_surface=16)
    out = _filled(_cabi.XrdNiceOut, p)
    dc = _filled(_cabi.XrdNiceDecoderGrads, p)
    grads = _filled(_cabi.XrdNiceGrads, p, d_color=C.pointer(dc)) if with_grads else None
    nb = lib.xrd_nice_workspace_bytes(R, 48, with_grads)
    assert lib.xrd_nice_step(C.byref(rays), grids, _nice_decoders(p), C.byref(cfg),
                             C.byref(out), _ref(grads), p, nb - 1, s) == E_WORKSPACE


@pytest.mark.parametrize('with_grads', [0, 1])
@pytest.mark.parametrize('R', [100, 1000])
def test_nice_coarse_step(env, R, with_grads):
    lib, p, s = env
    S = 32
    rays = _filled(_cabi.XrdRays, p, n_rays=R)
    grid = _filled(_cabi.XrdNiceGrid, p, nx=4, ny=5, nz=6)
    dec = _filled(_cabi.XrdNiceCoarseDecoder, p)
    cfg = _filled(_cabi.XrdNiceCoarseCfg, p, n_samples=S)
    out = _filled(_cabi.XrdNiceOut, p)
    nb = lib.xrd_nice_coarse_workspace_bytes(R, S, with_grads)
    assert lib.xrd_nice_coarse_step(C.byref(rays), C.byref(grid), C.byref(dec), C.byref(cfg),
                                    C.byref(out), p, p, p, with_grads, p, nb - 1,
                                    s) == E_WORKSPACE


@pytest.mark.parametrize('n', [10, 10000])
def test_nice_query(env, n):
    lib, p, s = env
    grids = (_cabi.XrdNiceGrid * 3)(*[_filled(_cabi.XrdNiceGrid, p, nx=4, ny=5, nz=6)] * 3)
    lo, hi = (C.c_double * 3)(0, 0, 0), (C.c_double * 3)(1, 1, 1)
    nb = lib.xrd_nice_query_workspace_bytes(n)
    assert lib.xrd_nice_query(p, n, grids, _nice_decoders(p), lo, hi, 2, p, p, nb - 1,
                              s) == E_WORKSPACE


@pytest.mark.parametrize('n,res', [(10, 0), (5000, 0), (3, 8)])
def test_voxfusion_query(env, n, res):
    lib, p, s = env
    vmap = _filled(_cabi.XrdVoxMap, p)
    dec = _filled(_cabi.XrdVoxDecoder, p)
    xyz = rgb = None if res else p
    lin = p if res else None
    nb = lib.xrd_voxfusion_query_workspace_bytes(n * res ** 3 if res else n)
    assert lib.xrd_voxfusion_query(C.byref(vmap), C.byref(dec), 0.2, n, p, res, lin, xyz, p,
                                   rgb, p, nb - 1, s) == E_WORKSPACE


@pytest.mark.parametrize('with_grads', [0, 1])
@pytest.mark.parametrize('R,Pn', [(5, 1024), (1024, 50000)])
def test_voxfusion_render(env, R, Pn, with_grads):
    lib, p, s = env
    rays = _filled(_cabi.XrdRays, p, n_rays=R)
    vmap = _filled(_cabi.XrdVoxMap, p)
    march = _filled(_cabi.XrdVoxMarch, p)
    mcfg = _cabi.XrdVoxMarchCfg(max_samples=64)
    dec = _filled(_cabi.XrdVoxDecoder, p)
    cfg = _cabi.XrdVoxRenderCfg(n_points=Pn, s_max=64, n_hit_rays=R)
    out = _filled(_cabi.XrdVoxOut, p)
    dd = _filled(_cabi.XrdVoxDecoderGrads, p)
    grads = _filled(_cabi.XrdVoxGrads, p, d_decoder=C.pointer(dd)) if with_grads else None
    nb = lib.xrd_voxfusion_render_workspace_bytes(R, Pn, with_grads)
    assert lib.xrd_voxfusion_render(C.byref(rays), C.byref(vmap), C.byref(march), C.byref(mcfg),
                                    C.byref(dec), C.byref(cfg), C.byref(out), _ref(grads), p,
                                    nb - 1, s) == E_WORKSPACE


@pytest.mark.parametrize('table_size', [1024, 1 << 20])
def test_pointslam_knn_build(env, table_size):
    lib, p, s = env
    nb = lib.xrd_pointslam_knn_build_workspace_bytes(table_size)
    assert lib.xrd_pointslam_knn_build(p, 100, 0.1, table_size, p, p, p, p, nb - 1,
                                       s) == E_WORKSPACE


@pytest.mark.parametrize('with_grads', [0, 1])
@pytest.mark.parametrize('R,stage', [(100, 0), (5000, 1)])
def test_pointslam_step(env, R, stage, with_grads):
    lib, p, s = env
    S = 5
    rays = _filled(_cabi.XrdRays, p, n_rays=R)
    index = _filled(_cabi.XrdPointIndex, p, n_points=100, cell=0.1, table_size=1024)
    feats = _filled(_cabi.XrdPointFeats, p)
    dec = _filled(_cabi.XrdNiceDecoder, p, c_dim=32, n_out=1)
    cdec = _filled(_cabi.XrdPointColorDecoder, p)
    cfg = _filled(_cabi.XrdPointCfg, p, stage=stage, is_mapping=1, n_surface=S)
    out = _filled(_cabi.XrdPointOut, p)
    cg = _filled(_cabi.XrdPointColorDecoderGrads, p)
    grads = _filled(_cabi.XrdPointGrads, p, color=C.pointer(cg)) if with_grads else None
    nb = lib.xrd_pointslam_workspace_bytes(R, S, stage, with_grads)
    assert lib.xrd_pointslam_step(C.byref(rays), C.byref(index), C.byref(feats), C.byref(dec),
                                  C.byref(cdec), C.byref(cfg), C.byref(out), _ref(grads), p,
                                  nb - 1, s) == E_WORKSPACE
