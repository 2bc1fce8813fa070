"""Corner pairs of the Co-SLAM hash table: trilinear corners k and k + 1 (x and x + 1) whose
entries form one 16-byte chunk (i1 == i0 ^ 1) get their table-gradient contributions from one
red.global.add.v4.f32, so the table gradient must be 16-byte aligned."""
import ctypes as C
import os
import shutil
import subprocess

import pytest
import torch

from helpers import coslam_pair, max_abs, rel_err

pytestmark = pytest.mark.gpu

XRD_E_SHAPE = -1


def _encode(model, table, x, feat, idx):
    from xrdslam_b200 import _cabi
    grid = model._grid_struct(table)
    return _cabi.lib().xrd_hashgrid_encode(C.byref(grid), x.data_ptr(), x.shape[0],
                                           feat.data_ptr() if feat is not None else None,
                                           idx.data_ptr() if idx is not None else None, None)


def _misaligned(t):
    """A copy of t whose data pointer is 8 bytes past a 16-byte boundary."""
    buf = torch.zeros(t.numel() + 4, dtype=t.dtype, device=t.device)
    v = buf[2:2 + t.numel()]
    assert v.data_ptr() % 16 == 8
    v.copy_(t.reshape(-1))
    return v.view_as(t)


def test_encode_corner_pairs_match_oracle(cuda_dev):
    """Points below 0 and above 1 (dense-level wrap) and both x parities on every hashed level:
    indices bit-exact, features within the fp32 tolerance; the features-only launch computes the
    same bits."""
    from oracle.tcnn_restated import hashgrid_indices
    from xrdslam_b200 import _cabi
    ora, model = coslam_pair(cuda_dev)
    g = torch.Generator().manual_seed(11)
    x = torch.rand(30000, 3, generator=g) * 1.6 - 0.3  # [-0.3, 1.3): in and outside the box
    idx_o, _ = hashgrid_indices(x, ora.embed_fn.table)
    xd = x.to(cuda_dev)
    table = model.embed_fn.params.detach()
    feat = torch.empty(x.shape[0], 32, device=cuda_dev)
    idx = torch.empty(x.shape[0], 16, 8, dtype=torch.int32, device=cuda_dev)
    _cabi.check('xrd_hashgrid_encode', _encode(model, table, xd, feat, idx))
    feat_only = torch.empty_like(feat)
    _cabi.check('xrd_hashgrid_encode', _encode(model, table, xd, feat_only, None))
    torch.cuda.synchronize()
    got = idx.cpu().to(torch.int64) & 0xFFFFFFFF
    assert torch.equal(got, idx_o)
    assert torch.equal(feat_only, feat)
    with torch.no_grad():
        f_o = ora.embed_fn(x)
    assert max_abs(feat, f_o) < 1e-6

    # the inputs exercise both kinds of corner pair on every level
    grid = model._grid_struct(table)
    i0, i1 = idx_o[:, :, 0::2], idx_o[:, :, 1::2]
    paired = i1 == (i0 ^ 1)
    outside = ((x < 0) | (x >= 1)).any(1)
    for l in range(16):
        assert paired[:, l].any() and (~paired[:, l]).any(), l
        if not grid.hashed[l]:
            assert (paired[outside, l]).any() and (~paired[outside, l]).any(), l
        else:  # x + 1 == x ^ 1 exactly for even x: about half of all pairs are one chunk
            assert 0.35 < paired[:, l].double().mean() < 0.65, l


def test_misaligned_table_gradient_rejected(cuda_dev):
    from xrdslam_b200 import _cabi
    _, model = coslam_pair(cuda_dev)
    lib = _cabi.lib()
    table = model.embed_fn.params.detach()
    cfg = model.config
    nb = lib.xrd_coslam_smoothness_workspace_bytes(cfg.trainging_smooth_pts)
    ws = torch.empty(nb, dtype=torch.uint8, device=cuda_dev)
    loss = torch.zeros(1, device=cuda_dev)
    r = (C.c_float * 6)(*([0.5] * 6))

    def smooth(tab, d_tab):
        grid = model._grid_struct(tab)
        return lib.xrd_coslam_smoothness(C.byref(grid), cfg.trainging_smooth_pts,
                                         cfg.trainging_smooth_vox, cfg.trainging_smooth_margin,
                                         1.0, r, loss.data_ptr(), d_tab.data_ptr(), 1.0,
                                         ws.data_ptr(), nb, None)
    assert smooth(table, _misaligned(torch.zeros_like(table))) == XRD_E_SHAPE
    d_ok = torch.zeros_like(table)
    assert smooth(table, d_ok) == 0
    # the table itself is read with 8-byte loads: no alignment beyond its element pair
    d_bad_tab = torch.zeros_like(table)
    assert smooth(_misaligned(table), d_bad_tab) == 0
    torch.cuda.synchronize()
    assert d_ok.abs().max() > 0
    assert rel_err(d_bad_tab, d_ok) < 1e-5  # the same sums, in another atomic order
    x = torch.rand(64, 3, device=cuda_dev)
    feat = torch.empty(64, 32, device=cuda_dev)
    assert _encode(model, _misaligned(table), x, feat, None) == 0


def test_table_gradient_scatters_use_red_v4():
    """k_fused, k_fused_g and k_smooth_bwd scatter paired corners with red.v4, the rest with red.v2."""
    from xrdslam_b200.build import LIB_PATH
    cuobjdump = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(cuobjdump):
        pytest.skip('cuobjdump not available')
    sass = subprocess.run([cuobjdump, '-sass', LIB_PATH], capture_output=True, text=True).stdout
    funcs = {}
    name = None
    for line in sass.splitlines():
        s = line.strip()
        if s.startswith('Function :'):
            name = s.split(':', 1)[1].strip()
            funcs[name] = []
        elif name:
            funcs[name].append(s)
    # gradient instantiations (BWD = true; their listing includes the non-inlined hash backward)
    # and the smoothness backward
    for kern in ('7k_fusedILb1', '9k_fused_gILb1', 'k_smooth_bwd'):
        bodies = ['\n'.join(b) for n, b in funcs.items() if kern in n]
        assert bodies, kern
        for body in bodies:
            assert 'REDG.E.ADD.F32x4' in body, kern
            assert 'REDG.E.ADD.F32x2' in body, kern
