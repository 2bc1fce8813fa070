"""The Hopper-native GEMM (csrc/mlp.cu: wgmma.mma_async tf32 + TMA + mbarrier, 3xTF32)
against float64 matmul and against the mma.sync path, on the shapes of the Vox-Fusion decoder and
the Point-SLAM colour trunk (forward and transposed-weight backward GEMMs, ragged N, masks)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

ACT = {0: lambda x: x, 1: torch.relu, 3: torch.sigmoid}


def run(dev, M, N, K, transA, act, mode, mask=False, addend=False, seed=0):
    from xrdslam_b200 import _cabi
    lib = _cabi.lib()
    g = torch.Generator().manual_seed(seed)
    A = torch.randn((K, M) if transA else (M, K), generator=g) / K ** 0.5
    Np = (N + 63) // 64 * 64
    B = torch.randn(K, Np, generator=g)
    bias = torch.randn(M, generator=g) * 0.1
    mk = torch.randn(M, Np, generator=g) if mask else None
    ad = torch.randn(M, Np, generator=g) if addend else None
    d = lambda t: t.to(dev).contiguous() if t is not None else None
    A_d, B_d, b_d, mk_d, ad_d = d(A), d(B), d(bias), d(mk), d(ad)
    C = torch.full((M, Np), float('nan'), device=dev)
    _cabi.check('mode', lib.xrd_debug_gemm_mode(mode))
    try:
        st = lib.xrd_debug_gemm(M, N, K, A_d.data_ptr(), A.shape[1], int(transA), B_d.data_ptr(), Np,
                                C.data_ptr(), Np, b_d.data_ptr(), act,
                                mk_d.data_ptr() if mask else None, Np,
                                ad_d.data_ptr() if addend else None, Np, None)
        _cabi.check('xrd_debug_gemm', st)
        torch.cuda.synchronize()
    finally:
        lib.xrd_debug_gemm_mode(1)
    Am = (A.t() if transA else A).double()
    ref = ACT[act](Am @ B.double()[:, :N] + bias.double()[:, None])
    if mask:
        ref = torch.where(mk[:, :N] > 0, ref, torch.zeros_like(ref))
    if addend:
        ref = ref + ad[:, :N].double()
    return C.cpu()[:, :N].double(), ref, C.cpu()[:, N:]


@pytest.mark.parametrize('M,N,K,transA,act', [
    (128, 4096, 128, 0, 1),      # trunk layer
    (128, 5000, 16, 0, 1),       # vox layer 0 (K = 16, ragged N)
    (128, 1111, 144, 0, 1),      # colour layer: K = 144 -> two-stage pipeline
    (128, 2048, 129, 1, 0),      # backward through sdf_out (transposed weights, K = 129)
    (144, 3000, 128, 1, 0),      # 144 rows = 128 (wgmma) + 16 (mma.sync)
    (64, 1024, 128, 0, 3),       # M < 128 (zero-padded rows)
    (32, 3000, 128, 0, 0),       # Point-SLAM 128 -> 32 neighbour layer
    (128, 150000, 128, 0, 1),    # benchmark-sized point count
])
def test_gemm_t5_matches_float64(cuda_dev, M, N, K, transA, act):
    got, ref, pad = run(cuda_dev, M, N, K, transA, act, mode=1)
    err = (got - ref).abs().max().item()
    assert err < 5e-6 * max(1.0, ref.abs().max().item()), err   # fp32-level (3xTF32)
    assert torch.isnan(pad).all()                               # columns >= N untouched
    legacy, _, _ = run(cuda_dev, M, N, K, transA, act, mode=3)
    assert (got - legacy).abs().max().item() < 1e-5 * max(1.0, ref.abs().max().item())


def test_gemm_t5_mask_and_addend(cuda_dev):
    got, ref, _ = run(cuda_dev, 128, 3333, 128, 1, 0, mode=1, mask=True, addend=True)
    assert (got - ref).abs().max().item() < 5e-6 * max(1.0, ref.abs().max().item())


def test_gemm_t5_sass_is_hopper_native():
    """The shipped library contains warpgroup MMAs, TMA loads and mbarrier waits (SASS mnemonics)."""
    import os
    import shutil
    import subprocess
    from xrdslam_b200.build import LIB_PATH
    cuobjdump = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(cuobjdump):
        pytest.skip('cuobjdump not available')
    sass = subprocess.run([cuobjdump, '-sass', LIB_PATH], capture_output=True, text=True).stdout
    for mn in ('HGMMA.64x128x8.F32.TF32', 'UTMALDG', 'SYNCS.PHASECHK'):
        assert mn in sass, mn


def test_gemm_t5_softplus_epilogue(cuda_dev):
    """Point-SLAM trunk epilogue: nn.Softplus(beta=100) in the wgmma kernel."""
    from xrdslam_b200 import _cabi
    lib = _cabi.lib()
    g = torch.Generator().manual_seed(3)
    M, N, K = 128, 4096 + 300, 128
    Np = (N + 63) // 64 * 64
    A = (torch.randn(M, K, generator=g) / K ** 0.5 * 0.05).to(cuda_dev)   # pre-activations ~ +-0.05:
    B = torch.randn(K, Np, generator=g).to(cuda_dev)                      # both softplus branches
    bias = (torch.randn(M, generator=g) * 0.01).to(cuda_dev)
    C = torch.empty(M, Np, device=cuda_dev)
    _cabi.check('gemm', lib.xrd_debug_gemm(M, N, K, A.data_ptr(), K, 0, B.data_ptr(), Np, C.data_ptr(), Np,
                                           bias.data_ptr(), 2, None, Np, None, Np, None))
    torch.cuda.synchronize()
    pre = A.double() @ B.double()[:, :N] + bias.double()[:, None]
    ref = torch.nn.functional.softplus(pre, beta=100, threshold=20)
    assert (pre * 100 > 20).any() and (pre * 100 < -5).any()
    assert (C[:, :N].double() - ref).abs().max().item() < 2e-6


def test_gemm_t5_act_out_and_accumulate(cuda_dev):
    """act_out receives the masked activation before the addend; accumulate adds into C."""
    from xrdslam_b200 import _cabi
    lib = _cabi.lib()
    g = torch.Generator().manual_seed(4)
    M, N, K = 96, 2048 + 77, 64
    Np = (N + 63) // 64 * 64
    d = lambda t: t.to(cuda_dev).contiguous()
    A, B = d(torch.randn(M, K, generator=g) / K ** 0.5), d(torch.randn(K, Np, generator=g))
    bias, mk, ad = d(torch.randn(M, generator=g) * 0.1), d(torch.randn(M, Np, generator=g)), \
        d(torch.randn(M, Np, generator=g))
    c0 = torch.randn(M, Np, generator=g)
    for mode in (1, 3):
        C, AO = d(c0.clone()), torch.full((M, Np), float('nan'), device=cuda_dev)
        lib.xrd_debug_gemm_mode(mode)
        try:
            _cabi.check('gemm', lib.xrd_debug_gemm_ex(
                M, N, K, A.data_ptr(), K, 0, B.data_ptr(), Np, C.data_ptr(), Np, bias.data_ptr(), 1,
                mk.data_ptr(), Np, ad.data_ptr(), Np, AO.data_ptr(), Np, 1, None))
            torch.cuda.synchronize()
        finally:
            lib.xrd_debug_gemm_mode(1)
        act = torch.relu(A.double() @ B.double()[:, :N] + bias.double()[:, None])
        act = torch.where(mk[:, :N] > 0, act, torch.zeros_like(act))
        e_ao = (AO[:, :N].double() - act).abs().max().item()
        assert e_ao < 5e-6 * max(1.0, act.abs().max().item()), ('act_out', mode, e_ao)
        ref = c0[:, :N].double().to(cuda_dev) + act + ad[:, :N].double()
        e_c = (C[:, :N].double() - ref).abs().max().item()
        assert e_c < 5e-6 * max(1.0, ref.abs().max().item()), ('C', mode, e_c)
        assert torch.equal(C[:, N:].cpu(), c0[:, N:]), ('pad', mode)   # columns >= N untouched


@pytest.mark.parametrize('nA,nB,P,masked', [
    (128, 128, 20000, False),    # trunk layer
    (144, 128, 7777, False),     # colour layer: two passes over A (128 + 16 rows), ragged P
    (16, 128, 5001, True),       # first layer, relu mask words
    (128, 129, 9000, False),     # 129 rows: a 128-row group and a 1-row group
    (128, 3, 6000, False),       # rgb head
    (32, 32, 100, True),         # one short chunk
])
def test_weight_gradient_kernels_match_float64(cuda_dev, nA, nB, P, masked):
    """dW[j][i] = sum_p B[j][p] A[i][p] (+ bias): tensor-core kernel (mode 1) and SIMT kernel
    (mode 0) against float64, accumulating into a non-zero output."""
    from xrdslam_b200 import _cabi
    lib = _cabi.lib()
    g = torch.Generator().manual_seed(nA * 1000 + nB)
    Pp = (P + 63) // 64 * 64
    A = torch.randn(nA, Pp, generator=g)
    B = torch.randn(nB, Pp, generator=g)
    A[:, P:] = float('nan')    # padding must never be read into the sums
    B[:, P:] = float('nan')
    mask = None
    Bm = B[:, :P].double()
    if masked:
        mask = torch.randint(0, 2 ** 31, ((nB + 31) // 32, P), generator=g, dtype=torch.int64).to(torch.int32)
        bits = torch.stack([(mask[j // 32].long() >> (j % 32)) & 1 for j in range(nB)]).double()
        Bm = Bm * bits
    ref = Bm @ A[:, :P].double().t()
    ref_b = Bm.sum(1)
    out0 = torch.randn(nB, nA, generator=g)
    b0 = torch.randn(nB, generator=g)
    # fp32 accumulation of P unit-variance products (|dW| ~ sqrt(P); the tensor-core accumulator
    # truncates): 4e-5 relative to that scale; one dropped or doubled point would be ~ 1
    tol = 4e-5 * P ** 0.5
    for mode in (1, 0):
        out, bias = out0.clone().to(cuda_dev), b0.clone().to(cuda_dev)
        A_d, B_d = A.to(cuda_dev), B.to(cuda_dev)
        m_d = mask.to(cuda_dev) if masked else None
        lib.xrd_debug_gemm_mode(mode)
        try:
            _cabi.check('dw', lib.xrd_debug_dw(nA, nB, P, Pp, A_d.data_ptr(), B_d.data_ptr(),
                                               m_d.data_ptr() if masked else None, out.data_ptr(),
                                               bias.data_ptr(), None))
            torch.cuda.synchronize()
        finally:
            lib.xrd_debug_gemm_mode(1)
        err = (out.cpu().double() - out0.double() - ref).abs().max().item()
        assert err < tol, (mode, err)
        errb = (bias.cpu().double() - b0.double() - ref_b).abs().max().item()
        assert errb < tol, (mode, errb)
