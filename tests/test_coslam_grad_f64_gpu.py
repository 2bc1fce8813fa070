"""Co-SLAM fused step (both kernels, all three precision modes) against the float64 replay of
oracle/coslam_f64.py: d_table per hash level and per entry, every weight element, every ray,
every loss term.  The whole-tensor relative L2 of test_coslam_gpu.py lets a fine hash level be
wrong by a quarter at precision 1, and a single ray by almost anything; these checks do not.

Gates (per precision mode): the worst ratio over all cases below, observed on one H100 80GB
HBM3 (identical for the tile and the grouped kernel), times about 4, and never above the
ceiling at which the mutations of test_coslam_f64_reference_cpu.py stop being flagged (the
level gate of mode 1 stays below the 1e-2 of a level scaled by 1.01):

  mode  level    entry    weight   ray      loss     rays with another sdf sign change
  0     2.0e-6   4.2e-7   3.1e-8   7.6e-9   1.4e-6   1 of 4097
  1     2.4e-3   3.2e-4   4.1e-5   1.0e-5   1.4e-6   1 of 4097
  2     1.8e-2   4.7e-4   4.6e-5   9.9e-6   3.8e-4   9 of 4096

Smoothness term (k_smooth_bwd), per lattice of LATTICES and margin 0.05.  T is the most
(point, corner) terms that land on one table entry, at level 0 .. level 15: the gather adds them
one atomic at a time, the box path sums at most that many per vertex in one thread.  The entry
gate is 2 (T + slabs + 16) 2^-24 of the bound A per level; the level and loss gates are about 4x
the worst observed over the automatic and the gather path, both entry points and the scaled
accumulation (H100 80GB HBM3, 700 W).  The mapping configuration p32 keeps its earlier gates on
the automatic path (level 1e-6, entry 2e-6, loss 3e-8).

  lattice   pts voxel      T           entry gate      entry  level (auto, gather)  gate   loss     gate
  p32        32 0.1      432..13  5.4e-05..4.4e-06  4.9e-07  9.7e-08 3.1e-07  1.3e-06  1.9e-08  7.5e-08
  p3          3 0.1        8..1   3.0e-06..2.1e-06  2.3e-07  1.7e-07 2.0e-07  8.0e-07  7.9e-08  3.2e-07
  p5          5 0.1       64..2   9.7e-06..2.3e-06  3.9e-07  1.2e-07 2.4e-07  9.6e-07  5.0e-08  2.0e-07
  p6          6 0.1      125..2   1.7e-05..2.4e-06  2.8e-07  1.1e-07 1.8e-07  7.4e-07  4.0e-08  1.6e-07
  p30        30 0.1      432..11  5.4e-05..4.2e-06  5.3e-07  1.1e-07 2.8e-07  1.2e-06  5.4e-08  2.2e-07
  p33        33 0.1      432..14  5.4e-05..4.5e-06  3.9e-07  1.0e-07 3.0e-07  1.3e-06  3.6e-08  1.5e-07
  p35        35 0.1      432..15  5.4e-05..4.8e-06  4.5e-07  1.0e-07 3.1e-07  1.3e-06  3.0e-08  1.3e-07
  p60        60 0.03   15660..69  1.9e-03..1.2e-05  2.6e-07  1.6e-07 1.6e-06  6.5e-06  5.7e-08  2.3e-07
  p76_v015   76 0.015 114480..201 1.4e-02..2.8e-05  2.7e-07  1.2e-06 4.3e-06  1.8e-05  2.4e-08  9.6e-08
  p76_v05    76 0.05    3456..76  4.2e-04..1.3e-05  3.5e-07  7.6e-07 7.5e-07  3.1e-06  1.6e-08  6.6e-08
  p40_v15    40 0.15     288..21  3.7e-05..5.6e-06  4.3e-07  1.1e-07 2.2e-07  8.8e-07  3.8e-08  1.6e-07
  p32_edge   32 0.1      432..13  5.4e-05..4.4e-06  5.6e-07  9.8e-08 2.6e-07  1.1e-06  3.2e-08  1.3e-07

The worst entry error stays near 5e-7 of A on every lattice, far inside the count-derived
gates: the bound assumes every addition rounds at the size of the whole sum.

The fp32 CPU oracle itself stays within level 4.5e-7, entry 1.7e-7, weight 1e-9, ray 3e-9,
loss 1e-7 of float64.
"""
import numpy as np
import pytest
import torch

from helpers import make_rays

pytestmark = pytest.mark.gpu

# ReLU ambiguity threshold |pre| / sum|terms| for the candidate's forward arithmetic:
# 3xTF32 (modes 0 and 1) rounds like fp32, plain TF32 (mode 2) has a 10-bit mantissa
AMB = {0: 1e-5, 1: 1e-5, 2: 2e-3}
GATES = {
    0: dict(level=1e-5, entry=2e-6, weight=1.5e-7, ray=3e-8, loss=6e-6),
    1: dict(level=8e-3, entry=1.3e-3, weight=2e-4, ray=4e-5, loss=6e-6),
    2: dict(level=8e-2, entry=2e-3, weight=2e-4, ray=4e-5, loss=1.5e-3),
}
KERNELS = {-1: 'tile', -2: 'grouped'}
LOSS_SCALE = (0.5, 2.0, 1.5, 0.25)
DEPTH_TRUNC = 4.0   # cam_depth_trunc of the depth-edge batch


def _batch(name):
    """(R, table amplitude, rays_o, rays_d, target_s, target_d, noise, loss_scale, depth_trunc)"""
    if name == 'bench':          # the benchmark's mapping batch: 4096 rays, table amplitude 0.1
        R, amp = 4096, 0.1
    elif name == 'tail':         # one ray in the last unit
        R, amp = 4097, 0.1
    elif name == 'groups':       # one unit more than 3 groups x 132 SMs (+ non-unit loss scale)
        R, amp = 793, 0.3
    elif name == 'one':
        R, amp = 1, 0.3
    elif name in ('outside', 'depth_edges', 'scaled'):
        R, amp = 1024, 0.3
    ro, rd, ts, td, noise = make_rays(R, seed=R + len(name))
    if name == 'outside':        # most samples outside the box: dense-level wrap, both pair kinds
        ro = ro * 12
    trunc = 100.0
    if name == 'depth_edges':
        trunc = DEPTH_TRUNC
        td[0::6] = 0
        td[1::6] = DEPTH_TRUNC
        td[2::6] = DEPTH_TRUNC + 0.7
    scale = LOSS_SCALE if name == 'scaled' else (1.0, 1.0, 1.0, 1.0)
    return R, amp, ro, rd, ts, td, noise, scale, trunc


CASES = ('bench', 'tail', 'groups', 'one', 'outside', 'depth_edges', 'scaled')


class _Refs:
    """Float64 replays, computed once per batch and shared by every kernel / precision mode."""
    def __init__(self, dev):
        self.dev = dev
        self.cache = {}

    def get(self, name):
        if name not in self.cache:
            from helpers import coslam_pair
            from oracle.coslam_f64 import replay_step
            R, amp, ro, rd, ts, td, noise, scale, trunc = _batch(name)
            ora, model = coslam_pair(self.dev, table_amp=amp, cam_depth_trunc=trunc)
            ora.cfg.depth_trunc = trunc
            with torch.no_grad():
                z = ora.sample_z(R, td, noise)
            ref = replay_step(ora, ro, rd, ts, td, z, loss_scale=scale, device=self.dev)
            self.cache[name] = dict(ora=ora, model=model, ref=ref, z=z, scale=scale,
                                    inp=(ro, rd, ts, td, noise))
        return self.cache[name]


@pytest.fixture(scope='module')
def refs(cuda_dev):
    return _Refs(cuda_dev)


def run_case(refs, name, kernel, mode, map_grads=True):
    """One fused step through JointEncoding._launch -> compare() report."""
    from oracle.coslam_f64 import compare
    c = refs.get(name)
    model, dev = c['model'], refs.dev
    model.config.rays_per_tile = kernel
    model.config.precision = mode
    ro, rd, ts, td, noise = (t.to(dev) for t in c['inp'])
    w = model._weights()
    out, g = model._launch(ro, rd, model.embed_fn.params, *w, ts, td, noise, with_grads=True,
                           need_ray_grads=True, loss_scale=list(c['scale']), map_grads=map_grads)
    torch.cuda.synchronize()
    assert torch.equal(out['z_vals'].cpu(), c['z'])            # the replay's fp32 input
    for k, v in g.items():
        if v is not None:
            assert bool(torch.isfinite(v).all()), k
    cand = dict(g, losses=out['losses'])
    return compare(c['ref'], cand, AMB[mode], cand_sdf=out['raw'][..., 3])


@pytest.mark.parametrize('mode', [0, 1, 2])
@pytest.mark.parametrize('kernel', [-1, -2])
@pytest.mark.parametrize('name', CASES)
def test_fused_step_vs_float64(refs, name, kernel, mode):
    from oracle.coslam_f64 import failures
    rep = run_case(refs, name, kernel, mode)
    # a handful of rays may see another sdf sign change; they are left out, not the batch
    assert rep['n_flip_rays'] <= max(2, refs.get(name)['ref']['R'] // 200), rep['n_flip_rays']
    bad = failures(rep, GATES[mode])
    assert not bad, (name, KERNELS[kernel], mode, bad)


@pytest.mark.parametrize('mode', [0, 1, 2])
@pytest.mark.parametrize('kernel', [-1, -2])
def test_pose_only_vs_float64(refs, kernel, mode):
    """Tracking pass (all map gradients NULL): the ray gradients alone."""
    from oracle.coslam_f64 import failures
    rep = run_case(refs, 'bench', kernel, mode, map_grads=False)
    assert 'level' not in rep and 'd_w_sdf0' not in rep and 'd_rays_d' in rep
    bad = failures(rep, GATES[mode])
    assert not bad, (KERNELS[kernel], mode, bad)


# ------------------------------------------------------------- smoothness ---
# k_smooth_bwd (plain fp32) against smoothness_replay, per lattice and per path: 'auto' lets a
# CTA interpolate from and gather into a shared-memory box of table entries where the box fits,
# 'gather' (xrd_debug_smooth_box_cap(0)) sends every level through the 8-corner gather and
# scatter.  Which levels take the box depends on the lattice and on the device's shared memory;
# the second path makes the gather a test input instead.
F32_U = 2.0 ** -24
RAND = (0.3, 0.7, 0.1, 0.9, 0.2, 0.5)
ONE_MINUS = float(np.nextafter(np.float32(1), np.float32(0)))     # the largest float below 1
EDGE_RAND = (0.0, ONE_MINUS, 0.0, ONE_MINUS, 0.0, ONE_MINUS)
MARGIN = 0.05
XRD_E_SHAPE = -1
# name: (sample points, voxel, smooth_rand); the lattice side is n = sample points - 1 and a CTA
# sweeps a slab of 4 x planes
LATTICES = {
    'p32': (32, 0.1, RAND),            # the mapping configuration: n % 4 = 3
    'p3': (3, 0.1, RAND),              # n = 2: one slab, fewer than 4 planes
    'p5': (5, 0.1, RAND),              # n = 4: one full slab
    'p6': (6, 0.1, RAND),              # n = 5: a last slab of one plane
    'p30': (30, 0.1, RAND),            # n % 4 = 1
    'p33': (33, 0.1, RAND),            # n % 4 = 0
    'p35': (35, 0.1, RAND),            # n % 4 = 2
    'p60': (60, 0.03, RAND),           # box and gather on the same level
    'p76_v015': (76, 0.015, RAND),     # the largest lattice (the smallest box) on dense cells
    'p76_v05': (76, 0.05, RAND),       # the largest lattice, no level fits the box
    'p40_v15': (40, 0.15, RAND),       # wider than the bound along z: cells wrap on both sides
    'p32_edge': (32, 0.1, EDGE_RAND),  # offsets and sub-voxel shifts at 0 and just below 1
}
PATHS = {'auto': -1, 'gather': 0}
# the mapping configuration on the automatic path keeps its gates (4x the observed worst)
SMOOTH_GATES = dict(level=1e-6, entry=2e-6, loss=3e-8)
# every other case: (level, loss) gates per lattice, about 4x the worst observed over both
# paths, both entry points and the scaled accumulation (module docstring); the entry gates
# follow from the number of terms (smooth_entry_gates)
SMOOTH_LEVEL_LOSS = {
    'p32': (1.3e-6, 7.5e-8), 'p3': (8e-7, 3.2e-7), 'p5': (9.6e-7, 2e-7), 'p6': (7.4e-7, 1.6e-7),
    'p30': (1.2e-6, 2.2e-7), 'p33': (1.3e-6, 1.5e-7), 'p35': (1.3e-6, 1.3e-7),
    'p60': (6.5e-6, 2.3e-7), 'p76_v015': (1.8e-5, 9.6e-8), 'p76_v05': (3.1e-6, 6.6e-8),
    'p40_v15': (8.8e-7, 1.6e-7), 'p32_edge': (1.1e-6, 1.3e-7),
}


def smooth_entry_gates(terms, n):
    """Per level: 2 (T + S + 16) 2^-24, with T the most (point, corner) terms that land on one
    table entry and S the slabs.  The gather adds T terms into the entry one atomic at a time;
    the box path sums at most T of them in one thread's fma chain and adds the result once per
    plane of a slab and once per slab.  16 covers the rounding of each point's own gradient."""
    slabs = -(-n // 4)
    return [2 * (t + slabs + 16) * F32_U for t in terms]


def smooth_ref(refs, name):
    """The float64 replay of one lattice (cached), on the table of the fused-step batches."""
    key = ('smooth', name)
    if key not in refs.cache:
        from helpers import coslam_pair
        from oracle.coslam_f64 import smoothness_replay
        if 'smooth_pair' not in refs.cache:
            refs.cache['smooth_pair'] = coslam_pair(refs.dev, table_amp=0.1)
        ora, model = refs.cache['smooth_pair']
        sp, vox, rnd = LATTICES[name]
        loss, g, A, lay, terms = smoothness_replay(
            ora, torch.tensor(rnd).reshape(2, 3), device=refs.dev, sample_points=sp, voxel=vox,
            margin=MARGIN, with_terms=True)
        refs.cache[key] = dict(model=model, loss=float(loss), g=g, A=A, lay=lay, terms=terms,
                               entry_gates=smooth_entry_gates(terms, sp - 1))
    return refs.cache[key]


def smooth_call(model, sp, vox, rnd, path='auto', dev_rand=False, weight=1.0, grad_scale=1.0,
                d_table=None, ws=None, loss_init=float('nan')):
    """One xrd_coslam_smoothness (host rand) or xrd_coslam_smoothness_dev (device rand) call
    on the model's table, synchronised -> (status, loss [1]).  loss starts at loss_init, so a
    loss the kernel never writes fails every comparison."""
    import ctypes as C
    from xrdslam_b200 import _cabi
    lib = _cabi.lib()
    table = model.embed_fn.params.detach()
    dev = table.device
    grid = model._grid_struct(table)
    loss = torch.full((1,), loss_init, dtype=torch.float32, device=dev)
    if ws is None:
        ws = _cabi.workspace(dev, 'coslam_smoothness', sp)
    if dev_rand:
        r_dev = torch.tensor(rnd, dtype=torch.float32, device=dev)
        fn, r = lib.xrd_coslam_smoothness_dev, r_dev.data_ptr()
    else:
        fn, r = lib.xrd_coslam_smoothness, (C.c_float * 6)(*rnd)
    prev = lib.xrd_debug_smooth_box_cap(PATHS[path])
    try:
        with torch.cuda.device(dev):
            st = fn(C.byref(grid), sp, vox, MARGIN, weight, r, _cabi.ptr(loss),
                    _cabi.ptr(d_table), grad_scale, _cabi.ptr(ws[0]), ws[1],
                    torch.cuda.current_stream(dev).cuda_stream)
    finally:
        lib.xrd_debug_smooth_box_cap(prev)
    torch.cuda.synchronize()
    return st, loss


def smoothness_report(c, loss, d_table, scale=1.0, before=None):
    """A kernel result against the replay times `scale`: per level the relative L2 of d_table
    (minus `before`) and the worst |g - g64| / A, and the relative loss error."""
    from oracle.coslam_f64 import level_slices
    g = d_table.double() - (before.double() if before is not None else 0.0)
    g64, A = c['g'] * scale, c['A'] * scale
    err = (g - g64).abs()
    lv, ent = [], []
    for a, b in level_slices(c['lay']):
        lv.append(float((g[a:b] - g64[a:b]).norm() / (g64[a:b].norm() + 1e-300)))
        e, Ab = err[a:b], A[a:b]
        bad = bool(((Ab == 0) & (e > 0)).any())
        ent.append(float('inf') if bad else float((e[Ab > 0] / Ab[Ab > 0]).max()))
    loss64 = c['loss'] * scale
    return dict(level=lv, entry=ent, loss=abs(float(loss) - loss64) / loss64)


def smooth_failures(c, rep, name, path, entry_factor=1.0):
    """Checks of a smoothness_report beyond the gates of its lattice (entry gates x factor)."""
    if name == 'p32' and path == 'auto' and entry_factor == 1.0:
        lg, sg = SMOOTH_GATES['level'], SMOOTH_GATES['loss']
        eg = [SMOOTH_GATES['entry']] * len(rep['entry'])
    else:
        lg, sg = SMOOTH_LEVEL_LOSS[name]
        eg = [entry_factor * v for v in c['entry_gates']]
    out = [f'level {l}: {v:.3g}' for l, v in enumerate(rep['level']) if not v <= lg]
    out += [f'entry level {l}: {v:.3g} > {eg[l]:.3g}' for l, v in enumerate(rep['entry'])
            if not v <= eg[l]]
    if not rep['loss'] <= sg:
        out.append(f"loss: {rep['loss']:.3g}")
    return out


def within_ulp(a, b):
    """|a - b| within one float ulp of the larger."""
    a, b = float(a), float(b)
    return abs(a - b) <= float(np.spacing(np.float32(max(abs(a), abs(b)))))


def _grad_run(refs, name, path, **kw):
    c = smooth_ref(refs, name)
    sp, vox, rnd = LATTICES[name]
    d = torch.zeros_like(c['model'].embed_fn.params.detach())
    st, loss = smooth_call(c['model'], sp, vox, rnd, path, d_table=d, **kw)
    assert st == 0, st
    return c, loss, d


def _check_vs_float64(refs, name, path):
    """d_table per level and per entry, and the loss, against the float64 replay."""
    c, loss, d = _grad_run(refs, name, path)
    bad = smooth_failures(c, smoothness_report(c, loss, d), name, path)
    assert not bad, (name, path, bad)


def test_smoothness_vs_float64(refs):
    """The mapping configuration (32 points, voxel 0.1) on the automatic path."""
    _check_vs_float64(refs, 'p32', 'auto')


@pytest.mark.parametrize('name, path', [
    pytest.param(n, p, id=f'{n}-{p}') for n in LATTICES for p in PATHS
    if (n, p) != ('p32', 'auto')])
def test_smoothness_lattice_vs_float64(refs, name, path):
    """Every other lattice, and the gather path, as test_smoothness_vs_float64."""
    _check_vs_float64(refs, name, path)


@pytest.mark.parametrize('name', list(LATTICES))
def test_smoothness_paths_agree_on_loss(refs, name):
    """Both paths interpolate with the same arithmetic and sum the loss per thread in the same
    order; only the double atomics of the per-CTA partials run in no fixed order."""
    _, l_auto, _ = _grad_run(refs, name, 'auto')
    _, l_gather, _ = _grad_run(refs, name, 'gather')
    assert within_ulp(l_auto, l_gather), (float(l_auto), float(l_gather))


@pytest.mark.parametrize('path', list(PATHS))
@pytest.mark.parametrize('name', list(LATTICES))
def test_smoothness_loss_only(refs, name, path):
    """d_table = NULL: the same loss as the gradient run, nothing else written."""
    c, l_grad, _ = _grad_run(refs, name, path)
    sp, vox, rnd = LATTICES[name]
    st, loss = smooth_call(c['model'], sp, vox, rnd, path)
    assert st == 0 and within_ulp(loss, l_grad), (st, float(loss), float(l_grad))


@pytest.mark.parametrize('name', list(LATTICES))
def test_smoothness_device_rand(refs, name):
    """xrd_coslam_smoothness_dev (the mapping graph's entry point, smooth_rand read on the
    device) against the host-rand entry point and the replay."""
    c, l_host, _ = _grad_run(refs, name, 'auto')
    _, l_dev, d_dev = _grad_run(refs, name, 'auto', dev_rand=True)
    assert within_ulp(l_dev, l_host), (float(l_dev), float(l_host))
    bad = smooth_failures(c, smoothness_report(c, l_dev, d_dev), name, 'device rand')
    assert not bad, (name, bad)


@pytest.mark.parametrize('path', list(PATHS))
@pytest.mark.parametrize('name', list(LATTICES))
def test_smoothness_scaled_accumulate(refs, name, path):
    """weight 0.37 and grad_scale 2.5 onto a non-zero d_table: the kernel adds
    weight * grad_scale * dL/dtable and writes weight * loss.  A touched entry starts at up to
    the gradient it receives, so the accumulation at most doubles the rounding (entry gate x2);
    an untouched one starts at a typical bound and must not change."""
    c = smooth_ref(refs, name)
    sp, vox, rnd = LATTICES[name]
    w, gs = np.float32(0.37), np.float32(2.5)
    A = c['A'] * (float(w) * float(gs))
    g64 = (c['g'] * (float(w) * float(gs))).abs()
    g = torch.Generator().manual_seed(sp)
    mag = torch.where(A > 0, g64, A[A > 0].median())
    u = torch.rand(A.numel(), generator=g, dtype=torch.float64).to(A.device) * 2 - 1
    before = (u * mag).float()
    d = before.clone()
    st, loss = smooth_call(c['model'], sp, vox, rnd, path, weight=float(w), grad_scale=float(gs),
                           d_table=d)
    assert st == 0, st
    rep = smoothness_report(c, loss, d, scale=float(w) * float(gs), before=before)
    rep['loss'] = abs(float(loss) - c['loss'] * float(w)) / (c['loss'] * float(w))
    bad = smooth_failures(c, rep, name, path, entry_factor=2.0)
    assert not bad, (name, path, bad)


@pytest.mark.parametrize('name', list(LATTICES))
def test_smoothness_workspace_reuse(refs, name):
    """Two calls on one workspace that starts as garbage give the same, right loss: the
    header (loss accumulator and CTA ticket) is reset every call."""
    from xrdslam_b200 import _cabi
    c = smooth_ref(refs, name)
    sp, vox, rnd = LATTICES[name]
    ws = _cabi.workspace(refs.dev, 'coslam_smoothness', sp)
    ws[0].fill_(0x5A)
    st1, l1 = smooth_call(c['model'], sp, vox, rnd, ws=ws)
    st2, l2 = smooth_call(c['model'], sp, vox, rnd, ws=ws)
    assert st1 == 0 and st2 == 0 and within_ulp(l1, l2), (float(l1), float(l2))
    assert abs(float(l1) - c['loss']) <= SMOOTH_LEVEL_LOSS[name][1] * c['loss'], float(l1)


@pytest.mark.parametrize('dev_rand', [False, True])
def test_smoothness_shape_limits(refs, dev_rand):
    """2 and 77 sample points are rejected and leave loss and d_table alone; 76 runs."""
    c = smooth_ref(refs, 'p32')
    model = c['model']
    for sp in (2, 77):
        d = torch.zeros_like(model.embed_fn.params.detach())
        st, loss = smooth_call(model, sp, 0.015, RAND, dev_rand=dev_rand, d_table=d,
                               loss_init=7.0)
        assert st == XRD_E_SHAPE and float(loss) == 7.0 and not bool(d.any()), (sp, st)
    st, loss = smooth_call(model, 76, 0.015, RAND, dev_rand=dev_rand, loss_init=7.0)
    assert st == 0 and float(loss) != 7.0 and np.isfinite(float(loss)), (st, float(loss))
