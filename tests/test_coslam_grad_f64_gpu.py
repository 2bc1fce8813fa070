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
  smoothness: level 2.6e-7, entry 4.9e-7, loss 7.3e-9

The fp32 CPU oracle itself stays within level 4.5e-7, entry 1.7e-7, weight 1e-9, ray 3e-9,
loss 1e-7 of float64.
"""
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


# smoothness (k_smooth_fwd / k_smooth_bwd, plain fp32): gates 4x the observed worst ratio
SMOOTH_GATES = dict(level=1e-6, entry=2e-6, loss=3e-8)


def smoothness_report(refs):
    from oracle.coslam_f64 import level_slices, smoothness_replay
    c = refs.get('bench')
    ora, model = c['ora'], c['model']
    rnd = torch.tensor([0.3, 0.7, 0.1, 0.9, 0.2, 0.5])
    loss64, g64, A, lay = smoothness_replay(ora, rnd.reshape(2, 3), device=refs.dev)
    loss, d_table = model._launch_smooth(model.embed_fn.params, rnd.tolist(), True, 1.0)
    torch.cuda.synchronize()
    g = d_table.double()
    err = (g - g64).abs()
    lv, ent = [], []
    for a, b in level_slices(lay):
        lv.append(float((g[a:b] - g64[a:b]).norm() / (g64[a:b].norm() + 1e-300)))
        e, Ab = err[a:b], A[a:b]
        bad = bool(((Ab == 0) & (e > 0)).any())
        ent.append(float('inf') if bad else float((e[Ab > 0] / Ab[Ab > 0]).max()))
    return dict(level=lv, entry=ent, loss=abs(float(loss) - float(loss64)) / float(loss64))


def test_smoothness_vs_float64(refs):
    rep = smoothness_report(refs)
    g = SMOOTH_GATES
    assert max(rep['level']) <= g['level'], rep['level']
    assert max(rep['entry']) <= g['entry'], rep['entry']
    assert rep['loss'] <= g['loss'], rep['loss']
