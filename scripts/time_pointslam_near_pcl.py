"""Time Point-SLAM's rendering_sample_near_pcl on the GPU: xrd_pointslam_sample_near_pcl alone,
and the colour-stage mapping step (forward + backward) with the option on and off, at the bench
shape (5000 rays x 5 samples, 40 000 cloud points) with 0 %, 5 % and 30 % zero-depth rays; and one
1200 x 680 render (ray_batch_size 3000 chunks, no gradients) with 30 % holes.  CUDA events after
a warm-up; prints one JSON object with the card and its power limit.

    python scripts/time_pointslam_near_pcl.py [--out results/time_near_pcl.json] [--reps 50]

Needs a CUDA device; no fallback."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                        '--format=csv,noheader'], capture_output=True, text=True).stdout
    return q.strip().splitlines()[0] if q.strip() else torch.cuda.get_device_name(0)


def scene(dev, R, n_points=40000, seed=0):
    """Rays from the origin onto a noisy surface 1.2-1.8 m away and a cloud on that surface."""
    g = torch.Generator().manual_seed(seed)
    rd = torch.nn.functional.normalize(torch.randn(R, 3, generator=g) *
                                       torch.tensor([0.4, 0.4, 0.05]) + torch.tensor([0, 0, -1.0]),
                                       dim=-1)
    d = torch.rand(R, generator=g) * 0.6 + 1.2
    m = n_points // 8
    src = torch.randint(0, R, (m,), generator=g)
    pos = ((rd[src] * d[src, None])[:, None, :] +
           torch.randn(m, 8, 3, generator=g) * 0.03).reshape(-1, 3)
    return torch.zeros(R, 3).to(dev), rd.to(dev), d.to(dev), pos


def model_for(dev, pos, on):
    from xrdslam_b200.camera import Camera
    from xrdslam_b200.conv_onet_pointslam import ConvOnet2Config
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', RuntimeWarning)
        model = ConvOnet2Config(rendering_sample_near_pcl=on).setup(
            camera=Camera(600., 600., 599.5, 339.5, 1200, 680))
    model.to(dev)
    g = torch.Generator().manual_seed(1)
    model.model_update(dev).set_cloud(pos, torch.randn(pos.shape[0], 32, generator=g) * 0.5,
                                      torch.randn(pos.shape[0], 32, generator=g) * 0.5)
    return model


def timed(fn, reps, warm=5):
    for _ in range(warm):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--reps', type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    dev = torch.device('cuda:0')
    R = 5000
    ro, rd, d, pos = scene(dev, R)
    res = {'card': card(), 'rays': R, 'points': int(pos.shape[0]), 'step_ms': {}, 'sampler_ms': {}}
    models = {on: model_for(dev, pos, on) for on in (False, True)}
    radius = torch.full((R,), 0.06, device=dev)
    for frac in (0.0, 0.05, 0.30):
        td = d.clone()
        td[torch.arange(R, device=dev) % 100 < int(frac * 100)] = 0
        far = torch.minimum(5 * td.mean(), torch.max(td * 1.2)).reshape(1).float()
        npc = models[True].neural_point_cloud
        res['sampler_ms'][f'{frac:.2f}'] = timed(
            lambda: npc.near_pcl_samples(ro, rd, td, far, 0.3, 5), a.reps)
        for on, model in models.items():
            cd = model.decoder.color_decoder

            def step():
                for p in [model.neural_point_cloud.geo_feats, model.neural_point_cloud.col_feats] + \
                        list(cd.parameters()):
                    p.grad = None
                inp = dict(rays_o=ro, rays_d=rd, target_d=td, target_s=torch.zeros(R, 3, device=dev),
                           stage='color', batch_dynamic_r=radius, is_mapping=True)
                out = model(inp)
                sum(model.get_loss_dict(out, inp, True).values()).backward()
            res['step_ms'][f'{"on" if on else "off"}_{frac:.2f}'] = timed(step, a.reps)
    # one 1200 x 680 render with 30 % holes, in ray_batch_size chunks as render_img runs it
    H, W = 680, 1200
    ro_f, rd_f, d_f, _ = scene(dev, H * W, seed=2)
    d_f[torch.arange(H * W, device=dev) % 10 < 3] = 0
    r_f = torch.full((H * W,), 0.06, device=dev)
    res['render_1200x680_ms'] = {}
    for on, model in models.items():
        def render():
            with torch.no_grad():
                for s in range(0, H * W, 3000):
                    model(dict(rays_o=ro_f[s:s + 3000], rays_d=rd_f[s:s + 3000],
                               target_d=d_f[s:s + 3000], target_s=None, stage='color',
                               batch_dynamic_r=r_f[s:s + 3000]))
        res['render_1200x680_ms']['on' if on else 'off'] = timed(render, 5, warm=1)
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or '.', exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
