"""Write tests/golden/nice_importance_step.npz from the reference's own ConvOnet (needs the
reference checkout): NICE-SLAM steps with stratified jitter and importance sampling.

The networks and grids are oracle.nice.NiceOracle(seed) copied into the reference's ConvOnet;
the reference runs under oracle.nice_importance.sample_pdf_without_device, since its
render_batch_ray passes a `device` keyword that its sample_pdf does not take.  Its draws --
torch.rand(z_vals.shape) for the jitter, then sample_pdf's torch.rand -- are recorded with the
outputs, the loss terms and the gradients of the grids, the colour decoder and the rays, so
that tests/test_nice_importance_cpu.py checks the restatement without the reference.

Usage: python tests/golden/make_golden_nice_importance.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

BOUND = np.array([[-2.0, 2.0], [-2.0, 2.0], [-2.0, 2.0]])
# name: (stage, is_mapping, n_importance, perturb)
CASES = {'perturb': ('color', True, 0, 1.0), 'det16': ('color', True, 16, 0.0),
         'rand16': ('color', False, 16, 1.0), 'fine_det5': ('fine', True, 5, 0.0),
         'coarse_rand8': ('coarse', True, 8, 1.0)}
SEED = 3


def oracle(coarse):
    from oracle.nice import NiceOracle
    with torch.random.fork_rng():
        torch.manual_seed(SEED)
        ora = NiceOracle(BOUND, seed=SEED, coarse=coarse)
    with torch.no_grad():
        for k in ora.grids:
            ora.grids[k].mul_(30.0)
    return ora


def rays(R=24):
    g = torch.Generator().manual_seed(SEED + 1)
    ro = (torch.rand(R, 3, generator=g) - 0.5) * 0.6
    rd = torch.nn.functional.normalize(torch.randn(R, 3, generator=g), dim=-1)
    td = torch.rand(R, 1, generator=g) * 1.5 + 0.3
    td[3::7] = 0
    ts = torch.rand(R, 3, generator=g)
    return ro, rd, ts, td


def color_tensors(d):
    t = [d.embedder._B]
    t += [x for i in range(5) for x in (d.pts_linears[i].weight, d.pts_linears[i].bias)]
    t += [x for i in range(5) for x in (d.fc_c[i].weight, d.fc_c[i].bias)]
    return t + [d.output_linear.weight, d.output_linear.bias]


def main():
    from oracle import ref_harness as H
    from oracle import nice_importance as NI
    ro, rd, ts, td = rays()
    R = ro.shape[0]
    rec = dict(rays_o=ro.numpy(), rays_d=rd.numpy(), target_s=ts.numpy(), target_d=td.numpy())
    for name, (stage, is_mapping, N, perturb) in CASES.items():
        coarse = stage == 'coarse'
        ora = oracle(coarse)
        ref = H.ref_conv_onet(BOUND, coarse=coarse, rendering_n_importance=N,
                              rendering_perturb=perturb)
        H.copy_nice_oracle_to_ref(ora, ref)
        for k in list(ref.grid_c):
            ref.grid_c[k] = ref.grid_c[k].detach().clone().requires_grad_(True)
        seed = 100 + N
        torch.manual_seed(seed)  # the reference's draws, in its order
        noise = torch.rand(R, 32) if perturb > 0 else None
        u = (torch.rand(R, N) if perturb > 0 else NI.det_u(N).expand(R, N)) if N > 0 else None
        r_o, r_d = ro.clone().requires_grad_(True), rd.clone().requires_grad_(True)
        torch.manual_seed(seed)
        with H.cuda_calls_are_noops(), NI.sample_pdf_without_device():
            out = ref.render_batch_ray(r_o, r_d, stage, gt_depth=td)
        ld = ora.loss_dict(out, ts, td, is_mapping, stage)  # conv_onet.py:145-185, restated
        sum(ld.values()).backward()
        p = name + '.'
        if noise is not None:
            rec[p + 'noise'] = noise.numpy()
        if u is not None:
            rec[p + 'u'] = u.contiguous().numpy()
        for k in ('rgb', 'depth', 'uncertainty'):
            rec[p + k] = out[k].detach().numpy()
        for k, v in ld.items():
            rec[p + 'loss.' + k] = np.array(float(v.detach()))
        for k, v in ref.grid_c.items():
            if v.grad is not None:
                rec[p + 'd_' + k] = v.grad.numpy()
        if stage == 'color':
            for i, t in enumerate(color_tensors(ref.decoder.color_decoder)):
                if t.grad is not None:
                    rec[p + f'd_color{i}'] = t.grad.numpy()
        rec[p + 'd_rays_o'], rec[p + 'd_rays_d'] = r_o.grad.numpy(), r_d.grad.numpy()
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'nice_importance_step.npz')
    np.savez_compressed(path, **rec)
    print(path, os.path.getsize(path))


if __name__ == '__main__':
    main()
