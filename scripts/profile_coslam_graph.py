"""Per-node breakdown of the captured Co-SLAM mapping iteration (the bench.py default workload).

    profile_coslam_graph.py [--steps N] [--warmup W] [--trace FILE]

Builds the mapping session exactly as `bench.py` does (same seed, frames, batch shape and
optimisers), replays the graph N times under torch.profiler (CUDA activities) with the L2
flushed between steps as in the timed leg, and prints, per device activity of one step (kernel
or memset node, in launch order), its median duration and its median start / end relative to
the first node of the step.  That places `k_fused_g` against the smoothness nodes on the side
branch.  The card's name, power limit and SM clock are printed with the numbers.
"""
import argparse
import collections
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

import bench


def card(index):
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    try:
        return subprocess.run(['nvidia-smi', '-i', str(index), f'--query-gpu={q}',
                               '--format=csv,noheader'], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as e:  # noqa
        return f'nvidia-smi unavailable ({e!r})'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=10)
    ap.add_argument('--trace', default=None, help='also keep the chrome trace here')
    args = ap.parse_args()

    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    algo, kfs, cur = bench.build_algorithm(dev, seed=1234)
    model = algo.model
    frames = kfs + [cur]
    K, W = args.steps, args.warmup
    algo.config.mapping_sample = bench.MAP_KF
    from xrdslam_b200.dp import MappingDataParallel
    dp = MappingDataParallel(bench.flat_params(model))
    dp.broadcast_params(0)
    model.dp = dp
    algo.setup_optimizers(K + W, frames, is_mapping=True)
    assert algo._graph_ok(frames), 'the bench workload runs as a captured graph'
    algo.config.min_sample_pixels = bench.MAP_CUR
    algo.bundle_adjust = True
    sess = algo.mapping_session(frames)
    sess.begin(frames)
    batches = [sess.make_resident_batch(frames) for _ in range(K + W)]
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    for i in range(W):
        sess.step_resident(i, batches[i])
    torch.cuda.synchronize()

    clocks = bench.ClockSampler(0)
    clocks.start()
    acts = [torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        for i in range(K):
            flush.zero_()
            sess.step_resident(W + i, batches[W + i])
        torch.cuda.synchronize()
    clk = clocks.stop()
    sess.end(frames)

    path = args.trace or os.path.join(tempfile.mkdtemp(), 'trace.json')
    prof.export_chrome_trace(path)
    with open(path) as f:
        ev = [e for e in json.load(f)['traceEvents']
              if e.get('ph') == 'X' and e.get('cat') in ('kernel', 'gpu_memset', 'gpu_memcpy')]
    ev.sort(key=lambda e: e['ts'])
    # steps are delimited by the 256 MB flush (the only fill kernel longer than 20 us)
    is_flush = lambda e: e['cat'] == 'kernel' and 'fill' in e['name'].lower() and e['dur'] > 20
    steps, cur_step = [], None
    for e in ev:
        if is_flush(e):
            cur_step = []
            steps.append(cur_step)
        elif cur_step is not None and e['cat'] != 'gpu_memcpy':  # the H2D scalar block
            cur_step.append(e)
    steps = [s for s in steps if s]
    sig = collections.Counter(tuple(e['name'] for e in s) for s in steps).most_common(1)[0][0]
    steps = [s for s in steps if tuple(e['name'] for e in s) == sig]
    dur = np.array([[e['dur'] for e in s] for s in steps])
    t0 = np.array([s[0]['ts'] for s in steps])[:, None]
    beg = np.array([[e['ts'] for e in s] for s in steps]) - t0
    end = beg + dur
    span = end.max(1)

    print(f'card: {card(0)}; SM clock during the run (NVML median / max): '
          f'{clk.get("sm_mhz")} / {clk.get("sm_max_mhz")} MHz, throttle {clk.get("reasons")}')
    print(f'{len(steps)} of {K} steps with the common node list; us, medians over those steps; '
          f'start / end relative to the first node of the step')
    print(f'{"node":<64} {"dur":>8} {"start":>8} {"end":>8}')
    for j, name in enumerate(sig):
        short = name if len(name) <= 64 else name[:61] + '...'
        print(f'{short:<64} {np.median(dur[:, j]):8.1f} {np.median(beg[:, j]):8.1f} '
              f'{np.median(end[:, j]):8.1f}')
    smooth = [j for j, n in enumerate(sig) if 'smooth' in n or 'Memset' in n]
    fused = [j for j, n in enumerate(sig) if 'k_fused_g' in n]
    print(f'step span (first node start .. last node end): {np.median(span):.1f} us')
    if smooth:
        print(f'smoothness kernels and memsets: {np.median(dur[:, smooth].sum(1)):.1f} us of kernel time, '
              f'{np.median(beg[:, smooth].min(1)):.1f} .. {np.median(end[:, smooth].max(1)):.1f} us')
    if fused:
        j = fused[0]
        print(f'k_fused_g: {np.median(beg[:, j]):.1f} .. {np.median(end[:, j]):.1f} us')


if __name__ == '__main__':
    main()
