"""Cost of categorical value heads (train_args['value_bins']) on one GPU.
  * each kernel alone (hrl_value_bins_expect, hrl_value_bins_fwd_bwd) at the cfg3 and cfg5-shard loss shapes with K = 51 and
    K = 255, two-hot and HL-Gauss: one CUDA graph of `--launches` launches per block, blocks timed with CUDA events, the best
    block kept; µs per launch and algorithmic GB/s against the 3.35 TB/s of the H100 SXM data sheet.  Algorithmic bytes: the
    expectation reads the logits and writes one value per row (4 K + 4 bytes a row); the cross-entropy reads the logits and
    writes their gradient (8 K bytes a row) and reads each column's target and mask (8 bytes a column);
  * the cfg4 LearnerStep (module path): the workload's net with the key off, and the same net with its value layer widened to
    51 outputs and the key on (a K = 51 value head): ms per step and launches per step, the two forms alternated over
    `--rounds` blocks.
The card's name, power limit and maximum SM clock are read in the same run.  Prints one JSON line.

    python scripts/bench_value_bins.py [--launches 200] [--steps 30] [--rounds 3] [--out FILE]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

from bench_diagnostics import time_block  # noqa: E402
from bench_distill import card  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
KERNEL_SHAPES = {       # B, T, P, Pa, burn_in: the loss shapes of cfg3 and of one shard of cfg5
    'cfg3': (256, 20, 2, 2, 4),
    'cfg5shard': (512, 64, 2, 1, 0),
}


def kernel(name, K, sigma_bins, launches, rounds):
    from handyrl_b200 import ops
    B, T, P, Pa, bi = KERNEL_SHAPES[name]
    spec = {'bins': K, 'low': -1.0, 'high': 1.0, 'symlog': False, 'sigma': sigma_bins * 2.0 / (K - 1)}
    g = torch.Generator().manual_seed(0)
    z = (torch.randn(B, T, Pa, K, generator=g) * 2).cuda()
    batch = {'observation_mask': (torch.rand(B, T, P, 1, generator=g) > 0.1).float().cuda()}
    buf = ops.LossBuffers(B, T, P, Pa, 4, True, False, 'cuda', value_bins={'value': spec})
    ops.bins_targets(buf)['value'].copy_(torch.rand(B, T, P, 1, generator=g) * 2 - 1)
    args = {'burn_in_steps': bi}
    out = torch.empty(B, T, Pa, 1, device='cuda')
    forms = {'expect': lambda: ops.value_bins_expect(z, spec, out=out, P=P),
             'fwd_bwd': lambda: ops.value_bins_fwd_bwd(z, 'value', spec, batch, args, buf)}
    rows, cols = B * T * Pa, B * T * P
    nbytes = {'expect': (4 * K + 4) * rows, 'fwd_bwd': 8 * K * rows + 8 * cols}
    res = {'B': B, 'T': T, 'P': P, 'Pa': Pa, 'K': K, 'sigma_bins': sigma_bins}
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    for form, fn in forms.items():
        with torch.cuda.stream(s):
            for _ in range(3):
                fn()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, stream=s):
                for _ in range(launches):
                    fn()
        times = []
        for _ in range(rounds):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            with torch.cuda.stream(s):
                e0.record()
                graph.replay()
                e1.record()
            e1.synchronize()
            times.append(e0.elapsed_time(e1) * 1e3 / launches)
        best = min(times)
        res[form] = {'us': times, 'best_us': best, 'algorithmic_bytes': nbytes[form],
                     'GB_per_s': nbytes[form] / (best * 1e-6) / 1e9, 'share_of_hbm': nbytes[form] / (best * 1e-6) / HBM_BYTES_PER_S}
    return res


def _widened_net(w, K):
    """The workload's net with its value layer (v_out) widened to K outputs: a K-logit value head."""
    import bench
    net = bench.make_net(w)
    torch.manual_seed(1)
    net.v_out = torch.nn.Linear(net.v_out.in_features, K)
    return net


def step(name, steps, rounds, K=51, warmup=10):
    import bench
    from handyrl_b200.train import LearnerStep, PackedBatch
    w = dict(bench.WORKLOADS[name])
    args = bench.train_args(w)
    example = bench.make_batch(w, 10_000)
    lr = 3e-8 * w['B'] * w['T']
    bins = {'value': {'bins': K, 'low': -1.0, 'high': 1.0}}
    steppers = {'off': LearnerStep(bench.make_net(w), args, example, lr=lr),
                'on': LearnerStep(_widened_net(w, K), dict(args, value_bins=bins), example, lr=lr)}
    batch = PackedBatch(steppers['off'].layout).fill(example).buffer.cuda()
    for st in steppers.values():
        time_block(st.stream, lambda i, st=st: st.step_resident(batch), warmup)
    res = {k: [] for k in steppers}
    for r in range(rounds):
        for k in (('off', 'on') if r % 2 == 0 else ('on', 'off')):
            st = steppers[k]
            res[k].append(time_block(st.stream, lambda i, st=st: st.step_resident(batch), steps))
    out = {'B': w['B'], 'T': w['T'], 'K': K, 'fused_tower': steppers['off'].engine is not None}
    for k, st in steppers.items():
        out[k] = {'ms_per_step': res[k], 'best_ms': min(res[k]), 'launches_per_step': st.launches_per_step}
        st.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--launches', type=int, default=200)
    ap.add_argument('--steps', type=int, default=30)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_value_bins.py measures on the GPU; there is none')
    kern = {}
    for name in KERNEL_SHAPES:
        for K in (51, 255):
            for sigma_bins in (0.0, 0.75):
                kern['%s_K%d_%s' % (name, K, 'hlgauss' if sigma_bins else 'twohot')] = kernel(name, K, sigma_bins, a.launches, a.rounds)
    res = {'card': card(), 'kernel': kern, 'step': {'cfg4': step('cfg4', a.steps, a.rounds)}}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
