"""Cost of gradient accumulation (train_args['gradient_accumulation'] = k) on one GPU: LearnerStep CUDA graphs on resident batches,
CUDA events around blocks of steps, the forms alternated over `--rounds` blocks and the best block of each kept; launches per
step of each form.
  * cfg2 (TicTacToe, fused tower) at B=512 with k = 1, 2, 4;
  * cfg4 (Hungry Geese, module path) at B=256 with k = 1, 4;
  * cfg5: the per-GPU shard of configs[4] (B=512, k = 1) against the whole batch on one GPU (B=4096, k = 8): ms per step,
    samples per second and peak allocated memory.  Skipped with a printed reason when the card has too little free memory.
    B=4096 at k = 1 is never attempted: its activations are 8x those of the shard (see the printed arithmetic).
Prints one JSON line.

    python scripts/bench_grad_accumulation.py [--steps 200] [--steps-cfg4 40] [--steps-cfg5 10] [--rounds 3] [--out FILE]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

from bench_bf16 import gpu_name_and_power  # noqa: E402
from bench_diagnostics import time_block  # noqa: E402

CFG5_FREE_BYTES = 48 << 30       # what the cfg5 comparison needs free: the 4 GiB batch, the shard's activations, both learners


def forms(name, B, ks, steps, rounds, warmup, ring_size):
    import bench
    from handyrl_b200.train import LearnerStep, PackedBatch
    w = dict(bench.WORKLOADS[name], B=B)
    args = bench.train_args(w)
    example = bench.make_batch(w, 10_000)
    steppers = {k: LearnerStep(bench.make_net(w), args, example, lr=3e-8 * B * w['T'], gradient_accumulation=k) for k in ks}
    layout = steppers[ks[0]].layout
    ring = [PackedBatch(layout).fill(bench.make_batch(w, 20_000 + i)).buffer.cuda() for i in range(ring_size)]
    torch.cuda.synchronize()
    res = {k: [] for k in ks}
    for k, st in steppers.items():
        time_block(st.stream, lambda i, st=st: st.step_resident(ring[i % len(ring)]), warmup)
    for r in range(rounds):
        for k in (ks if r % 2 == 0 else ks[::-1]):
            st = steppers[k]
            res[k].append(time_block(st.stream, lambda i, st=st: st.step_resident(ring[i % len(ring)]), steps))
    out = {'B': B, 'T': w['T'], 'steps_per_block': steps, 'fused_tower': steppers[ks[0]].engine is not None}
    for k, st in steppers.items():
        out['k%d' % k] = {'ms_per_step': res[k], 'best_ms': min(res[k]), 'launches_per_step': st.launches_per_step}
        st.close()
    return out


def cfg5(steps, rounds, warmup):
    """The shard (B=512, k=1) and the whole configs[4] batch on one GPU (B=4096, k=8), one learner at a time so that each peak is
    its own."""
    import gc
    import bench
    from handyrl_b200.train import LearnerStep, PackedBatch
    free, total = torch.cuda.mem_get_info()
    per_sample = 32 * 32 * 32 * 4          # the first convolution's output of nets.WideActionNet, fp32
    arithmetic = {'first_conv_output_bytes_B4096_k1': per_sample * 4096 * 64, 'packed_batch_bytes_B4096': None}
    if free < CFG5_FREE_BYTES:
        return {'skipped': 'free memory %.1f GiB < %.1f GiB needed' % (free / 2 ** 30, CFG5_FREE_BYTES / 2 ** 30), **arithmetic}
    out = {'free_bytes_at_start': free}
    for B, k in ((512, 1), (4096, 8)):
        w = dict(bench.WORKLOADS['cfg5shard'], B=B)
        example = bench.make_batch(w, 10_000)
        gc.collect()
        torch.cuda.empty_cache()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        st = LearnerStep(bench.make_net(w), bench.train_args(w), example, lr=3e-8 * B * w['T'], gradient_accumulation=k)
        batch = PackedBatch(st.layout).fill(example).buffer.cuda()
        del example
        time_block(st.stream, lambda i: st.step_resident(batch), warmup)
        times = [time_block(st.stream, lambda i: st.step_resident(batch), steps) for _ in range(rounds)]
        torch.cuda.synchronize()
        best = min(times)
        out['B%d_k%d' % (B, k)] = {'ms_per_step': times, 'best_ms': best, 'samples_per_s': B * w['T'] / (best * 1e-3),
                                   'peak_allocated_bytes': torch.cuda.max_memory_allocated() - base,
                                   'packed_batch_bytes': st.layout.nbytes, 'launches_per_step': st.launches_per_step}
        arithmetic['packed_batch_bytes_B4096'] = st.layout.nbytes * 4096 // B
        st.close()
        del st, batch
    out.update(arithmetic)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=200)
    ap.add_argument('--steps-cfg4', type=int, default=40)
    ap.add_argument('--steps-cfg5', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--configs', default='cfg2,cfg4,cfg5')
    ap.add_argument('--out', default=None)
    opt = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_grad_accumulation needs a GPU'
    import __graft_entry__
    __graft_entry__.build()
    out = {'gpu': gpu_name_and_power()}
    todo = opt.configs.split(',')
    if 'cfg2' in todo:
        out['cfg2'] = forms('cfg2', 512, (1, 2, 4), opt.steps, opt.rounds, opt.warmup, 16)
    if 'cfg4' in todo:
        out['cfg4'] = forms('cfg4', 256, (1, 4), opt.steps_cfg4, opt.rounds, opt.warmup, 8)
    if 'cfg5' in todo:
        out['cfg5'] = cfg5(opt.steps_cfg5, opt.rounds, min(opt.warmup, 3))
    line = json.dumps(out)
    print(line)
    if opt.out:
        os.makedirs(os.path.dirname(os.path.abspath(opt.out)), exist_ok=True)
        with open(opt.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
