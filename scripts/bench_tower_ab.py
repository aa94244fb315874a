"""A/B of two builds of the CUDA library on the flagship workload (cfg2: TicTacToe BoardNet on the fused tower, B=512 T=32).

    python scripts/bench_tower_ab.py --old OLD/libhrl_b200.so --new handyrl_b200/libhrl_b200.so [--blocks 3] [--steps 300]

Each arm runs in a subprocess of its own that points `_capi.LIB_PATH` at its library before the library is first loaded, and
the arms alternate (old, new, old, new, ...) so that both see the same state of the machine.  Per block and arm:
  * the three tensor-core products of one tower layer alone (`bench.time_tower_products`: forward, input gradient, weight
    gradient; 20 launches in a CUDA graph, replayed 5 times);
  * the cfg2 learner step (`LearnerStep.step_resident`, captured in a CUDA graph) over a ring of resident batches larger than
    L2, timed with CUDA events over --steps steps after --warmup steps;
  * the card's name, power limit and maximum SM clock.
The first block's runs also take ONE step from the seeded initial weights on the same batch and write its six loss sums and
the updated flat parameters; the two arms must agree bit for bit.  Prints min / median / max of every time per arm and one
JSON line with everything.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def gpu_info():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else 'unknown'
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def run_arm(opt):
    """One arm in this process: load opt.arm as the library, time, optionally dump the first step's results."""
    sys.path.insert(0, ROOT)
    from handyrl_b200 import _capi
    _capi.LIB_PATH = os.path.abspath(opt.arm)
    import numpy as np
    import torch
    import bench
    from handyrl_b200.train import LearnerStep, PackedBatch

    w = bench.WORKLOADS['cfg2']
    torch.cuda.set_device(0)
    device = torch.device('cuda', 0)
    B, T = w['B'], w['T']
    stepper = LearnerStep(bench.make_net(w), bench.train_args(w), bench.make_batch(w, 10_000), lr=3e-8 * B * T, device=device,
                          use_graph=True)
    assert stepper.engine is not None, 'cfg2 must run on the fused tower engine'
    nbytes = stepper.layout.nbytes
    R = min(96, max(8, int(2 * bench.L2_BYTES / nbytes) + 1))
    ring = torch.empty((R, nbytes), dtype=torch.uint8, device=device)
    for i in range(R):
        ring[i].copy_(PackedBatch(stepper.layout).fill(bench.make_batch(w, 20_000 + i)).buffer)
    torch.cuda.synchronize()

    stepper.step_resident(ring[0])          # the first step: seeded weights, the same batch in both arms
    stepper.stream.synchronize()
    if opt.dump:
        np.savez(opt.dump, losses=stepper.last_losses.detach().cpu().numpy(), params=stepper.state.flat_param.detach().cpu().numpy())

    for i in range(opt.warmup):
        stepper.step_resident(ring[(1 + i) % R])
    stepper.stream.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(stepper.stream):
        e0.record()
    for i in range(opt.steps):
        stepper.step_resident(ring[(1 + opt.warmup + i) % R])
    with torch.cuda.stream(stepper.stream):
        e1.record()
    stepper.stream.synchronize()
    step_ms = e0.elapsed_time(e1) / opt.steps
    products = bench.time_tower_products(stepper.engine, device)
    res = {'lib': opt.arm, 'gpu': gpu_info(), 'step_ms': step_ms,
           'products_us': {k.split(' (')[0]: v['kernel_us'] for k, v in products.items()}}
    print('ARM ' + json.dumps(res), flush=True)


def spread(xs):
    return {'min': min(xs), 'median': statistics.median(xs), 'max': max(xs)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--old', help='library of the base build')
    ap.add_argument('--new', help='library of the build under test')
    ap.add_argument('--blocks', type=int, default=3)
    ap.add_argument('--steps', type=int, default=300)
    ap.add_argument('--warmup', type=int, default=30)
    ap.add_argument('--arm', help=argparse.SUPPRESS)
    ap.add_argument('--dump', help=argparse.SUPPRESS)
    opt = ap.parse_args()
    if opt.arm:
        return run_arm(opt)
    if not (opt.old and opt.new):
        ap.error('--old and --new are required')

    runs = {'old': [], 'new': []}
    with tempfile.TemporaryDirectory() as tmp:
        dumps = {}
        for block in range(opt.blocks):
            for name in ('old', 'new'):
                cmd = [sys.executable, os.path.abspath(__file__), '--arm', getattr(opt, name), '--steps', str(opt.steps),
                       '--warmup', str(opt.warmup)]
                if block == 0:
                    dumps[name] = os.path.join(tmp, name + '.npz')
                    cmd += ['--dump', dumps[name]]
                out = subprocess.run(cmd, capture_output=True, text=True)
                if out.returncode != 0:
                    sys.stderr.write(out.stdout + out.stderr)
                    raise SystemExit('arm %s failed in block %d' % (name, block))
                line = [ln for ln in out.stdout.splitlines() if ln.startswith('ARM ')][-1]
                r = json.loads(line[4:])
                runs[name].append(r)
                print('block %d %-3s step %.4f ms  %s' % (block, name, r['step_ms'],
                                                         '  '.join('%s %.1f us' % kv for kv in r['products_us'].items())), flush=True)
        import numpy as np
        a, b = np.load(dumps['old']), np.load(dumps['new'])
        identical = {k: bool(a[k].shape == b[k].shape and np.array_equal(a[k].view(np.uint32), b[k].view(np.uint32)))
                     for k in ('losses', 'params')}
        max_abs = {k: float(np.max(np.abs(a[k].astype(np.float64) - b[k].astype(np.float64)))) if a[k].shape == b[k].shape else None
                   for k in ('losses', 'params')}

    summary = {'gpu': sorted({r['gpu'] for rs in runs.values() for r in rs}), 'blocks': opt.blocks, 'steps': opt.steps,
               'bit_identical_first_step': identical, 'max_abs_diff_first_step': max_abs}
    for name in ('old', 'new'):
        rs = runs[name]
        summary[name] = {'lib': getattr(opt, name), 'step_ms': spread([r['step_ms'] for r in rs]),
                         'products_us': {k: spread([r['products_us'][k] for r in rs]) for k in rs[0]['products_us']}}
        s = summary[name]['step_ms']
        print('%-3s step ms  min %.4f  median %.4f  max %.4f' % (name, s['min'], s['median'], s['max']))
        for k, v in summary[name]['products_us'].items():
            print('%-3s %-16s us  min %.1f  median %.1f  max %.1f' % (name, k, v['min'], v['median'], v['max']))
    print('first step bit-identical: %s  (max |diff| %s)' % (identical, max_abs))
    print(json.dumps(summary), flush=True)


if __name__ == '__main__':
    main()
