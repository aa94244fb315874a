"""Guard against non-finite optimiser steps on the GPU: hrl_clip_adam_step, hrl_step_commit and hrl_weight_ema given a skip
flag against the same entry points without one and ATen, in eager launches and CUDA graphs; and a learner that meets a batch
with a NaN in it is left bit for bit as if that batch had never been drawn (fused tower, module path, recurrent net; graph and
eager; the epoch hand-off, the Trainer, sharded ranks).  NaN and Inf only ever enter as data values."""
import bz2
import copy
import os
import pickle
import re
import socket
import sys
import tempfile
import threading
import time

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT

pytestmark = pytest.mark.gpu

NAN, INF = float('nan'), float('inf')
EXTRA = 8                                   # tail words behind the gradients (the learner pads its 6 loss sums to 8)
HP = (4.0, 0.9, 0.999, 1e-8, 1e-5)           # max_norm, beta1, beta2, eps, weight_decay


# ---------------------------------------------------------------------------------------------------------------- kernels
def _bucket(n, seed):
    """Optimiser state over n words and a gradient bucket [n gradients | EXTRA tail words, the first 6 loss sums]."""
    g = torch.Generator().manual_seed(seed)
    grad = torch.cat([0.05 * torch.randn(n, generator=g), torch.tensor([0.5, 0.2, 0.0, 1.3, 0.9, 48.0, 0.0, 0.0])])
    return {'param': torch.randn(n, generator=g).cuda(), 'grad': grad.cuda(),
            'm': (0.01 * torch.randn(n, generator=g)).cuda(), 'v': (0.001 * torch.rand(n, generator=g)).cuda(),
            'lr': torch.tensor([1e-3], device='cuda'), 'step': torch.tensor([7], dtype=torch.int64, device='cuda'),
            'gnorm': torch.full((1,), -1.0, device='cuda'), 'diag': torch.arange(4, dtype=torch.float64, device='cuda'),
            'skip': torch.full((1,), 7, dtype=torch.int32, device='cuda')}


def _clone(b):
    return {k: v.clone() for k, v in b.items()}


def _optimise(b, form, diag=False, n_tail=6):
    """hrl_grad_sumsq + hrl_clip_adam_step in one of its three forms on bucket b, in place, on the current stream: guarded
    (a skip flag and the first n_tail tail words, with or without diag), diag, or plain."""
    from handyrl_b200 import ops
    from handyrl_b200._capi import check, lib
    n = b['param'].numel()
    partials = torch.zeros(lib().hrl_sumsq_num_partials(), device='cuda')
    s = ops._stream_ptr()
    p = ops._ptr
    check(lib().hrl_grad_sumsq(p(b['grad']), n, p(partials), s))
    fixed = (p(b['param']), p(b['grad']), p(b['m']), p(b['v']), n, p(partials), p(b['lr']), p(b['step'])) + HP + (p(b['gnorm']),)
    diag_accum = p(b['diag']) if diag else None
    if form == 'guarded':
        check(lib().hrl_clip_adam_step(*fixed, diag_accum, p(b['grad'][n:]), n_tail, p(b['skip']), s))
    else:
        check(lib().hrl_clip_adam_step(*fixed, diag_accum, None, 0, None, s))


def _assert_same(a, b, keys=('param', 'm', 'v', 'step', 'gnorm', 'diag'), what=''):
    for k in keys:
        assert torch.equal(a[k], b[k]) or (k == 'gnorm' and torch.equal(a[k].isnan(), b[k].isnan()) and a[k].isnan().all()), \
            '%s: %s differs' % (what, k)


SIZES = [1, 4, 5, 257, 1031, 29008, 116928, 231604]     # TicTacToe, Geese and Geister buckets, and small ones


@pytest.mark.parametrize('diag', [False, True], ids=['plain', 'diag'])
@pytest.mark.parametrize('n', SIZES)
def test_guarded_step_is_bit_identical_on_finite_buckets(n, diag):
    start = _bucket(n, n)
    want, got = _clone(start), _clone(start)
    for _ in range(3):                                     # repeated calls: the step count moves alike
        _optimise(want, 'plain', diag)
        _optimise(got, 'guarded', diag)
    torch.cuda.synchronize()
    _assert_same(want, got, what='n=%d' % n)
    assert int(got['skip']) == 0 and int(got['step']) == 10
    if not diag:
        assert torch.equal(got['diag'], start['diag'])


def _rejected_cases(n):
    cases = []
    for pos in (0, n // 2, n - 1):
        for val in (NAN, INF, -INF):
            cases.append(('grad[%d]=%g' % (pos, val), pos, val))
    cases.append(('grad[%d]=1e20 (fp32 sum of squares overflows)' % (n // 3), n // 3, 1e20))
    for i in range(6):
        for val in (NAN, INF, -INF):
            cases.append(('tail[%d]=%g' % (i, val), n + i, val))
    return cases


@pytest.mark.parametrize('diag', [False, True], ids=['plain', 'diag'])
@pytest.mark.parametrize('n', [5, 29008, 231604])
def test_a_rejected_step_writes_nothing_and_counts_nothing(n, diag):
    start = _bucket(n, 3 * n)
    clean = _clone(start)
    _optimise(clean, 'guarded', diag)
    for what, pos, val in _rejected_cases(n):
        b = _clone(start)
        b['grad'][pos] = val
        _optimise(b, 'guarded', diag)
        torch.cuda.synchronize()
        assert int(b['skip']) == 1, what
        _assert_same(b, start, keys=('param', 'm', 'v', 'step', 'diag'), what=what)
        if pos >= n:                                         # a finite gradient: its norm is written as usual
            assert torch.equal(b['gnorm'], clean['gnorm']), what
        else:
            assert not torch.isfinite(b['gnorm']).any(), what
        # a good call after the rejected one equals a good call with nothing before it
        b['grad'].copy_(start['grad'])
        _optimise(b, 'guarded', diag)
        torch.cuda.synchronize()
        assert int(b['skip']) == 0, what
        _assert_same(b, clean, what=what + ', then a good call')


def test_only_the_tail_entries_asked_for_are_checked():
    n = 1031
    start = _bucket(n, 1)
    start['grad'][n + 6] = NAN                                # padding behind the six loss sums
    b = _clone(start)
    _optimise(b, 'guarded', n_tail=6)
    torch.cuda.synchronize()
    assert int(b['skip']) == 0
    b = _clone(start)
    _optimise(b, 'guarded', n_tail=7)
    torch.cuda.synchronize()
    assert int(b['skip']) == 1 and torch.equal(b['param'], start['param'])


@pytest.mark.parametrize('n_tail', [6, 22])
@pytest.mark.parametrize('nbytes', [0, 5, 16, 1000, 4103])
def test_commit_accumulates_like_aten_or_restores_and_counts(n_tail, nbytes):
    from handyrl_b200 import ops
    g = torch.Generator().manual_seed(nbytes + n_tail)
    tail = torch.randn(n_tail, generator=g).cuda()
    accum0 = torch.cat([torch.randn(n_tail, generator=g, dtype=torch.float64) * 1e3, torch.tensor([2.0], dtype=torch.float64)]).cuda()
    state0 = torch.randint(0, 256, (nbytes,), generator=g, dtype=torch.uint8).cuda()
    saved = torch.randint(0, 256, (nbytes,), generator=g, dtype=torch.uint8).cuda()
    pair = (state0.clone(), saved) if nbytes else (None, None)

    # accepted: the two ATen adds of the unguarded learner, bit for bit; the buffers and the count untouched
    want = accum0.clone()
    want[:6].add_(tail[:6].clone())
    if n_tail > 6:
        want[6:n_tail].add_(tail[6:n_tail])
    accum = accum0.clone()
    skip = torch.zeros(1, dtype=torch.int32, device='cuda')
    ops.step_commit(skip, tail, accum[:n_tail], accum[n_tail:], *pair)
    torch.cuda.synchronize()
    assert torch.equal(accum, want)
    if nbytes:
        assert torch.equal(pair[0], state0)

    # rejected: the sums untouched, the count up by one, the saved bytes back in place
    accum = accum0.clone()
    skip.fill_(1)
    ops.step_commit(skip, tail, accum[:n_tail], accum[n_tail:], *pair)
    torch.cuda.synchronize()
    assert torch.equal(accum[:n_tail], accum0[:n_tail]) and float(accum[n_tail]) == 3.0
    if nbytes:
        assert torch.equal(pair[0], saved)


@pytest.mark.parametrize('n', [3, 29008])
def test_guarded_average_is_a_no_op_on_a_rejected_step(n):
    from handyrl_b200 import ops
    g = torch.Generator().manual_seed(n)
    avg0, x = torch.randn(n, generator=g).cuda(), torch.randn(n, generator=g).cuda()
    step = torch.tensor([5], dtype=torch.int64, device='cuda')
    skip = torch.zeros(1, dtype=torch.int32, device='cuda')
    for seeded in (False, True):
        want, got = avg0.clone(), avg0.clone()
        ops.weight_ema_update(want, x, step, 0.9, seeded)
        ops.weight_ema_update(got, x, step, 0.9, seeded, skip=skip)
        torch.cuda.synchronize()
        assert torch.equal(got, want)
    skip.fill_(1)
    got = avg0.clone()
    ops.weight_ema_update(got, x, step, 0.9, False, skip=skip)
    torch.cuda.synchronize()
    assert torch.equal(got, avg0)


def test_the_three_kernels_in_one_graph_replay_like_eager_launches():
    from handyrl_b200 import ops
    n, nb = 29008, 1000
    start = _bucket(n, 17)
    g = torch.Generator().manual_seed(18)
    grads, moves = [], []
    for i in range(8):                       # good, bad, good, bad, ...: NaN, Inf in a gradient, Inf in a loss, overflow
        gr = start['grad'].cpu().clone()
        gr[:n] = 0.05 * torch.randn(n, generator=g)
        bad = [(5, NAN), (n - 1, INF), (n + 4, INF), (100, 1e20)]
        if i % 2:
            pos, val = bad[(i // 2) % 4]
            gr[pos] = val
        grads.append(gr.cuda())
        moves.append(torch.randint(0, 256, (nb,), generator=g, dtype=torch.uint8).cuda())

    def make():
        b = _clone(start)
        b.update(accum=torch.zeros(7, dtype=torch.float64, device='cuda'), avg=b['param'].clone(),
                 buffers=torch.randint(0, 256, (nb,), generator=torch.Generator().manual_seed(3), dtype=torch.uint8).cuda(),
                 saved=torch.zeros(nb, dtype=torch.uint8, device='cuda'), moved=torch.zeros(nb, dtype=torch.uint8, device='cuda'))
        return b

    def body(b):                             # the learner's order: save the buffers, the forward moves them, step, commit, average
        b['saved'].copy_(b['buffers'])
        b['buffers'].copy_(b['moved'])
        _optimise(b, 'guarded')
        ops.step_commit(b['skip'], b['grad'][n:n + 6], b['accum'][:6], b['accum'][6:], b['buffers'], b['saved'])
        ops.weight_ema_update(b['avg'], b['param'], b['step'], 0.9, False, skip=b['skip'])

    eager = make()
    for gr, mv in zip(grads, moves):
        eager['grad'].copy_(gr)
        eager['moved'].copy_(mv)
        body(eager)
    graphed = make()
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=stream):
        body(graphed)
    with torch.cuda.stream(stream):
        for gr, mv in zip(grads, moves):
            graphed['grad'].copy_(gr)
            graphed['moved'].copy_(mv)
            graph.replay()
    stream.synchronize()
    torch.cuda.synchronize()
    for k in ('param', 'm', 'v', 'step', 'accum', 'avg', 'buffers', 'skip'):
        assert torch.equal(graphed[k], eager[k]), k
    assert int(eager['step']) == 7 + 4 and float(eager['accum'][6]) == 4.0
    assert torch.isfinite(eager['param']).all() and torch.isfinite(eager['avg']).all()


# ---------------------------------------------------------------------------------------------------------------- learner
with open(os.path.join(GOLDEN, 'step_cases.pkl'), 'rb') as f:
    STEP_CASES = pickle.load(f)
with open(os.path.join(GOLDEN, 'net_step_cases.pkl'), 'rb') as f:
    NET_CASES = pickle.load(f)
KINDS = ['tictactoe', 'geese', 'geister']


def _setup(kind):
    """(net factory, args, [three good batches], lr): the fused-tower TicTacToe net, the module-path Geese net or the recurrent
    Geister net."""
    if kind == 'tictactoe':
        from handyrl_b200.nets import tictactoe_net, load_state_by_order
        from handyrl_b200.synthetic import synthetic_batch
        c = STEP_CASES[sorted(STEP_CASES)[0]]
        B, T, P, A = c['dims']
        args = c['args']
        batches = [synthetic_batch(B, T, P, A, turn_based=args['turn_based_training'], observation=args['observation'], seed=60 + s)
                   for s in range(3)]
        return (lambda: load_state_by_order(tictactoe_net(), c['state0'])), args, batches, c['lr']
    from conftest import net_case_setup
    name = [n for n in sorted(NET_CASES) if NET_CASES[n]['net'] == kind][0]
    c = NET_CASES[name]
    _, batches = net_case_setup(c)
    return (lambda: net_case_setup(c)[0]), c['args'], list(batches[:3]), c['lr']


def _poisoned(batch, args):
    """The batch with NaN in one observation element of one window, at a trained step where a player has the turn."""
    from handyrl_b200.batch import tree_leaves
    bad = {k: (copy.deepcopy(v) if k == 'observation' else v) for k, v in batch.items()}
    burn = args.get('burn_in_steps', 0)
    tm = batch['turn_mask'][:, burn:].reshape(batch['turn_mask'].shape[0], -1, batch['turn_mask'].shape[2])
    b, t, p = [int(x) for x in (tm > 0).nonzero()[0]]
    leaf = tree_leaves(bad['observation'])[0]
    leaf[b, burn + t, p if leaf.shape[2] > 1 else 0].view(-1)[0] = NAN
    return bad


def _template(kind):
    from handyrl_b200 import nets
    return {'tictactoe': nets.tictactoe_net, 'geese': nets.geese_net, 'geister': nets.geister_net}[kind]()


def _run(kind, order, guard, use_graph=True, time_loss_kernel=False, diagnostics=False, weight_ema=None, save_optimizer=False,
         keep=False):
    """Steps over the batches named in `order` ('b0', 'b1', 'b2', 'bad'); returns the learner's state (and the stepper when
    `keep`)."""
    from handyrl_b200.train import LearnerStep
    make, args, good, lr = _setup(kind)
    batches = {'b0': good[0], 'b1': good[1], 'b2': good[2], 'bad': _poisoned(good[1], args)}
    st = LearnerStep(make(), dict(args, skip_nonfinite=guard, diagnostics=diagnostics, weight_ema=weight_ema,
                                  save_optimizer=save_optimizer),
                     good[0], lr=lr, use_graph=use_graph, time_loss_kernel=time_loss_kernel, cudnn_benchmark=False)
    assert (st.engine is not None) == (kind == 'tictactoe') and st.skip_nonfinite == bool(guard)
    for name in order:
        st.step(st.new_packed().fill(batches[name]))
    st.stream.synchronize()
    out = {'bytes': st.state.bytes.cpu(), 'm': st.opt.exp_avg.cpu(), 'v': st.opt.exp_avg_sq.cpu(),
           'steps': int(st.opt.step_count), 'accum': st.accum.cpu(), 'launches': st.launches_per_step,
           'avg': st.avg_bytes.cpu() if st.avg is not None else None,
           'skipped': float(st.skipped) if st.skipped is not None else None, 'last': st.read_losses()}
    if keep:
        return out, st
    st.close()
    return out


@pytest.fixture
def deterministic_cudnn():
    # the Geese stem (17 input channels) stays on cuDNN: pin deterministic algorithms so that runs compare bit for bit
    old = torch.backends.cudnn.deterministic
    torch.backends.cudnn.deterministic = True
    yield
    torch.backends.cudnn.deterministic = old


def _assert_learners_equal(a, b, n_sums, what):
    for k in ('bytes', 'm', 'v', 'avg'):
        if a[k] is not None or b[k] is not None:
            assert torch.equal(a[k], b[k]), '%s: %s differs' % (what, k)
    assert a['steps'] == b['steps'], what
    assert torch.equal(a['accum'][:n_sums], b['accum'][:n_sums]), '%s: the sums differ' % what


@pytest.mark.parametrize('kind', KINDS)
def test_good_batches_train_alike_with_the_key_on_or_off(kind, deterministic_cudnn):
    off = _run(kind, ['b0', 'b1', 'b2'], False)
    on = _run(kind, ['b0', 'b1', 'b2'], True)
    _assert_learners_equal(off, on, 6, kind)
    assert on['skipped'] == 0.0 and off['skipped'] is None
    assert on['accum'].numel() == off['accum'].numel() + 1
    assert on['launches'] == off['launches'] + 1
    assert on['steps'] == 3


@pytest.mark.parametrize('kind', KINDS)
def test_the_bad_batch_poisons_an_unguarded_learner(kind, deterministic_cudnn):
    from handyrl_b200.batch import tree_leaves
    _, args, good, _ = _setup(kind)
    bad = _poisoned(good[1], args)
    assert sum(int(torch.isnan(t).sum()) for t in tree_leaves(bad['observation'])) == 1
    assert not any(torch.isnan(t).any() for t in tree_leaves(good[1]['observation']))      # the good batch is left alone
    out = _run(kind, ['b0', 'bad'], False)
    assert not torch.isfinite(out['bytes'][:out['m'].numel() * 4].view(torch.float32)).all()


@pytest.mark.parametrize('kind,use_graph', [('tictactoe', True), ('geese', True), ('geister', True), ('tictactoe', False)],
                         ids=['tictactoe', 'geese', 'geister', 'tictactoe-eager'])
def test_a_rejected_batch_leaves_the_learner_as_if_never_drawn(kind, use_graph, deterministic_cudnn):
    opts = dict(use_graph=use_graph, diagnostics=True, weight_ema=0.7)
    with_bad = _run(kind, ['b0', 'b1', 'bad', 'b2'], True, **opts)
    without = _run(kind, ['b0', 'b1', 'b2'], True, **opts)
    n_sums = with_bad['accum'].numel() - 1               # loss sums and diagnostics sums; the last slot counts rejections
    _assert_learners_equal(with_bad, without, n_sums, kind)
    assert with_bad['skipped'] == 1.0 and without['skipped'] == 0.0
    assert with_bad['steps'] == 3
    assert torch.isfinite(with_bad['bytes'][:with_bad['m'].numel() * 4].view(torch.float32)).all()
    assert with_bad['avg'] is not None and float(with_bad['accum'][6:6 + 20].abs().sum()) > 0


def test_the_loss_kernel_split_rejects_alike(deterministic_cudnn):
    graph = _run('tictactoe', ['b0', 'bad', 'b1'], True)
    split = _run('tictactoe', ['b0', 'bad', 'b1'], True, time_loss_kernel=True)
    _assert_learners_equal(graph, split, 7, 'time_loss_kernel')
    assert split['skipped'] == 1.0


def test_last_losses_show_the_rejected_step():
    # the rejected step's raw sums, as an unguarded learner computes them (the fused tower's ReLU may keep them finite while
    # the gradient is not)
    on = _run('tictactoe', ['b0', 'bad'], True)
    off = _run('tictactoe', ['b0', 'bad'], False)
    assert on['skipped'] == 1.0
    assert torch.equal(torch.tensor(list(on['last'].values())).nan_to_num(7.0), torch.tensor(list(off['last'].values())).nan_to_num(7.0))


@pytest.mark.parametrize('kind', ['tictactoe', 'geese'])
def test_end_epoch_hands_over_the_count_and_prints_the_line(kind, capsys, deterministic_cudnn):
    from handyrl_b200.train import LOSS_KEYS
    out, st = _run(kind, ['b0', 'b1', 'bad', 'b2'], True, save_optimizer=True, keep=True)
    heads = ['p'] + (['v'] if st.loss_buf.dvalue is not None else []) + (['r'] if st.loss_buf.dreturn is not None else []) + \
        ['ent', 'total']
    capsys.readouterr()
    pending = st.end_epoch(4, 4, 3e-8, _template(kind), heads)
    model, sums = pending.resolve()
    lines = capsys.readouterr().out.splitlines()
    assert pending.skipped == 1
    assert lines[-1] == 'skipped = 1 of 4 steps: non-finite loss or gradient'
    loss = [l for l in lines if l.startswith('loss = ')]
    assert len(loss) == 1 and lines.index(loss[0]) < len(lines) - 1
    assert all(np.isfinite(float(v)) for v in re.findall(r':(-?[0-9.]+|nan|-?inf)', loss[0]))
    assert all(np.isfinite(sums[k]) for k in LOSS_KEYS)
    state = pending.optim_state
    assert all(int(s['step']) == 3 for s in state['optimizer']['state'].values())
    assert all(torch.isfinite(s['exp_avg']).all() and torch.isfinite(s['exp_avg_sq']).all()
               for s in state['optimizer']['state'].values())
    assert all(torch.isfinite(v).all() for v in model.state_dict().values() if v.is_floating_point())
    # the next epoch starts from a zero count
    st.step(st.new_packed().fill(_setup(kind)[2][0]))
    st.stream.synchronize()
    assert float(st.skipped) == 0.0
    st.close()


# ---------------------------------------------------------------------------------------------------------------- trainer
def _poison_episode(ep):
    """A copy of an episode (compressed moments) whose every observation holds a NaN."""
    ep = copy.deepcopy(ep)
    blocks = []
    for blob in ep['moment']:
        moments = pickle.loads(bz2.decompress(blob))
        for m in moments:
            for p, o in m['observation'].items():
                if o is not None:
                    o = np.array(o, copy=True)
                    o.reshape(-1)[0] = np.nan
                    m['observation'][p] = o
        blocks.append(bz2.compress(pickle.dumps(moments)))
    ep['moment'] = blocks
    return ep


def _wait_steps(tr, n, timeout=300):
    t0 = time.time()
    while tr.steps < n:
        assert time.time() - t0 < timeout, 'the trainer made %d of %d steps' % (tr.steps, n)
        time.sleep(0.01)


def test_trainer_survives_an_episode_with_a_nan(capsys):
    from handyrl_b200.nets import tictactoe_net
    from handyrl_b200.train import Trainer
    with open(os.path.join(GOLDEN, 'batch_cases.pkl'), 'rb') as f:
        case = pickle.load(f)['tictactoe']
    args = dict(case['args'], batch_size=8, minimum_episodes=4, num_batchers=1, **{'lambda': 0.7},
                entropy_regularization=0.1, entropy_regularization_decay=0.1, policy_target='UPGO', value_target='VTRACE',
                gpu_replay=True, num_gpus=1, skip_nonfinite=True)
    episodes = list(case['episodes'])
    episodes[3] = _poison_episode(episodes[3])
    benchmark = torch.backends.cudnn.benchmark          # the Trainer's learner turns cuDNN autotuning on for the process
    tr = Trainer(args, tictactoe_net())
    tr.episodes.extend(episodes)
    th = threading.Thread(target=tr.run, daemon=True)
    th.start()
    models = []
    try:
        for target in (20, 40):              # epochs of at least 20 steps: one in eight windows comes from the bad episode
            _wait_steps(tr, target)
            models.append(tr.update()[0])
    finally:
        tr.stop()
        th.join(timeout=10)
        torch.backends.cudnn.benchmark = benchmark
    for model in models:
        for k, v in model.state_dict().items():
            if v.is_floating_point():
                assert torch.isfinite(v).all(), k
    lines = capsys.readouterr().out.splitlines()
    assert any(re.fullmatch(r'skipped = [1-9][0-9]* of [1-9][0-9]* steps: non-finite loss or gradient', l) for l in lines)
    losses = [l for l in lines if l.startswith('loss = ')]
    assert losses and not any('nan' in l for l in losses)


# ---------------------------------------------------------------------------------------------------------------- multi-GPU
NGPU = torch.cuda.device_count() if torch.cuda.is_available() else 0
MG_ARGS = {'turn_based_training': True, 'observation': False, 'gamma': 0.8, 'lambda': 0.7, 'burn_in_steps': 0, 'forward_steps': 8,
           'entropy_regularization': 0.1, 'entropy_regularization_decay': 0.1, 'policy_target': 'UPGO', 'value_target': 'VTRACE',
           'skip_nonfinite': True}
MG_DIMS = (16, 8, 2, 9)


def _mg_rank(rank, world, port, out_dir):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    from handyrl_b200.multigpu import shard_batch, shard_bounds
    from handyrl_b200.nets import BoardNet
    from handyrl_b200.synthetic import synthetic_batch
    from handyrl_b200.train import LearnerStep
    torch.cuda.set_device(rank)
    dist.init_process_group('nccl', init_method='tcp://127.0.0.1:%d' % port, rank=rank, world_size=world,
                            device_id=torch.device('cuda', rank))
    B, T, P, A = MG_DIMS
    full = [synthetic_batch(B, T, P, A, turn_based=True, observation=False, seed=700 + s) for s in range(3)]
    bad = {k: (v.clone() if k == 'observation' else v) for k, v in full[1].items()}
    lo, _ = shard_bounds(B, 1, world)
    bad['observation'][lo, 0, 0].view(-1)[0] = float('nan')           # only in rank 1's shard
    res = {}
    for peer in (True, False):
        torch.manual_seed(11)
        st = LearnerStep(BoardNet(norm=False), MG_ARGS, shard_batch(full[0], rank, world), lr=1e-3,
                         device=torch.device('cuda', rank), process_group=dist.group.WORLD, peer_allreduce=peer)
        for b in (full[0], bad, full[2]):
            st.step(st.new_packed().fill(shard_batch(b, rank, world)))
        st.stream.synchronize()
        res[peer] = {'bytes': st.state.bytes.cpu(), 'm': st.opt.exp_avg.cpu(), 'steps': int(st.opt.step_count),
                     'skipped': float(st.skipped), 'sums': st.accum.cpu()}
        st.close()
    with open(os.path.join(out_dir, 'rank%d.pkl' % rank), 'wb') as f:
        pickle.dump(res, f)
    dist.barrier()
    torch.cuda.synchronize()
    dist.destroy_process_group()


@pytest.mark.skipif(NGPU < 2, reason='needs at least 2 GPUs')
def test_a_nan_in_one_shard_makes_every_rank_reject():
    import torch.multiprocessing as mp
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        port = s.getsockname()[1]
    out_dir = tempfile.mkdtemp(prefix='hrl_guard_')
    mp.spawn(_mg_rank, args=(2, port, out_dir), nprocs=2, join=True)
    res = [pickle.load(open(os.path.join(out_dir, 'rank%d.pkl' % r), 'rb')) for r in range(2)]
    for peer in (True, False):
        for r in range(2):
            assert res[r][peer]['skipped'] == 1.0 and res[r][peer]['steps'] == 2, (peer, r)
            assert torch.isfinite(res[r][peer]['m']).all()
        for k in ('bytes', 'm', 'sums'):
            assert torch.equal(res[0][peer][k], res[1][peer][k]), (peer, k)
