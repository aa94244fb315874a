"""Moving average of the learner's weights on the GPU: hrl_weight_ema against a float64 recurrence of its rule, graph replays, no side
effect on training, the per-epoch hand-off, the Trainer's files and restart seed, and sharded learners."""
import os
import pickle
import socket
import sys
import tempfile
import threading

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT

pytestmark = pytest.mark.gpu


def rule_weight(t, decay, seeded):
    """w of the rule, in fp32 like the kernel: max(1 - d, 1 / t), or 1 - d once seeded."""
    keep = np.float32(1) - np.float32(decay)
    return float(keep if seeded else max(keep, np.float32(1) / np.float32(max(t, 1))))


def recurrence(xs, decay, seed=None, t0=0):
    """float64 average over the live states xs (after steps t0 + 1, t0 + 2, ...); starts from `seed` when given."""
    a = np.zeros_like(xs[0], dtype=np.float64) if seed is None else np.asarray(seed, np.float64).copy()
    for i, x in enumerate(xs):
        w = rule_weight(t0 + i + 1, decay, seed is not None)
        a = a + w * (np.asarray(x, np.float64) - a)
    return a


def assert_near(got, ref, err=''):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    bad = np.abs(got - ref) > 1e-6 + 1e-5 * np.abs(ref)
    assert not bad.any(), '%s: %d of %d off, worst %g' % (err, bad.sum(), bad.size, np.abs(got - ref).max())


# ---------------------------------------------------------------------------------------------------------------- the kernel
@pytest.mark.parametrize('seeded', [False, True], ids=['fresh', 'seeded'])
@pytest.mark.parametrize('decay', [0.9, 0.999])
@pytest.mark.parametrize('n', [1, 3, 5, 1027, 29008])
def test_kernel_against_a_float64_recurrence(n, decay, seeded):
    from handyrl_b200 import ops
    g = torch.Generator().manual_seed(n)
    start = torch.randn(n, generator=g)
    avg = start.cuda()
    step = torch.zeros(1, dtype=torch.int64, device='cuda')       # the optimiser's counter, on the device
    xs = [torch.randn(n, generator=g) + 0.5 for _ in range(50)]
    x_dev = torch.empty(n, device='cuda')
    got = []
    for x in xs:
        step.add_(1)
        x_dev.copy_(x)
        ops.weight_ema_update(avg, x_dev, step, decay, seeded)
        got.append(avg.cpu().numpy())
    torch.cuda.synchronize()
    seed = start.numpy() if seeded else None
    for k in (1, 2, 10, 50):
        want = recurrence([x.numpy() for x in xs[:k]], decay, seed=seed)
        assert_near(got[k - 1], want, 'n=%d d=%g after %d steps' % (n, decay, k))
    if not seeded:
        assert np.array_equal(got[0], xs[0].numpy())              # the first step copies


def test_kernel_in_a_graph_replays_like_eager_launches():
    from handyrl_b200 import ops
    n, K, decay = 29008, 20, 0.99
    g = torch.Generator().manual_seed(5)
    xs = [torch.randn(n, generator=g).cuda() for _ in range(K)]
    start = torch.randn(n, generator=g).cuda()
    eager = start.clone()
    step = torch.zeros(1, dtype=torch.int64, device='cuda')
    for x in xs:
        step.add_(1)
        ops.weight_ema_update(eager, x, step, decay, False)
    graphed, x_in = start.clone(), torch.empty(n, device='cuda')
    step_g = torch.zeros(1, dtype=torch.int64, device='cuda')
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    before = ops.LAUNCHES['n']
    with torch.cuda.graph(graph, stream=stream):
        step_g.add_(1)
        ops.weight_ema_update(graphed, x_in, step_g, decay, False)
    assert ops.LAUNCHES['n'] - before == 1
    with torch.cuda.stream(stream):
        for x in xs:
            x_in.copy_(x)
            graph.replay()
    stream.synchronize()
    torch.cuda.synchronize()
    assert int(step_g) == K
    assert torch.equal(graphed, eager)


def test_kernel_refuses_bad_arguments():
    from handyrl_b200 import ops, _capi
    a, step = torch.zeros(8, device='cuda'), torch.zeros(1, dtype=torch.int64, device='cuda')
    calls = [(a, a, bad) for bad in (0.0, 1.0, -0.5, float('nan'))]
    calls += [(a, torch.zeros(7, device='cuda'), 0.9), (a[1:], a[:7], 0.9)]       # sizes differ; not 16-byte aligned
    raised = []

    def refused():           # the library's error text is per thread: keep the main thread's clean
        for avg, x, d in calls:
            try:
                ops.weight_ema_update(avg, x, step, d, False)
            except _capi.HrlError:
                raised.append(True)

    th = threading.Thread(target=refused)
    th.start()
    th.join()
    assert len(raised) == len(calls)
    assert torch.equal(a.cpu(), torch.zeros(8))


# ---------------------------------------------------------------------------------------------------------------- learner step
with open(os.path.join(GOLDEN, 'step_cases.pkl'), 'rb') as f:
    STEP_CASES = pickle.load(f)
with open(os.path.join(GOLDEN, 'net_step_cases.pkl'), 'rb') as f:
    NET_CASES = pickle.load(f)
NSTEPS = 5
DECAY = 0.7          # w = 1, 1/2, 1/3, then 1 - d: both regimes of the rule within five steps


def _setup(kind):
    """(net factory, args, [batches], lr) of a fused-tower TicTacToe case or a module-path Geese case."""
    if kind == 'tictactoe':
        from handyrl_b200.nets import tictactoe_net, load_state_by_order
        from handyrl_b200.synthetic import synthetic_batch
        c = STEP_CASES[sorted(STEP_CASES)[0]]
        B, T, P, A = c['dims']
        args = c['args']
        batches = [synthetic_batch(B, T, P, A, turn_based=args['turn_based_training'], observation=args['observation'], seed=40 + s)
                   for s in range(NSTEPS)]
        return (lambda: load_state_by_order(tictactoe_net(), c['state0'])), args, batches, c['lr']
    from conftest import net_case_setup
    name = [n for n in sorted(NET_CASES) if NET_CASES[n]['net'] == 'geese'][0]
    c = NET_CASES[name]
    _, batches = net_case_setup(c)
    batches = (batches * NSTEPS)[:NSTEPS]
    return (lambda: net_case_setup(c)[0]), c['args'], batches, c['lr']


def _run(kind, decay, use_graph, per_step=False):
    from handyrl_b200.train import LearnerStep
    make, args, batches, lr = _setup(kind)
    st = LearnerStep(make(), dict(args, weight_ema=decay), batches[0], lr=lr, use_graph=use_graph, cudnn_benchmark=False)
    assert (st.engine is not None) == (kind == 'tictactoe')
    states = []
    for b in batches:
        st.step(st.new_packed().fill(b))
        if per_step:
            states.append(st.cpu_state_dict())
    st.stream.synchronize()
    out = {'live': st.cpu_state_dict(), 'm': st.opt.exp_avg.cpu(), 'v': st.opt.exp_avg_sq.cpu(), 'sums': st.accum.cpu(),
           'steps': int(st.opt.step_count), 'launches': st.launches_per_step, 'states': states,
           'avg': st.ema_state_dict() if decay else None, 'has_avg': st.avg is not None}
    st.close()
    return out


@pytest.fixture
def deterministic_cudnn():
    # the Geese stem (17 input channels) stays on cuDNN: pin deterministic algorithms so that runs compare bit for bit
    old = torch.backends.cudnn.deterministic
    torch.backends.cudnn.deterministic = True
    yield
    torch.backends.cudnn.deterministic = old


@pytest.mark.parametrize('kind', ['tictactoe', 'geese'])
def test_averaging_leaves_training_alone_and_follows_the_rule(kind, deterministic_cudnn):
    off = _run(kind, None, use_graph=True)
    on = _run(kind, DECAY, use_graph=True)
    assert not off['has_avg'] and on['has_avg']
    for k in off['live']:
        assert torch.equal(off['live'][k], on['live'][k]), k
    for k in ('m', 'v', 'sums'):
        assert torch.equal(off[k], on[k]), k
    assert on['launches'] == off['launches'] + 1
    assert on['steps'] == NSTEPS
    eager = _run(kind, DECAY, use_graph=False, per_step=True)
    assert eager['launches'] == on['launches']
    for k in on['live']:
        assert torch.equal(eager['live'][k], on['live'][k]), 'graph and eager live weights differ: %s' % k
    for k in on['avg']:
        assert torch.equal(eager['avg'][k], on['avg'][k]), 'graph and eager averages differ: %s' % k
    assert list(on['avg']) == list(on['live'])
    n_f32 = 0
    for k, v in eager['avg'].items():
        if v.dtype == torch.float32:          # parameters and BatchNorm running statistics
            want = recurrence([s[k].numpy() for s in eager['states']], DECAY)
            assert_near(v.numpy(), want, k)
            n_f32 += 1
        else:                                 # int64 buffers: the live model's
            assert torch.equal(v, eager['live'][k]), k
    assert n_f32 > 0 and any(k.endswith('running_var') for k in eager['avg'])
    assert any(v.dtype == torch.int64 for v in eager['avg'].values())


@pytest.mark.parametrize('kind', ['tictactoe', 'geese'])
def test_end_epoch_hands_over_the_average(kind, deterministic_cudnn):
    from handyrl_b200 import nets
    from handyrl_b200.train import LearnerStep
    make, args, batches, lr = _setup(kind)
    st = LearnerStep(make(), dict(args, weight_ema=0.9), batches[0], lr=lr, cudnn_benchmark=False)
    for b in batches:
        st.step(st.new_packed().fill(b))
    want = st.ema_state_dict()
    template = nets.tictactoe_net() if kind == 'tictactoe' else nets.geese_net()
    pending = st.end_epoch(len(batches), NSTEPS, 3e-8, template, ['p', 'v', 'ent', 'total'])
    model, sums = pending.resolve()
    got = pending.ema_state
    assert list(got) == list(template.state_dict())
    for k in got:
        assert torch.equal(got[k], want[k]), k
    fresh = nets.tictactoe_net() if kind == 'tictactoe' else nets.geese_net()
    fresh.load_state_dict(got, strict=True)
    # the returned model is the live one
    live = st.cpu_state_dict()
    for k, v in model.state_dict().items():
        assert torch.equal(v, live[k]), k
    st.close()


# ---------------------------------------------------------------------------------------------------------------- trainer
def _trainer_args(**extra):
    with open(os.path.join(GOLDEN, 'batch_cases.pkl'), 'rb') as f:
        case = pickle.load(f)['tictactoe']
    args = dict(case['args'], batch_size=8, minimum_episodes=4, num_batchers=1, **{'lambda': 0.7},
                entropy_regularization=0.1, entropy_regularization_decay=0.1, policy_target='UPGO', value_target='VTRACE',
                gpu_replay=True, num_gpus=1, **extra)
    return args, case['episodes']


def _two_epochs(args, episodes):
    from handyrl_b200.nets import tictactoe_net
    from handyrl_b200.train import Trainer
    tr = Trainer(args, tictactoe_net())
    tr.episodes.extend(episodes)
    th = threading.Thread(target=tr.run, daemon=True)
    th.start()
    try:
        tr.update()
        tr.update()
    finally:
        tr.stop()
        th.join(timeout=10)
    return tr


def test_trainer_writes_and_resumes_the_average(tmp_path, monkeypatch):
    from handyrl_b200.nets import tictactoe_net
    from handyrl_b200.train import Trainer
    monkeypatch.chdir(tmp_path)
    decay = 0.9
    args, episodes = _trainer_args(weight_ema=decay)
    tr = _two_epochs(args, episodes)
    assert sorted(os.listdir('models')) == ['1.ema.pth', '2.ema.pth', 'latest.ema.pth']
    latest, second = torch.load('models/latest.ema.pth'), torch.load('models/2.ema.pth')
    assert all(torch.equal(latest[k], second[k]) for k in second)
    fresh = tictactoe_net()
    fresh.load_state_dict(second, strict=True)
    launches_on = tr.stepper.launches_per_step

    # a run restarted at epoch 2 resumes from 2.ema.pth: after its first step, avg = d seed + (1 - d) live
    tr = Trainer(dict(args, restart_epoch=2), tictactoe_net())
    tr.episodes.extend(episodes)
    try:
        tr._start_stepper()
        st = tr.stepper
        assert st.avg_seeded
        st.step(st.new_packed().fill(tr.batcher._make()))
        avg, live = st.ema_state_dict(), st.cpu_state_dict()
    finally:
        tr.stop()
    for k, v in avg.items():
        if v.dtype == torch.float32:
            want = decay * second[k].double() + (1 - decay) * live[k].double()
            assert_near(v.numpy(), want.numpy(), k)
        else:
            assert torch.equal(v, live[k]), k

    # without the key: no file, and the step has one launch fewer
    (tmp_path / 'off').mkdir()
    monkeypatch.chdir(tmp_path / 'off')
    args_off, _ = _trainer_args()
    tr = _two_epochs(args_off, episodes)
    assert os.listdir('.') == []
    assert tr.stepper.avg is None and tr.ema_files is None
    assert tr.stepper.launches_per_step == launches_on - 1


# ---------------------------------------------------------------------------------------------------------------- multi-GPU
NGPU = torch.cuda.device_count() if torch.cuda.is_available() else 0
MG_ARGS = {'turn_based_training': True, 'observation': False, 'gamma': 0.8, 'lambda': 0.7, 'burn_in_steps': 0, 'forward_steps': 8,
           'entropy_regularization': 0.1, 'entropy_regularization_decay': 0.1, 'policy_target': 'UPGO', 'value_target': 'VTRACE',
           'weight_ema': 0.9}
MG_DIMS = (16, 8, 2, 9)


def _mg_rank(rank, world, port, out_dir):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    from handyrl_b200.multigpu import shard_batch
    from handyrl_b200.nets import BoardNet
    from handyrl_b200.synthetic import synthetic_batch
    from handyrl_b200.train import LearnerStep
    torch.cuda.set_device(rank)
    dist.init_process_group('nccl', init_method='tcp://127.0.0.1:%d' % port, rank=rank, world_size=world,
                            device_id=torch.device('cuda', rank))
    B, T, P, A = MG_DIMS
    full = [synthetic_batch(B, T, P, A, turn_based=True, observation=False, seed=900 + s) for s in range(3)]
    res = {}
    for helpers_average in (False, True):
        torch.manual_seed(11)
        # helper ranks as multigpu.py builds them (no average), then with one of their own
        decay = None if (rank == 0 or helpers_average) else 0
        st = LearnerStep(BoardNet(norm=False), MG_ARGS, shard_batch(full[0], rank, world), lr=1e-3,
                         device=torch.device('cuda', rank), process_group=dist.group.WORLD, weight_ema=decay)
        for b in full:
            st.step(st.new_packed().fill(shard_batch(b, rank, world)))
        res[helpers_average] = {'has_avg': st.avg is not None, 'live': st.cpu_state_dict(),
                                'avg': st.ema_state_dict() if st.avg is not None else None}
        st.close()
    with open(os.path.join(out_dir, 'rank%d.pkl' % rank), 'wb') as f:
        pickle.dump(res, f)
    dist.barrier()
    torch.cuda.synchronize()
    dist.destroy_process_group()


@pytest.mark.skipif(NGPU < 2, reason='needs at least 2 GPUs')
def test_only_rank0_averages_and_helpers_do_not_change_it():
    import torch.multiprocessing as mp
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        port = s.getsockname()[1]
    out_dir = tempfile.mkdtemp(prefix='hrl_ema_')
    mp.spawn(_mg_rank, args=(2, port, out_dir), nprocs=2, join=True)
    res = [pickle.load(open(os.path.join(out_dir, 'rank%d.pkl' % r), 'rb')) for r in range(2)]
    assert res[0][False]['has_avg'] and not res[1][False]['has_avg'] and res[1][True]['has_avg']
    for k in res[0][False]['avg']:
        assert torch.equal(res[0][False]['avg'][k], res[0][True]['avg'][k]), k
    for k in res[0][False]['live']:           # every rank holds the same weights
        assert torch.equal(res[0][False]['live'][k], res[1][False]['live'][k]), k
