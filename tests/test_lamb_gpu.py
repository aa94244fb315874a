"""The LAMB optimiser on the GPU (train_args['optimizer'] = 'lamb', ops.FlatLamb, hrl_clip_lamb_step): the kernels against the
float64 restatement (tests/lamb_ref.py) on the reference nets' bucket layouts, reproducibility under graph replay, the learner
against the eager CPU step with LAMB in place of Adam, the key off, the non-finite guard, the checkpoint round trip and the
sharded step."""
import os
import pickle
import sys
import tempfile

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from lamb_ref import Lamb64, lamb_step

pytestmark = pytest.mark.gpu

with open(os.path.join(GOLDEN, 'step_cases.pkl'), 'rb') as f:
    STEP_CASES = pickle.load(f)
with open(os.path.join(GOLDEN, 'net_step_cases.pkl'), 'rb') as f:
    NET_CASES = pickle.load(f)
NETS = ['tictactoe', 'geister', 'geese']
HP = dict(max_norm=4.0, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-5)
LR, LR_SCALE, T0 = 1e-3, 2.0, 4          # T0: the step count before the step under test


@pytest.fixture
def deterministic_cudnn():
    old = (torch.backends.cudnn.deterministic, torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.deterministic = True
    yield
    torch.backends.cudnn.deterministic, torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


# ---------------------------------------------------------------------------------------------------------------- kernels


def _shapes(name):
    from handyrl_b200 import nets
    net = {'tictactoe': nets.tictactoe_net, 'geister': nets.geister_net, 'geese': nets.geese_net}[name]()
    return [tuple(p.shape) for p in net.parameters()]


def _start(name, clip, seed=5):
    """Random weights (tensor 1 all zero: r = 1), moments and gradients on the bucket layout of net `name`; the gradient's
    norm is 40 (clip active) or 1 (inactive)."""
    g = torch.Generator().manual_seed(seed)
    numels = [int(np.prod(s)) for s in _shapes(name)]
    n = sum(numels)
    w = 0.5 * torch.randn(n, generator=g)
    w[numels[0]:numels[0] + numels[1]] = 0.0
    grad = torch.randn(n, generator=g)
    grad *= (40.0 if clip else 1.0) / float(grad.norm())
    return {'numels': numels, 'w': w, 'g': grad, 'm': 0.01 * torch.randn(n, generator=g), 'v': 1e-4 * torch.rand(n, generator=g)}


def _optimiser(start, form):
    """A FlatLamb over CUDA parameters of the start's shapes, its buffers set to `start`, in `form` ('plain', 'diag', 'guard')."""
    from handyrl_b200 import ops
    params = [torch.nn.Parameter(torch.zeros(k, device='cuda')) for k in start['numels']]
    opt = ops.FlatLamb(params, lr=LR, lr_scale=LR_SCALE, extra=8, **HP)
    n = opt.n
    with torch.no_grad():
        opt.flat_param[:n].copy_(start['w'])
        opt.flat_grad[:n].copy_(start['g'])
        opt.exp_avg[:n].copy_(start['m'])
        opt.exp_avg_sq[:n].copy_(start['v'])
    opt.step_count.fill_(T0)
    opt.ratio = torch.zeros(len(params), device='cuda')
    if form == 'diag':
        opt.diag = torch.zeros(4, dtype=torch.float64, device='cuda')
    if form == 'guard':
        opt.skip = torch.full((1,), 7, dtype=torch.int32, device='cuda')
        opt.guard_tail = 6
    return opt


def _split(flat, numels):
    out, off = [], 0
    for k in numels:
        out.append(flat[off:off + k])
        off += k
    return out


def _state(opt):
    torch.cuda.synchronize()
    return {'w': opt.flat_param.cpu(), 'm': opt.exp_avg.cpu(), 'v': opt.exp_avg_sq.cpu(), 'step': int(opt.step_count),
            'ratio': opt.ratio.cpu(), 'gnorm': opt.grad_norm.cpu()}


@pytest.mark.parametrize('form', ['diag', 'guard'])
@pytest.mark.parametrize('clip', [True, False], ids=['clip', 'noclip'])
@pytest.mark.parametrize('name', NETS)
def test_kernel_matches_the_float64_restatement(name, clip, form):
    """Weights, moments and each tensor's ratio against lamb_ref.lamb_step on the fp32 inputs: the moments and ratios to 1e-5,
    the weights to 1e-6 of their size and each tensor's step to 1e-3 of its largest element (the fp32 rounding of w)."""
    start = _start(name, clip)
    opt = _optimiser(start, form)
    opt.step()
    got = _state(opt)
    nm = start['numels']
    w, m, v, r, norm = lamb_step(_split(start['w'], nm), _split(start['g'], nm), _split(start['m'], nm), _split(start['v'], nm),
                                 T0 + 1, LR, LR_SCALE, **HP)
    assert (norm > 4.0) == clip
    assert got['step'] == T0 + 1
    assert abs(float(got['gnorm']) - norm) <= 1e-5 * norm
    np.testing.assert_allclose(got['ratio'].numpy(), r, rtol=1e-5)
    assert r[1] == 1.0 and float(got['ratio'][1]) == 1.0                # the all-zero tensor
    w0 = _split(start['w'].double().numpy(), nm)
    for i, (gw, gm, gv) in enumerate(zip(_split(got['w'].double().numpy(), nm), _split(got['m'].double().numpy(), nm),
                                         _split(got['v'].double().numpy(), nm))):
        np.testing.assert_allclose(gm, m[i], rtol=1e-5, atol=1e-6 * np.abs(m[i]).max(), err_msg='m of tensor %d' % i)
        np.testing.assert_allclose(gv, v[i], rtol=1e-5, atol=1e-6 * np.abs(v[i]).max(), err_msg='v of tensor %d' % i)
        np.testing.assert_allclose(gw, w[i], rtol=1e-6, atol=1e-6 * np.abs(w[i]).max(), err_msg='w of tensor %d' % i)
        step = w[i] - w0[i]
        np.testing.assert_allclose(gw - w0[i], step, rtol=1e-3, atol=1e-3 * np.abs(step).max(), err_msg='step of tensor %d' % i)
    n = opt.n
    assert (got['w'][n:] == 0).all() and (got['m'][n:] == 0).all() and (got['v'][n:] == 0).all()    # padding
    if form == 'diag':
        d = opt.diag.cpu().tolist()
        assert d[0] == float(got['gnorm']) and d[2] == (1.0 if clip else 0.0) and d[3] == 1.0
    else:
        assert int(opt.skip) == 0


@pytest.mark.parametrize('name', NETS)
def test_a_rejected_kernel_step_writes_nothing(name):
    start = _start(name, True)
    want = _state(_optimiser(start, 'guard'))
    for where in ('grad', 'tail'):
        opt = _optimiser(start, 'guard')
        opt.flat_grad[3 if where == 'grad' else opt.n_pad + 2] = float('nan')
        opt.step()
        got = _state(opt)
        assert int(opt.skip) == 1, where
        for k in ('w', 'm', 'v', 'ratio'):
            assert torch.equal(got[k], want[k]), (where, k)
        assert got['step'] == T0


def test_repeated_launches_and_graph_replays_are_bit_identical():
    start = _start('geese', True)
    a, b = _optimiser(start, 'plain'), _optimiser(start, 'plain')
    a.step()
    b.step()
    assert all(torch.equal(x, y) for x, y in zip(_state(a).values(), _state(b).values()) if torch.is_tensor(x))
    eager, graphed = _optimiser(start, 'guard'), _optimiser(start, 'guard')
    for _ in range(20):
        eager.step()
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=stream):
        graphed.step()
    with torch.cuda.stream(stream):
        for _ in range(20):
            graph.replay()
    stream.synchronize()
    e, g = _state(eager), _state(graphed)
    assert e['step'] == g['step'] == T0 + 20
    for k in ('w', 'm', 'v', 'ratio', 'gnorm'):
        assert torch.equal(e[k], g[k]), k
    assert torch.equal(eager.chunk_sums, graphed.chunk_sums) and torch.equal(eager.update, graphed.update)


# ---------------------------------------------------------------------------------------------------------------- learner


def _case(kind):
    """(net factory, args, [three batches], lr): the fused-tower TicTacToe net or the recurrent Geister net."""
    if kind == 'tictactoe':
        from handyrl_b200.nets import tictactoe_net, load_state_by_order
        from handyrl_b200.synthetic import synthetic_batch
        c = STEP_CASES[sorted(STEP_CASES)[0]]
        B, T, P, A = c['dims']
        args = c['args']
        batches = [synthetic_batch(B, T, P, A, turn_based=args['turn_based_training'], observation=args['observation'], seed=40 + s)
                   for s in range(3)]
        return (lambda: load_state_by_order(tictactoe_net(), c['state0'])), args, batches, c['lr']
    from conftest import net_case_setup
    c = NET_CASES[[n for n in sorted(NET_CASES) if NET_CASES[n]['net'] == kind][0]]
    _, batches = net_case_setup(c)
    return (lambda: net_case_setup(c)[0]), c['args'], list(batches[:3]), c['lr']


def _learn(kind, optimizer='lamb', use_graph=True, batches=None, **kw):
    from handyrl_b200.train import LearnerStep
    make, args, good, lr = _case(kind)
    args = dict(args, **kw.pop('args', {}))
    if optimizer is not None:
        args['optimizer'] = optimizer
    st = LearnerStep(make(), args, good[0], lr=lr, use_graph=use_graph, cudnn_benchmark=False, **kw)
    losses = []
    for b in (good if batches is None else batches):
        st.step(st.new_packed().fill(b))
        losses.append(st.read_losses())
    st.stream.synchronize()
    return st, losses


def _image(st):
    st.stream.synchronize()
    return {'bytes': st.state.bytes.cpu(), 'm': st.opt.exp_avg.cpu(), 'v': st.opt.exp_avg_sq.cpu(), 'step': int(st.opt.step_count)}


def _same(a, b):
    return [k for k in a if not (torch.equal(a[k], b[k]) if torch.is_tensor(a[k]) else a[k] == b[k])]


@pytest.mark.parametrize('kind', ['tictactoe', 'geister'])
def test_three_learner_steps_match_the_cpu_step_with_lamb(kind, deterministic_cudnn):
    """LearnerStep with the key against oracle.torch_learner.CpuLearner with Lamb64 in place of Adam, to the bounds of the
    Adam step tests (test_step_gpu); eager and graph runs bit for bit."""
    from oracle.torch_learner import CpuLearner
    from conftest import noise_driven
    from handyrl_b200 import ops
    make, args, batches, lr = _case(kind)
    ref = CpuLearner(make(), args, lr=lr)
    ref.opt = Lamb64(ref.params, lr=lr, **{k: HP[k] for k in ('betas', 'eps', 'weight_decay')})
    graph, losses = _learn(kind)
    assert graph.optimizer == {'name': 'lamb', 'lr_scale': 1.0} and isinstance(graph.opt, ops.FlatLamb)
    for s, (b, got) in enumerate(zip(batches, losses)):
        want, dcnt = ref.step(b)
        scale = max(abs(v) for v in want.values())
        for k, v in want.items():
            assert abs(got[k] - v) <= (1 + s) * 1e-4 * scale + 1e-4, (s, k, got[k], v)
        assert got['dcnt'] == dcnt
    final = graph.cpu_state_dict()
    case = {'net': kind}
    for key, vr in ref.net.state_dict().items():
        v = final[key]
        if noise_driven(case, key):
            continue
        if v.dtype.is_floating_point:
            bad = np.abs(v.numpy() - vr.numpy()) > 5e-5 + 1e-3 * np.abs(vr.numpy())
            assert bad.mean() <= 1e-3, '%s: %d of %d elements differ' % (key, bad.sum(), bad.size)
            np.testing.assert_allclose(v.numpy(), vr.numpy(), rtol=1e-3, atol=2 * lr * len(batches) + 5e-5, err_msg=key)
        else:
            assert int(v) == int(vr), key
    eager, eager_losses = _learn(kind, use_graph=False)
    assert eager_losses == losses and _same(_image(eager), _image(graph)) == []
    eager.close()
    graph.close()


def test_key_off_is_adam_bit_for_bit_and_lamb_adds_one_launch(deterministic_cudnn):
    """The key absent, None and 'adam' run the same launches to the same bits; 'lamb' takes one launch more per step."""
    runs = {}
    for key, args in (('absent', {}), (None, {'optimizer': None}), ('adam', {'optimizer': 'adam'}), ('lamb', {'optimizer': 'lamb'})):
        st, losses = _learn('tictactoe', optimizer=None, args=args)
        runs[key] = (st.launches_per_step, losses, _image(st), type(st.opt).__name__, st.optimizer)
        st.close()
    base = runs['absent']
    assert base[3] == 'FlatAdam' and base[4] == {'name': 'adam'}
    for key in (None, 'adam'):
        assert runs[key][0] == base[0] and runs[key][1] == base[1] and _same(runs[key][2], base[2]) == [] and runs[key][3] == 'FlatAdam'
    assert runs['lamb'][3] == 'FlatLamb' and runs['lamb'][0] == base[0] + 1
    assert _same(runs['lamb'][2], base[2]) != []


@pytest.mark.parametrize('kind', ['tictactoe', 'geister'])
def test_a_poisoned_step_leaves_the_lamb_learner_untouched(kind, deterministic_cudnn):
    from test_nonfinite_guard_gpu import _poisoned
    _, args, good, _ = _case(kind)
    bad = _poisoned(good[1], args)
    with_bad, _ = _learn(kind, batches=[good[0], bad], args={'skip_nonfinite': True})
    without, _ = _learn(kind, batches=[good[0]], args={'skip_nonfinite': True})
    assert float(with_bad.skipped) == 1.0 and int(with_bad.opt.skip) == 1
    assert _same(_image(with_bad), _image(without)) == []
    assert _image(with_bad)['step'] == 1
    with_bad.close()
    without.close()


def test_checkpoint_round_trip_continues_bit_for_bit(deterministic_cudnn):
    """optimizer_state_dict() after 2 steps, loaded with the weights into a fresh LAMB learner: its third step equals the
    uninterrupted learner's bit for bit.  An Adam learner refuses the file, and a LAMB learner an Adam file, changing nothing."""
    from handyrl_b200.train import LearnerStep
    make, args, batches, lr = _case('tictactoe')
    whole, _ = _learn('tictactoe')
    first, _ = _learn('tictactoe', batches=batches[:2])
    saved, weights = first.optimizer_state_dict(), first.cpu_state_dict()
    assert saved['algorithm'] == 'lamb' and saved['lr_scale'] == 1.0
    first.close()
    net = make()
    net.load_state_dict(weights)
    resumed = LearnerStep(net, dict(args, optimizer='lamb'), batches[0], lr=lr, cudnn_benchmark=False)
    resumed.load_optimizer_state(saved)
    resumed.step(resumed.new_packed().fill(batches[2]))
    assert _same(_image(resumed), _image(whole)) == []
    adam = LearnerStep(make(), args, batches[0], lr=lr, cudnn_benchmark=False)
    before = adam.optimizer_state_dict()
    with pytest.raises(ValueError):
        adam.load_optimizer_state(saved)
    after = adam.optimizer_state_dict()
    assert 'algorithm' not in after and sorted(after) == sorted(before)
    assert all(torch.equal(before['optimizer']['state'][i][k], after['optimizer']['state'][i][k])
               for i in before['optimizer']['state'] for k in before['optimizer']['state'][i])
    lamb = LearnerStep(make(), dict(args, optimizer='lamb'), batches[0], lr=lr, cudnn_benchmark=False)
    image = _image(lamb)
    with pytest.raises(ValueError):
        lamb.load_optimizer_state(before)
    assert _same(_image(lamb), image) == []
    for st in (whole, resumed, adam, lamb):
        st.close()


# ---------------------------------------------------------------------------------------------------------------- ranks

NGPU = torch.cuda.device_count() if torch.cuda.is_available() else 0


def _rank_main(rank, world, port, out_dir):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    import torch.distributed as dist
    from handyrl_b200.multigpu import shard_batch
    from handyrl_b200.train import LearnerStep
    from test_multi_gpu import ARGS, _batch, _net, _run_steps
    args = dict(ARGS, optimizer='lamb')
    torch.cuda.set_device(rank)
    dist.init_process_group('nccl', init_method='tcp://127.0.0.1:%d' % port, rank=rank, world_size=world,
                            device_id=torch.device('cuda', rank))
    res = {}
    full = [_batch(s) for s in range(3)]
    for mode in ('peer', 'nccl'):
        st = LearnerStep(_net(), args, shard_batch(full[0], rank, world), lr=1e-3, device=torch.device('cuda', rank),
                         process_group=dist.group.WORLD, peer_allreduce=(mode == 'peer'))
        losses, w = _run_steps(st, [shard_batch(b, rank, world) for b in full])
        gathered = [torch.empty_like(w).cuda() for _ in range(world)]
        dist.all_gather(gathered, w.cuda())
        res[mode] = {'losses': losses, 'weights': w.numpy(), 'ranks_identical': all(torch.equal(g, gathered[0]) for g in gathered)}
        st.close()
    if rank == 0:
        single = LearnerStep(_net(), args, full[0], lr=1e-3, device=torch.device('cuda', 0))
        losses, w = _run_steps(single, full)
        res['single'] = {'losses': losses, 'weights': w.numpy()}
    with open(os.path.join(out_dir, 'rank%d.pkl' % rank), 'wb') as f:
        pickle.dump(res, f)
    dist.barrier()
    torch.cuda.synchronize()
    dist.destroy_process_group()


@pytest.mark.skipif(NGPU < 2, reason='needs at least 2 GPUs')
def test_sharded_lamb_step_keeps_ranks_identical_and_equals_the_full_batch_step():
    """As test_multi_gpu.test_sharded_step_equals_full_batch_step, with the key on, on 2 ranks."""
    import torch.multiprocessing as mp
    from test_multi_gpu import _free_port
    world = 2
    out_dir = tempfile.mkdtemp(prefix='hrl_lamb_')
    mp.spawn(_rank_main, args=(world, _free_port(), out_dir), nprocs=world, join=True)
    res = [pickle.load(open(os.path.join(out_dir, 'rank%d.pkl' % r), 'rb')) for r in range(world)]
    single = res[0]['single']
    for mode in ('peer', 'nccl'):
        for r in range(world):
            assert res[r][mode]['ranks_identical'], (mode, r)
            assert np.array_equal(res[r][mode]['weights'], res[0][mode]['weights']), (mode, r)
        for s in range(3):
            got, ref = res[0][mode]['losses'][s], single['losses'][s]
            scale = max(abs(v) for v in ref.values())
            for k, v in ref.items():
                assert abs(got[k] - v) <= 1e-5 * scale + 1e-6, (mode, s, k, got[k], v)
        diff = np.abs(res[0][mode]['weights'] - single['weights'])
        assert (diff > 1e-6).mean() <= 1e-3 and diff.max() <= 1e-4, (mode, (diff > 1e-6).sum(), diff.max())
