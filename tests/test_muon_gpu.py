"""The Muon optimiser on the GPU (train_args['optimizer'] = 'muon', ops.FlatMuon, hrl_clip_muon_step): the kernel against the
float64 restatement (tests/muon_ref.py) on the shipped nets' bucket layouts and the envelope's edge shapes, reproducibility
under graph replay, the learner against the eager CPU step with Muon in place of Adam, the key off, the learner's options,
the non-finite guard, the checkpoint round trip and the sharded step.

Bounds on O (derived on the CPU by running the restatement with the kernel's arithmetic -- bf16 operands, fp32
accumulation in another order, fp32 epilogues -- on every matrix shape of the shipped nets and the edge shapes, four seeds
each):
  * against the bf16 mode of the restatement, only the fp32 accumulation order and the bf16 rounding flips it causes differ.
    A flip moves an element by one bf16 ulp, at most 2^-7 of its size, and later iterations carry it on; the worst seen was
    0.019 max|O|.  Bound: 2^-5 max|O| (four ulps at the largest element).
  * against the float64 restatement the bf16 roundings themselves count; the worst seen was 0.040 max|O| (2 x 2) and a
    singular value 0.038 outside the float64 band.  Bound: 2^-4 max|O|, and the band widened by 2^-4.
"""
import os
import pickle
import sys
import tempfile

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from muon_ref import Muon64, matrix_view, orthogonalise

pytestmark = pytest.mark.gpu

with open(os.path.join(GOLDEN, 'step_cases.pkl'), 'rb') as f:
    STEP_CASES = pickle.load(f)
with open(os.path.join(GOLDEN, 'net_step_cases.pkl'), 'rb') as f:
    NET_CASES = pickle.load(f)
NETS = ['tictactoe', 'geister', 'geese']
EDGES = {'2x2': [(2, 2), (2,)], 'tall': [(5,), (576, 128), (3, 2)], 'largest': [(128, 64, 3, 3), (128,)]}
HP = dict(max_norm=4.0, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-5)
LR, LR_SCALE, T0 = 1e-3, 2.0, 4          # T0: the step count before the step under test
BF16_BOUND, F64_BOUND = 2.0 ** -5, 2.0 ** -4


@pytest.fixture
def deterministic_cudnn():
    old = (torch.backends.cudnn.deterministic, torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.deterministic = True
    yield
    torch.backends.cudnn.deterministic, torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


# ---------------------------------------------------------------------------------------------------------------- kernel


def _shapes(name):
    if name in EDGES:
        return EDGES[name]
    from handyrl_b200 import nets
    net = {'tictactoe': nets.tictactoe_net, 'geister': nets.geister_net, 'geese': nets.geese_net}[name]()
    return [tuple(p.shape) for p in net.parameters()]


def _start(name, clip, seed=5):
    """Random weights, moments and gradients on the bucket layout of `name`; the gradient's norm is 40 (clip active) or 1.
    The Muon-owned words' exp_avg_sq is zero, as a Muon learner keeps it."""
    from handyrl_b200.ops import muon_plan
    g = torch.Generator().manual_seed(seed)
    shapes = _shapes(name)
    kinds = muon_plan(shapes)[0]
    numels = [int(np.prod(s)) for s in shapes]
    n = sum(numels)
    grad = torch.randn(n, generator=g)
    grad *= (40.0 if clip else 1.0) / float(grad.norm())
    v = 1e-4 * torch.rand(n, generator=g)
    off = 0
    for k, kind in zip(numels, kinds):
        if kind == 'matrix':
            v[off:off + k] = 0.0
        off += k
    return {'shapes': shapes, 'kinds': kinds, 'numels': numels, 'w': 0.5 * torch.randn(n, generator=g), 'g': grad,
            'm': 0.01 * torch.randn(n, generator=g), 'v': v}


def _optimiser(start, form, muon=True):
    """A FlatMuon (or FlatAdam) over CUDA parameters of the start's shapes, its buffers set to `start`, in `form`
    ('plain', 'diag', 'guard')."""
    from handyrl_b200 import ops
    params = [torch.nn.Parameter(torch.zeros(s, device='cuda')) for s in start['shapes']]
    opt = ops.FlatMuon(params, lr=LR, lr_scale=LR_SCALE, extra=8, **HP) if muon else ops.FlatAdam(params, lr=LR, extra=8, **HP)
    n = opt.n
    with torch.no_grad():
        opt.flat_param[:n].copy_(start['w'])
        opt.flat_grad[:n].copy_(start['g'])
        opt.exp_avg[:n].copy_(start['m'])
        opt.exp_avg_sq[:n].copy_(start['v'])
    opt.step_count.fill_(T0)
    if muon:
        opt.ortho = torch.full((opt.n_pad,), 7.0, device='cuda')
    if form == 'diag':
        opt.diag = torch.zeros(4, dtype=torch.float64, device='cuda')
    if form == 'guard':
        opt.skip = torch.full((1,), 7, dtype=torch.int32, device='cuda')
        opt.guard_tail = 6
    return opt


def _state(opt):
    torch.cuda.synchronize()
    st = {'w': opt.flat_param.cpu(), 'm': opt.exp_avg.cpu(), 'v': opt.exp_avg_sq.cpu(), 'step': int(opt.step_count),
          'gnorm': opt.grad_norm.cpu()}
    if getattr(opt, 'ortho', None) is not None:
        st['o'] = opt.ortho.cpu()
    return st


def _check_kernel_step(start, form):
    opt = _optimiser(start, form)
    opt.step()
    got = _state(opt)
    adam = _optimiser(start, form, muon=False)
    adam.step()
    want_adam = _state(adam)
    assert got['step'] == T0 + 1 and torch.equal(got['gnorm'], want_adam['gnorm'])
    gnorm = np.float32(got['gnorm'].item())
    coef = np.minimum(np.float32(4.0) / (gnorm + np.float32(1e-6)), np.float32(1.0))
    off = 0
    for shape, kind, k in zip(start['shapes'], start['kinds'], start['numels']):
        span = slice(off, off + k)
        off += k
        if kind != 'matrix':
            for key in ('w', 'm', 'v'):                       # Adam-owned words: hrl_clip_adam_step bit for bit
                assert torch.equal(got[key][span], want_adam[key][span]), (shape, key)
            assert (got['o'][span] == 7.0).all()
            continue
        r, c = matrix_view(shape)
        g32 = start['g'][span].numpy() * coef
        m32 = np.float32(0.95) * start['m'][span].numpy() + g32        # numpy float32: one rounding per operation
        n32 = g32 + np.float32(0.95) * m32
        assert np.array_equal(got['m'][span].numpy(), m32), shape
        assert (got['v'][span] == 0).all()
        o = got['o'][span].double().numpy().reshape(r, c)
        ref_bf16 = orthogonalise(n32.astype(np.float64).reshape(r, c), bf16=True)
        ref64 = orthogonalise(n32.astype(np.float64).reshape(r, c))
        err_bf16, err64 = np.abs(o - ref_bf16).max(), np.abs(o - ref64).max()
        assert err_bf16 <= BF16_BOUND * np.abs(ref_bf16).max(), (shape, err_bf16, np.abs(ref_bf16).max())
        assert err64 <= F64_BOUND * np.abs(ref64).max(), (shape, err64, np.abs(ref64).max())
        s, s64 = np.linalg.svd(o, compute_uv=False), np.linalg.svd(ref64, compute_uv=False)
        assert s64.min() - F64_BOUND <= s.min() and s.max() <= s64.max() + F64_BOUND, (shape, s.min(), s.max(), s64.min(), s64.max())
        # the update on the kernel's own O, in fp32 operation by operation
        w32, o32 = start['w'][span].numpy(), got['o'][span].numpy()
        scale = np.float32(LR_SCALE * 0.2 * np.sqrt(max(r, c)))
        want_w = w32 - np.float32(LR) * (scale * o32 + np.float32(HP['weight_decay']) * w32)
        np.testing.assert_array_max_ulp(got['w'][span].numpy(), want_w, maxulp=1)
    n = opt.n
    for key in ('w', 'm', 'v'):
        assert (got[key][n:] == 0).all()                       # padding
    if form == 'diag':
        d = opt.diag.cpu().tolist()
        assert torch.equal(opt.diag.cpu(), adam.diag.cpu()) and d[3] == 1.0
    elif form == 'guard':
        assert int(opt.skip) == 0


@pytest.mark.parametrize('form', ['diag', 'guard'])
@pytest.mark.parametrize('clip', [True, False], ids=['clip', 'noclip'])
@pytest.mark.parametrize('name', NETS)
def test_kernel_matches_adam_and_the_restatement(name, clip, form):
    _check_kernel_step(_start(name, clip), form)


@pytest.mark.parametrize('name', sorted(EDGES))
def test_kernel_on_the_edge_shapes(name):
    _check_kernel_step(_start(name, True), 'plain')


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
        for k in ('w', 'm', 'v', 'o'):
            assert torch.equal(got[k], want[k]), (where, k)
        assert got['step'] == T0


def test_repeated_launches_and_graph_replays_are_bit_identical():
    start = _start('geister', True)
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
    for k in ('w', 'm', 'v', 'o', 'gnorm'):
        assert torch.equal(e[k], g[k]), k


# ---------------------------------------------------------------------------------------------------------------- learner


def _case(kind):
    """(net factory, args, [three batches], lr): the fused-tower TicTacToe net, the recurrent Geister net or the Geese net."""
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


def _learn(kind, optimizer='muon', use_graph=True, batches=None, **kw):
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


def _check_weights(kind, got, want, owned, lr, steps):
    """A learner's weights after `steps` steps against the CPU step's.  Muon-owned tensors: each step moves one by
    lr * 0.2 sqrt(max(r, k)) O with |O| <= 1.25, and the kernel's O is within F64_BOUND max|O| of the float64 one, so each
    step may differ by lr * 0.2 sqrt(max(r, k)) * 1.25 * F64_BOUND, plus the fp32 slack of the Adam tests.  Adam-owned
    tensors after one step: the Adam step tests' bounds, since the step's gradient comes from identical weights.  After
    more steps the Muon-owned weights already differ by the bf16 bound above, so the gradients differ, and Adam, which
    divides by sqrt(v), can turn a small gradient difference on an element whose gradient is near zero into a step of the
    other sign: up to 2 lr per element per step, the bound the Adam tests also allow, with no limit on how many elements."""
    from conftest import noise_driven
    case = {'net': kind}
    for key, vr in want.items():
        v = got[key]
        if noise_driven(case, key):
            continue
        if not v.dtype.is_floating_point:
            assert int(v) == int(vr), key
        elif key in owned:
            r, c = matrix_view(v.shape)
            atol = steps * lr * 0.2 * np.sqrt(max(r, c)) * 1.25 * F64_BOUND + 5e-5
            np.testing.assert_allclose(v.numpy(), vr.numpy(), rtol=1e-3, atol=atol, err_msg=key)
        else:
            if steps == 1:
                bad = np.abs(v.numpy() - vr.numpy()) > 5e-5 + 1e-3 * np.abs(vr.numpy())
                assert bad.mean() <= 1e-3, '%s: %d of %d elements differ' % (key, bad.sum(), bad.size)
            np.testing.assert_allclose(v.numpy(), vr.numpy(), rtol=1e-3, atol=2 * lr * steps + 5e-5, err_msg=key)


@pytest.mark.parametrize('kind', NETS)
def test_three_learner_steps_match_the_cpu_step_with_muon(kind, deterministic_cudnn):
    """LearnerStep with the key against oracle.torch_learner.CpuLearner with Muon64 in place of Adam; eager and graph runs bit
    for bit.  Losses to the bounds of the Adam step tests; weights after the first and the third step to the bounds of
    _check_weights."""
    from oracle.torch_learner import CpuLearner
    from handyrl_b200 import ops
    make, args, batches, lr = _case(kind)

    def reference():
        ref = CpuLearner(make(), args, lr=lr)
        ref.opt = Muon64(ref.params, lr=lr, **{k: HP[k] for k in ('betas', 'eps', 'weight_decay')})
        return ref

    one, _ = _learn(kind, batches=batches[:1])
    ref = reference()
    ref.step(batches[0])
    _check_weights(kind, one.cpu_state_dict(), ref.net.state_dict(), set(one.opt.muon_params), lr, 1)
    one.close()
    ref = reference()
    graph, losses = _learn(kind)
    assert graph.optimizer == {'name': 'muon', 'lr_scale': 1.0} and isinstance(graph.opt, ops.FlatMuon)
    for s, (b, got) in enumerate(zip(batches, losses)):
        want, dcnt = ref.step(b)
        scale = max(abs(v) for v in want.values())
        for k, v in want.items():
            assert abs(got[k] - v) <= (1 + s) * 1e-4 * scale + 1e-4, (s, k, got[k], v)
        assert got['dcnt'] == dcnt
    owned = set(graph.opt.muon_params)
    assert owned
    _check_weights(kind, graph.cpu_state_dict(), ref.net.state_dict(), owned, lr, len(batches))
    eager, eager_losses = _learn(kind, use_graph=False)
    assert eager_losses == losses and _same(_image(eager), _image(graph)) == []
    eager.close()
    graph.close()


def test_key_off_is_adam_bit_for_bit_and_muon_adds_at_most_two_launches(deterministic_cudnn):
    runs = {}
    for key, args in (('absent', {}), (None, {'optimizer': None}), ('adam', {'optimizer': 'adam'}), ('muon', {'optimizer': 'muon'})):
        st, losses = _learn('tictactoe', optimizer=None, args=args)
        runs[key] = (st.launches_per_step, losses, _image(st), type(st.opt).__name__, st.optimizer)
        st.close()
    base = runs['absent']
    assert base[3] == 'FlatAdam' and base[4] == {'name': 'adam'}
    for key in (None, 'adam'):
        assert runs[key][0] == base[0] and runs[key][1] == base[1] and _same(runs[key][2], base[2]) == [] and runs[key][3] == 'FlatAdam'
    assert runs['muon'][3] == 'FlatMuon' and base[0] <= runs['muon'][0] <= base[0] + 2
    assert _same(runs['muon'][2], base[2]) != []


OPTIONS = {'diagnostics': {'diagnostics': True}, 'gradient_accumulation': {'gradient_accumulation': 2},
           'weight_ema': {'weight_ema': 0.9}, 'save_optimizer': {'save_optimizer': True}, 'tensor_cores_bf16': {'tensor_cores': 'bf16'}}


@pytest.mark.parametrize('option', sorted(OPTIONS))
def test_learner_options_with_muon(option, deterministic_cudnn):
    """Each option with the key on: graph and eager runs agree bit for bit, three steps count, Muon's words keep a zero
    exp_avg_sq, and the option's own state is there."""
    graph, losses = _learn('tictactoe', args=OPTIONS[option])
    eager, eager_losses = _learn('tictactoe', use_graph=False, args=OPTIONS[option])
    assert eager_losses == losses and _same(_image(eager), _image(graph)) == []
    img = _image(graph)
    assert img['step'] == 3 and torch.isfinite(img['m']).all()
    d = graph.optimizer_state_dict()
    assert d['algorithm'] == 'muon' and d['muon_params'] == graph.opt.muon_params
    for i, name in enumerate(d['param_names']):
        if name in graph.opt.muon_params:
            assert (d['optimizer']['state'][i]['exp_avg_sq'] == 0).all(), name
    if option == 'diagnostics':
        assert graph.opt.diag is not None and float(graph.opt.diag[3]) == 3.0
    if option == 'weight_ema':
        assert graph.avg is not None and torch.isfinite(graph.avg).all()
        assert torch.equal(graph.avg.cpu(), eager.avg.cpu())
    if option == 'gradient_accumulation':
        assert len(graph._micro) == 2
    if option == 'tensor_cores_bf16':
        assert graph.tensor_cores == 'bf16'
    eager.close()
    graph.close()


@pytest.mark.parametrize('kind', ['tictactoe', 'geister'])
def test_a_poisoned_step_leaves_the_muon_learner_untouched(kind, deterministic_cudnn):
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
    """optimizer_state_dict() after 2 steps, loaded with the weights into a fresh Muon learner: its third step equals the
    uninterrupted learner's bit for bit.  An Adam learner refuses the file, and a Muon learner an Adam file, changing nothing."""
    from handyrl_b200.train import LearnerStep
    make, args, batches, lr = _case('tictactoe')
    whole, _ = _learn('tictactoe')
    first, _ = _learn('tictactoe', batches=batches[:2])
    saved, weights = first.optimizer_state_dict(), first.cpu_state_dict()
    assert saved['algorithm'] == 'muon' and saved['lr_scale'] == 1.0 and saved['muon_params'] == first.opt.muon_params
    first.close()
    net = make()
    net.load_state_dict(weights)
    resumed = LearnerStep(net, dict(args, optimizer='muon'), batches[0], lr=lr, cudnn_benchmark=False)
    resumed.load_optimizer_state(saved)
    resumed.step(resumed.new_packed().fill(batches[2]))
    assert _same(_image(resumed), _image(whole)) == []
    adam = LearnerStep(make(), args, batches[0], lr=lr, cudnn_benchmark=False)
    before = adam.optimizer_state_dict()
    with pytest.raises(ValueError):
        adam.load_optimizer_state(saved)
    after = adam.optimizer_state_dict()
    assert 'algorithm' not in after and sorted(after) == sorted(before)
    muon = LearnerStep(make(), dict(args, optimizer='muon'), batches[0], lr=lr, cudnn_benchmark=False)
    image = _image(muon)
    with pytest.raises(ValueError):
        muon.load_optimizer_state(before)
    assert _same(_image(muon), image) == []
    for st in (whole, resumed, adam, muon):
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
    args = dict(ARGS, optimizer='muon')
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
def test_sharded_muon_step_keeps_ranks_identical_and_equals_the_full_batch_step():
    """As test_multi_gpu.test_sharded_step_equals_full_batch_step, with the key on, on 2 ranks.  The sharded and full-batch
    gradients differ in fp32 summation order only; Muon's bf16 iterations can turn that into a bf16 flip of O, so the
    weights may differ by lr * 0.2 sqrt(288) * 1.25 * BF16_BOUND per step on a few elements."""
    import torch.multiprocessing as mp
    from test_multi_gpu import _free_port
    world = 2
    out_dir = tempfile.mkdtemp(prefix='hrl_muon_')
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
                assert abs(got[k] - v) <= 1e-4 * scale + 1e-5, (mode, s, k, got[k], v)
        diff = np.abs(res[0][mode]['weights'] - single['weights'])
        assert diff.max() <= 3 * 1e-3 * 0.2 * np.sqrt(288) * 1.25 * BF16_BOUND + 1e-5, (mode, diff.max())
