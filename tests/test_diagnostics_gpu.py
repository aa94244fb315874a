"""Learner diagnostics on the GPU: the sums of hrl_loss_fwd_bwd_diag against the float64 reference for every golden case, kernel
variant and recurrence form; no side effect on losses, gradients or weights; the LearnerStep / FlatAdam accumulation; the Trainer's
per-epoch line; sharded sums."""
import os
import pickle
import re
import socket
import sys
import tempfile

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT, case_args, load_cases
from diag_oracle import compare, diagnostics

pytestmark = pytest.mark.gpu

LOSS_CASES = load_cases('loss_cases.npz')
VARIANTS = ['rows-direct', 'rows-staged', 'bulk', 'element', 'group']
_ORACLE = {}
ARGS = {'turn_based_training': True, 'observation': False, 'gamma': 0.8, 'lambda': 0.7, 'burn_in_steps': 0,
        'entropy_regularization': 0.1, 'entropy_regularization_decay': 0.1, 'policy_target': 'UPGO', 'value_target': 'VTRACE'}


def to_dev(d):
    return {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in d.items()}


def split(case):
    batch = {k[3:]: v for k, v in case.items() if k.startswith('in.')}
    outs = {k[4:]: v for k, v in case.items() if k.startswith('out.')}
    return batch, outs


def run_both(outs, batch, args, tuning=None):
    """(plain call, diagnostics call) on the same inputs, each with its own buffers."""
    from handyrl_b200 import ops
    plain = ops.loss_fwd_bwd(outs, batch, args, tuning=tuning)
    diag = ops.loss_fwd_bwd(outs, batch, args, tuning=tuning, diagnostics=True)
    torch.cuda.synchronize()
    return plain, diag


def assert_same_outputs(a, b):
    assert torch.equal(a.losses, b.losses)
    assert torch.equal(a.dpolicy, b.dpolicy)
    for k in ('dvalue', 'dreturn'):
        x, y = getattr(a, k), getattr(b, k)
        assert (x is None) == (y is None) and (x is None or torch.equal(x, y)), k


@pytest.mark.parametrize('recurrence', ['serial', 'scan'])
@pytest.mark.parametrize('variant', VARIANTS)
@pytest.mark.parametrize('name', sorted(LOSS_CASES))
def test_golden_cases_every_variant_and_recurrence(name, variant, recurrence):
    case = LOSS_CASES[name]
    batch, outs = split(case)
    args = case_args(case['meta'])
    if name not in _ORACLE:
        _ORACLE[name] = diagnostics(batch, outs, args)
    want, near = _ORACLE[name]
    plain, diag = run_both(to_dev(outs), to_dev(batch), args, tuning={'variant': variant, 'recurrence': recurrence})
    assert_same_outputs(plain, diag)
    got = diag.diagnostics.cpu().numpy()
    compare(got, want, near, err='%s/%s/%s' % (name, variant, recurrence))
    assert np.all(got[16:] == 0)           # the optimiser's entries


FULL = [  # the full-size shapes of test_loss_gpu.py
    dict(id='cfg2', B=512, T=32, P=2, A=9, turn_based=True, observation=False, has_return=False,
         policy_target='UPGO', value_target='VTRACE', reward_kind='zero', burn_in=0),
    dict(id='cfg2_sim', B=512, T=32, P=2, A=9, turn_based=False, observation=False, has_return=False,
         policy_target='UPGO', value_target='VTRACE', reward_kind='zero', burn_in=0),
    dict(id='cfg3_geister', B=256, T=20, P=2, A=214, turn_based=True, observation=True, has_return=True,
         policy_target='TD', value_target='TD', reward_kind='step', burn_in=4),
    dict(id='cfg4_geese', B=256, T=32, P=4, A=4, turn_based=False, observation=False, has_return=False,
         policy_target='VTRACE', value_target='VTRACE', reward_kind='zero', burn_in=0),
    dict(id='cfg5_shard', B=512, T=64, P=2, A=512, turn_based=True, observation=False, has_return=False,
         policy_target='UPGO', value_target='VTRACE', reward_kind='zero', burn_in=0),
]


@pytest.mark.parametrize('cfg', FULL, ids=[c['id'] for c in FULL])
def test_full_size_parity_determinism_and_split(cfg):
    from handyrl_b200 import ops
    from handyrl_b200.synthetic import synthetic_batch, synthetic_outputs
    cfg = dict(cfg)
    cfg.pop('id')
    has_return = cfg.pop('has_return')
    args = {'turn_based_training': cfg['turn_based'], 'observation': cfg['observation'], 'gamma': 0.8, 'lambda': 0.7,
            'burn_in_steps': cfg['burn_in'], 'entropy_regularization': 0.1, 'entropy_regularization_decay': 0.1,
            'policy_target': cfg.pop('policy_target'), 'value_target': cfg.pop('value_target')}
    batch = synthetic_batch(cfg['B'], cfg['T'], cfg['P'], cfg['A'], turn_based=cfg['turn_based'], observation=cfg['observation'],
                            reward_kind=cfg['reward_kind'], burn_in=cfg['burn_in'], seed=0, with_obs=False)
    outs = synthetic_outputs(batch, has_value=True, has_return=has_return, seed=1)
    db, do = {k: v.cuda() for k, v in batch.items()}, {k: v.cuda() for k, v in outs.items()}
    plain, diag = run_both(do, db, args)
    assert_same_outputs(plain, diag)
    got = diag.diagnostics.cpu().numpy().astype(np.float64)
    want, near = diagnostics({k: v.numpy() for k, v in batch.items()}, {k: v.numpy() for k, v in outs.items()}, args)
    compare(got, want, near)
    again = ops.loss_fwd_bwd(do, db, args, diagnostics=True)
    torch.cuda.synchronize()
    assert torch.equal(again.diagnostics.cpu(), diag.diagnostics.cpu())           # a second launch is bit-identical
    h = cfg['B'] // 2
    parts = []
    for sl in (slice(0, h), slice(h, None)):
        r = ops.loss_fwd_bwd({k: v[sl].contiguous() for k, v in do.items()}, {k: v[sl].contiguous() for k, v in db.items()}, args,
                             diagnostics=True)
        torch.cuda.synchronize()
        parts.append(r.diagnostics.cpu().numpy().astype(np.float64))
    np.testing.assert_allclose(parts[0] + parts[1], got, rtol=1e-6, atol=1e-5)    # shards add up to the whole batch


@pytest.mark.parametrize('cluster', [1, 2, 4, 8])
def test_bulk_cluster_sizes_and_bf16_io(cluster):
    from handyrl_b200.synthetic import synthetic_batch, synthetic_outputs
    batch = synthetic_batch(64, 32, 2, 512, seed=3, with_obs=False)     # (a window a single CTA can hold, for cluster 1)
    outs = synthetic_outputs(batch, seed=4)
    db, do = {k: v.cuda() for k, v in batch.items()}, {k: v.cuda() for k, v in outs.items()}
    tuning = {'variant': 'bulk', 'cluster': cluster}
    plain, diag = run_both(do, db, ARGS, tuning=tuning)
    assert_same_outputs(plain, diag)
    want, near = diagnostics({k: v.numpy() for k, v in batch.items()}, {k: v.numpy() for k, v in outs.items()}, ARGS)
    compare(diag.diagnostics.cpu().numpy(), want, near, err='cluster %d' % cluster)
    half = dict(do, policy=do['policy'].to(torch.bfloat16))
    plain16, diag16 = run_both(half, db, ARGS, tuning=tuning)
    assert_same_outputs(plain16, diag16)
    widened = dict(do, policy=half['policy'].float())
    _, diag32 = run_both(widened, db, ARGS, tuning=tuning)
    assert torch.equal(diag16.diagnostics, diag32.diagnostics)     # bf16 I/O: everything in between is the fp32 arithmetic


# ---------------------------------------------------------------------------------------------------------------- learner step
with open(os.path.join(GOLDEN, 'step_cases.pkl'), 'rb') as f:
    STEP_CASES = pickle.load(f)
with open(os.path.join(GOLDEN, 'net_step_cases.pkl'), 'rb') as f:
    NET_CASES = pickle.load(f)
NSTEPS = 4


def _setup(kind):
    """(net factory, args, [batches]) of a fused-tower TicTacToe case or a module-path Geese case."""
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


@pytest.mark.parametrize('kind', ['tictactoe', 'geese'])
def test_learner_step_accumulates_and_leaves_the_weights_alone(kind):
    from handyrl_b200 import ops
    from handyrl_b200.train import LearnerStep
    make, args, batches, lr = _setup(kind)
    weights, launches = {}, {}
    # the Geese stem (17 input channels) stays on cuDNN, whose autotuner may pick differently summing algorithms in two
    # steppers: pin deterministic algorithms so that two runs can be compared bit for bit
    old = torch.backends.cudnn.deterministic
    torch.backends.cudnn.deterministic = True
    for on in (False, True):
        st = LearnerStep(make(), dict(args, diagnostics=on), batches[0], lr=lr, use_graph=True, cudnn_benchmark=False)
        assert (st.engine is not None) == (kind == 'tictactoe')
        for b in batches:
            st.step(st.new_packed().fill(b))
        weights[on] = st.cpu_state_dict()
        launches[on] = st.launches_per_step
        if on:
            graph_sums = np.array([v for v in st.pop_diagnostics().values()])
            summary = ops.summarize_diagnostics(graph_sums)
        else:
            assert st.diag_accum is None and st.opt.diag is None and st.loss_buf.diagnostics is None
        st.close()
    assert launches[True] == launches[False]
    for k in weights[False]:
        assert torch.equal(weights[False][k], weights[True][k]), k
    # eager steps, one diagnostics read per step: the per-step sums add up to the graph's epoch sums (on the same pinned
    # cuDNN algorithms: an autotuned pick sums the Geese stem in another order)
    st = LearnerStep(make(), args, batches[0], lr=lr, use_graph=False, diagnostics=True, cudnn_benchmark=False)
    total, norms = np.zeros(ops.NUM_DIAG), []
    for b in batches:
        st.step(st.new_packed().fill(b))
        total += np.array(list(st.pop_diagnostics().values()))
        norms.append(float(st.opt.grad_norm))
        assert float(st.loss_buf.diagnostics[0]) == st.read_losses()['dcnt']          # n_pol == dcnt
    st.close()
    torch.backends.cudnn.deterministic = old
    np.testing.assert_allclose(graph_sums, total, rtol=1e-6, atol=1e-6)
    norms = np.array(norms, np.float32).astype(np.float64)
    i = {k: n for n, k in enumerate(ops.DIAG_KEYS)}
    assert total[i['steps']] == NSTEPS and graph_sums[i['steps']] == NSTEPS
    np.testing.assert_allclose(total[i['gnorm']], norms.sum(), rtol=1e-12)
    np.testing.assert_allclose(total[i['gnorm2']], (norms * norms).sum(), rtol=1e-12)
    assert total[i['gclip']] == (norms > st.opt.max_norm).sum()
    assert {'rho', 'clip', 'kl', 'adv', 'adv_sd', 'ev_v', 'gnorm', 'gclip'} <= set(summary)


@pytest.mark.parametrize('on', [False, True], ids=['off', 'on'])
def test_trainer_prints_one_diagnostics_line_per_loss_line(on, capsys):
    import threading
    from handyrl_b200.nets import tictactoe_net
    from handyrl_b200.train import Trainer
    with open(os.path.join(GOLDEN, 'batch_cases.pkl'), 'rb') as f:
        case = pickle.load(f)['tictactoe']
    args = dict(case['args'], batch_size=8, minimum_episodes=4, num_batchers=1, **{'lambda': 0.7},
                entropy_regularization=0.1, entropy_regularization_decay=0.1, policy_target='UPGO', value_target='VTRACE',
                gpu_replay=True, num_gpus=1)
    if on:
        args['diagnostics'] = True
    tr = Trainer(args, tictactoe_net())
    tr.episodes.extend(case['episodes'])
    th = threading.Thread(target=tr.run, daemon=True)
    th.start()
    tr.update()
    tr.update()
    tr.stop()
    th.join(timeout=10)
    lines = capsys.readouterr().out.splitlines()
    loss_at = [n for n, l in enumerate(lines) if l.startswith('loss = ')]
    diag_at = [n for n, l in enumerate(lines) if l.startswith('diagnostics = ')]
    assert len(loss_at) >= 2
    if not on:
        assert diag_at == []
        return
    assert diag_at == [n + 1 for n in loss_at]
    pat = re.compile(r'diagnostics = ((?:[a-z_]+:-?(?:[0-9.]+(?:e[+-]?[0-9]+)?|nan|inf) ?)+)')
    for n in diag_at:
        m = pat.fullmatch(lines[n])
        assert m, lines[n]
        fields = dict(kv.split(':') for kv in m.group(1).split())
        assert {'rho', 'clip', 'kl', 'adv', 'ev_v', 'gnorm', 'gclip'} <= set(fields), fields
        assert 0.0 <= float(fields['clip']) <= 1.0 and 0.0 <= float(fields['gclip']) <= 1.0


# ---------------------------------------------------------------------------------------------------------------- multi-GPU
NGPU = torch.cuda.device_count() if torch.cuda.is_available() else 0
MG_ARGS = dict(ARGS, forward_steps=8, diagnostics=True)
MG_DIMS = (16, 8, 2, 9)


def _mg_net():
    from handyrl_b200.nets import BoardNet
    torch.manual_seed(11)
    return BoardNet(norm=False)


def _mg_batch(s):
    from handyrl_b200.synthetic import synthetic_batch
    B, T, P, A = MG_DIMS
    return synthetic_batch(B, T, P, A, turn_based=True, observation=False, seed=900 + s)


def _mg_rank(rank, world, port, out_dir):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    from handyrl_b200.multigpu import shard_batch
    from handyrl_b200.train import LearnerStep
    torch.cuda.set_device(rank)
    dist.init_process_group('nccl', init_method='tcp://127.0.0.1:%d' % port, rank=rank, world_size=world,
                            device_id=torch.device('cuda', rank))
    full = [_mg_batch(s) for s in range(3)]
    st = LearnerStep(_mg_net(), MG_ARGS, shard_batch(full[0], rank, world), lr=1e-3, device=torch.device('cuda', rank),
                     process_group=dist.group.WORLD)
    for b in full:
        st.step(st.new_packed().fill(shard_batch(b, rank, world)))
    res = {'sharded': st.pop_diagnostics()}
    st.close()
    if rank == 0:
        single = LearnerStep(_mg_net(), MG_ARGS, full[0], lr=1e-3, device=torch.device('cuda', 0))
        for b in full:
            single.step(single.new_packed().fill(b))
        res['single'] = single.pop_diagnostics()
    with open(os.path.join(out_dir, 'rank%d.pkl' % rank), 'wb') as f:
        pickle.dump(res, f)
    dist.barrier()
    torch.cuda.synchronize()
    dist.destroy_process_group()


@pytest.mark.skipif(NGPU < 2, reason='needs at least 2 GPUs')
def test_sharded_diagnostics_equal_the_full_batch_ones():
    import torch.multiprocessing as mp
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        port = s.getsockname()[1]
    out_dir = tempfile.mkdtemp(prefix='hrl_diag_')
    mp.spawn(_mg_rank, args=(2, port, out_dir), nprocs=2, join=True)
    res = [pickle.load(open(os.path.join(out_dir, 'rank%d.pkl' % r), 'rb')) for r in range(2)]
    assert res[0]['sharded'] == res[1]['sharded']          # every rank accumulates the same (all-reduced) values
    single = res[0]['single']
    for k, v in single.items():
        assert abs(res[0]['sharded'][k] - v) <= 1e-5 * abs(v) + 1e-5, (k, res[0]['sharded'][k], v)
