"""The replay with the checkpoints (train_args['save_replay']) on the GPU: a learner restored from an epoch's files draws the
same batches and continues bit for bit, the key changes nothing about the step, and the Trainer writes the files, ends its
writer with stop(), restarts from them without waiting for new episodes and never synchronises the step stream for them."""
import os
import threading
import time

import pytest
import torch

from test_optimizer_state_gpu import _trainer_args

pytestmark = pytest.mark.gpu

N_FIRST, N_MORE, K = 14, 6, 6          # steps on the backlog, steps after the ring has wrapped, steps compared
HEADS = ['p', 'v', 'ent', 'total']
DIHEDRAL = {'group': 'dihedral', 'board': [3, 3]}
CASES = {'plain': {}, 'symmetry': {'symmetry': DIHEDRAL}, 'prioritized': {'prioritized_replay': True},
         'everything': {'prioritized_replay': True, 'symmetry': DIHEDRAL, 'validation_rate': 0.2, 'weight_ema': 0.9,
                        'skip_nonfinite': True}}


def _wait(cond, timeout=30.0):
    t0 = time.monotonic()
    while not cond():
        if time.monotonic() - t0 > timeout:
            return False
        time.sleep(0.005)
    return True


def _learner(args, episodes, restore=None, weights=None):
    """A LearnerStep and a running GpuBatcher on a deque holding `episodes`; the net starts from `weights` when given."""
    from handyrl_b200.nets import tictactoe_net
    from handyrl_b200.train import Batcher, EpisodeDeque, GpuBatcher, LearnerStep
    dq = EpisodeDeque()
    dq.extend(episodes)
    torch.manual_seed(0)
    net = tictactoe_net()
    if weights is not None:
        net.load_state_dict(weights, strict=True)
    st = LearnerStep(net, args, Batcher(args, dq)._make(), lr=1e-4, cudnn_benchmark=False)
    gb = GpuBatcher(args, dq, st.device, restore=restore)
    gb.run()
    assert _wait(gb.ready)
    return st, gb, dq


def _step(st, gb, record=None):
    """One training step (and, with validation, one pass on a held-out batch with the live and the averaged weights); with
    `record`, the bytes of every gathered batch, the importance weights and the loss sums are appended to it."""
    def keep(*tensors):
        if record is not None:
            st.stream.synchronize()
            record.extend(t.clone() for t in tensors)

    from handyrl_b200.batch import tree_leaves
    gb.fill(st)         # every tensor of the batch (not the buffer's bytes: its alignment padding is never written)
    keep(*tree_leaves(st.dev), *([st.prio_state.win_weight] if st.prio_state is not None else []))
    st.step_in_place()
    keep(st.last_losses)
    if st.validation and gb.validation_ready():
        gb.fill_validation(st)
        keep(*tree_leaves(st.dev))
        st.validate_in_place()
        if st.avg is not None:
            st.validate_in_place(averaged=True)


def _final(st, gb):
    st.stream.synchronize()
    out = [st.state.bytes, st.opt.exp_avg, st.opt.exp_avg_sq, st.opt.step_count, st.opt.lr, st.ema, st.accum]
    if st.avg is not None:
        out.append(st.avg)
    if st.validation:
        out.append(st.val_accum_all)
    if st.prio_state is not None:           # by position, oldest first: the restored ring hands out other slots
        slots, _ = gb.replay.positions()
        out += [st.prio_state.prio[torch.from_numpy(slots).to(st.device)], st.prio_state.max_prio]
    return [t.clone() for t in out]


@pytest.mark.parametrize('case', list(CASES))
def test_a_restored_learner_continues_bit_for_bit(case, tmp_path):
    from handyrl_b200.nets import tictactoe_net
    from handyrl_b200.synthetic import tictactoe_episodes
    from handyrl_b200.train import ReplayCheckpoints, load_replay_file, replay_file, restore_priorities
    args, _ = _trainer_args(batch_size=16, maximum_episodes=150, replay_capacity_steps=700, seed=5, save_replay=True,
                            save_optimizer=True, **CASES[case])
    episodes = tictactoe_episodes(260, seed=9)
    st, gb, dq = _learner(args, episodes[:200])
    assert (st.prio_snap is not None) == ('prioritized_replay' in CASES[case])
    for _ in range(N_FIRST):
        _step(st, gb)
    dq.extend(episodes[200:])                         # the feeder stores them while nothing samples: the ring wraps
    assert _wait(lambda: gb.fed == len(episodes))
    for _ in range(N_MORE):
        _step(st, gb)
    steps = N_FIRST + N_MORE
    pending = st.end_epoch(steps, steps, 3e-8, tictactoe_net(), HEADS)
    model, _ = pending.resolve()
    snap = gb.snapshot()
    assert (pending.priority_state is not None) == (st.prio_state is not None)
    path = ReplayCheckpoints(str(tmp_path)).write(1, replay_file(snap, pending.priority_state, None, steps, 1))

    # the ring has wrapped and evicted: the file holds what is resident, not what arrived
    resident = len(gb.replay) + (len(gb.val_replay) if gb.val_replay is not None else 0)
    assert len(snap['episodes']) == resident < len(episodes)
    assert gb.replay.handles[0].first_step > gb.replay.handles[-1].first_step
    kept = [e for e in episodes if any(e is s for s in snap['episodes'])]
    assert all(a is b for a, b in zip(kept, snap['episodes']))                  # oldest first, in arrival order
    assert int((snap['serials'] >= 0).sum()) == len(gb.replay)
    assert snap['serials'][snap['serials'] >= 0].tolist() == gb.replay.positions()[1].tolist()

    run_a = []
    for _ in range(K):
        _step(st, gb, run_a)
    run_a += _final(st, gb)
    gb.stop()
    st.close()

    d = load_replay_file(path, leaf_shapes=[(3, 3, 3)], actions=9)
    st2, gb2, _ = _learner(args, d['episodes'], restore=d, weights=model.state_dict())
    st2.load_optimizer_state(pending.optim_state)
    if st2.avg is not None:
        st2.seed_weight_ema(pending.ema_state)
    st2.warm_up()
    gb2.restore_sampler(d['sampler'])
    restored = restore_priorities(st2, gb2, d)
    assert (restored > 0) == (st2.prio_state is not None)
    assert len(gb2.replay) == len(gb.replay) and gb2.replay.handles[0].first_step == 0       # same episodes, other rows
    if gb.val_replay is not None:
        assert len(gb2.val_replay) == len(gb.val_replay) > 0
    run_b = []
    for _ in range(K):
        _step(st2, gb2, run_b)
    run_b += _final(st2, gb2)
    gb2.stop()
    st2.close()

    assert len(run_a) == len(run_b) > 3 * K
    different = [i for i, (a, b) in enumerate(zip(run_a, run_b)) if not torch.equal(a, b)]
    assert different == []
    if st.prio_state is not None:
        assert float(run_a[-1]) >= 1.0 and not torch.all(run_a[-2] == 1.0)      # learned priorities were in play


def test_without_the_restore_the_batches_differ(tmp_path):
    """The comparison above can fail: the same episodes under a freshly seeded sampler give other batches."""
    from handyrl_b200.synthetic import tictactoe_episodes
    args, _ = _trainer_args(batch_size=16, maximum_episodes=150, replay_capacity_steps=700, seed=5, save_replay=True)
    episodes = tictactoe_episodes(80, seed=9)
    runs = []
    for restore in (True, False):
        st, gb, _ = _learner(args, episodes)
        for _ in range(3):
            _step(st, gb)
        snap = gb.snapshot()
        rec = []
        _step(st, gb, rec)
        st2, gb2, _ = _learner(args, snap['episodes'])
        st2.warm_up()
        if restore:
            gb2.restore_sampler(snap['sampler'])
        rec2 = []
        _step(st2, gb2, rec2)
        runs.append(all(torch.equal(a, b) for a, b in zip(rec[:-1], rec2[:-1])))        # the batch; the weights differ
        for s, g in ((st, gb), (st2, gb2)):
            g.stop()
            s.close()
    assert runs == [True, False]


# ---------------------------------------------------------------------------------------------------------------- trainer
def _run(tr, updates, feed=(), check_sync=False):
    """`updates` epochs of a Trainer on its own thread, then stop(); the last update() is watched for synchronisations of
    the step stream when check_sync."""
    tr.episodes.extend(feed)
    th = threading.Thread(target=tr.run, daemon=True)
    th.start()
    calls, out = [], []
    try:
        for i in range(updates):
            if i == 1:
                assert _wait(lambda: tr.gpu_batcher.fed >= len(tr.episodes))
            if check_sync and i == updates - 1:
                stream_cls = type(tr.stepper.stream)
                real = stream_cls.synchronize
                stream_cls.synchronize = lambda self: (calls.append(self), real(self))[1]
                try:
                    out.append(tr.update())
                finally:
                    stream_cls.synchronize = real
            else:
                out.append(tr.update())
    finally:
        tr.stop()
        th.join(timeout=20)
    assert not th.is_alive()
    assert not any(s is tr.stepper.stream for s in calls)
    return out


def test_the_key_off_changes_nothing_and_on_adds_no_launch(tmp_path, monkeypatch):
    from handyrl_b200.nets import tictactoe_net
    from handyrl_b200.synthetic import tictactoe_episodes
    from handyrl_b200.train import Trainer
    episodes = tictactoe_episodes(40, seed=2)
    launches = {}
    for on in (False, True):
        (tmp_path / str(on)).mkdir()
        monkeypatch.chdir(tmp_path / str(on))
        args, _ = _trainer_args(prioritized_replay=True, seed=3, **({'save_replay': True} if on else {}))
        before = set(threading.enumerate())
        tr = Trainer(args, tictactoe_net())
        _run(tr, 2, episodes)
        launches[on] = tr.stepper.launches_per_step
        assert set(threading.enumerate()) - before == set()
        if on:
            assert sorted(os.listdir('models')) == ['1.replay.pth', '2.replay.pth']
        else:
            assert os.listdir('.') == []
            assert tr.replay_files is None and tr.stepper.prio_snap is None and tr.gpu_batcher.replay.resident is None
            assert [e.name for e in tr.stepper._handoff] == ['state', 'losses']
    assert launches[True] == launches[False]


def test_trainer_writes_the_files_and_a_restart_resumes_from_them(tmp_path, monkeypatch, capsys):
    from handyrl_b200.nets import tictactoe_net
    from handyrl_b200.synthetic import tictactoe_episodes
    from handyrl_b200.train import Trainer
    monkeypatch.chdir(tmp_path)
    args, _ = _trainer_args(save_replay=True, save_optimizer=True, prioritized_replay=True, validation_rate=0.2, seed=3,
                            replay_ratio=64)
    episodes = tictactoe_episodes(60, seed=21)
    before = set(threading.enumerate())
    tr = Trainer(args, tictactoe_net())
    (model, _), (_, steps2), _ = _run(tr, 3, episodes, check_sync=True)
    assert set(threading.enumerate()) - before == set()                     # the writer ended with stop()
    assert tr.replay_files.thread is None and tr.replay_files.last_error is None
    # the newest two replay files; every epoch's optimiser state
    assert sorted(os.listdir('models')) == ['1.optim.pth', '2.optim.pth', '2.replay.pth', '3.optim.pth', '3.replay.pth',
                                            'latest.optim.pth']
    d = torch.load('models/2.replay.pth')
    assert d['epoch'] == 2 and d['steps'] == steps2 == torch.load('models/2.optim.pth')['schedule']['steps']
    held = int((d['serials'] < 0).sum())
    assert len(d['episodes']) == len(episodes) and 0 < held < len(episodes)
    assert all(a == b for a, b in zip(d['episodes'], episodes))
    saved = dict(zip(d['priorities']['serial'].tolist(), d['priorities']['priority'].tolist()))
    train_serials = [s for s in d['serials'].tolist() if s >= 0]
    assert 0 < len(saved) <= len(train_serials) and set(saved) <= set(train_serials)
    assert any(p != 1.0 for p in saved.values()) and d['sampler']['prio_batches'] == steps2
    assert d['limiter']['stored'] == sum(e['steps'] for e, s in zip(episodes, d['serials'].tolist()) if s >= 0)
    torch.save(model.state_dict(), 'models/2.pth')

    # restarted at epoch 2 with no new episode: it trains at once, from the file's state
    capsys.readouterr()
    net = tictactoe_net()
    net.load_state_dict(torch.load('models/2.pth'))
    tr2 = Trainer(dict(args, restart_epoch=2), net)
    lines = capsys.readouterr().out.splitlines()
    assert lines == ['restored replay: %d episodes (%d held out), %d steps, priorities: yes'
                     % (len(episodes), held, sum(e['steps'] for e in episodes))]
    assert len(tr2.episodes) == len(episodes) >= args['minimum_episodes']
    # up to the first batch by hand, to look at the restored state before a step moves it
    tr2._start_stepper()
    gb = tr2.gpu_batcher
    assert _wait(gb.ready)
    tr2._finish_restore()
    assert tr2.restored is None and tr2.steps == steps2
    assert [ep for _, ep in gb.replay.resident] == [e for e, s in zip(d['episodes'], d['serials'].tolist()) if s >= 0]
    assert [ep for _, ep in gb.val_replay.resident] == [e for e, s in zip(d['episodes'], d['serials'].tolist()) if s < 0]
    assert gb.prio_batches == steps2 and gb.rng.bit_generator.state == d['sampler']['rng']
    got = tr2.stepper.priority_state_dict()
    slots, serials = gb.replay.positions()
    assert got['max_prio'] == d['priorities']['max_prio']
    for slot, serial, old in zip(slots.tolist(), serials.tolist(), train_serials):      # both oldest first
        if old in saved:
            assert int(got['slot_serial'][slot]) == serial and float(got['priority'][slot]) == saved[old]
        else:                           # the sampler had not seen it when the file was taken: it starts at max_prio
            assert int(got['slot_serial'][slot]) != serial
    assert tr2.replay_ratio_stats()['restored'] == d['limiter']
    (_, steps3), = _run(tr2, 1)
    out = capsys.readouterr().out.splitlines()
    assert out[0] == 'waiting training' and out[1] == 'started training'
    assert steps3 > steps2
    assert sorted(f for f in os.listdir('models') if 'replay' in f) == ['2.replay.pth', '3.replay.pth']
    assert torch.load('models/3.replay.pth')['steps'] == steps3                   # epoch 3, written again by this run
