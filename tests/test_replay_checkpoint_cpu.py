"""The replay with the checkpoints (train_args['save_replay']), without a GPU: the key, the resident lists beside the replay
directory, the file (round trip in both wire formats, atomic write, retention, numbering), a Trainer that starts from a file,
what a bad file does, and the mapping of saved priorities onto a restored ring."""
import os
import subprocess
import sys
import threading

import numpy as np
import pytest
import torch



def _episodes(n, seed=1, flat=()):
    """n TicTacToe episodes in the reference's wire format; those at the positions in `flat` in the flat one, moments dropped."""
    from handyrl_b200.synthetic import tictactoe_episodes
    from handyrl_b200.wire import pack_episode
    eps = tictactoe_episodes(n, seed=seed)
    return [pack_episode(e, drop_moments=True) if i in flat else e for i, e in enumerate(eps)]


def _snapshot(eps, held=()):
    serials = torch.tensor([-1 if i in held else 100 + i for i in range(len(eps))])
    return {'episodes': list(eps), 'serials': serials, 'capacity_steps': 500, 'maximum_episodes': 64,
            'sampler': {'rng': np.random.default_rng(5).bit_generator.state, 'val_rng': np.random.default_rng(6).bit_generator.state,
                        'sym_rng': None, 'prio_batches': 7}}


# ---------------------------------------------------------------------------------------------------------------- the key
def test_the_key_parses():
    from handyrl_b200.train import save_replay
    for off in ({}, {'save_replay': None}, {'save_replay': False}, {'save_replay': 0}):
        assert save_replay(off) is None
    assert save_replay({'save_replay': True}) == {'every': 1, 'keep': 2}
    assert save_replay({'save_replay': 5}) == {'every': 5, 'keep': 2}
    assert save_replay({'save_replay': {'every': 3, 'keep': 0}}) == {'every': 3, 'keep': 0}
    assert save_replay({'save_replay': {'keep': 4}}) == {'every': 1, 'keep': 4}


@pytest.mark.parametrize('bad', [-1, 1.5, 2.0, 'yes', [1], {'every': 0}, {'every': True}, {'keep': -1}, {'keep': 1.0},
                                 {'each': 2}, float('nan')])
def test_a_bad_key_raises_when_the_trainer_is_built(bad):
    from handyrl_b200.nets import tictactoe_net
    from handyrl_b200.train import Trainer, save_replay
    with pytest.raises(ValueError):
        save_replay({'save_replay': bad})
    with pytest.raises(ValueError):
        Trainer({'batch_size': 4, 'forward_steps': 4, 'save_replay': bad}, tictactoe_net())


def test_the_key_needs_the_gpu_replay():
    from handyrl_b200.train import Trainer, save_replay
    with pytest.raises(ValueError, match='gpu_replay'):
        save_replay({'save_replay': True, 'gpu_replay': False})
    with pytest.raises(ValueError, match='gpu_replay'):
        Trainer({'batch_size': 4, 'forward_steps': 4, 'save_replay': 2, 'gpu_replay': False}, torch.nn.Identity())
    assert save_replay({'save_replay': 0, 'gpu_replay': False}) is None


def test_without_the_key_the_trainer_has_no_writer_and_no_numbering():
    from handyrl_b200.train import Trainer
    before = threading.active_count()
    tr = Trainer({'batch_size': 4, 'forward_steps': 4}, torch.nn.Identity())
    assert tr.save_replay is None and tr.replay_files is None and tr.checkpoint_files is None and tr.restored is None
    on = Trainer({'batch_size': 4, 'forward_steps': 4, 'save_replay': True}, torch.nn.Identity())
    assert on.replay_files is not None and on.replay_files.thread is None      # the writer thread starts with the first file
    assert on.checkpoint_files is not None and on.ema_files is None and on.optim_files is None
    assert threading.active_count() == before


# ---------------------------------------------------------------------------------------------------------------- resident lists
def test_the_resident_list_follows_the_directory():
    from handyrl_b200.replay import DeviceReplay
    from handyrl_b200.wire import episode_to_flat
    eps = _episodes(60, seed=3)
    for capacity, max_episodes in ((60, 50), (400, 5)):          # evict by steps (the ring wraps), by episode count
        replay = DeviceReplay(capacity, max_episodes, device='cpu', track=True)
        stored = []
        for lo in range(0, len(eps), 4):
            chunk = eps[lo:lo + 4]
            handles = replay.commit(replay.stage([episode_to_flat(e) for e in chunk], chunk))
            stored += list(zip(chunk, handles))
            live = replay.handles
            assert len(replay.resident) == len(live) == len(replay)
            # the newest len(live) stored episodes, in order: same objects, same rows
            assert all(r is e for r, (e, _) in zip(replay.resident, stored[-len(live):]))
            assert live == [h for _, h in stored[-len(live):]]
            slots, serials = replay.positions()
            first = len(stored) - len(live)
            assert serials.tolist() == list(range(first, len(stored)))             # serial = the order of storing
            assert np.array_equal(replay._serial[slots], serials) and len(set(slots.tolist())) == len(live)
        assert len(replay) < len(eps) and (replay.write < capacity)
    plain = DeviceReplay(60, 50, device='cpu')
    plain.add(eps[0])
    assert plain.resident is None
    with pytest.raises(ValueError):
        replay.stage([episode_to_flat(eps[0])], eps[:2])


# ---------------------------------------------------------------------------------------------------------------- the file
def test_the_file_round_trips_both_wire_formats_and_loads_without_the_package(tmp_path):
    from handyrl_b200.train import ReplayCheckpoints, load_replay_file, replay_file
    from handyrl_b200.wire import episode_to_flat
    eps = _episodes(12, flat={1, 4, 7})
    assert 'flat' in eps[1] and eps[1]['moment'] == [] and 'flat' not in eps[0]
    state = {'slot_serial': torch.tensor([105, -1, 3, 100, 111]), 'priority': torch.tensor([0.5, 1.0, 0.7, 0.2, 0.9]),
             'max_prio': 1.25}
    limiter = {'limit': 4.0, 'trained': 640, 'stored': 200, 'waited': 0.5, 'waiting': False}
    files = ReplayCheckpoints(str(tmp_path / 'models'))
    path = files.write(3, replay_file(_snapshot(eps, held={2}), state, limiter, steps=77, epoch=3))
    assert path == str(tmp_path / 'models' / '3.replay.pth') and os.listdir(tmp_path / 'models') == ['3.replay.pth']
    d = load_replay_file(path, leaf_shapes=[(3, 3, 3)], actions=9)
    assert d['format'] == 1 and d['steps'] == 77 and d['epoch'] == 3 and d['limiter'] == limiter
    assert d['capacity_steps'] == 500 and d['maximum_episodes'] == 64
    assert d['serials'].dtype == torch.int64 and d['serials'].tolist() == [100, 101, -1] + list(range(103, 112))
    # keyed by serial: the slot without an episode, the evicted serial 3 are gone; serial 102 is held out, so never there
    assert d['priorities']['serial'].tolist() == [100, 105, 111]
    assert d['priorities']['priority'].tolist() == pytest.approx([0.2, 0.5, 0.9]) and d['priorities']['max_prio'] == 1.25
    assert d['sampler']['prio_batches'] == 7 and d['sampler']['sym_rng'] is None
    rng = np.random.default_rng()
    rng.bit_generator.state = d['sampler']['rng']
    assert rng.random() == np.random.default_rng(5).random()
    for got, want in zip(d['episodes'], eps):
        assert got == want                                           # bytes, dicts and numbers: exactly as they arrived
        a, b = episode_to_flat(got), episode_to_flat(want)
        assert np.array_equal(a.action, b.action) and np.array_equal(a.outcome, b.outcome)
    # plain torch.load in a process that never imports this package
    code = ("import sys, torch; d = torch.load(sys.argv[1]); assert not any(m.startswith('handyrl') for m in sys.modules); "
            "print(len(d['episodes']), d['format'], d['priorities']['serial'].tolist())")
    out = subprocess.run([sys.executable, '-c', code, path], capture_output=True, text=True, cwd=str(tmp_path))
    assert out.returncode == 0, out.stderr
    assert out.stdout.split('\n')[0] == '12 1 [100, 105, 111]'
    # without prioritised replay there are no priorities
    assert replay_file(_snapshot(eps))['priorities'] is None


def test_an_interrupted_write_leaves_no_file(tmp_path, monkeypatch):
    from handyrl_b200 import train
    files = train.ReplayCheckpoints(str(tmp_path))
    obj = train.replay_file(_snapshot(_episodes(3)))

    def interrupted(src, dst):
        assert os.path.exists(src) and not src.endswith('.replay.pth') and not os.path.exists(dst)     # written under another name
        raise OSError('interrupted before the rename')

    monkeypatch.setattr(train.os, 'replace', interrupted)
    with pytest.raises(OSError):
        files.write(1, obj)
    assert os.listdir(tmp_path) == [] and files.written == []
    monkeypatch.undo()
    files.write(1, obj)
    assert os.listdir(tmp_path) == ['1.replay.pth']


def test_retention_keeps_the_newest_and_never_a_foreign_file(tmp_path):
    from handyrl_b200.train import ReplayCheckpoints, replay_file
    obj = replay_file(_snapshot(_episodes(2)))
    foreign = tmp_path / '1.replay.pth'                  # an earlier run's file, and the Learner's own checkpoints
    foreign.write_bytes(b'earlier run')
    (tmp_path / '2.pth').write_bytes(b'model')
    files = ReplayCheckpoints(str(tmp_path), keep=2)
    for epoch in (2, 3, 4, 5):
        files.write(epoch, obj)
    assert sorted(os.listdir(tmp_path)) == ['1.replay.pth', '2.pth', '4.replay.pth', '5.replay.pth']
    assert foreign.read_bytes() == b'earlier run'
    everything = ReplayCheckpoints(str(tmp_path / 'all'), keep=0)
    for epoch in range(1, 6):
        everything.write(epoch, obj)
    assert len(os.listdir(tmp_path / 'all')) == 5


def test_the_writer_thread_keeps_at_most_one_waiting_and_ends_with_close(tmp_path, monkeypatch):
    from handyrl_b200 import train
    files = train.ReplayCheckpoints(str(tmp_path), keep=0)
    obj = train.replay_file(_snapshot(_episodes(2)))
    gate, started = threading.Event(), threading.Event()
    real_save = torch.save

    def slow_save(o, f):
        started.set()
        assert gate.wait(20)
        real_save(o, f)

    monkeypatch.setattr(train.torch, 'save', slow_save)
    before = threading.active_count()
    files.submit(1, obj)                          # returns at once; the writer is now inside the (held) save of epoch 1
    assert started.wait(20) and threading.active_count() == before + 1
    files.submit(2, obj)
    files.submit(3, obj)                          # replaces epoch 2, which still waited
    assert files.replaced == 1 and files.queued[0] == 3
    gate.set()
    files.close()                                 # writes what waits, then joins
    assert sorted(os.listdir(tmp_path)) == ['1.replay.pth', '3.replay.pth']
    assert files.thread is None and threading.active_count() == before
    with pytest.raises(RuntimeError):
        files.submit(4, obj)


# ---------------------------------------------------------------------------------------------------------------- trainer
class _Pending:
    """What Trainer.update() reads of a PendingModel."""

    def __init__(self, snapshot, steps):
        self.replay, self.priority_state, self.steps = snapshot, None, steps
        self.ema_state = self.optim_state = self.replay_ratio = None
        self.batch_cnt = 4

    def resolve(self):
        return 'model', {'dcnt': 10.0}


def _fake_pending():
    from handyrl_b200 import train
    return type('P', (train.PendingModel,), {'__init__': _Pending.__init__, 'resolve': _Pending.resolve})


def test_update_numbers_the_files_like_the_other_checkpoints(tmp_path, monkeypatch):
    from handyrl_b200.train import Trainer
    monkeypatch.chdir(tmp_path)
    eps = _episodes(4)
    tr = Trainer({'batch_size': 4, 'forward_steps': 4, 'save_replay': {'every': 3, 'keep': 0}, 'restart_epoch': 4},
                 torch.nn.Identity())
    Pending = _fake_pending()
    for k in range(6):                            # epochs 5 .. 10: every third NUMBER, i.e. 6 and 9
        tr.update_queue.put((Pending(_snapshot(eps), 100 + k), 100 + k))
        assert tr.update() == ('model', 100 + k)
        assert tr.checkpoint_files.epoch == 5 + k
    tr.stop()
    assert sorted(os.listdir('models')) == ['6.replay.pth', '9.replay.pth']
    d = torch.load('models/9.replay.pth')
    assert d['epoch'] == 9 and d['steps'] == 104 and len(d['episodes']) == 4
    assert tr.replay_files.thread is None


def test_a_restarted_trainer_starts_from_the_file(tmp_path, monkeypatch, capsys):
    from handyrl_b200.train import ReplayCheckpoints, Trainer, replay_file
    monkeypatch.chdir(tmp_path)
    eps = _episodes(10, flat={3})
    limiter = {'limit': 2.0, 'trained': 64, 'stored': 70, 'waited': 0.0, 'waiting': False}
    ReplayCheckpoints('models').write(7, replay_file(_snapshot(eps, held={1, 5}), None, limiter, steps=900, epoch=7))
    args = {'batch_size': 4, 'forward_steps': 4, 'minimum_episodes': 8, 'num_batchers': 1, 'save_replay': True,
            'restart_epoch': 7, 'replay_ratio': 2}
    capsys.readouterr()
    tr = Trainer(args, torch.nn.Identity())
    assert capsys.readouterr().out.splitlines() == [
        'restored replay: 10 episodes (2 held out), %d steps, priorities: no' % sum(e['steps'] for e in eps)]
    assert list(tr.episodes) == eps and tr.restored is not None
    assert tr.replay_ratio_stats()['restored'] == limiter and tr.replay_ratio_stats()['stored'] == 0
    # a listener attached now sees what the Learner appends next, and the deque trims as the Learner trims it
    seen = []
    tr.episodes.listener = seen.append
    tr.episodes.append(eps[0])
    tr.episodes.popleft()
    assert seen == [eps[0]] and len(tr.episodes) == 10
    # run() finds minimum_episodes satisfied: it does not wait for new episodes (a parameterless model trains nothing)
    th = threading.Thread(target=tr.run, daemon=True)
    th.start()
    model, steps = tr.update()
    tr.stop()
    th.join(timeout=10)
    assert not th.is_alive() and model is tr.model
    assert capsys.readouterr().out.splitlines()[0] == 'waiting training'

    # the listeners of an EpisodeDeque see preloaded episodes as they see appended ones
    from handyrl_b200.train import EpisodeDeque
    dq, seen = EpisodeDeque(), []
    dq.listener = seen.append
    dq.extend(eps)
    assert seen == eps

    # no file for the epoch: one line, then an empty replay as without the key; key off: the file is not even looked for
    tr = Trainer(dict(args, restart_epoch=8), torch.nn.Identity())
    assert capsys.readouterr().out.splitlines() == ['handyrl_b200: no %s, the replay starts empty'
                                                    % os.path.join('models', '8.replay.pth')]
    assert len(tr.episodes) == 0 and tr.restored is None
    off = Trainer({k: v for k, v in args.items() if k != 'save_replay'}, torch.nn.Identity())
    assert capsys.readouterr().out == '' and len(off.episodes) == 0 and 'restored' not in off.replay_ratio_stats()


def test_a_file_that_does_not_fit_raises_and_loads_nothing(tmp_path, monkeypatch):
    from handyrl_b200.nets import tictactoe_net
    from handyrl_b200.train import ReplayCheckpoints, Trainer, load_replay_file, replay_file
    monkeypatch.chdir(tmp_path)
    eps = _episodes(5)
    files = ReplayCheckpoints('models', keep=0)
    good = replay_file(_snapshot(eps))
    undecodable = [dict(eps[0], moment=[b'not bz2'])] + eps[1:]
    cases = {1: dict(good, format=2), 2: {k: v for k, v in good.items() if k != 'sampler'},
             3: dict(good, serials=good['serials'][:-1]), 4: dict(good, episodes=eps[:-1] + [{'steps': 3}]),
             5: dict(good, episodes=undecodable), 6: [1, 2, 3]}
    for epoch, obj in cases.items():
        files.write(epoch, obj)
    (tmp_path / 'models' / '7.replay.pth').write_bytes(b'truncated')
    for epoch in range(1, 8):
        path = os.path.join('models', '%d.replay.pth' % epoch)
        with pytest.raises(ValueError) as err:
            load_replay_file(path)
        assert path in str(err.value)
        with pytest.raises(ValueError):
            Trainer({'batch_size': 4, 'forward_steps': 4, 'save_replay': True, 'restart_epoch': epoch}, torch.nn.Identity())
    files.write(8, good)
    assert len(load_replay_file('models/8.replay.pth')['episodes']) == 5
    for wrong in (dict(leaf_shapes=[(3, 4, 4)]), dict(leaf_shapes=[(3, 3, 3), (2,)]), dict(actions=7)):
        with pytest.raises(ValueError, match='8.replay.pth'):
            load_replay_file('models/8.replay.pth', **wrong)
    # the Trainer checks the episodes against its net: another board, another action count
    tr = Trainer.__new__(Trainer)
    tr.model = tictactoe_net()
    tr.params = list(tr.model.parameters())
    tr._check_fits_net(eps[0], 'f')
    tr.model.training or pytest.fail('the check leaves the net in training mode as it found it')
    tr.model = torch.nn.Sequential(torch.nn.Flatten(), torch.nn.Linear(5, 9))
    tr.params = list(tr.model.parameters())
    with pytest.raises(ValueError, match='observations'):
        tr._check_fits_net(eps[0], 'f')

    class SevenActions(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.fc = torch.nn.Linear(27, 7)

        def forward(self, x, hidden=None):
            return {'policy': self.fc(x.flatten(1))}

    tr.model = SevenActions()
    tr.params = list(tr.model.parameters())
    with pytest.raises(ValueError, match='9 actions, the net has 7'):
        tr._check_fits_net(eps[0], 'f')


# ---------------------------------------------------------------------------------------------------------------- priorities
def test_saved_priorities_map_onto_the_restored_ring():
    from handyrl_b200 import priority
    # the saved ring: serials 40..47 resident (position 2 and 6 of the list are held out), slot state with leftovers
    saved_serials = np.array([40, 41, -1, 42, 43, 44, -1, 45, 46, 47])
    slot_serial = np.array([44, 45, 46, -1, 12, 39, 40, 41, 42, 43])       # 47 is resident but the sampler has not seen it
    prio = np.arange(10, dtype=np.float32) / 10 + 0.05
    img = priority.image(slot_serial, prio, 2.5, saved_serials)
    assert img['serial'].tolist() == [40, 41, 42, 43, 44, 45, 46] and img['max_prio'] == 2.5          # 12 and 39 were evicted
    assert img['priority'].tolist() == pytest.approx([0.65, 0.75, 0.85, 0.95, 0.05, 0.15, 0.25])
    # the restored ring kept the training episodes from list position 3 on (the two oldest did not fit) and then stored
    # two new episodes; it gave them slots 0.. and serials 0..
    positions = np.array([3, 4, 5, 7, 8, 9, -1, -1])
    slots, serials = np.arange(8), np.arange(8)
    s, ser, p = priority.restore_entries(img, saved_serials, positions, slots, serials)
    assert s.tolist() == [0, 1, 2, 3, 4] and ser.tolist() == [0, 1, 2, 3, 4]       # 42 43 44 45 46; 47 and the new ones: none
    assert p.tolist() == pytest.approx([0.85, 0.95, 0.05, 0.15, 0.25])
    assert len(set(s.tolist())) == len(s)
    # a ring that wrapped its directory: slots are not positions
    s, ser, p = priority.restore_entries(img, saved_serials, np.array([8, 0]), np.array([9, 0]), np.array([30, 31]))
    assert (s.tolist(), ser.tolist()) == ([9, 0], [30, 31]) and p.tolist() == pytest.approx([0.25, 0.65])
    # a held-out position has serial -1 and gets nothing; nothing saved gives nothing
    s, _, _ = priority.restore_entries(img, saved_serials, np.array([2, 6]), np.array([0, 1]), np.array([0, 1]))
    assert s.size == 0
    empty = priority.image(np.full(4, -1), np.ones(4, np.float32), 1.0, saved_serials)
    assert empty['serial'].size == 0
    assert priority.restore_entries(empty, saved_serials, positions, slots, serials)[0].size == 0
    # one episode cannot get two priorities, and two episodes cannot share a saved position
    with pytest.raises(ValueError):
        priority.restore_entries(img, saved_serials, np.array([3, 3]), np.array([0, 1]), np.array([0, 1]))
    with pytest.raises(ValueError):
        priority.restore_entries(dict(img, serial=np.array([40, 40, 42, 43, 44, 45, 46])), saved_serials, positions, slots, serials)
    with pytest.raises(ValueError):
        priority.restore_entries(img, saved_serials, np.array([10]), np.array([0]), np.array([0]))
