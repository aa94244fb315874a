"""Replay ratio limit on the GPU: the drop-in Trainer with the TicTacToe BoardNet on an EpisodeDeque that a producer fills in
bursts trains up to the limit and not past it (within one step, or one chunk with several GPUs), held-out episodes give no
credit, update() returns while the trainer waits for credit, and without the key the learner step is the same."""
import os
import pickle
import re
import threading
import time

import pytest
import torch

from conftest import GOLDEN

pytestmark = pytest.mark.gpu

NGPU = torch.cuda.device_count() if torch.cuda.is_available() else 0
R = 4.0                 # samples trained per stored step: an episode of 5-9 steps pays for about half a batch


def _args(**extra):
    with open(os.path.join(GOLDEN, 'batch_cases.pkl'), 'rb') as f:
        case = pickle.load(f)['tictactoe']
    return dict(case['args'], batch_size=8, minimum_episodes=4, num_batchers=1, **{'lambda': 0.7}, seed=5,
                entropy_regularization=0.1, entropy_regularization_decay=0.1, policy_target='UPGO', value_target='VTRACE',
                gpu_replay=True, num_gpus=1, **extra)


def _credit(episodes, rate):
    """Steps of the episodes that enter the training replay (held-out ones give no credit)."""
    from handyrl_b200.replay import held_out
    from handyrl_b200.wire import episode_to_flat
    return sum(ep['steps'] for ep in episodes if not held_out(episode_to_flat(ep), rate))


def _settle(tr, stored, chunk=1, timeout=180.0):
    """Wait until the feeder has stored `stored` steps and the trainer waits for credit with less than one step (chunk) of it
    left unspent.  A limiter that under-trains never gets there."""
    spb = tr.limiter.samples_per_batch
    t0 = time.monotonic()
    while True:
        s = tr.limiter.snapshot()
        if s['stored'] == stored and s['waiting'] and s['trained'] + chunk * spb > R * s['stored']:
            return s
        assert time.monotonic() - t0 < timeout, ('never settled', s, stored)
        time.sleep(0.01)


def _update_returns(tr, timeout=60.0):
    out = []
    u = threading.Thread(target=lambda: out.append(tr.update()), daemon=True)
    u.start()
    u.join(timeout)
    assert not u.is_alive(), 'update() did not return while the trainer waited for credit'
    return out[0]


def _bursts(tr, episodes, rate, chunk, sizes):
    """The backlog (sizes[0] episodes) is already in tr.episodes; feed the rest in bursts of sizes[1:] and check the bound
    after each.  After every other burst update() ends two epochs: the first spent the burst's credit and ends without another
    step, the second has no credit and lets one step (chunk) through over the limit."""
    spb = tr.limiter.samples_per_batch
    stored = _credit(episodes[:sizes[0]], rate)
    i = sizes[0]
    forced = False
    for n, size in enumerate(sizes):
        if n:
            tr.episodes.extend(episodes[i:i + size])
            stored += _credit(episodes[i:i + size], rate)
            i += size
        s = _settle(tr, stored, chunk)
        # within the limit (plus the forced step, which the next burst's credit pays first) and within one step of it
        assert R * stored - chunk * spb < s['trained'] <= R * stored + (chunk * spb if forced else 0), (n, s, stored)
        assert s['trained'] == tr.steps * spb and tr.steps % chunk == 0
        if n % 2 == 1:
            _update_returns(tr)
            before = tr.steps
            _, steps = _update_returns(tr)
            assert steps == before + chunk
            s = _settle(tr, stored, chunk)
            assert R * stored < s['trained'] <= R * stored + chunk * spb, (n, s, stored)
            forced = True
    return stored


@pytest.mark.parametrize('rate', [None, 0.5], ids=['all_trained', 'validation_rate'])
def test_trainer_trains_up_to_the_limit_after_each_burst(rate, capsys):
    from handyrl_b200.nets import tictactoe_net
    from handyrl_b200.synthetic import tictactoe_episodes
    from handyrl_b200.train import Trainer
    episodes = tictactoe_episodes(120, seed=17)
    tr = Trainer(_args(replay_ratio=R, validation_rate=rate), tictactoe_net())
    sizes = [8, 20, 20, 20, 20, 20]
    tr.episodes.extend(episodes[:sizes[0]])
    assert _credit(episodes[:sizes[0]], rate) > 0
    th = threading.Thread(target=tr.run, daemon=True)
    th.start()
    try:
        stored = _bursts(tr, episodes, rate, 1, sizes)
        _update_returns(tr)
        out = capsys.readouterr().out
        stats = tr.replay_ratio_stats()
        launches = tr.stepper.launches_per_step
    finally:
        tr.stop()
        th.join(timeout=30)
    assert not th.is_alive()
    assert stored == stats['stored'] and stats['limit'] == R
    if rate is not None:
        assert stored < sum(ep['steps'] for ep in episodes[:sum(sizes)])      # held-out episodes gave no credit
        assert tr.gpu_batcher.validation_ready()
    lines = out.splitlines()
    ratio_lines = [i for i, l in enumerate(lines) if l.startswith('replay_ratio = ')]
    assert len(ratio_lines) >= 6, out
    for i in ratio_lines:
        assert re.fullmatch(r'replay_ratio = (\d+\.\d )?limit:4 waited:[01]\.\d\d', lines[i]), lines[i]
        assert lines[i - 1].startswith('loss = '), out
    assert sum(l.startswith('replay_ratio = ') for l in lines) == sum(l.startswith('loss = ') for l in lines)
    if rate is not None:
        assert any(l.startswith('validation = ') and lines[i - 1].startswith('replay_ratio = ')
                   for i, l in enumerate(lines)), out
    # the key does not touch the learner step
    plain = Trainer(_args(validation_rate=rate), tictactoe_net())
    plain.episodes.extend(episodes[:sizes[0]])
    th = threading.Thread(target=plain.run, daemon=True)
    th.start()
    try:
        plain.update()
        plain_out = capsys.readouterr().out
    finally:
        plain.stop()
        th.join(timeout=30)
    assert plain.limiter is None and plain.replay_ratio_stats() is None
    assert plain.stepper.launches_per_step == launches
    assert 'replay_ratio' not in plain_out and 'loss = ' in plain_out


@pytest.mark.skipif(NGPU < 2, reason='needs at least 2 GPUs')
def test_sharded_trainer_commands_whole_chunks_within_the_limit():
    from handyrl_b200.nets import tictactoe_net
    from handyrl_b200.synthetic import tictactoe_episodes
    from handyrl_b200.train import Trainer
    chunk = 4
    args = _args(replay_ratio=R, multi_gpu_chunk=chunk)
    args['num_gpus'] = 2
    episodes = tictactoe_episodes(120, seed=23)
    tr = Trainer(args, tictactoe_net())
    assert tr.world == 2
    sizes = [16, 30, 30, 30]
    tr.episodes.extend(episodes[:sizes[0]])
    th = threading.Thread(target=tr.run, daemon=True)
    th.start()
    try:
        _bursts(tr, episodes, None, chunk, sizes)
    finally:
        tr.stop()
        th.join(timeout=60)
    assert not th.is_alive()
