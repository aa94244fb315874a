"""Replay ratio limit without a GPU: the key's checks, the limiter's arithmetic (allowed steps from stored steps, backlog
credit, chunks, the epoch figures), the printed line, and the Trainer's own loop on fakes of the step and the feeder: a waiting
trainer wakes when steps are stored, update() gets one step through, stop() ends a waiting trainer."""
import re
import threading
import time

import numpy as np
import pytest
import torch

from handyrl_b200._capi import NUM_LOSS
from handyrl_b200.train import PendingModel

HEADS = ['p', 'v', 'ent', 'total']


@pytest.mark.parametrize('value', [-1, -0.5, float('-inf'), float('inf'), float('nan'), True, 'x', '32', [32], {'r': 32}])
def test_refused_values(value):
    from handyrl_b200.train import replay_ratio
    with pytest.raises(ValueError):
        replay_ratio({'replay_ratio': value})


def test_off_and_accepted_values():
    from handyrl_b200.train import replay_ratio
    for off in ({}, {'replay_ratio': None}, {'replay_ratio': 0}, {'replay_ratio': 0.0}, {'replay_ratio': False}):
        assert replay_ratio(off) is None
    assert replay_ratio({'replay_ratio': 32}) == 32.0
    assert replay_ratio({'replay_ratio': 0.25}) == 0.25
    assert replay_ratio({'replay_ratio': np.float64(8)}) == 8.0
    assert replay_ratio({'replay_ratio': 4, 'gpu_replay': False}) == 4.0


@pytest.mark.parametrize('bad', [-1, True, 'fast'])
def test_trainer_refuses_a_bad_key_before_touching_a_device(bad):
    from handyrl_b200.nets import tictactoe_net
    from handyrl_b200.train import Trainer
    with pytest.raises(ValueError):
        Trainer({'batch_size': 4, 'forward_steps': 4, 'replay_ratio': bad}, tictactoe_net())


def test_allowed_steps_follow_the_stored_steps():
    from handyrl_b200.train import ReplayRatioLimiter
    lim = ReplayRatioLimiter(4, 8 * 8)              # r = 4, batch_size 8 x forward_steps 8 = 64 samples per batch
    assert not lim.allows(1)
    lim.store(15)                                  # 60 samples of credit: less than one batch
    assert not lim.allows(1)
    lim.store(1)                                   # 64: exactly one
    assert lim.allows(1) and not lim.allows(2)
    lim.drew()
    assert lim.trained == 64 and not lim.allows(1)
    lim.store(48)                                  # 64 stored steps -> 256 samples: three more batches
    for _ in range(3):
        assert lim.allows(1)
        lim.drew()
    assert not lim.allows(1) and lim.trained == 4 * lim.stored


def test_fractional_limit():
    from handyrl_b200.train import ReplayRatioLimiter
    lim = ReplayRatioLimiter(0.5, 10)
    lim.store(19)
    assert not lim.allows(1)
    lim.store(1)
    assert lim.allows(1) and not lim.allows(2)


def test_backlog_credit_is_spent_at_once():
    from handyrl_b200.train import ReplayRatioLimiter
    lim = ReplayRatioLimiter(32, 6 * 8)
    lim.store(7 * 100)                             # a backlog of 100 episodes of 7 steps: 22400 samples, 466 batches
    for _ in range(22400 // 48):
        assert lim.acquire(1, lambda: True)        # credit: returns at once, without waiting
        lim.drew()
    assert lim.waited == 0.0
    assert not lim.acquire(1, lambda: True)


def test_chunks_pass_only_whole():
    from handyrl_b200.train import ReplayRatioLimiter
    lim = ReplayRatioLimiter(1, 10)
    lim.store(39)                                  # three batches of credit, a chunk of four does not fit
    assert lim.allows(3) and not lim.allows(4)
    assert lim.acquire(4, lambda: True) is False   # interrupted: no credit for the whole chunk
    lim.store(1)
    assert lim.acquire(4, lambda: True) is True    # credit wins over the interrupt


def test_epoch_figures_and_line():
    from handyrl_b200.train import ReplayRatioLimiter, replay_ratio_line
    now = [100.0]
    lim = ReplayRatioLimiter(32, 48, clock=lambda: now[0])
    lim.store(50)                                  # before the first epoch starts: counts in it
    lim.start_epoch()
    lim.start_epoch()                              # only the first call starts the clock
    for _ in range(20):
        lim.drew()
    now[0] = 104.0
    ep = lim.end_epoch()
    assert ep == {'trained': 960, 'stored': 50, 'ratio': 960 / 50, 'limit': 32.0, 'waited': 0.0, 'wall': 4.0}
    assert replay_ratio_line(ep) == 'replay_ratio = 19.2 limit:32 waited:0.00'
    lim.waited += 1.0                              # what acquire() adds
    lim.drew()
    now[0] = 108.0
    ep = lim.end_epoch()                           # nothing stored in this epoch: no ratio
    assert ep['trained'] == 48 and ep['stored'] == 0 and ep['ratio'] is None and ep['waited'] == 0.25
    assert replay_ratio_line(ep) == 'replay_ratio = limit:32 waited:0.25'
    assert replay_ratio_line(dict(ep, ratio=31.74, limit=0.5, waited=0.43)) == 'replay_ratio = 31.7 limit:0.5 waited:0.43'
    assert lim.snapshot() == {'limit': 32.0, 'trained': 21 * 48, 'stored': 50, 'waited': 1.0, 'waiting': False}


def test_the_line_is_not_a_loss_line():
    from handyrl_b200.train import replay_ratio_line
    line = replay_ratio_line({'ratio': 31.7, 'limit': 32.0, 'waited': 0.43})
    assert line == 'replay_ratio = 31.7 limit:32 waited:0.43'
    assert not line.startswith('loss')             # the reference's scripts/loss_plot.py takes line.startswith('loss')


def _report(replay_ratio=None, skip=False):
    host = torch.zeros(NUM_LOSS + (1 if skip else 0), dtype=torch.float64)
    host[:NUM_LOSS] = torch.tensor([51.2, 23.1, 0.0, 184.3, 56.1, 100.0], dtype=torch.float64)
    if skip:
        host[-1] = 2
    pm = PendingModel(None, None, None, host, HEADS, None, skip_nonfinite=skip, batch_cnt=10)
    pm.replay_ratio = replay_ratio
    pm.report()


def test_pending_model_prints_the_line_after_the_loss_and_skipped_lines(capsys):
    _report()
    plain = capsys.readouterr().out
    assert 'replay_ratio' not in plain
    _report(skip=True)
    skipped = capsys.readouterr().out
    stats = {'trained': 960, 'stored': 30, 'ratio': 32.0, 'limit': 32.0, 'waited': 0.5, 'wall': 1.0}
    _report(stats)
    assert capsys.readouterr().out == plain + 'replay_ratio = 32.0 limit:32 waited:0.50\n'
    _report(stats, skip=True)
    assert capsys.readouterr().out == skipped + 'replay_ratio = 32.0 limit:32 waited:0.50\n'


# ---------------------------------------------------------------------------------------------------- the Trainer's loop
class _Pending(PendingModel):
    """What LearnerStep.end_epoch hands over, without a device: report() prints the lines, resolve() returns a placeholder."""

    def __init__(self, batch_cnt):
        host = torch.zeros(NUM_LOSS, dtype=torch.float64)
        host[:] = batch_cnt                        # dcnt > 0: update() takes the epoch
        super().__init__(None, None, None, host, HEADS, None, batch_cnt=batch_cnt)

    def resolve(self):
        return 'model', self.report()


class _Stepper:
    def __init__(self):
        self.steps = 0
        self.stream = type('S', (), {'synchronize': lambda self: None})()

    def step_in_place(self):
        self.steps += 1

    def end_epoch(self, batch_cnt, steps, default_lr, template, heads):
        return _Pending(batch_cnt)


class _Batcher:
    def ready(self):
        return True

    def fill(self, stepper):
        pass

    def validation_ready(self):
        return False

    def stop(self):
        pass


SPB = 6 * 8


def _trainer(ratio=4):
    """A Trainer whose step and GPU batcher are fakes: train() / run() / update() / stop() are the real ones."""
    from handyrl_b200.train import Trainer
    tr = Trainer({'batch_size': 6, 'forward_steps': 8, 'minimum_episodes': 0, 'num_batchers': 1, 'replay_ratio': ratio},
                 torch.nn.Identity())
    tr.params = [torch.zeros(1)]
    tr.stepper, tr.gpu_batcher = _Stepper(), _Batcher()
    tr.cpu_template, tr.heads = None, HEADS
    return tr


def _until(cond, timeout=10.0):
    t0 = time.monotonic()
    while not cond():
        if time.monotonic() - t0 > timeout:
            return False
        time.sleep(0.002)
    return True


def test_trainer_waits_for_credit_and_wakes_when_steps_are_stored(capsys):
    tr = _trainer(ratio=4)
    lim = tr.limiter
    assert lim.samples_per_batch == SPB
    th = threading.Thread(target=tr.run, daemon=True)
    lim.store(24)                                  # the backlog: 96 samples, two batches
    th.start()
    try:
        assert _until(lambda: lim.waiting)
        assert tr.steps == 2 and tr.stepper.steps == 2
        time.sleep(0.2)
        assert tr.steps == 2                       # no credit, no step

        def feeder():                              # what GpuBatcher._feed does after each commit
            for _ in range(5):
                lim.store(7)
                time.sleep(0.02)

        f = threading.Thread(target=feeder)
        f.start()
        f.join()
        stored = 24 + 35
        assert _until(lambda: lim.waiting and tr.steps == stored * 4 // SPB)
        assert tr.steps * SPB <= 4 * stored < (tr.steps + 1) * SPB     # within the limit, and not one step under it
        model, steps = tr.update()                 # the epoch has steps: update() ends it without another
        assert model == 'model' and steps == tr.steps == stored * 4 // SPB
        out = capsys.readouterr().out
        assert re.search(r'^replay_ratio = (\d+\.\d) limit:4 waited:(0\.\d\d|1\.00)$', out, re.M), out
        ep = tr.replay_ratio_stats()['epoch']
        assert ep['trained'] == steps * SPB and ep['stored'] == stored
        assert '%.1f' % ep['ratio'] in out
    finally:
        tr.stop()
        th.join(timeout=5)
    assert not th.is_alive()


def test_update_gets_one_step_through_an_epoch_without_credit():
    tr = _trainer(ratio=4)
    lim = tr.limiter
    th = threading.Thread(target=tr.run, daemon=True)
    th.start()
    try:
        assert _until(lambda: lim.waiting)
        assert tr.steps == 0
        for k in range(1, 4):                      # each update() forces one step over the limit, no more
            result = []
            u = threading.Thread(target=lambda: result.append(tr.update()))
            u.start()
            u.join(timeout=5)
            assert not u.is_alive() and result[0][1] == k
            assert _until(lambda: lim.waiting)
            assert tr.steps == k and lim.trained == k * SPB and lim.stored == 0
        lim.store(3 * SPB // 4)                    # credit for three batches: it pays the three forced steps first
        time.sleep(0.2)
        assert tr.steps == 3
        lim.store(SPB // 4)
        assert _until(lambda: tr.steps == 4 and lim.waiting)
        stats = tr.replay_ratio_stats()
        assert stats['trained'] == 4 * SPB and stats['stored'] == SPB and stats['waiting']
        assert stats['epoch']['trained'] == SPB and stats['epoch']['ratio'] is None
    finally:
        tr.stop()
        th.join(timeout=5)
    assert not th.is_alive()


def test_stop_ends_a_waiting_trainer_promptly():
    tr = _trainer(ratio=4)
    lim = tr.limiter
    tr.limiter.poll = 30.0                         # only the notification can end the wait in time
    th = threading.Thread(target=tr.run, daemon=True)
    th.start()
    assert _until(lambda: lim.waiting)
    t0 = time.monotonic()
    tr.stop()
    th.join(timeout=5)
    assert not th.is_alive() and time.monotonic() - t0 < 2.0
    assert tr.steps == 0 and lim.waited > 0


def test_update_wakes_a_waiting_trainer_promptly():
    tr = _trainer(ratio=4)
    tr.limiter.poll = 30.0
    th = threading.Thread(target=tr.run, daemon=True)
    th.start()
    try:
        assert _until(lambda: tr.limiter.waiting)
        t0 = time.monotonic()
        _, steps = tr.update()
        assert steps == 1 and time.monotonic() - t0 < 2.0
    finally:
        tr.stop()
        th.join(timeout=5)


def test_host_batcher_path_counts_the_deque_appends():
    """gpu_replay: False -- every episode appended to Trainer.episodes is stored; evictions do not lower the count."""
    from handyrl_b200.train import Trainer
    tr = Trainer({'batch_size': 6, 'forward_steps': 8, 'replay_ratio': 2, 'gpu_replay': False}, torch.nn.Identity())
    tr.episodes.extend([{'steps': 5}, {'steps': 9}])
    tr.episodes.append({'steps': 7})
    tr.episodes.popleft()
    assert tr.limiter.stored == 21
    plain = Trainer({'batch_size': 6, 'forward_steps': 8, 'gpu_replay': False}, torch.nn.Identity())
    assert plain.limiter is None and plain.episodes.listener is None and plain.replay_ratio_stats() is None
