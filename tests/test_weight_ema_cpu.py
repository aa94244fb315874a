"""Moving average of the learner's weights, without a GPU: the C ABI mirror of hrl_weight_ema, the decay check, the file names and
epoch numbers of the averaged checkpoints, and that a written averaged state_dict loads strictly into a fresh net."""
import ctypes
import os
import queue
import re
import threading

import pytest
import torch

from handyrl_b200.train import PendingModel

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ARGS = {'batch_size': 4, 'forward_steps': 2, 'num_batchers': 1, 'minimum_episodes': 1, 'maximum_episodes': 10}


def test_header_declares_and_binding_mirrors_hrl_weight_ema():
    from handyrl_b200 import _capi
    C = ctypes
    text = re.sub(r'\s+', ' ', re.sub(r'/\*.*?\*/', '', open(os.path.join(ROOT, 'include', 'hrl_b200.h')).read(), flags=re.S))
    assert ('int hrl_weight_ema(float *avg, const float *state, int64_t n, const int64_t *step, float decay, int32_t seeded, '
            'void *stream);') in text
    assert _capi.HRL_ABI_VERSION == 2
    res, argt = _capi.SYMBOLS['hrl_weight_ema']
    assert res is C.c_int
    assert argt == [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_float, C.c_int32, C.c_void_p]


def test_library_exports_hrl_weight_ema_and_refuses_bad_arguments():
    import __graft_entry__ as g
    g.build()
    from handyrl_b200._capi import lib
    got = []

    def refused():      # argument checks fail before anything touches a device
        buf, step = (ctypes.c_float * 8)(), (ctypes.c_int64 * 1)()
        got.append((lib().hrl_weight_ema(None, None, 4, None, 0.9, 0, None), lib().hrl_last_error()))
        got.append((lib().hrl_weight_ema(buf, buf, 4, step, 1.0, 0, None), lib().hrl_last_error()))

    th = threading.Thread(target=refused)         # the error text is per thread: keep this one's clean
    th.start()
    th.join()
    assert got[0][0] != 0 and b'hrl_weight_ema' in got[0][1]
    assert got[1][0] != 0 and b'decay' in got[1][1]


@pytest.mark.parametrize('bad', [1.0, 1.5, -0.1, float('nan'), True, '0.99', [0.9]])
def test_a_decay_outside_the_open_unit_interval_is_refused(bad):
    from handyrl_b200.train import LearnerStep, Trainer, weight_ema_decay
    with pytest.raises(ValueError):
        weight_ema_decay(bad)
    with pytest.raises(ValueError):
        Trainer(dict(ARGS, weight_ema=bad), torch.nn.Identity())
    with pytest.raises(ValueError):            # checked before the model goes to a device
        LearnerStep(torch.nn.Linear(2, 2), dict(ARGS, weight_ema=bad), None, lr=1e-3)
    with pytest.raises(ValueError):
        LearnerStep(torch.nn.Linear(2, 2), ARGS, None, lr=1e-3, weight_ema=bad)


def test_no_decay_means_no_averaging():
    from handyrl_b200.train import Trainer, weight_ema_decay
    for off in (None, 0, 0.0, False):
        assert weight_ema_decay(off) is None
    assert weight_ema_decay(0.999) == 0.999
    assert Trainer(ARGS, torch.nn.Identity()).ema_files is None
    assert Trainer(dict(ARGS, weight_ema=0), torch.nn.Identity()).ema_files is None
    assert Trainer(dict(ARGS, weight_ema=0.9), torch.nn.Identity()).ema_files is not None


class _Epoch(PendingModel):
    """Stands in for the PendingModel of one epoch: what resolve() hands back, with its averaged state_dict."""

    def __init__(self, dcnt, tag):        # (no device copy to wait for)
        self.dcnt, self.tag, self.batch_cnt = dcnt, tag, 1
        self.ema_state = {'w': torch.full((2,), float(tag))}

    def resolve(self):
        return 'model%d' % self.tag, {'dcnt': self.dcnt}


def _trainer_with_epochs(epochs, **extra):
    """A Trainer whose queue holds the given epochs (its update() runs on the host alone)."""
    from handyrl_b200.train import Trainer
    tr = Trainer(dict(ARGS, **extra), torch.nn.Identity())
    tr.update_queue = queue.Queue()
    for i, e in enumerate(epochs):
        tr.update_queue.put((e, 10 * (i + 1)))
    return tr


def test_files_are_numbered_like_the_learners_models(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    # epochs 2 and 4 have no sample with a turn in them: update() skips them, and they get no number
    tr = _trainer_with_epochs([_Epoch(5, 1), _Epoch(0, 2), _Epoch(3, 3), _Epoch(0, 4), _Epoch(0, 5), _Epoch(7, 6)], weight_ema=0.9)
    got = [tr.update() for _ in range(3)]
    assert got == [('model1', 10), ('model3', 30), ('model6', 60)]
    files = sorted(os.listdir('models'))
    assert files == ['1.ema.pth', '2.ema.pth', '3.ema.pth', 'latest.ema.pth']
    for epoch, tag in ((1, 1), (2, 3), (3, 6)):
        assert torch.equal(torch.load(os.path.join('models', '%d.ema.pth' % epoch))['w'], torch.full((2,), float(tag)))
    assert torch.equal(torch.load(os.path.join('models', 'latest.ema.pth'))['w'], torch.full((2,), 6.0))


def test_a_restarted_run_continues_the_numbering_and_finds_its_seed(tmp_path, monkeypatch):
    from handyrl_b200.train import AveragedCheckpoints
    monkeypatch.chdir(tmp_path)
    assert AveragedCheckpoints(0).seed_path() is None
    assert AveragedCheckpoints(7).seed_path() is None           # no file to resume from: a fresh average
    os.makedirs('models')
    torch.save({'w': torch.zeros(2)}, os.path.join('models', '7.ema.pth'))
    assert AveragedCheckpoints(7).seed_path() == os.path.join('models', '7.ema.pth')
    assert AveragedCheckpoints(0).seed_path() is None            # restart_epoch 0 never seeds
    tr = _trainer_with_epochs([_Epoch(0, 1), _Epoch(2, 2), _Epoch(2, 3)], weight_ema=0.999, restart_epoch=7)
    tr.update()
    tr.update()
    assert sorted(os.listdir('models')) == ['7.ema.pth', '8.ema.pth', '9.ema.pth', 'latest.ema.pth']
    assert torch.equal(torch.load(os.path.join('models', '8.ema.pth'))['w'], torch.full((2,), 2.0))


def test_without_the_key_update_writes_nothing(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    tr = _trainer_with_epochs([_Epoch(3, 1)])
    assert tr.update() == ('model1', 10)
    assert not os.path.exists('models')


@pytest.mark.parametrize('net', ['tictactoe_net', 'geese_net'])
def test_an_averaged_state_dict_loads_strictly_into_a_fresh_net(net, tmp_path, monkeypatch):
    """The hand-off rebuilds the averaged state_dict from a host image of StateStore.bytes whose fp32 words hold the average; the
    file it writes must load with strict=True (the Learner's --eval, aux_swa.py)."""
    from handyrl_b200 import nets
    from handyrl_b200.train import AveragedCheckpoints, StateStore
    monkeypatch.chdir(tmp_path)
    torch.manual_seed(0)
    model = getattr(nets, net)()
    keys = list(model.state_dict().keys())
    store = StateStore(model, 'cpu')
    flat = torch.zeros(store.n_pad)
    off = 0
    for k, p in model.named_parameters():           # what FlatAdam does on the device
        flat[off:off + p.numel()] = p.detach().reshape(-1)
        off += p.numel()
    store.bytes[:4 * store.n_pad] = flat.view(torch.uint8)
    store.index_params(model)
    live = store.bytes.clone()
    avg = torch.zeros_like(live)
    avg[:store.i_off] = (live[:store.i_off].view(torch.float32) * 0.5).view(torch.uint8)
    state = store.state_dict_from(store.averaged_bytes(avg, live), keys)
    assert list(state) == keys
    path = AveragedCheckpoints(0).save(state)
    fresh = getattr(nets, net)()
    fresh.load_state_dict(torch.load(path), strict=True)
    for k, v in model.state_dict().items():
        if v.dtype == torch.float32:
            assert torch.equal(fresh.state_dict()[k], v * 0.5), k
        else:                                        # int64 buffers (num_batches_tracked): the live model's
            assert torch.equal(fresh.state_dict()[k], v), k
    assert any(v.dtype == torch.int64 for v in model.state_dict().values())
