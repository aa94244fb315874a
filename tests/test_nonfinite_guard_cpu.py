"""Guard against non-finite optimiser steps, without a GPU: the C ABI mirror of hrl_clip_adam_step, hrl_step_commit and
hrl_weight_ema (their skip flags), how train_args['skip_nonfinite'] is read, the `skipped = ...` line, and the accumulator
layout PendingModel reads."""
import ctypes
import itertools
import os
import re
import threading

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C = ctypes

DECLS = {
    'hrl_clip_adam_step': (
        'int hrl_clip_adam_step(float *param, const float *grad, float *exp_avg, float *exp_avg_sq, int64_t n, '
        'const float *partials, const float *lr, int64_t *step, double max_norm, double beta1, double beta2, double eps, '
        'double weight_decay, float *grad_norm_out , double *diag_accum , const float *tail, int32_t n_tail, int32_t *skip , '
        'void *stream);',
        [C.c_void_p] * 4 + [C.c_int64] + [C.c_void_p] * 3 + [C.c_double] * 5 +
        [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    'hrl_step_commit': (
        'int hrl_step_commit(const int32_t *skip, const float *tail, int32_t n_tail, double *accum, double *skip_count, '
        'void *state, const void *saved, int64_t nbytes, void *stream);',
        [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    'hrl_weight_ema': (
        'int hrl_weight_ema(float *avg, const float *state, int64_t n, const int64_t *step, float decay, int32_t seeded, '
        'const int32_t *skip , void *stream);',
        [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_float, C.c_int32, C.c_void_p, C.c_void_p]),
}


@pytest.mark.parametrize('name', sorted(DECLS))
def test_header_declares_and_binding_mirrors(name):
    from handyrl_b200 import _capi
    text = re.sub(r'\s+', ' ', re.sub(r'/\*.*?\*/', '', open(os.path.join(ROOT, 'include', 'hrl_b200.h')).read(), flags=re.S))
    decl, argtypes = DECLS[name]
    assert decl in text
    assert _capi.HRL_ABI_VERSION == 3
    res, argt = _capi.SYMBOLS[name]
    assert res is C.c_int
    assert argt == argtypes


def test_library_refuses_bad_arguments_before_touching_a_device():
    import __graft_entry__ as g
    g.build()
    from handyrl_b200._capi import lib
    got = []

    def refused():      # the error text is per thread: keep this one's clean
        f, d, i, i64 = (C.c_float * 8)(), (C.c_double * 8)(), (C.c_int32 * 1)(), (C.c_int64 * 1)()
        got.append((lib().hrl_clip_adam_step(None, f, f, f, 8, f, f, i64, 4.0, 0.9, 0.999, 1e-8, 1e-5, None, None, f, 6, i,
                                             None), lib().hrl_last_error()))
        got.append((lib().hrl_clip_adam_step(f, f, f, f, 8, f, f, i64, 4.0, 0.9, 0.999, 1e-8, 1e-5, None, None, None, 6, i,
                                             None), lib().hrl_last_error()))      # guarded, but no tail to check
        got.append((lib().hrl_step_commit(None, f, 6, d, d, None, None, 0, None), lib().hrl_last_error()))
        got.append((lib().hrl_step_commit(i, f, 6, d, d, None, None, 16, None), lib().hrl_last_error()))
        got.append((lib().hrl_weight_ema(None, f, 8, i64, 0.9, 0, i, None), lib().hrl_last_error()))

    th = threading.Thread(target=refused)
    th.start()
    th.join()
    assert len(got) == 5
    for (status, err), name in zip(got, ['hrl_clip_adam_step', 'hrl_clip_adam_step', 'hrl_step_commit', 'hrl_step_commit',
                                         'hrl_weight_ema']):
        assert status != 0 and name.encode() in err, (name, status, err)


def test_how_the_key_is_read():
    from handyrl_b200.train import nonfinite_guard
    for off in ({}, {'skip_nonfinite': False}, {'skip_nonfinite': None}, {'skip_nonfinite': 0}):
        assert nonfinite_guard(off) is False
    for on in ({'skip_nonfinite': True}, {'skip_nonfinite': 1}):
        assert nonfinite_guard(on) is True


def test_the_skipped_line():
    from handyrl_b200.train import skipped_line
    line = skipped_line(3, 1200)
    assert line == 'skipped = 3 of 1200 steps: non-finite loss or gradient'
    assert not line.startswith('loss')         # the reference's loss plot reads lines starting with 'loss'


class _Done:
    def synchronize(self):
        pass


def _pending(host, diagnostics, guard, batch_cnt=4):
    from handyrl_b200.train import PendingModel
    return PendingModel(None, _Done(), None, torch.tensor(host, dtype=torch.float64), ['p', 'v', 'ent', 'total'], None,
                        diagnostics=diagnostics, skip_nonfinite=guard, batch_cnt=batch_cnt)


LOSSES = [1.0, 2.0, 0.0, 3.0, 4.0, 8.0]


@pytest.mark.parametrize('diagnostics', [False, True], ids=['plain', 'diagnostics'])
def test_accumulator_layout_with_and_without_the_guard(diagnostics, capsys):
    from handyrl_b200._capi import NUM_DIAG
    diag = [0.0] * NUM_DIAG if diagnostics else []

    p = _pending(LOSSES + diag, diagnostics, False)           # guard off: the layout of before
    sums = p.report()
    assert sums['dcnt'] == 8.0 and p.skipped == 0 and (p.diagnostics is not None) == diagnostics
    out = capsys.readouterr().out.splitlines()
    assert out[0].startswith('loss = ') and not any(l.startswith('skipped') for l in out)
    assert len(out) == (2 if diagnostics else 1)

    p = _pending(LOSSES + diag + [0.0], diagnostics, True)    # guard on, nothing rejected: the same lines
    p.report()
    assert p.skipped == 0
    assert capsys.readouterr().out.splitlines() == out

    p = _pending(LOSSES + diag + [2.0], diagnostics, True, batch_cnt=4)
    sums = p.report()
    assert p.skipped == 2 and sums['dcnt'] == 8.0
    got = capsys.readouterr().out.splitlines()
    assert got == out + ['skipped = 2 of 4 steps: non-finite loss or gradient']

    with pytest.raises(ValueError):           # the layout is told, not guessed from the length
        _pending(LOSSES + diag, diagnostics, True).report()


def test_the_line_is_printed_when_the_epoch_has_no_samples(capsys):
    p = _pending([0.0] * 6 + [3.0], False, True, batch_cnt=3)
    sums = p.report()
    assert sums['dcnt'] == 0 and p.skipped == 3
    assert capsys.readouterr().out.splitlines() == ['skipped = 3 of 3 steps: non-finite loss or gradient']


@pytest.mark.parametrize('diagnostics,guard,distill', list(itertools.product([False, True], repeat=3)))
def test_accumulator_layout_of_every_option_set(diagnostics, guard, distill, capsys):
    """accum_layout: [loss | distill | diag | skipped] from slot 0, each part there exactly when its option is on, without a
    gap or an overlap; the tail (loss, distill, the loss pass's diagnostics) is its head; PendingModel reads n slots."""
    from handyrl_b200 import ops
    from handyrl_b200._capi import NUM_DIAG, NUM_LOSS, NUM_LOSS_DIAG
    from handyrl_b200.train import NUM_DISTILL, PendingModel, accum_layout
    lay = accum_layout(diagnostics, guard, distill)
    parts = [(lay.loss, True, NUM_LOSS), (lay.distill, distill, NUM_DISTILL), (lay.diag, diagnostics, NUM_DIAG),
             (lay.skipped, guard, 1)]
    at = 0
    for part, on, size in parts:
        assert (part is not None) == on
        if on:
            assert part == slice(at, at + size)
            at += size
    assert at == lay.n
    loss_pass = lay.distill.stop if distill else NUM_LOSS
    assert lay.n_tail == loss_pass + (NUM_LOSS_DIAG if diagnostics else 0)
    assert not diagnostics or lay.diag.start == loss_pass

    host = [float(i + 1) for i in range(lay.n)]
    p = PendingModel(None, _Done(), None, torch.tensor(host, dtype=torch.float64), ['p', 'v', 'ent', 'total'], None,
                     diagnostics=diagnostics, skip_nonfinite=guard, batch_cnt=1000, distill=distill)
    sums = p.report()
    capsys.readouterr()
    assert list(sums.values()) == host[:NUM_LOSS]
    assert p.diagnostics == (ops.summarize_diagnostics(host[lay.diag]) if diagnostics else None)
    assert p.skipped == (int(host[-1]) if guard else 0)
    assert p.distill == ({'kl': host[NUM_LOSS], 'term': host[NUM_LOSS + 1]} if distill else None)
    for wrong in (host[:-1], host + [0.0]):
        with pytest.raises(ValueError):
            PendingModel(None, _Done(), None, torch.tensor(wrong, dtype=torch.float64), ['p'], None, diagnostics=diagnostics,
                         skip_nonfinite=guard, distill=distill).report()
