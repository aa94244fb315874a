"""Policy distillation (train_args['distill'], handyrl_b200/distill.py) without a GPU: the key's parsing and errors, the
teacher's loading, the float64 reference of the term against autograd of the reference loss, the annealing schedule,
forward_raw's train=False, the printed line, the C struct mirror and the kernel's register budget."""
import ctypes
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import case_args, load_cases
from handyrl_b200 import distill
from handyrl_b200.nets import BoardNet
from oracle.torch_learner import loss_from_raw

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOSS_CASES = load_cases('loss_cases.npz')


@pytest.fixture
def teacher_file(tmp_path):
    torch.manual_seed(3)
    path = str(tmp_path / '7.pth')
    torch.save(BoardNet().state_dict(), path)
    return path


def small_board_net():
    return BoardNet(width=8, depth=1)


# ----------------------------------------------------------------------------------------------------------- parsing

@pytest.mark.parametrize('value', ['absent', None, False, 0, 0.0])
def test_off_forms(value):
    args = {} if value == 'absent' else {'distill': value}
    assert distill.config(args) is None


def test_defaults_and_values(teacher_file):
    spec = distill.config({'distill': {'teacher': teacher_file}})
    assert spec == {'teacher': teacher_file, 'net': None, 'coef': 1.0, 'anneal_steps': 0}
    spec = distill.config({'distill': {'teacher': teacher_file, 'coef': 0, 'anneal_steps': 100,
                                       'net': 'test_distill_cpu:small_board_net'}})
    assert spec['coef'] == 0.0 and spec['anneal_steps'] == 100 and spec['net'] is not None


@pytest.mark.parametrize('value', [True, 1, 2.5, 'models/1.pth', ['models/1.pth'], {}])
def test_other_values_raise(value):
    with pytest.raises(ValueError, match='distill'):
        distill.config({'distill': value})


@pytest.mark.parametrize('extra, match', [
    ({'alpha': 1}, 'unknown key'),
    ({'coef': -1}, 'coef'), ({'coef': float('nan')}, 'coef'), ({'coef': float('inf')}, 'coef'), ({'coef': True}, 'coef'),
    ({'coef': '1'}, 'coef'),
    ({'anneal_steps': -1}, 'anneal_steps'), ({'anneal_steps': 1.5}, 'anneal_steps'), ({'anneal_steps': True}, 'anneal_steps'),
    ({'net': 'no_such_package_xyz.mod:fn'}, 'does not import'), ({'net': 'handyrl_b200.nets:no_such_fn'}, 'does not import'),
    ({'net': 'handyrl_b200.distill:DEFAULTS'}, 'not callable'), ({'net': 'handyrl_b200.nets'}, 'module:function'),
])
def test_bad_entries_raise(teacher_file, extra, match):
    with pytest.raises(ValueError, match=match):
        distill.config({'distill': dict({'teacher': teacher_file}, **extra)})


def test_missing_or_unreadable_teacher_names_the_file(tmp_path):
    missing = str(tmp_path / 'none.pth')
    with pytest.raises(ValueError, match=re.escape(missing)):
        distill.config({'distill': {'teacher': missing}})
    with pytest.raises(ValueError, match=re.escape(str(tmp_path))):
        distill.config({'distill': {'teacher': str(tmp_path)}})           # a directory is not a file
    with pytest.raises(ValueError, match='teacher'):
        distill.config({'distill': {'teacher': 3}})
    garbage = tmp_path / 'garbage.pth'
    garbage.write_bytes(b'not a checkpoint')
    spec = distill.config({'distill': {'teacher': str(garbage)}})
    with pytest.raises(ValueError, match=re.escape(str(garbage))):
        distill.teacher_net(spec, BoardNet())


def test_state_dict_must_load_strictly(teacher_file, tmp_path):
    spec = distill.config({'distill': {'teacher': teacher_file}})
    with pytest.raises(ValueError, match=re.escape(teacher_file)):
        distill.teacher_net(spec, BoardNet(width=16))                    # other shapes
    partial = str(tmp_path / 'partial.pth')
    state = BoardNet().state_dict()
    state.pop('stem.bias')
    torch.save(state, partial)
    with pytest.raises(ValueError, match=re.escape(partial)):
        distill.teacher_net(distill.config({'distill': {'teacher': partial}}), BoardNet())
    not_dict = str(tmp_path / 'list.pth')
    torch.save([1, 2], not_dict)
    with pytest.raises(ValueError, match=re.escape(not_dict)):
        distill.teacher_net(distill.config({'distill': {'teacher': not_dict}}), BoardNet())


def test_teacher_is_a_loaded_copy_in_eval_mode(teacher_file):
    student = BoardNet()
    student.train()
    teacher = distill.teacher_net(distill.config({'distill': {'teacher': teacher_file}}), student)
    assert teacher is not student and not teacher.training and student.training
    want = torch.load(teacher_file)
    for k, v in teacher.state_dict().items():
        assert torch.equal(v, want[k])
    assert all(not p.requires_grad for p in teacher.parameters())
    assert any(not torch.equal(a, b) for a, b in zip(student.state_dict().values(), teacher.state_dict().values()))


def test_net_builds_a_different_architecture(tmp_path):
    path = str(tmp_path / 'small.pth')
    torch.save(small_board_net().state_dict(), path)
    spec = distill.config({'distill': {'teacher': path, 'net': 'test_distill_cpu:small_board_net'}})
    teacher = distill.teacher_net(spec, BoardNet())
    assert teacher.stem.out_channels == 8 and len(teacher.tower) == 1


# ----------------------------------------------------------------------------------------------------------- schedule

def test_schedule():
    spec = {'coef': 0.5, 'anneal_steps': 100}
    assert distill.coefficient(spec, 0) == 0.5
    assert distill.coefficient(spec, 50) == pytest.approx(0.25, abs=0)
    assert distill.coefficient(spec, 100) == 0.0
    assert distill.coefficient(spec, 1000) == 0.0
    assert distill.coefficient({'coef': 0.5, 'anneal_steps': 0}, 10 ** 9) == 0.5


def test_line():
    assert distill.line(4.12, 3.09, 100.0) == 'distill = kl:0.0412 term:0.0309'
    assert not distill.line(1, 1, 1).startswith('loss')


# ----------------------------------------------------------------------------------------------------------- reference

def _as_double(batch):
    return {k: (torch.from_numpy(v).double() if v.dtype != np.int64 else torch.from_numpy(v)) for k, v in batch.items()}


def _case(name, pad=False, weights=False, seed=0):
    case = LOSS_CASES[name]
    batch = _as_double({k[3:]: v for k, v in case.items() if k.startswith('in.')})
    student = torch.from_numpy(case['out.policy']).double()
    g = torch.Generator().manual_seed(seed)
    teacher = student + torch.randn(student.shape, generator=g, dtype=torch.float64)
    if pad:     # the last window ends early: its pad rows have no turn and every action masked
        B, T = batch['turn_mask'].shape[:2]
        cut = T // 2
        batch['turn_mask'][-1, cut:] = 0
        batch['observation_mask'][-1, cut:] = 0
        batch['episode_mask'][-1, cut:] = 0
        batch['action_mask'][-1, cut:] = 1e32
    w = torch.rand(batch['turn_mask'].shape[0], generator=g, dtype=torch.float64) * 2 if weights else None
    return case, batch, student, teacher, w


def _kl_by_autograd_law(raw_s, raw_t, batch, args, w):
    """The law written out on its own: the reference's mask epilogue, then sum w * KL_row * tm broadcast like ent * tm."""
    bi = args.get('burn_in_steps', 0)

    def epi(raw):
        z = raw * batch['turn_mask']
        if z.size(2) > 1 and batch['action'].size(2) == 1:
            z = z.sum(2, keepdim=True)
        z = z - batch['action_mask']
        return z[:, bi:] if (bi > 0 and z.size(1) > 1) else z
    tm = batch['turn_mask'][:, bi:] if (bi > 0 and raw_s.size(1) > 1) else batch['turn_mask']
    lps, lpt = F.log_softmax(epi(raw_s), -1), F.log_softmax(epi(raw_t), -1).detach()
    pt = lpt.exp()
    row = (pt * (lpt - lps)).nan_to_num(0.0).sum(-1)                      # (B, T', Pa)
    cell = row * tm.squeeze(-1)                                           # broadcast exactly like ent * tm
    if w is not None:
        cell = cell * w.view(-1, 1, 1)
    return cell.sum()


@pytest.mark.parametrize('name, pad, weights', [
    ('alt_UPGO_VTRACE', False, False), ('sim_UPGO_VTRACE', False, False), ('obs_TD_MC', True, True),
    ('burnin_alt', True, True), ('burnin_obs', False, True), ('geese4', True, False), ('alt4', False, True),
    ('wide', True, True), ('t1', False, True), ('solo1', True, True),
])
def test_reference_against_autograd(name, pad, weights):
    case, batch, student, teacher, w = _case(name, pad, weights)
    args = case_args(case['meta'])
    coef = 0.7
    raw = student.clone().requires_grad_(True)
    losses, _ = loss_from_raw({'policy': raw}, batch, args)
    (g_rl,) = torch.autograd.grad(losses['total'], raw)
    raw2 = student.clone().requires_grad_(True)
    losses2, _ = loss_from_raw({'policy': raw2}, batch, args)
    kl_auto = _kl_by_autograd_law(raw2, teacher, batch, args, w)
    (g_all,) = torch.autograd.grad(losses2['total'] + coef * kl_auto, raw2)
    kl, grad = distill.reference(student, teacher, batch, args, coef, window_weight=w)
    assert torch.isfinite(grad).all() and torch.isfinite(kl)
    assert float(kl) == pytest.approx(float(kl_auto.detach()), rel=1e-12, abs=1e-12)
    torch.testing.assert_close(grad, g_all - g_rl, rtol=0, atol=1e-12)
    assert float(kl) > 0
    bi = args['burn_in_steps']
    if bi > 0:
        assert (grad[:, :bi] == 0).all()


@pytest.mark.parametrize('name', ['alt_UPGO_VTRACE', 'sim_UPGO_VTRACE', 'burnin_obs', 'geese4'])
def test_teacher_equal_to_student_gives_zero(name):
    case, batch, student, _, w = _case(name, pad=True, weights=True)
    kl, grad = distill.reference(student, student.clone(), batch, case_args(case['meta']), 1.0, window_weight=w)
    assert abs(float(kl)) < 1e-12 and grad.abs().max() < 1e-12


def test_rows_of_weight_zero_add_nothing():
    case, batch, student, teacher, _ = _case('alt_UPGO_VTRACE', pad=True)
    args = case_args(case['meta'])
    w = torch.ones(batch['turn_mask'].shape[0], dtype=torch.float64)
    w[0] = 0
    teacher2 = teacher.clone()
    teacher2[0] = teacher[0] + 5            # the zero-weight window's teacher changes nothing
    teacher2[-1, 5:] = 1e30                 # nor do the pad rows' logits
    kl, grad = distill.reference(student, teacher, batch, args, 1.0, window_weight=w)
    kl2, grad2 = distill.reference(student, teacher2, batch, args, 1.0, window_weight=w)
    assert float(kl) == float(kl2) and torch.equal(grad, grad2)
    assert (grad[0] == 0).all() and (grad[-1, 5:] == 0).all()


# ----------------------------------------------------------------------------------------------------------- forward_raw

class _RecurrentStub(torch.nn.Module):
    """Records the mode of every call."""

    def __init__(self):
        super().__init__()
        self.lin = torch.nn.Linear(2, 3)
        self.modes = []

    def init_hidden(self, batch_size=None):
        return torch.zeros(tuple(batch_size or []) + (2,))

    def forward(self, x, hidden):
        self.modes.append(self.training)
        return {'policy': self.lin(x + hidden), 'hidden': hidden + 1}


@pytest.mark.parametrize('train, want_after', [(False, False), (True, True)])
def test_forward_raw_train_flag(train, want_after):
    from handyrl_b200.train import forward_raw
    B, T, P = 2, 5, 2
    batch = {'observation': torch.randn(B, T, 1, 2), 'action': torch.zeros(B, T, 1, 1, dtype=torch.int64),
             'observation_mask': torch.ones(B, T, P, 1)}
    net = _RecurrentStub().eval()
    args = {'turn_based_training': True, 'observation': False, 'burn_in_steps': 2}
    kw = {} if train else {'train': False}
    with torch.no_grad():
        out = forward_raw(net, net.init_hidden([B, P]), batch, args, **kw)
    assert out['policy'].shape == (B, T, 1, 3)
    assert net.modes == [False, False] + [want_after] * 3
    assert net.training == want_after


# ----------------------------------------------------------------------------------------------------------- boundary

def test_struct_layout_matches_header():
    from handyrl_b200 import _capi
    fields = ['A', 'burn_in', 'policy_raw', 'window_weight', 'step_count', 'coef', 'anneal_steps', 'dpolicy_raw', 'sums',
              'workspace', 'workspace_bytes', 'io_bf16']
    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "hrl_b200.h"\nint main(){printf("%zu\\n", sizeof(HrlDistillArgs));' +
           ''.join('printf("%%zu\\n", offsetof(HrlDistillArgs, %s));' % f for f in fields) + 'return 0;}\n')
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, 's.c')
        open(c, 'w').write(src)
        exe = os.path.join(d, 's')
        subprocess.run(['gcc', '-I', os.path.join(ROOT, 'include'), c, '-o', exe], check=True)
        got = [int(x) for x in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    want = [ctypes.sizeof(_capi.HrlDistillArgs)] + [getattr(_capi.HrlDistillArgs, f).offset for f in fields]
    assert got == want


def test_kernel_does_not_spill():
    """Every width of the distillation kernel (lanes per row 4, 8, 16, 32) compiles for sm_90a without spills or a stack."""
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    if not (os.path.exists(nvcc) or shutil.which(nvcc)):
        pytest.skip('nvcc is not available')
    with tempfile.TemporaryDirectory() as d:
        cmd = [nvcc, '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '-c', '-Xptxas', '-v',
               '-o', os.path.join(d, 'distill_kernel.o'), os.path.join(ROOT, 'handyrl_b200', 'csrc', 'distill_kernel.cu')]
        res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    widths, cur = {}, None
    for line in res.stderr.splitlines():
        m = re.search(r'distill_kernelILi(\d+)EE', line)
        if 'Compiling entry function' in line:
            cur = int(m.group(1)) if m else None
            continue
        s = re.search(r'(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads', line)
        if s and cur is not None:
            widths[cur] = tuple(int(x) for x in s.groups())
    assert widths == {4: (0, 0, 0), 8: (0, 0, 0), 16: (0, 0, 0), 32: (0, 0, 0)}
