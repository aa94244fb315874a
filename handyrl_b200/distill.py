"""Policy distillation from a teacher net (train_args['distill']): "kickstarting" (Schmitt et al. 2018).

A new run -- a wider tower, other heads, a recurrent net -- can be pulled toward the policy of a trained model instead of
starting from zero.  The learner adds an annealed term c_n * KL(teacher || student) on the policy rows it already trains; the
coefficient decays to zero, after which the RL loss alone trains the net.

The law (INTEGRATION.md), with epi(raw) the mask epilogue of oracle/torch_learner.py:loss_from_raw (raw * turn_mask, summed
over players when Pa = 1 and the net has P > 1 rows, minus action_mask, then the burn-in cut):
  zS = epi(student raw policy), zT = epi(teacher raw policy), pT = softmax(zT) (no gradient), log pS = log_softmax(zS)
  KL_row = sum_a pT * (log pT - log pS)                    (terms with pT = 0 add 0)
  kl     = sum_{b,t,p} w_b * KL_row * tm                   (broadcast like ent * tm; w_b the prioritised-replay weight)
  c_n    = c0 * max(0, 1 - n / N)   (c0 when N = 0; n = the optimiser's step count before the step)
  total += c_n * kl

The term and its gradient run in their own kernel after the fused loss (hrl_distill_fwd_bwd, csrc/distill_kernel.cu).  This
module parses the key, builds and loads the teacher and holds the host float64 reference of the term.
"""
import copy
import importlib
import numbers
import os

import numpy as np
import torch

DEFAULTS = {'teacher': None, 'net': None, 'coef': 1.0, 'anneal_steps': 0}


def config(args, teacher_given=False):
    """train_args['distill'] -> {'teacher': path, 'net': callable or None, 'coef': float, 'anneal_steps': int}, or None when
    the feature is off (key absent, None, False or 0).  Raises ValueError for any other value, True, an unknown key, a
    missing or unreadable teacher file, a `net` that does not import or is not callable, a negative or non-finite coef and
    an anneal_steps that is not an integer >= 0.  teacher_given: the caller holds the teacher net already, so 'teacher' may
    be absent (it is None in the result)."""
    value = args.get('distill')
    if value is None or value is False or (isinstance(value, numbers.Number) and not isinstance(value, bool) and value == 0):
        return None
    if not isinstance(value, dict):
        raise ValueError("train_args['distill'] must be off (absent, None, False, 0) or a dict with a 'teacher' path; got %r"
                         % (value,))
    unknown = sorted(set(value) - set(DEFAULTS), key=str)
    if unknown:
        raise ValueError("train_args['distill']: unknown key(s) %s (known: teacher, net, coef, anneal_steps)" % unknown)
    spec = dict(DEFAULTS)
    spec.update(value)
    path = spec['teacher']
    if path is None and teacher_given:
        pass
    elif not isinstance(path, (str, os.PathLike)):
        raise ValueError("train_args['distill']['teacher'] must be the path of a saved state_dict; got %r" % (path,))
    else:
        path = os.fspath(path)
        if not os.path.isfile(path) or not os.access(path, os.R_OK):
            raise ValueError("train_args['distill']: teacher file %s is missing or unreadable" % path)
        spec['teacher'] = path
    spec['net'] = _resolve_net(spec['net'])
    c = spec['coef']
    if isinstance(c, bool) or not isinstance(c, numbers.Real) or not np.isfinite(float(c)) or float(c) < 0:
        raise ValueError("train_args['distill']['coef'] must be a finite number >= 0; got %r" % (c,))
    spec['coef'] = float(c)
    n = spec['anneal_steps']
    if isinstance(n, bool) or not isinstance(n, numbers.Integral) or n < 0:
        raise ValueError("train_args['distill']['anneal_steps'] must be an integer >= 0; got %r" % (n,))
    spec['anneal_steps'] = int(n)
    return spec


def _resolve_net(net):
    """None, or a 'package.module:function' string -> the function it names."""
    if net is None:
        return None
    if not isinstance(net, str) or net.count(':') != 1:
        raise ValueError("train_args['distill']['net'] must be a 'package.module:function' string; got %r" % (net,))
    mod, name = net.split(':')
    try:
        fn = getattr(importlib.import_module(mod), name)
    except (ImportError, AttributeError) as e:
        raise ValueError("train_args['distill']['net'] = %r does not import: %s" % (net, e)) from None
    if not callable(fn):
        raise ValueError("train_args['distill']['net'] = %r is not callable" % net)
    return fn


def teacher_net(spec, student):
    """The teacher nn.Module of a parsed spec on the host, in eval mode, its weights loaded strict=True from spec['teacher']:
    spec['net']() when given, else a deep copy of `student` (the student as built, before any rewrite of the learner).
    Raises ValueError naming the file when it does not unpickle as a state_dict or does not load into the net."""
    net = spec['net']() if spec['net'] is not None else copy.deepcopy(student)
    if not isinstance(net, torch.nn.Module):
        raise ValueError("train_args['distill']['net'] returned %s, not a torch.nn.Module" % type(net).__name__)
    path = spec['teacher']
    try:
        state = torch.load(path, map_location='cpu', weights_only=True)
    except Exception as e:          # noqa: BLE001 -- any failure to read the file is the user's file, not our bug
        raise ValueError('train_args[\'distill\']: cannot read the teacher state_dict %s: %s' % (path, e)) from None
    if not isinstance(state, dict):
        raise ValueError("train_args['distill']: %s holds a %s, not a state_dict" % (path, type(state).__name__))
    try:
        net.load_state_dict(state, strict=True)
    except Exception as e:          # noqa: BLE001
        raise ValueError("train_args['distill']: the state_dict %s does not load into the teacher net: %s" % (path, e)) from None
    net.eval()
    for p in net.parameters():
        p.requires_grad_(False)
    return net


def coefficient(spec, n):
    """c_n = c0 * max(0, 1 - n / N), or c0 when N = 0, at optimiser step count n (float64)."""
    c0, N = float(spec['coef']), int(spec['anneal_steps'])
    if N == 0:
        return c0
    return c0 * max(0.0, 1.0 - float(n) / N)


def line(kl, term, dcnt):
    """'distill = kl:0.0412 term:0.0309': the epoch's sums of kl and c_n * kl over its dcnt, as the Trainer prints them."""
    return 'distill = kl:%.4f term:%.4f' % (kl / dcnt, term / dcnt)


def _epilogue(raw, batch, bi):
    tm4 = batch['turn_mask'].double()
    z = raw.double() * tm4
    if z.size(2) > 1 and batch['action'].size(2) == 1:
        z = z.sum(2, keepdim=True)
    z = z - batch['action_mask'].double()
    return z[:, bi:] if (bi > 0 and z.size(1) > 1) else z


def reference(student, teacher, batch, args, coef, window_weight=None):
    """Host float64 reference of the term: (kl, grad), kl the sum of the law above and grad = d(coef * kl) / d student, shaped
    like `student` (B, T, Pa, A) with zeros on burn-in rows.  `coef` is c_n; the batch tensors and the logits may live on any
    device and are read as float64."""
    bi = int(args.get('burn_in_steps', 0))
    cut = (bi > 0 and student.size(1) > 1)
    zs, zt = _epilogue(student, batch, bi), _epilogue(teacher, batch, bi)
    tm = batch['turn_mask'].double()
    tm = (tm[:, bi:] if cut else tm).squeeze(-1)                              # (B, T', P)
    lps, lpt = torch.log_softmax(zs, -1), torch.log_softmax(zt, -1)
    ps, pt = lps.exp(), lpt.exp()
    kl_row = torch.where(pt > 0, pt * (lpt - lps), torch.zeros_like(pt)).sum(-1)      # (B, T', Pa)
    w = torch.ones(student.size(0), dtype=torch.float64, device=zs.device) if window_weight is None else window_weight.double()
    # the row's weight f: kl_row * tm broadcast over P and summed (Pa = 1), or row by row (Pa = P)
    f = tm.sum(-1, keepdim=True) if kl_row.size(2) == 1 else tm
    f = f * w.view(-1, 1, 1)
    kl = torch.where(f != 0, kl_row * f, torch.zeros_like(kl_row)).sum()
    dz = coef * torch.where((f != 0).unsqueeze(-1), f.unsqueeze(-1) * (ps - pt), torch.zeros_like(ps))   # d(c kl) / d zS
    # chain rule through the epilogue: zS = raw * sum_p tm (Pa = 1) or raw * tm (Pa = P)
    s = tm.sum(-1, keepdim=True) if kl_row.size(2) == 1 else tm
    g = dz * s.unsqueeze(-1)
    grad = torch.zeros(student.shape, dtype=torch.float64, device=zs.device)
    grad[:, (bi if cut else 0):] = g
    return kl, grad
