"""TEST INFRASTRUCTURE -- Python front end of the CPU oracle (oracle/hrl_oracle.c).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs
may import this module.  Parity status: pinned by tests/test_oracle.py against the
reference's own outputs in tests/golden/.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from handyrl_b200._capi import HrlLossArgs, ALGO_ID, NUM_LOSS, LOSS_KEYS

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, '_build', 'libhrl_oracle.so')
_lib = None


def build(force=False):
    srcs = [os.path.join(_HERE, f) for f in ('hrl_oracle.c', 'hrl_oracle_impl.h')]
    srcs.append(os.path.join(_HERE, '..', 'include', 'hrl_b200.h'))
    if force or not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in srcs):
        subprocess.run(['make', '-C', _HERE, '-B'], check=True, capture_output=True)
    return _SO


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        _lib.hrl_oracle_clip_adam.restype = C.c_double
        _lib.hrl_oracle_clip_adam.argtypes = [C.c_void_p] * 4 + [C.c_int64, C.c_double, C.c_int64] + [C.c_double] * 5
    return _lib


class _Out32(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ('dpolicy_raw', 'dvalue_raw', 'dreturn_raw', 'losses', 'target_value',
                                          'target_return', 'advantage', 'logp', 'rho', 'entropy')]


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _f32(x):
    return None if x is None else np.ascontiguousarray(np.asarray(x, dtype=np.float32))


def loss(batch, outputs, args, dtype=np.float32):
    """Oracle for compute_loss + autograd.

    batch / outputs: dicts of numpy arrays (or torch CPU tensors) in the reference layout;
    args: the reference's train_args dict (lambda, gamma, entropy_*, *_target,
    turn_based_training, burn_in_steps).  Returns a dict with losses (floats), grads and taps.
    """
    g = lambda k: np.asarray(batch[k])
    amask = _f32(g('action_mask'))
    B, T, Pa, A = amask.shape
    P = g('turn_mask').shape[2]
    keep = {}
    a = HrlLossArgs()
    a.B, a.T, a.P, a.Pa, a.A = B, T, P, Pa, A
    a.burn_in = int(args.get('burn_in_steps', 0))
    a.value_target = ALGO_ID[args['value_target']]
    a.policy_target = ALGO_ID[args['policy_target']]
    a.two_player_zero_sum = int(bool(args['turn_based_training']) and P == 2)
    a.lambda_ = args['lambda']
    a.gamma = args['gamma']
    a.entropy_regularization = args['entropy_regularization']
    a.entropy_regularization_decay = args['entropy_regularization_decay']

    def put(field, arr):
        keep[field] = arr
        setattr(a, field, _ptr(arr))

    put('policy_raw', _f32(outputs['policy']))
    put('value_raw', _f32(outputs.get('value')))
    put('return_raw', _f32(outputs.get('return')))
    put('action_mask', amask)
    put('action', np.ascontiguousarray(g('action').astype(np.int64)))
    put('selected_prob', _f32(g('selected_prob')))
    put('reward', _f32(g('reward')))
    put('ret', _f32(g('return')))
    put('turn_mask', _f32(g('turn_mask')))
    put('observation_mask', _f32(g('observation_mask')))
    put('episode_mask', _f32(g('episode_mask')))
    put('progress', _f32(g('progress')))
    put('outcome', _f32(g('outcome')))

    o = _Out32()
    res = {
        'dpolicy_raw': np.zeros((B, T, Pa, A), dtype),
        'dvalue_raw': np.zeros((B, T, Pa, 1), dtype) if 'value' in outputs else None,
        'dreturn_raw': np.zeros((B, T, Pa, 1), dtype) if 'return' in outputs else None,
        'losses': np.zeros(NUM_LOSS, dtype),
        'target_value': np.zeros((B, T, P, 1), dtype), 'target_return': np.zeros((B, T, P, 1), dtype),
        'advantage': np.zeros((B, T, P, 1), dtype), 'logp': np.zeros((B, T, Pa, 1), dtype),
        'rho': np.zeros((B, T, Pa, 1), dtype), 'entropy': np.zeros((B, T, Pa), dtype),
    }
    for k, v in res.items():
        setattr(o, k, _ptr(v))
    fn = lib().hrl_oracle_loss_f32 if dtype == np.float32 else lib().hrl_oracle_loss_f64
    rc = fn(C.byref(a), C.byref(o))
    if rc != 0:
        raise ValueError('oracle rejected the arguments (%d)' % rc)
    res['loss'] = {k: float(res['losses'][i]) for i, k in enumerate(LOSS_KEYS)}
    return res


def compute_target(algo, values, returns, rewards, lmb, gamma, rhos, cs, masks, dtype=np.float32):
    """Oracle for handyrl.losses.compute_target on (B,T,P,1) arrays."""
    returns = _f32(returns)
    ref = _f32(values) if values is not None else _f32(masks)
    B, T, P = ref.shape[:3]
    Tr = returns.shape[1]
    rhos, cs = _f32(rhos), _f32(cs)
    Pr = rhos.shape[2] if rhos is not None else 1
    values, rewards, masks = _f32(values), _f32(rewards), _f32(masks)
    tg = np.zeros((B, T, P, 1), dtype)
    ad = np.zeros((B, T, P, 1), dtype)
    fn = lib().hrl_oracle_compute_target_f32 if dtype == np.float32 else lib().hrl_oracle_compute_target_f64
    fn.argtypes = [C.c_int] * 6 + [C.c_void_p] * 3 + [C.c_double, C.c_double] + [C.c_void_p] * 5
    rc = fn(ALGO_ID[algo], B, T, P, Tr, Pr, _ptr(values), _ptr(returns), _ptr(rewards), lmb, gamma,
            _ptr(rhos), _ptr(cs), _ptr(masks), _ptr(tg), _ptr(ad))
    if rc != 0:
        raise ValueError('oracle rejected the arguments (%d)' % rc)
    return tg, ad


def clip_adam(param, grad, m, v, lr, step, max_norm=4.0, b1=0.9, b2=0.999, eps=1e-8, wd=1e-5):
    """In-place oracle for clip_grad_norm_ + Adam.step on flat fp32 arrays; returns the grad norm."""
    for x in (param, grad, m, v):
        assert x.dtype == np.float32 and x.flags.c_contiguous
    return lib().hrl_oracle_clip_adam(_ptr(param), _ptr(grad), _ptr(m), _ptr(v), param.size, lr, step,
                                      max_norm, b1, b2, eps, wd)


def board_conv(x, w, b=None):
    """Reference of a stride-1 "same" convolution over a small board (what torch.nn.functional.conv2d computes inside the
    user's net, reference envs/tictactoe.py:20-31): plain float64 loops over taps, NCHW.  Checker of the tensor-core dense
    path (hrl_board_expand + hrl_gemm_fused) in __graft_entry__.smoke() and the tests."""
    x = np.asarray(x, np.float64)
    w = np.asarray(w, np.float64)
    N, Cin, H, W = x.shape
    Cout, _, kh, kw = w.shape
    xp = np.zeros((N, Cin, H + kh - 1, W + kw - 1))
    xp[:, :, kh // 2:kh // 2 + H, kw // 2:kw // 2 + W] = x
    y = np.zeros((N, Cout, H, W))
    for a in range(kh):
        for c in range(kw):
            y += np.einsum('nihw,oi->nohw', xp[:, :, a:a + H, c:c + W], w[:, :, a, c])
    if b is not None:
        y += np.asarray(b, np.float64).reshape(1, Cout, 1, 1)
    return y
