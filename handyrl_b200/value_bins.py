"""Categorical value heads (train_args['value_bins']): a value or return head that predicts a distribution over bins and trains
by cross-entropy, in place of the scalar head regressed with squared error (value) or smooth-L1 (return).

Two-hot targets (MuZero, DreamerV3) and HL-Gauss targets (Farebrother et al., "Stop Regressing", ICML 2024); symlog bins give
an unbounded return head a fixed support.

    train_args['value_bins'] = {
        'value':  {'bins': 51, 'low': -1.0, 'high': 1.0},                                   # sigma 0: two-hot
        'return': {'bins': 101, 'low': -8.0, 'high': 8.0, 'symlog': True, 'sigma': 0.12},   # HL-Gauss in symlog space
    }

The law (INTEGRATION.md, include/hrl_b200.h), with K bins:
  bins         D = (high - low) / (K - 1), centres c_k = low + k D, edges e_k = low + (k - 1/2) D
  transform    s(y) = sign(y) log(1 + |y|) with symlog, else y;  s^-1(m) = sign(m) (exp|m| - 1)
  expectation  p = softmax(z), v = s^-1(sum_k p_k c_k): what the fused loss reads as the head's raw output
  target       x = clamp(s(y), low, high);  two-hot (sigma = 0): j = min(floor((x - low) / D), K - 2), u = (x - c_j) / D,
               pi_j = 1 - u, pi_j+1 = u;  HL-Gauss (sigma > 0): pi_k = [Phi((e_k+1 - x)/sigma) - Phi((e_k - x)/sigma)] / Z,
               Z = Phi((e_K - x)/sigma) - Phi((e_0 - x)/sigma)
  loss         L = sum over trained columns (b, t, p) of w_b om_btp (-sum_k pi_k(y_btp) log p_k(z_btq)), q = p (Pa = P) or 0,
               y the fused loss's targets['value'] / targets['return'];  dz_btq = sum_p w_b om_btp (p - pi(y_btp))

L takes the head's place in the loss sums (HRL_LOSS_V / HRL_LOSS_R) and in the total.  The expectation and the cross-entropy
run in their own kernels around the fused loss (csrc/value_bins_kernel.cu).  This module parses the key and holds the host
float64 reference of the law and the expectation the replay applies to stored K-vector values.
"""
import math
import numbers

import numpy as np
import torch

HEADS = ('value', 'return')
KEYS = ('bins', 'low', 'high', 'symlog', 'sigma')
MAX_BINS = 1024


def _real(v):
    return isinstance(v, numbers.Real) and not isinstance(v, bool) and math.isfinite(float(v))


def config(args):
    """train_args['value_bins'] -> {head: {'bins': K, 'low', 'high', 'symlog', 'sigma'}} for the categorical heads, or None when
    the feature is off (key absent, None, False or 0).  Raises ValueError for any other value: True, a non-dict, an empty dict,
    a head other than 'value' / 'return', an unknown key, bins not an integer in [2, 1024], low / high not finite or low >= high,
    symlog not a bool, sigma not finite or negative."""
    value = args.get('value_bins')
    if value is None or value is False or (isinstance(value, numbers.Number) and not isinstance(value, bool) and value == 0):
        return None
    if not isinstance(value, dict) or not value:
        raise ValueError("train_args['value_bins'] must be off (absent, None, False, 0) or a non-empty dict with 'value' and/or "
                         "'return' entries; got %r" % (value,))
    unknown = sorted(set(value) - set(HEADS), key=str)
    if unknown:
        raise ValueError("train_args['value_bins']: unknown head(s) %s (known: value, return)" % unknown)
    out = {}
    for head in HEADS:
        if head not in value:
            continue
        spec = value[head]
        name = "train_args['value_bins'][%r]" % head
        if not isinstance(spec, dict):
            raise ValueError('%s must be a dict with bins, low and high; got %r' % (name, spec))
        unknown = sorted(set(spec) - set(KEYS), key=str)
        if unknown:
            raise ValueError('%s: unknown key(s) %s (known: %s)' % (name, unknown, ', '.join(KEYS)))
        for k in ('bins', 'low', 'high'):
            if k not in spec:
                raise ValueError('%s needs %r' % (name, k))
        K = spec['bins']
        if isinstance(K, bool) or not isinstance(K, numbers.Integral) or not 2 <= K <= MAX_BINS:
            raise ValueError("%s['bins'] must be an integer in [2, %d]; got %r" % (name, MAX_BINS, K))
        low, high = spec['low'], spec['high']
        if not (_real(low) and _real(high)) or not float(low) < float(high):
            raise ValueError('%s: low and high must be finite numbers with low < high; got %r, %r' % (name, low, high))
        symlog = spec.get('symlog', False)
        if not isinstance(symlog, (bool, np.bool_)):
            raise ValueError("%s['symlog'] must be a bool; got %r" % (name, symlog))
        sigma = spec.get('sigma', 0.0)
        if not _real(sigma) or float(sigma) < 0:
            raise ValueError("%s['sigma'] must be a finite number >= 0; got %r" % (name, sigma))
        out[head] = {'bins': int(K), 'low': float(low), 'high': float(high), 'symlog': bool(symlog), 'sigma': float(sigma)}
    return out


def centres(spec):
    """The K bin centres c_k = low + k D (float64)."""
    K = spec['bins']
    delta = (spec['high'] - spec['low']) / (K - 1)
    return spec['low'] + delta * np.arange(K, dtype=np.float64)


def symlog(y):
    return np.sign(y) * np.log1p(np.abs(y))


def symexp(m):
    return np.sign(m) * np.expm1(np.abs(m))


def expectation(logits, spec):
    """v = s^-1(sum_k softmax(z)_k c_k) of (..., K) logits, as a float64 numpy array shaped (...)."""
    z = np.asarray(logits, dtype=np.float64)
    z = z - z.max(-1, keepdims=True)
    e = np.exp(z)
    mean = (e * centres(spec)).sum(-1) / e.sum(-1)
    return symexp(mean) if spec['symlog'] else mean


def _phi(u):
    return torch.special.ndtr(torch.from_numpy(np.asarray(u, dtype=np.float64))).numpy()


def target_distribution(y, spec):
    """pi of the law for targets y (any shape) -> float64 (..., K)."""
    y = np.asarray(y, dtype=np.float64)
    K, low, high, sigma = spec['bins'], spec['low'], spec['high'], spec['sigma']
    delta = (high - low) / (K - 1)
    x = np.clip(symlog(y) if spec['symlog'] else y, low, high)
    if sigma == 0:
        j = np.minimum(np.floor((x - low) / delta).astype(np.int64), K - 2)
        u = (x - (low + j * delta)) / delta
        pi = np.zeros(x.shape + (K,), np.float64)
        np.put_along_axis(pi, j[..., None], (1 - u)[..., None], -1)
        np.put_along_axis(pi, j[..., None] + 1, u[..., None], -1)
        return pi
    edges = low + (np.arange(K + 1, dtype=np.float64) - 0.5) * delta
    cdf = _phi((edges - x[..., None]) / sigma)
    return (cdf[..., 1:] - cdf[..., :-1]) / (cdf[..., -1:] - cdf[..., :1])


def reference(logits, target, observation_mask, spec, burn_in=0, window_weight=None):
    """Host float64 reference of one head: {'v': the expectation (B, T, Pa), 'pi': (B, T, P, K), 'loss': L, 'dz': dL/dz
    (B, T, Pa, K), zero on rows that are not trained}.  logits (B, T, Pa, K); target and observation_mask (B, T, P) or
    (B, T, P, 1); window_weight (B,) or None.  Any device, read as float64."""
    z = torch.as_tensor(logits).detach().double().cpu()
    y = torch.as_tensor(target).detach().double().cpu().reshape(z.shape[0], z.shape[1], -1)
    om = torch.as_tensor(observation_mask).detach().double().cpu().reshape(y.shape)
    B, T, Pa, K = z.shape
    P = y.shape[2]
    w = torch.ones(B, dtype=torch.float64) if window_weight is None else torch.as_tensor(window_weight).detach().double().cpu()
    pi = torch.from_numpy(target_distribution(y.numpy(), spec))                             # (B, T, P, K)
    logp = torch.log_softmax(z, -1)
    lp = logp.expand(B, T, P, K) if Pa == 1 else logp                                       # row q of column p
    c = om * w.view(-1, 1, 1)
    trained = torch.ones(T, dtype=torch.float64)
    if burn_in > 0 and T > 1:
        trained[:burn_in] = 0
    c = c * trained.view(1, -1, 1)
    ce = -(pi * lp).sum(-1)                                                                 # (B, T, P)
    loss = torch.where(c != 0, c * ce, torch.zeros_like(ce)).sum()
    g = c.unsqueeze(-1) * (logp.exp().expand(B, T, P, K) if Pa == 1 else logp.exp()) - c.unsqueeze(-1) * pi
    g = torch.where((c != 0).unsqueeze(-1), g, torch.zeros_like(g))
    dz = g.sum(2, keepdim=True) if Pa == 1 else g
    return {'v': torch.from_numpy(expectation(z.numpy(), spec)), 'pi': pi, 'loss': float(loss), 'dz': dz}


def check_net_heads(value_bins, outs, bins=True):
    """ValueError unless every categorical head of the parsed key is among the net's outputs `outs` (a dict of tensors), with
    K logits in its last dimension when `bins`."""
    if value_bins is None:
        return
    for head, spec in value_bins.items():
        if head not in outs:
            raise ValueError("train_args['value_bins'][%r]: the net has no %r head (its outputs: %s)"
                             % (head, head, sorted(k for k in outs if k != 'hidden')))
        if not bins:
            continue
        K = outs[head].shape[-1]
        if K != spec['bins']:
            raise ValueError("train_args['value_bins'][%r] has %d bins, but the net's %r head outputs %d value(s) per row"
                             % (head, spec['bins'], head, K))


def reduce_values(values, observed, spec):
    """The replay's ingest: (S, Ps, K) stored head logits -> (S, Ps, 1) float32 expectations where `observed` (S, Ps), 0
    elsewhere (the reference's default for a player without a value)."""
    v = expectation(values, spec)
    return np.where(observed, v, 0.0).astype(np.float32)[..., None]
