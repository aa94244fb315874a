"""GPU-native (H100, sm_90a) learner hot path behind the reference's Python surface.

Same public names as handyrl/train.py for the path
    Batcher.batch -> forward_prediction -> compute_loss -> backward -> optimizer.step
(reference train.py:127-400), different machinery:

  * the net runs ONCE per step and returns raw outputs; the mask epilogue, the whole of
    compute_loss / compose_losses / losses.py AND their backward run in one CUDA kernel
    (ops.loss_fwd_bwd -> csrc/loss_kernel.cu) that hands autograd closed-form gradients;
  * parameters and gradients live in one flat bucket: one NCCL all-reduce(SUM) per step when
    sharded over GPUs, then clip+Adam in two launches (csrc/optim_kernel.cu);
  * the whole step (H2D copies, net forward, loss kernel, net backward, all-reduce, optimiser)
    is captured in a CUDA graph and replayed; the host never synchronises inside an epoch
    (the reference does 4-6 .item() syncs per step, train.py:200, 375-376).
"""
import collections
import copy
import functools
import numbers
import os
import pickle
import queue
import threading
import time
import traceback
from collections import deque

import numpy as np
import torch

from . import ops, fastnet, priority, symmetry
from . import distill as distill_mod
from . import value_bins as value_bins_mod
from .batch import tree_map, tree_leaves, make_batch, gather_windows, sample_window, reduce_values
from ._capi import DIAG_KEYS, LOSS_KEYS, NUM_DIAG, NUM_LOSS, NUM_LOSS_DIAG


# --------------------------------------------------------------------------- forward

def _call_model(model, obs, hidden):
    return model(obs, hidden)


def _as_format(o, memory_format):
    if memory_format is not None and o.dim() == 4:
        return o.contiguous(memory_format=memory_format)
    return o


def forward_raw(model, hidden, batch, args, memory_format=None, train=True):
    """Run the net over a batch and return its RAW outputs shaped (B, T, Pa, ...).

    Feed-forward nets see all B*T*Pa observations at once; recurrent nets are stepped over T
    with the hidden state masked by observation_mask, burn-in steps without gradient and in
    eval mode, exactly as the reference does (train.py:142-174) -- but WITHOUT the mask
    epilogue of train.py:176-184, which the fused loss kernel applies on the fly.  train=False keeps a net in eval mode
    after burn-in too (a distillation teacher): the steps t >= burn_in then leave the mode as it is.
    """
    observations = batch['observation']
    B, T, Pa = batch['action'].shape[:3]

    if hidden is None:
        flat = tree_map(lambda o: _as_format(o.flatten(0, 2), memory_format), observations)
        outs = _call_model(model, flat, None)
        return {k: v.unflatten(0, (B, T, Pa)) for k, v in outs.items() if k != 'hidden' and v is not None}

    alternating = args['turn_based_training'] and not args['observation']
    burn_in = args['burn_in_steps']
    per_step = {}
    omask_all = batch['observation_mask']
    for t in range(T):
        obs_t = tree_map(lambda o: _as_format(o[:, t].flatten(0, 1), memory_format), observations)
        om = omask_all[:, t]                                                   # (B, P, 1)

        def gate(h):
            return om.view(*h.shape[:2], *([1] * (h.dim() - 2)))

        fused = om.is_cuda and om.dtype == torch.float32          # one kernel per hidden leaf instead of mul + sum / blend chains
        if fused:
            visible = tree_map(lambda h: ops.hidden_visible(h, om, alternating), hidden)
            if not alternating:
                visible = tree_map(lambda h: h.flatten(0, 1), visible)
        else:
            visible = tree_map(lambda h: h * gate(h), hidden)
            if alternating:
                visible = tree_map(lambda h: h.sum(1), visible)                # only the turn player observes
            else:
                visible = tree_map(lambda h: h.flatten(0, 1), visible)
        if t < burn_in:
            model.eval()
            with torch.no_grad():
                out_t = _call_model(model, obs_t, visible)
        else:
            if train and not model.training:
                model.train()
            out_t = _call_model(model, obs_t, visible)
        new_hidden = out_t.pop('hidden', None)
        for k, v in out_t.items():
            if v is not None:
                per_step.setdefault(k, []).append(v.unflatten(0, (B, Pa)))
        new_hidden = tree_map(lambda h: h.unflatten(0, (B, Pa)), new_hidden)
        if fused:
            hidden = tree_map(lambda h, nh: ops.hidden_blend(h, nh, om), hidden, new_hidden)
        else:
            hidden = tree_map(lambda h, nh: h * (1 - gate(h)) + nh * gate(h), hidden, new_hidden)
    return {k: torch.stack(v, dim=1) for k, v in per_step.items()}


def forward_prediction(model, hidden, batch, args):
    """API-compatible with handyrl.train.forward_prediction: raw outputs + the mask epilogue
    (train.py:176-184) as torch ops.  NOT used by the learner below (the epilogue is fused into
    the loss kernel); kept so code written against the reference keeps importing."""
    outs = forward_raw(model, hidden, batch, args)
    Pa = batch['action'].shape[2]
    masked = {}
    for k, o in outs.items():
        if k == 'policy':
            o = o * batch['turn_mask']
            if o.size(2) > 1 and Pa == 1:
                o = o.sum(2, keepdim=True)
            masked[k] = o - batch['action_mask']
        else:
            masked[k] = o * batch['observation_mask']
    return masked


# --------------------------------------------------------------------------- loss

class _FusedLoss(torch.autograd.Function):
    """total = fused_loss(policy_raw, value_raw?, return_raw?); backward returns the closed-form
    gradients the kernel already produced, scaled by grad_output."""

    @staticmethod
    def forward(ctx, batch, args, keys, *heads):
        outs = dict(zip(keys, [h.detach() for h in heads]))
        buf = ops.loss_fwd_bwd(outs, batch, args)
        grads = {'policy': buf.dpolicy, 'value': buf.dvalue, 'return': buf.dreturn}
        ctx.save_for_backward(*[grads[k] for k in keys])
        ctx.mark_non_differentiable(buf.losses)
        total = buf.losses[4].clone()
        return total, buf.losses

    @staticmethod
    def backward(ctx, g_total, _g_losses):
        return (None, None, None) + tuple(g * g_total for g in ctx.saved_tensors)


def compute_loss(batch, model, hidden, args):
    """Drop-in for handyrl.train.compute_loss (train.py:218-267): returns
    ({'p','v','r','ent','total'} 0-d tensors, dcnt float).  `total` is differentiable.  Categorical heads
    (train_args['value_bins']) are trained by LearnerStep and Trainer only: with that key on this raises ValueError."""
    if value_bins_mod.config(args) is not None:
        raise ValueError("train_args['value_bins']: the drop-in compute_loss trains scalar heads only; categorical heads train "
                         "through LearnerStep or Trainer")
    outs = forward_raw(model, hidden, batch, args)
    keys = [k for k in ('policy', 'value', 'return') if k in outs]
    total, vec = _FusedLoss.apply(batch, args, keys, *[outs[k] for k in keys])
    losses = {'p': vec[0]}
    if 'value' in outs:
        losses['v'] = vec[1]
    if 'return' in outs:
        losses['r'] = vec[2]
    losses['ent'] = vec[3]
    losses['total'] = total
    return losses, float(vec[5].item())     # the reference also synchronises here (train.py:200)


# --------------------------------------------------------------------------- one learner step

def obs_rows(obs):
    return tree_leaves(obs)[0].shape[0]


def _align(x, a=256):
    return (x + a - 1) // a * a


class BatchLayout:
    """Byte layout of one replay batch packed into a single buffer (one H2D copy per step).
    `value` (the behaviour value, train.py:117) is left out: nothing on the hot path reads it."""

    SKIP = ('value',)

    def __init__(self, example_batch):
        self.entries = []      # (key path tuple, shape, dtype, offset)
        off = 0

        def walk(tree, path):
            nonlocal off
            if isinstance(tree, dict):
                for k, v in tree.items():
                    walk(v, path + (k,))
            elif isinstance(tree, (list, tuple)):
                for i, v in enumerate(tree):
                    walk(v, path + (i,))
            else:
                self.entries.append((path, tuple(tree.shape), tree.dtype, off))
                off = _align(off + tree.numel() * tree.element_size())

        for k, v in example_batch.items():
            if k not in self.SKIP:
                walk(v, (k,))
        self.template = {k: v for k, v in example_batch.items() if k not in self.SKIP}
        self.nbytes = off
        self.payload_bytes = sum(int(torch.tensor(sh).prod()) * torch.empty(0, dtype=dt).element_size()
                                 for _, sh, dt, _ in self.entries)

    def views(self, buf):
        """Tree of tensors (same nesting as the batch) aliasing the flat uint8 buffer `buf`."""
        flat = {}
        for path, shape, dtype, off in self.entries:
            n = int(torch.tensor(shape).prod()) * torch.empty(0, dtype=dtype).element_size()
            flat[path] = buf[off:off + n].view(dtype).view(shape)

        def build(tree, path):
            if isinstance(tree, dict):
                return type(tree)((k, build(v, path + (k,))) for k, v in tree.items())
            if isinstance(tree, (list, tuple)):
                return type(tree)(build(v, path + (i,)) for i, v in enumerate(tree))
            return flat[path]

        return build(self.template, ())


class PackedBatch:
    """A replay batch in ONE pinned host buffer; `tensors` alias it in the reference's dict layout."""

    def __init__(self, layout):
        self.layout = layout
        self.buffer = torch.empty(layout.nbytes, dtype=torch.uint8).pin_memory()
        self.tensors = layout.views(self.buffer)
        self.in_flight = None      # CUDA event: the H2D copy reading this buffer has completed

    def fill(self, host_batch):
        for d, s in zip(tree_leaves(self.tensors), tree_leaves({k: host_batch[k] for k in self.tensors})):
            d.copy_(s)
        return self

    def wait_reusable(self):
        if self.in_flight is not None:
            self.in_flight.synchronize()
            self.in_flight = None


class StateStore:
    """Everything `model.state_dict()` holds, in ONE device allocation: [fp32 parameters, padded to 4 | fp32 buffers
    (BatchNorm running statistics) | int64 buffers (num_batches_tracked)].  Parameters and buffers are re-pointed
    into it, so the per-epoch model hand-off to the workers (train.py:385-387) is one device-to-device snapshot on
    the step stream plus one device-to-host copy on a side stream instead of a `model.cpu()` of every tensor."""

    def __init__(self, model, device):
        params = list(model.parameters())
        self.n = sum(p.numel() for p in params)
        self.n_pad = (self.n + 3) // 4 * 4
        named = list(model.named_buffers())
        fbufs = [(k, b) for k, b in named if b.dtype == torch.float32]
        ibufs = [(k, b) for k, b in named if b.dtype == torch.int64]
        self.loose = [(k, b) for k, b in named if b.dtype not in (torch.float32, torch.int64)]   # copied one by one
        nf = sum(b.numel() for _, b in fbufs)
        ni = sum(b.numel() for _, b in ibufs)
        self.f_off = 4 * self.n_pad
        self.i_off = (self.f_off + 4 * nf + 7) // 8 * 8
        self.nbytes = self.i_off + 8 * ni
        self.bytes = torch.zeros(max(self.nbytes, 16), dtype=torch.uint8, device=device)
        self.flat_param = self.bytes[:4 * self.n_pad].view(torch.float32)
        fview = self.bytes[self.f_off:self.f_off + 4 * nf].view(torch.float32)
        iview = self.bytes[self.i_off:self.i_off + 8 * ni].view(torch.int64)
        self.where = {}           # state_dict key -> (view name, offset in elements, shape)
        with torch.no_grad():
            for view, tag, bufs in ((fview, 'f', fbufs), (iview, 'i', ibufs)):
                off = 0
                for k, b in bufs:
                    n = b.numel()
                    view[off:off + n].copy_(b.reshape(-1))
                    b.data = view[off:off + n].view(b.shape)
                    self.where[k] = (tag, off, tuple(b.shape))
                    off += n
        self._params = params

    def index_params(self, model):
        """Call after FlatAdam re-pointed the parameters into flat_param (same order as model.parameters())."""
        off = 0
        for k, p in model.named_parameters():
            self.where[k] = ('p', off, tuple(p.shape))
            off += p.numel()

    def state_dict_from(self, host_bytes, keys):
        """Rebuild {key: CPU tensor} from a host copy of `bytes` (fresh storage per tensor)."""
        views = {'p': host_bytes[:4 * self.n_pad].view(torch.float32),
                 'f': host_bytes[self.f_off:self.i_off].view(torch.float32) if self.i_off > self.f_off else None,
                 'i': host_bytes[self.i_off:self.nbytes].view(torch.int64) if self.nbytes > self.i_off else None}
        out = {}
        for k in keys:
            if k in self.where:
                tag, off, shape = self.where[k]
                n = 1
                for d in shape:
                    n *= d
                out[k] = views[tag][off:off + n].clone().view(shape)
        return out

    def averaged_bytes(self, host_avg, host_bytes):
        """A host image of `bytes` holding the moving average: the fp32 words [0, i_off) are already in `host_avg` (a host
        buffer of the size of `bytes`), the int64 buffers are taken from the live image `host_bytes`."""
        host_avg[self.i_off:self.nbytes].copy_(host_bytes[self.i_off:self.nbytes])
        return host_avg


def weight_ema_decay(value):
    """train_args['weight_ema'] -> the decay of the weights' moving average, or None when averaging is off (key absent, 0 or
    None).  Anything else outside (0, 1) raises ValueError."""
    if value is None or (isinstance(value, numbers.Real) and value == 0):
        return None
    if not isinstance(value, numbers.Real) or not 0.0 < float(value) < 1.0:
        raise ValueError("train_args['weight_ema'] must be a decay in (0, 1) (e.g. 0.999), or 0 / None for no averaging; got %r"
                         % (value,))
    return float(value)


def validation_rate(args):
    """train_args['validation_rate'] -> the fraction r of episodes held out of training for the validation loss, or None when
    validation is off (key absent, 0 or None).  Anything else outside (0, 1) raises ValueError, and so does the key together
    with gpu_replay: False (the held-out split lives in the GPU replay)."""
    value = args.get('validation_rate')
    if value is None or (isinstance(value, numbers.Real) and value == 0):
        return None
    if isinstance(value, bool) or not isinstance(value, numbers.Real) or not 0.0 < float(value) < 1.0:
        raise ValueError("train_args['validation_rate'] must be a fraction in (0, 1) (e.g. 0.05), or 0 / None for no validation; "
                         "got %r" % (value,))
    if not args.get('gpu_replay', True):
        raise ValueError("train_args['validation_rate'] needs the GPU replay (gpu_replay: True): the held-out episodes are kept there")
    return float(value)


def replay_ratio(args):
    """train_args['replay_ratio'] -> the cap r on samples trained per step stored in the training replay, or None when the
    limit is off (key absent, 0 or None).  A negative, NaN or infinite value, True and anything that is not a number raise
    ValueError."""
    value = args.get('replay_ratio')
    if value is None or (isinstance(value, numbers.Real) and value == 0):
        return None
    if isinstance(value, bool) or not isinstance(value, numbers.Real) or not 0.0 < float(value) < float('inf'):
        raise ValueError("train_args['replay_ratio'] must be a positive number of samples trained per stored step (e.g. 32), "
                         "or 0 / None for no limit; got %r" % (value,))
    return float(value)


def gradient_accumulation(args):
    """train_args['gradient_accumulation'] -> k, the number of micro-batches each batch is trained as (one optimiser step per
    batch); 1 when accumulation is off (key absent, None, 0 or 1).  True, a negative value and anything that is not an integer
    raise ValueError."""
    return micro_batch_count(args.get('gradient_accumulation'))


def micro_batch_count(value):
    """The checks of gradient_accumulation() on a value: None or 0 -> 1, an integer k >= 1 -> k, anything else ValueError."""
    if value is None:
        return 1
    if isinstance(value, bool) or not isinstance(value, numbers.Integral) or value < 0:
        raise ValueError("train_args['gradient_accumulation'] must be an integer k >= 1 of micro-batches per batch, or 0 / None "
                         "for none; got %r" % (value,))
    return max(1, int(value))


class ReplayRatioLimiter:
    """The Trainer's samples-per-insert limit (train_args['replay_ratio'] = r), counted on the host from numbers it already
    has: `trained`, the samples of the batches drawn (drew(): batch_size * forward_steps each, the global batch without
    burn-in), and `stored`, the steps of the episodes that entered the training replay (store(), called by the feeder after
    each commit).  Evictions never lower `stored`: it counts inserts.  acquire(n) holds the trainer thread until n more
    batches fit,

        trained + n * samples_per_batch <= r * stored,

    on a condition that store() signals (and a short poll), so it never touches the device and never blocks the feeder.
    Both counts start at zero with the object, and the per-epoch figures of the printed line come from end_epoch()."""

    def __init__(self, ratio, samples_per_batch, poll=0.05, clock=time.monotonic):
        self.ratio, self.samples_per_batch = float(ratio), int(samples_per_batch)
        self.poll, self.clock = poll, clock
        self.cond = threading.Condition()
        self.trained = self.stored = 0
        self.waited = 0.0                 # seconds the trainer thread spent in acquire() without credit
        self.waiting = False
        self._mark = None                 # (trained, stored, waited, clock) at the start of the running epoch

    def allows(self, n=1):
        return self.trained + n * self.samples_per_batch <= self.ratio * self.stored

    def store(self, steps):
        with self.cond:
            self.stored += int(steps)
            self.cond.notify_all()

    def drew(self, batches=1):
        with self.cond:
            self.trained += batches * self.samples_per_batch

    def wake(self):
        """Make a waiting acquire() look at its interrupt() now (the Trainer calls it from update() and stop())."""
        with self.cond:
            self.cond.notify_all()

    def acquire(self, n, interrupt):
        """Wait until n more batches fit (returns True) or, without that credit, until interrupt() is true (returns False)."""
        with self.cond:
            if self.allows(n):
                return True
            t0 = self.clock()
            self.waiting = True
            try:
                while not self.allows(n):
                    if interrupt():
                        return False
                    self.cond.wait(self.poll)
                return True
            finally:
                self.waiting = False
                self.waited += self.clock() - t0

    def start_epoch(self):
        """Start the first epoch's clock (later epochs start where the previous one ended); its counts start at zero, so the
        first epoch's stored steps include the backlog."""
        with self.cond:
            if self._mark is None:
                self._mark = (0, 0, 0.0, self.clock())

    def end_epoch(self):
        """The running epoch's figures, and start the next: {'trained': samples, 'stored': steps, 'ratio': trained / stored
        (None when nothing was stored), 'limit': r, 'waited': the fraction of the epoch's wall time spent waiting for credit,
        'wall': the epoch's wall time in seconds}."""
        with self.cond:
            now = self.clock()
            trained0, stored0, waited0, t0 = self._mark if self._mark is not None else (0, 0, 0.0, now)
            self._mark = (self.trained, self.stored, self.waited, now)
            trained, stored, waited = self.trained - trained0, self.stored - stored0, self.waited - waited0
        wall = now - t0
        return {'trained': trained, 'stored': stored, 'ratio': trained / stored if stored else None, 'limit': self.ratio,
                'waited': min(1.0, waited / wall) if wall > 0 else 0.0, 'wall': wall}

    def snapshot(self):
        with self.cond:
            return {'limit': self.ratio, 'trained': self.trained, 'stored': self.stored, 'waited': self.waited,
                    'waiting': self.waiting}


def replay_ratio_line(stats):
    """'replay_ratio = 31.7 limit:32 waited:0.43': an epoch's trained samples over the steps stored during it (left out when
    nothing was stored), the limit, and the fraction of its wall time the trainer waited for credit (ReplayRatioLimiter.end_epoch)."""
    head = '%.1f ' % stats['ratio'] if stats['ratio'] is not None else ''
    return 'replay_ratio = %slimit:%g waited:%.2f' % (head, stats['limit'], stats['waited'])


def save_replay(args):
    """train_args['save_replay'] -> {'every': n, 'keep': k}: the replay is saved with every n-th numbered epoch and the run keeps
    the newest k files it wrote (0: all), or None when the key is off (absent, None, False or 0).  True is n = 1; a positive
    integer is n; {'every': n, 'keep': k} sets both (defaults 1 and 2).  Anything else raises ValueError, and so does the key
    with gpu_replay: False (the saved set is what the GPU replay holds)."""
    value = args.get('save_replay')
    if value is None or value is False or (isinstance(value, numbers.Integral) and not isinstance(value, bool) and value == 0):
        return None
    spec = {'every': 1, 'keep': 2}
    if isinstance(value, dict):
        unknown = sorted(set(value) - set(spec), key=str)
        if unknown:
            raise ValueError("train_args['save_replay']: unknown key(s) %s (known: every, keep)" % unknown)
        spec.update(value)
    elif value is not True:
        spec['every'] = value
    for k, least in (('every', 1), ('keep', 0)):
        v = spec[k]
        if isinstance(v, bool) or not isinstance(v, numbers.Integral) or v < least:
            raise ValueError("train_args['save_replay']: %s must be an integer >= %d; got %r" % (k, least, v))
        spec[k] = int(v)
    if not args.get('gpu_replay', True):
        raise ValueError("train_args['save_replay'] needs the GPU replay (gpu_replay: True): it saves what that replay holds")
    return spec


_save_replay_spec = save_replay       # for the constructors whose `save_replay` argument shadows the parser

REPLAY_FORMAT = 1


def replay_file(snapshot, priority_state=None, limiter=None, steps=0, epoch=0):
    """The dict of a models/<epoch>.replay.pth file (plain containers and tensors: it loads with torch.load alone):

        {'format': 1,
         'episodes': [episode, ...],    the episodes resident in the training and held-out rings, oldest first, as they arrived
         'serials': int64 tensor,       the DeviceReplay serial of each, -1 for a held-out episode
         'capacity_steps', 'maximum_episodes': int,
         'sampler': {'rng', 'val_rng', 'sym_rng' (or None): numpy bit_generator.state dicts, 'prio_batches': int},
         'priorities': None or {'serial': int64 tensor, 'priority': float32 tensor, 'max_prio': float}  (priority.image),
         'limiter': None or ReplayRatioLimiter.snapshot(), 'steps': Trainer.steps, 'epoch': int}

    snapshot: GpuBatcher.snapshot(); priority_state: LearnerStep.priority_state_dict() / PendingModel.priority_state."""
    prio = None
    if priority_state is not None:
        img = priority.image(priority_state['slot_serial'].numpy(), priority_state['priority'].numpy(),
                             priority_state['max_prio'], snapshot['serials'].numpy())
        prio = {'serial': torch.from_numpy(img['serial']), 'priority': torch.from_numpy(img['priority']),
                'max_prio': img['max_prio']}
    return dict(snapshot, format=REPLAY_FORMAT, priorities=prio, limiter=limiter, steps=int(steps), epoch=int(epoch))


def load_replay_file(path, leaf_shapes=None, actions=None):
    """Read a replay file and check it: a known 'format', every entry present, one serial per episode, every episode a dict
    with its step count and one of the two wire formats, the first episode decodable, and -- when given -- its observation
    leaf shapes and action count equal to `leaf_shapes` (a list of tuples) and `actions`.  Raises ValueError naming the file."""
    from .wire import episode_to_flat
    try:
        d = torch.load(path, map_location='cpu')
    except Exception as e:
        raise ValueError('%s: not a readable replay file (%s)' % (path, e))
    if not isinstance(d, dict) or d.get('format') != REPLAY_FORMAT:
        raise ValueError('%s: unknown replay file format %r (this version reads %d)'
                         % (path, d.get('format') if isinstance(d, dict) else type(d).__name__, REPLAY_FORMAT))
    missing = [k for k in ('episodes', 'serials', 'capacity_steps', 'maximum_episodes', 'sampler', 'priorities') if k not in d]
    if missing:
        raise ValueError('%s: no %s entry' % (path, ', '.join(missing)))
    eps = d['episodes']
    if not isinstance(eps, list) or len(d['serials']) != len(eps):
        raise ValueError('%s: %d serials for %s episodes' % (path, len(d['serials']), len(eps) if isinstance(eps, list) else 'no'))
    for i, ep in enumerate(eps):
        if not isinstance(ep, dict) or not isinstance(ep.get('steps'), numbers.Integral) or ep['steps'] <= 0 \
                or 'outcome' not in ep or not ('flat' in ep or ep.get('moment')):
            raise ValueError('%s: episode %d is not an episode in either wire format' % (path, i))
    if eps:
        try:
            fe = episode_to_flat(eps[0])
            shapes, A = [tuple(l.shape[2:]) for l in tree_leaves(fe.obs)], int(fe.amask.shape[-1])
        except Exception as e:
            raise ValueError('%s: the episodes do not decode (%s: %s)' % (path, type(e).__name__, e))
        if leaf_shapes is not None and shapes != [tuple(sh) for sh in leaf_shapes]:
            raise ValueError('%s: observations of shape %s, expected %s' % (path, shapes, [tuple(sh) for sh in leaf_shapes]))
        if actions is not None and A != int(actions):
            raise ValueError('%s: %d actions, expected %d' % (path, A, int(actions)))
    return d


class ReplayCheckpoints:
    """Writes models/<epoch>.replay.pth files off the caller's thread.  submit(epoch, obj) returns at once: one writer thread
    (started by the first submit) torch.saves obj to a temporary name in the directory and renames it, so a file that exists
    is complete.  While a write runs at most one submission waits: a newer one replaces it.  After each write the files this
    object wrote beyond the newest `keep` are deleted (keep = 0: none); files it did not write are never touched.  close()
    writes what still waits and joins the thread."""

    def __init__(self, directory='models', keep=2):
        self.directory, self.keep = directory, int(keep)
        self.cond = threading.Condition()
        self.queued = None
        self.closed = False
        self.thread = None
        self.written = []           # paths this object wrote and has not deleted, oldest first
        self.replaced = 0           # submissions a newer one overtook
        self.last_error = None

    def path(self, epoch):
        return os.path.join(self.directory, '%s.replay.pth' % epoch)

    def write(self, epoch, obj):
        """Write one file now, on this thread; returns its path."""
        os.makedirs(self.directory, exist_ok=True)
        path = self.path(epoch)
        tmp = path + '.tmp'
        try:
            torch.save(obj, tmp)
            os.replace(tmp, path)
        except BaseException:
            if os.path.exists(tmp):
                os.remove(tmp)
            raise
        if path in self.written:
            self.written.remove(path)
        self.written.append(path)
        while self.keep and len(self.written) > self.keep:
            old = self.written.pop(0)
            if os.path.exists(old):
                os.remove(old)
        return path

    def submit(self, epoch, obj):
        with self.cond:
            if self.closed:
                raise RuntimeError('ReplayCheckpoints is closed')
            if self.queued is not None:
                self.replaced += 1
            self.queued = (epoch, obj)
            if self.thread is None:
                self.thread = threading.Thread(target=self._run, daemon=True)
                self.thread.start()
            self.cond.notify_all()

    def _run(self):
        while True:
            with self.cond:
                while self.queued is None and not self.closed:
                    self.cond.wait()
                if self.queued is None:
                    return
                epoch, obj = self.queued
                self.queued = None
            try:
                self.write(epoch, obj)
            except Exception as e:          # a full disk must not end the run: the next epoch tries again
                self.last_error = e
                traceback.print_exc()

    def close(self):
        with self.cond:
            self.closed = True
            self.cond.notify_all()
        if self.thread is not None:
            self.thread.join()
            self.thread = None


def optimizer_config(value):
    """train_args['optimizer'] -> {'name': 'adam'} (key absent, None or 'adam': clip + Adam, ops.FlatAdam) or
    {'name': 'lamb', 'lr_scale': s} ('lamb', or {'name': 'lamb', 'lr_scale': s} with s a finite number > 0, default 1.0:
    clip + LAMB, ops.FlatLamb).  Anything else -- another name, another dict key, a bad lr_scale -- raises ValueError."""
    if value is None or (isinstance(value, str) and value == 'adam'):
        return {'name': 'adam'}
    if isinstance(value, str) and value == 'lamb':
        return {'name': 'lamb', 'lr_scale': 1.0}
    if not isinstance(value, dict):
        raise ValueError("train_args['optimizer'] must be 'adam', 'lamb' or {'name': 'lamb', 'lr_scale': s}; got %r" % (value,))
    unknown = sorted(str(k) for k in value if k not in ('name', 'lr_scale'))
    if unknown:
        raise ValueError("train_args['optimizer']: unknown key(s) %s (known: name, lr_scale)" % ', '.join(unknown))
    if value.get('name') != 'lamb':
        raise ValueError("train_args['optimizer']: the dict form is {'name': 'lamb', 'lr_scale': s}; got name %r"
                         % (value.get('name'),))
    s = value.get('lr_scale', 1.0)
    if isinstance(s, bool) or not isinstance(s, numbers.Real) or not 0.0 < float(s) < float('inf'):
        raise ValueError("train_args['optimizer']: lr_scale must be a finite number > 0; got %r" % (s,))
    return {'name': 'lamb', 'lr_scale': float(s)}


def nonfinite_guard(args):
    """train_args['skip_nonfinite'] -> whether optimiser steps whose loss or gradient is not finite are rejected on the device
    (key absent, False or None: off)."""
    return bool(args.get('skip_nonfinite'))


# the distillation sums [kl, c_n * kl] (distill.py)
NUM_DISTILL = 2

AccumLayout = collections.namedtuple('AccumLayout', 'loss distill diag skipped n_tail n')


def accum_layout(diagnostics=False, skip_nonfinite=False, distill=False):
    """The AccumLayout of the learner's float64 epoch accumulator (LearnerStep.accum) with these options on: the slices
    `loss`, `distill`, `diag` and `skipped` (None when their option is off) and the size `n`.  Its first n_tail slots are
    the step's float32 tail at the same offsets -- each row of LearnerStep.loss_rows and the gradient bucket's extra slots
    start with it -- so a step adds its whole tail to the accumulator in one piece:

        tail         [loss NUM_LOSS | distill NUM_DISTILL, when distilling | the loss pass's diagnostics NUM_LOSS_DIAG]
        accumulator  [tail | the optimiser's diagnostics NUM_DIAG - NUM_LOSS_DIAG | skipped 1, with the guard]

    `diag` is both kinds of diagnostics in DIAG_KEYS order."""
    d = NUM_LOSS + (NUM_DISTILL if distill else 0)
    n = d + (NUM_DIAG if diagnostics else 0)
    return AccumLayout(loss=slice(0, NUM_LOSS), distill=slice(NUM_LOSS, d) if distill else None,
                       diag=slice(d, n) if diagnostics else None, skipped=slice(n, n + 1) if skip_nonfinite else None,
                       n_tail=d + (NUM_LOSS_DIAG if diagnostics else 0), n=n + (1 if skip_nonfinite else 0))


def skipped_line(skipped, steps):
    """'skipped = 3 of 1200 steps: non-finite loss or gradient': the steps of an epoch the guard rejected."""
    return 'skipped = %d of %d steps: non-finite loss or gradient' % (skipped, steps)


def loss_line(name, sums, heads):
    """'<name> = p:0.512 v:0.231 ent:1.843 total:0.561': each head's sum over the sums' own sample count dcnt, as the Trainer
    prints its training loss (train.py:392)."""
    return '%s = %s' % (name, ' '.join([k + ':' + '%.3f' % (sums[k] / sums['dcnt']) for k in heads]))


class AveragedCheckpoints:
    """Files written next to the Learner's checkpoints (reference train.py:441-454): models/<epoch>.<suffix>.pth and
    models/latest.<suffix>.pth, in the Learner's relative `models` directory, written with torch.save.  <epoch> is the number
    the Learner gives the model handed back with them: restart_epoch + the models handed back so far.  One object numbers
    every kind of file (the moving average of the weights, 'ema'; the optimiser state, 'optim'), so the files of one epoch
    share <epoch>.  `suffix` is the kind path(), seed_path() and save() use when not told otherwise."""

    def __init__(self, restart_epoch=0, directory='models', suffix='ema'):
        self.directory = directory
        self.suffix = suffix
        self.restart_epoch = int(restart_epoch or 0)
        self.epoch = self.restart_epoch

    def path(self, epoch, suffix=None):
        return os.path.join(self.directory, '%s.%s.pth' % (epoch, suffix or self.suffix))

    def seed_path(self, suffix=None):
        """The file of this kind a restarted run resumes from (models/<restart_epoch>.<suffix>.pth), or None."""
        if self.restart_epoch > 0 and os.path.exists(self.path(self.restart_epoch, suffix)):
            return self.path(self.restart_epoch, suffix)
        return None

    def save(self, state_dict):
        """Write the file of the default kind for the next epoch; returns its path."""
        return self.save_epoch({self.suffix: state_dict})[self.suffix]

    def save_epoch(self, files):
        """Write the files of the next epoch, {suffix: object to torch.save}; returns {suffix: path}."""
        self.epoch += 1
        if files:
            os.makedirs(self.directory, exist_ok=True)
        for suffix, obj in files.items():
            torch.save(obj, self.path(self.epoch, suffix))
            torch.save(obj, self.path('latest', suffix))
        return {suffix: self.path(self.epoch, suffix) for suffix in files}


class OptimizerStateFormat:
    """The learner's optimiser state as a plain dict that loads without this package:

        {'optimizer': what torch.optim.Adam(net.parameters(), lr, betas, eps, weight_decay).state_dict() holds after a step:
                      'state': {i: {'step', 'exp_avg', 'exp_avg_sq'}} shaped like parameter i, 'param_groups': [one group],
         'param_names': [names in net.named_parameters() order],
         'schedule': {'steps': int, 'data_cnt_ema': float, 'lr': float},
         'max_norm': float}

    Parameter i is the i-th of net.parameters(), words [off_i, off_i + numel_i) of FlatAdam's flat buckets; the words from n
    up to n_pad are padding, not part of the format, and zero after a load.  'step' is the number of optimiser steps taken
    (FlatAdam.step_count), a float32 tensor as torch keeps it.  'schedule' holds what the next step uses: the learning rate
    and the data-count average it came from (the device's float32 values), and the step count it was scheduled at.

    A LAMB learner (optimizer_config(...)['name'] == 'lamb', `optimizer`) adds two top-level entries, 'algorithm': 'lamb'
    and 'lr_scale': float; its moments and step mean what Adam's do.  A dict without 'algorithm' is an Adam dict, and an Adam
    learner writes exactly the entries above.  unpack() refuses a dict of the other algorithm; lr_scale is not compared."""

    def __init__(self, named_params, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-5, max_norm=4.0, optimizer=None):
        self.names, self.shapes, self.offsets = [], [], []
        off = 0
        for k, p in named_params:
            self.names.append(k)
            self.shapes.append(tuple(p.shape))
            self.offsets.append(off)
            off += p.numel()
        self.n = off
        self.n_pad = (off + 3) // 4 * 4
        self.betas = (float(betas[0]), float(betas[1]))
        self.eps, self.weight_decay, self.max_norm = float(eps), float(weight_decay), float(max_norm)
        self.optimizer = optimizer if optimizer is not None else {'name': 'adam'}

    def _spans(self):
        for name, shape, off in zip(self.names, self.shapes, self.offsets):
            n = 1
            for d in shape:
                n *= d
            yield name, shape, off, n

    def to_dict(self, exp_avg, exp_avg_sq, step, lr, data_cnt_ema, steps):
        """The dict of flat CPU moments (at least n words each), the step count and the schedule; fresh storage per tensor."""
        dummies = [torch.zeros(1, requires_grad=True) for _ in self.names]       # the param group exactly as torch writes it
        groups = torch.optim.Adam(dummies, lr=float(lr), betas=self.betas, eps=self.eps,
                                  weight_decay=self.weight_decay).state_dict()['param_groups']
        state = {}
        for i, (_, shape, off, n) in enumerate(self._spans()):
            state[i] = {'step': torch.tensor(float(step), dtype=torch.float32),
                        'exp_avg': exp_avg[off:off + n].clone().view(shape),
                        'exp_avg_sq': exp_avg_sq[off:off + n].clone().view(shape)}
        d = {'optimizer': {'state': state, 'param_groups': groups},
             'param_names': list(self.names),
             'schedule': {'steps': int(steps), 'data_cnt_ema': float(data_cnt_ema), 'lr': float(lr)},
             'max_norm': self.max_norm}
        if self.optimizer['name'] == 'lamb':
            d['algorithm'], d['lr_scale'] = 'lamb', self.optimizer['lr_scale']
        return d

    def check_algorithm(self, d):
        """Raise ValueError when the dict `d` was written by the other optimiser (its 'algorithm' entry, absent: Adam)."""
        got, want = d.get('algorithm', 'adam'), self.optimizer['name']
        if got != want:
            raise ValueError('optimiser state: written by %s, the learner runs %s (train_args[\'optimizer\'])' % (got, want))

    def unpack(self, d):
        """Check a dict of this format against the net and the optimiser's settings and return its flat form
        (exp_avg, exp_avg_sq: float32 CPU tensors of n_pad words with zero padding; step; lr; data_cnt_ema; steps).
        Raises KeyError (an entry or a parameter name missing or extra) or ValueError (a shape, betas, eps, weight_decay or
        max_norm that differs, or a dict of the other algorithm: check_algorithm)."""
        self.check_algorithm(d)
        for key in ('optimizer', 'param_names', 'schedule', 'max_norm'):
            if key not in d:
                raise KeyError('optimiser state: no %r entry' % key)
        names = list(d['param_names'])
        missing = [k for k in self.names if k not in names]
        extra = [k for k in names if k not in self.names]
        if missing or extra or len(names) != len(self.names):
            raise KeyError('optimiser state: parameter names differ from the net\'s (missing: %s; extra or repeated: %s)'
                           % (', '.join(missing) or '-', ', '.join(extra) or '-'))
        groups = d['optimizer']['param_groups']
        if len(groups) != 1:
            raise ValueError('optimiser state: %d parameter groups, the learner has one' % len(groups))
        group = groups[0]
        got = {'betas': tuple(float(b) for b in group['betas']), 'eps': float(group['eps']),
               'weight_decay': float(group['weight_decay']), 'max_norm': float(d['max_norm'])}
        want = {'betas': self.betas, 'eps': self.eps, 'weight_decay': self.weight_decay, 'max_norm': self.max_norm}
        for key in want:
            if got[key] != want[key]:
                raise ValueError('optimiser state: %s is %r, the learner\'s %r' % (key, got[key], want[key]))
        state = d['optimizer']['state']
        index = {k: i for i, k in enumerate(names)}
        m, v = torch.zeros(self.n_pad), torch.zeros(self.n_pad)
        steps_seen = set()
        for name, shape, off, n in self._spans():
            s = state.get(index[name])
            if s is None:
                raise KeyError('optimiser state: no state for parameter %d (%s)' % (index[name], name))
            for key, flat in (('exp_avg', m), ('exp_avg_sq', v)):
                src = torch.as_tensor(s[key])
                if tuple(src.shape) != shape:
                    raise ValueError('optimiser state: %s of %s has shape %s, the parameter %s'
                                     % (key, name, tuple(src.shape), shape))
                flat[off:off + n] = src.reshape(-1).to(torch.float32)
            steps_seen.add(float(s['step']))
        if len(steps_seen) != 1:
            raise ValueError('optimiser state: the parameters have different step counts %s' % sorted(steps_seen))
        sched = d['schedule']
        return m, v, int(round(steps_seen.pop())), float(group['lr']), float(sched['data_cnt_ema']), int(sched['steps'])


class PendingModel:
    """The model of a finished epoch, still on its way to the host.  `resolve()` (called by Trainer.update() on the
    Learner's thread) waits for the side-stream copy only, prints the epoch's loss line, rebuilds the CPU model in
    eval mode and caches its pickled bytes on it (the Learner pickles the model for every worker request,
    train.py:605-615).  `host` maps the names of LearnerStep's hand-off entries to their pinned host copies.  With a moving
    average of the weights ('avg'), it also leaves the averaged state_dict, keyed like the model's, in `ema_state`; with the
    optimiser state ('optim', the optim_snap layout), it leaves that state in the OptimizerStateFormat dict in `optim_state`,
    scheduled at step count `steps`.  With validation passes ('val'), it prints their lines after the loss line and leaves
    their sums in `validation` (what LearnerStep.pop_validation() returns).  `host_losses` holds the learner's accumulator in
    the layout `diagnostics`, `skip_nonfinite` and
    `distill` give (accum_layout, in `slots`); with the guard, the number of the epoch's `batch_cnt` steps that were rejected is left
    in `skipped` and, when it is not zero, printed (skipped_line) after the loss and diagnostics lines.  The Trainer sets
    `replay_ratio` to the epoch's ReplayRatioLimiter.end_epoch() figures under train_args['replay_ratio'], and report() prints
    them (replay_ratio_line) after those lines and before the validation lines.  Under train_args['save_replay'] the Trainer
    sets `replay` to the GpuBatcher.snapshot() taken at the boundary, and with the priorities ('prio', the prio_snap layout)
    resolve() leaves them in `priority_state` (what LearnerStep.priority_state_dict() returns).  With distillation
    (`distill`), the accumulator holds the epoch's sums of kl and c_n * kl: report() leaves them in `distill` and prints
    distill.line() after the loss and diagnostics lines and before the skipped line."""

    def __init__(self, stepper, done_event, host_state, host_losses, heads, template, host=None, steps=0, diagnostics=False,
                 skip_nonfinite=False, batch_cnt=0, distill=False):
        self.stepper, self.done, self.host_state, self.host_losses = stepper, done_event, host_state, host_losses
        self.heads, self.template, self.host, self.steps = heads, template, host or {}, steps
        self.slots, self.batch_cnt = accum_layout(diagnostics, skip_nonfinite, distill), batch_cnt
        self.distill = None
        self.ema_state = None
        self.optim_state = None
        self.validation = None
        self.skipped = 0
        self.replay_ratio = None
        self.replay = None
        self.priority_state = None

    def report(self):
        """Read the epoch's sums from the host copy (already arrived) and print the epoch's lines; returns the loss sums."""
        host = self.host_losses.tolist()
        slots = self.slots
        if len(host) != slots.n:
            raise ValueError('PendingModel: %d accumulator slots, the layout has %d' % (len(host), slots.n))
        sums = dict(zip(LOSS_KEYS, host[slots.loss]))
        dcnt = sums['dcnt']
        self.diagnostics = ops.summarize_diagnostics(host[slots.diag]) if slots.diag is not None else None
        self.skipped = int(host[slots.skipped][0]) if slots.skipped is not None else 0
        if slots.distill is not None:
            self.distill = dict(zip(('kl', 'term'), host[slots.distill]))
        if dcnt > 0:
            print(loss_line('loss', sums, self.heads))
            if self.diagnostics is not None:
                print(ops.format_diagnostics(self.diagnostics))
            if self.distill is not None:
                print(distill_mod.line(self.distill['kl'], self.distill['term'], dcnt))
        if self.skipped:
            print(skipped_line(self.skipped, self.batch_cnt))
        if self.replay_ratio is not None:
            print(replay_ratio_line(self.replay_ratio))
        if 'val' in self.host:
            self.validation = self.stepper.validation_sums(self.host['val'].tolist())
            for name, val in self.validation.items():
                if val['dcnt'] > 0:
                    print(loss_line(name, val, self.heads))
        return sums

    def resolve(self):
        self.done.synchronize()
        sums = self.report()
        tpl, stepper = self.template, self.stepper
        keys = list(tpl.state_dict().keys())
        state = stepper._state_dict_of(self.host_state)
        if 'avg' in self.host:
            avg = stepper._state_dict_of(stepper.state.averaged_bytes(self.host['avg'], self.host_state))
            self.ema_state = collections.OrderedDict((k, avg[k]) for k in keys)
        if 'optim' in self.host:
            self.optim_state = stepper.optimizer_state_from(self.host['optim'], self.steps)
        if 'prio' in self.host:
            self.priority_state = stepper.priority_state_from(self.host['prio'])
        tpl.load_state_dict({k: state[k] for k in keys})
        tpl.eval()
        blob = pickle.dumps(tpl)
        model = pickle.loads(blob)                        # == copy.deepcopy(tpl), and leaves the bytes for the workers
        attach_pickle_cache(model, blob)
        return model, sums


def attach_pickle_cache(model, blob):
    """pickle.dumps(model) / copy.deepcopy(model) of this instance replay `blob` instead of walking the module tree:
    the instance-level __reduce_ex__ makes every later pickle of the (immutable until the next epoch) model a memcpy.
    What the workers unpickle is the plain nn.Module that `blob` holds."""
    object.__setattr__(model, '__reduce_ex__', lambda protocol, _b=blob: (pickle.loads, (_b,)))
    return model


# LearnerStep._handoff: end_epoch fills the device buffer `snap` on the step stream by `copies`, (view of snap, live tensor)
# pairs, runs `after()`, and carries snap to the start of PendingModel.host[name], pinned memory of `room` (or snap's) elements
_Handoff = collections.namedtuple('_Handoff', 'name snap copies after room', defaults=(None, None))


def tensor_core_mode(value):
    """train_args['tensor_cores'] -> the precision of the net's products on this library's kernels: True (the default: 3xTF32
    tensor-core products, fp32-class accuracy), False (fp32 SIMT kernels) or 'bf16' (tensor-core products on bf16 operands,
    rounded after their fp32 transform, fp32 accumulation).  Any other value reads as bool(value)."""
    if isinstance(value, str) and value == 'bf16':
        return 'bf16'
    return bool(value)


class LearnerStep:
    """One replay batch -> one optimiser step.

    tensor_cores (default: train_args['tensor_cores'], True): the precision of the net's products, tensor_core_mode(); the
    step runs the mode in `self.tensor_cores` (True, False or 'bf16').  'bf16' covers every product of the fused tower and of
    the rewritten small-board convolutions, in the step and in validation passes alike; layers left on cuDNN / cuBLAS keep
    following allow_tf32.

    step(packed):  ONE H2D copy of the packed pinned batch -> [CUDA graph: net forward ->
    fused loss fwd+bwd kernel -> net backward -> (all-reduce SUM) -> clip + Adam].
    The six loss sums land in `last_losses` / `loss_accum` on the device; nothing in here
    synchronises the host.

    diagnostics (default: train_args['diagnostics'], off): the loss pass also takes the learner diagnostics sums
    (ops.DIAG_KEYS), which ride the gradient bucket behind the loss sums, and the optimiser adds its pre-clip norm
    statistics; both accumulate in `diag_accum` (float64, on the device) until end_epoch / pop_diagnostics.  Losses,
    gradients and weights are the same with and without.

    weight_ema (default: train_args['weight_ema'], off): a decay d in (0, 1).  Every step ends with one more launch that
    updates a moving average of the fp32 state (parameters and BatchNorm buffers, StateStore bytes [0, i_off)) on the
    device: a <- a + w (x - a), w = max(1 - d, 1 / t) at optimiser step t, or 1 - d once seeded (seed_weight_ema).
    end_epoch hands it over with the model (PendingModel.ema_state); ema_state_dict() reads it now.  Training itself is
    the same with and without.

    save_optimizer (default: train_args['save_optimizer'], off): end_epoch also hands over the optimiser state the next
    step uses (Adam's moments and step count, the learning rate and the data-count average of its schedule) in the
    OptimizerStateFormat dict (PendingModel.optim_state), by the same device-to-device snapshot and side-stream copy as the
    model.  optimizer_state_dict() reads it now; load_optimizer_state() resumes from it.  The step itself is the same with
    and without.

    validation (default: whether train_args['validation_rate'] is set, off): validate_in_place() evaluates the batch in
    self.dev with the current weights -- net forward in training mode (BatchNorm on batch statistics, as in the step), then the
    forward-only loss kernel (ops.loss_fwd) -- and adds the six loss sums to `val_accum`; validate_in_place(averaged=True)
    does the same with the moving average of the weights into `val_ema_accum`.  No backward, no optimiser step, no
    all-reduce, and the learner is left bit for bit as it was: the StateStore bytes (weights, BatchNorm running statistics,
    num_batches_tracked) are saved and restored around the pass on the device.  In graph mode each form is one more CUDA
    graph sharing the step graph's memory pool; `launches_per_validation` counts its launches.  end_epoch hands the sums
    over with the loss sums (PendingModel.validation); pop_validation() reads them now.

    train_args['prioritized_replay'] (priority.py): the step owns the priority state (`prio_state`, a priority.PriorityState:
    the per-slot priorities and the per-window slot, serial and weight buffers the sampler fills), because the captured graph
    bakes in its pointers.  The loss pass scales window b's terms and gradients by prio_state.win_weight[b] and writes the
    advantage tap, and the step ends with one more launch (ops.priority_update, after the optimiser: it reads the guard's flag)
    that stores the windows' priorities.  With the weights at 1 and the serials at -1 (as built, and so during the warm-up and
    capture steps) the weights train exactly as without the key and no priority moves.

    skip_nonfinite (default: train_args['skip_nonfinite'], off): a step whose pre-clip gradient norm or one of whose six loss
    sums is not finite is rejected on the device (ops.FlatAdam.skip, hrl_clip_adam_step with a skip flag), and the learner is left
    bit for bit as if its batch had never been drawn: weights, Adam's moments and step count, the BatchNorm buffers (saved by
    one device-to-device copy at the start of every step and put back by hrl_step_commit), the epoch's loss and diagnostics
    sums and the weight average.  Only the count of rejected steps (`skipped`, the accumulator's last slot; handed over as
    PendingModel.skipped) goes up, and last_losses still holds the rejected step's sums.  `steps` and the host's batch counts
    keep counting batches drawn; a rejected batch adds nothing to dcnt.  One more launch per step.  Validation passes are not
    guarded.

    save_replay (default: whether train_args['save_replay'] is set, off): with prioritized_replay, end_epoch also hands over the
    per-slot priorities, their serials and max_prio (PendingModel.priority_state), by the same device-to-device snapshot and
    side-stream copy.  priority_state_dict() reads them now; load_priority_state() writes saved ones.  The step is the same
    with and without.

    gradient_accumulation (default: train_args['gradient_accumulation'], 1): an integer k >= 1 that divides the batch B.  Every
    step consumes one batch of B windows and takes one optimiser step, running the net, the loss kernel and the net's
    backward over the k micro-batches dev[i*B/k:(i+1)*B/k] (`_micro`) in order, each adding its gradient into the bucket;
    the micro-batches' loss (and diagnostics) sums are then folded into the bucket tail (one device copy at k = 1, one
    ops.sum_rows launch otherwise), and the all-reduce, the optimiser and the rest of the step run once.  k = 1 is the whole
    batch as one micro-batch.  The net is sized for B/k windows, so its activations (and the recurrent hidden state) take
    1/k of the memory.  The gradient is the full batch's up to fp32 summation order, except that BatchNorm normalises each
    micro-batch with its own statistics and moves its running statistics once per micro-batch (k per step) -- the step k
    ranks of B/k windows would take.  `micro_batches` is k; launches_per_step counts all k micro-batches.  Validation
    passes run in the same micro-batches; time_loss_kernel needs k = 1.

    distill (default: train_args['distill'], off; distill.py) and teacher (an nn.Module, or None: built from the key's file,
    distill.teacher_net): policy distillation.  Each micro-batch first runs the teacher -- in eval mode, under no_grad, on the
    module path (optimize_small_boards in the step's tensor_cores mode, its own channels-last probe, forward_raw with its own
    init_hidden and train=False), never on the fused tower -- then the student, the fused loss kernel, one more launch
    (ops.distill_fwd_bwd) that adds c_n * KL(teacher || student) to the policy gradient and to the loss row's total, and the
    backward.  Its two sums [kl, c_n * kl] follow the loss sums in the loss row, the bucket tail and the accumulator
    (`distill_accum`; accum_layout); the teacher's weights are in no bucket, hand-off or checkpoint.  With c_n = 0 the step
    is bit for bit the step without the key.  Validation passes are unchanged.

    optimizer (default: train_args['optimizer'], Adam; optimizer_config): 'lamb' or {'name': 'lamb', 'lr_scale': s} runs the
    optimiser step as clip + LAMB (ops.FlatLamb, hrl_clip_lamb_step: Adam's moments, one trust ratio |w_i| / |u_i| per
    parameter tensor, the step lr * s * r_i * u) in place of clip + Adam, in step() and in the peer all-reduce path alike: one
    more launch per step.  `self.optimizer` is the parsed setting.  The moments, step count, guard, diagnostics, weight
    average, gradient accumulation and the hand-off are the same; the saved optimiser state carries 'algorithm': 'lamb'
    (OptimizerStateFormat), and load_optimizer_state() refuses a file of the other algorithm.

    value_bins (default: train_args['value_bins'], off; value_bins.py): categorical value / return heads.  The key is parsed
    here, and a probe call of the net on one observation checks that it outputs every listed head (ValueError otherwise); the
    first forward of warm_up() checks that each such head has K logits in its last dimension (ValueError otherwise -- so a
    net with one-output heads, such as the fused tower's, is refused).  Each micro-batch then runs, after the net's forward,
    one ops.value_bins_expect launch per categorical head (the expectation the fused loss reads in place of the head), the
    fused loss with that head's term and gradient left to the next launch, and one ops.value_bins_fwd_bwd launch per head
    (the cross-entropy: its sum replaces the head's loss sum and joins the total, its logit gradient goes to the net's
    backward).  Validation passes run the forward-only forms.  With the key off nothing of this runs.

    A feature that adds device state registers it in __init__, where it allocates it: in `_mutable` (or `_zeroed`) when a
    step or validation pass changes it, so that the capture's warm-up leaves it as it was, and in `_handoff` (a _Handoff)
    when the epoch boundary carries it to the host; end_epoch, _snapshot and _restore have no per-feature code.
    """

    def __init__(self, model, args, example_batch, lr, device=None, process_group=None, use_graph=True,
                 max_norm=4.0, weight_decay=1e-5, time_loss_kernel=False, channels_last=True, cudnn_benchmark=True,
                 small_boards=True, peer_allreduce=None, allow_tf32=None, fused_tower=True, tensor_cores=None, diagnostics=None,
                 weight_ema=None, save_optimizer=None, validation=None, skip_nonfinite=None, save_replay=None,
                 gradient_accumulation=None, distill=None, teacher=None, optimizer=None, value_bins=None):
        self.optimizer = optimizer_config(args.get('optimizer') if optimizer is None else optimizer)
        self.value_bins = value_bins_mod.config({'value_bins': value_bins} if value_bins is not None else args)
        self.distill = distill_mod.config({'distill': distill} if distill is not None else args, teacher_given=teacher is not None)
        if self.distill is None and teacher is not None:
            self.distill = distill_mod.config({'distill': {}}, teacher_given=True)
        if self.distill is not None and teacher is None:
            teacher = distill_mod.teacher_net(self.distill, model)      # the default net copies the student before any rewrite
        self.teacher = teacher
        k = micro_batch_count(args.get('gradient_accumulation') if gradient_accumulation is None else gradient_accumulation)
        if k > 1 and example_batch['action'].shape[0] % k:
            raise ValueError('gradient_accumulation = %d does not divide the batch of %d windows' % (k, example_batch['action'].shape[0]))
        if k > 1 and time_loss_kernel:
            raise ValueError('time_loss_kernel times the loss kernel of a whole batch: it needs gradient_accumulation = 1')
        self.micro_batches = k
        self.save_replay = bool(_save_replay_spec(args) is not None if save_replay is None else save_replay)
        self.weight_ema = weight_ema_decay(args.get('weight_ema') if weight_ema is None else weight_ema)
        rate = validation_rate(args)
        symmetry.config(args)           # malformed train_args['symmetry'] fails here; the gather applies it, not the step
        self.priority = priority.config(args)
        self.validation = bool(rate is not None if validation is None else validation)
        self.save_optimizer = bool(args.get('save_optimizer', False) if save_optimizer is None else save_optimizer)
        self.skip_nonfinite = nonfinite_guard(args) if skip_nonfinite is None else bool(skip_nonfinite)
        self.device = torch.device(device if device is not None else 'cuda')
        self.args = args
        if diagnostics is None:
            diagnostics = bool(args.get('diagnostics', False))
        self.diagnostics = diagnostics
        self.slots = accum_layout(diagnostics, self.skip_nonfinite, self.teacher is not None)    # accumulator and bucket tail
        # the learner owns its precision contract (1e-5 of the reference's fp32 arithmetic): PyTorch's default lets
        # cuDNN convolutions run on TF32 tensor cores (10-bit mantissa).  train_args['allow_tf32'] = True opts out.
        if allow_tf32 is None:
            allow_tf32 = bool(args.get('allow_tf32', False))
        self.allow_tf32 = allow_tf32
        torch.backends.cudnn.allow_tf32 = allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = allow_tf32
        self.model = model.to(self.device)
        if self.value_bins is not None:         # a categorical head the net does not output: refused before anything runs
            value_bins_mod.check_net_heads(self.value_bins, self._probe_outputs(example_batch), bins=False)
        # cuDNN's default heuristics pick FFT / NCHW-spatial kernels that are 5x slower than its NHWC
        # implicit-GEMM kernels on the tiny boards of these games; NHWC + autotune is a pure layout choice
        # tiny boards: convolutions as one SGEMM, BatchNorm as fused reductions (fastnet.py); NCHW stays as is
        self.engine = None          # hand-scheduled fused forward/backward for recognised architectures (tower.py)
        # train_args['tensor_cores'] = False: the small-board dense products stay on fp32 SIMT kernels (strict fp32 summation);
        # 'bf16': the same tensor-core products on bf16 operands (tensor_core_mode)
        self.tensor_cores = tensor_core_mode(args.get('tensor_cores', True) if tensor_cores is None else tensor_cores)
        tensor_cores = self.tensor_cores
        fused_tower = fused_tower and tensor_cores
        self.rewritten = fastnet.optimize_small_boards(self.model, tensor_cores=tensor_cores) if small_boards else 0
        if self.rewritten and channels_last:
            channels_last = not self._uses_dense_convs(example_batch)       # dense products want NCHW-flat activations
        self.memory_format = torch.channels_last if channels_last else None
        if channels_last:
            self.model = self.model.to(memory_format=torch.channels_last)
        if cudnn_benchmark:
            torch.backends.cudnn.benchmark = True
        self.model.train()
        self.teacher_format = None
        self.launches_per_teacher = 0
        if self.teacher is not None:
            self.teacher = self.teacher.to(self.device).eval()
            self.teacher.requires_grad_(False)
            teacher_rewritten = fastnet.optimize_small_boards(self.teacher, tensor_cores=tensor_cores) if small_boards else 0
            teacher_cl = channels_last and not (teacher_rewritten and self._uses_dense_convs(example_batch, self.teacher))
            self.teacher_format = torch.channels_last if teacher_cl else None
            if teacher_cl:
                self.teacher = self.teacher.to(memory_format=torch.channels_last)
        self.time_loss_kernel = time_loss_kernel
        self.kernel_events = []
        self._timed_loss = None          # time_loss_kernel: the loss kernel launched between the two step graphs
        self.pg = process_group
        self.world = torch.distributed.get_world_size(process_group) if process_group is not None else 1
        params = [p for p in self.model.parameters()]
        # gradient exchange: fused one-shot all-reduce over NVLink peer memory (default when sharded), or NCCL
        if peer_allreduce is None:
            peer_allreduce = self.world > 1 and os.environ.get('HRL_PEER_ALLREDUCE', '1') != '0'
        self.peer = ops.PeerAllReduce(self.pg, self.device) if (peer_allreduce and self.world > 1) else None
        self.state = StateStore(self.model, self.device)
        bucket = dict(lr=lr, weight_decay=weight_decay, max_norm=max_norm, extra=self.slots.n_tail,
                      grad_alloc=self.peer.alloc if self.peer is not None else None, param_storage=self.state.flat_param)
        if self.optimizer['name'] == 'lamb':
            self.opt = ops.FlatLamb(params, lr_scale=self.optimizer['lr_scale'], **bucket)
        else:
            self.opt = ops.FlatAdam(params, **bucket)
        self.state.index_params(self.model)
        self.optim_format = OptimizerStateFormat(self.model.named_parameters(), betas=self.opt.betas, eps=self.opt.eps,
                                                 weight_decay=weight_decay, max_norm=max_norm, optimizer=self.optimizer)
        self.schedule_steps = 0          # the step count the current learning rate was scheduled at
        # what a step or a validation pass changes and the capture's warm-up must leave as it was: _snapshot clones `_mutable`,
        # _restore copies the clones back into the same tensors (the graphs bake their pointers) and zeroes `_zeroed`.
        # StateStore's bytes and loose buffers hold every parameter and buffer, i.e. the model's whole state_dict
        self._mutable = [self.state.bytes] + [b for _, b in self.state.loose] + \
            [self.opt.exp_avg, self.opt.exp_avg_sq, self.opt.step_count]
        self._zeroed = []
        snap = torch.empty_like(self.state.bytes)
        self.acc_snap = torch.zeros(self.slots.n, dtype=torch.float64, device=self.device)       # filled by epoch_schedule
        self._handoff = [_Handoff('state', snap, [(snap, self.state.bytes)]), _Handoff('losses', self.acc_snap, [])]
        self.avg_bytes = self.avg = None       # moving average of the fp32 state: a copy of bytes [0, i_off)
        self.avg_seeded = False
        if self.weight_ema is not None:
            self.avg_bytes = self.state.bytes[:self.state.i_off].clone()
            self.avg = self.avg_bytes.view(torch.float32)
            self._mutable.append(self.avg)
            snap = torch.empty_like(self.avg_bytes)     # on the host an image of `bytes`, which averaged_bytes completes
            self._handoff.append(_Handoff('avg', snap, [(snap, self.avg_bytes)], room=self.state.bytes.numel()))
        self.copy_stream = torch.cuda.Stream(device=self.device)
        self._handoff_slots = None
        self._handoff_i = 0
        self._last_done = None
        self._staging = None
        self._staging_i = 0
        self._captured = False
        self.launches_per_step = 0
        self.ema = torch.full((1,), float(example_batch['action'].shape[0] * args.get('forward_steps', 1)) * self.world,
                              dtype=torch.float32, device=self.device)
        self.optim_snap = None           # optimiser state of the epoch hand-off (_optim_views)
        if self.save_optimizer:
            self.optim_snap = self._optim_image(self.device)
            self._handoff.append(_Handoff('optim', self.optim_snap, self._optim_copies(self.optim_snap)))
        # validation sums [live (NUM_LOSS) | averaged (NUM_LOSS)] and the state saved around a pass
        self.val_accum_all = self.val_accum = self.val_ema_accum = self.val_saved = None
        self.val_buf = None
        self.val_graphs = {}
        self.launches_per_validation = 0
        if self.validation:
            self.val_accum_all = torch.zeros(2 * NUM_LOSS, dtype=torch.float64, device=self.device)
            self.val_accum = self.val_accum_all[:NUM_LOSS]
            if self.avg is not None:
                self.val_ema_accum = self.val_accum_all[NUM_LOSS:]
            self._zeroed.append(self.val_accum_all)
            snap = torch.zeros_like(self.val_accum_all)
            self._handoff.append(_Handoff('val', snap, [(snap, self.val_accum_all)], after=self.val_accum_all.zero_))
            self.val_saved = torch.empty_like(self.state.bytes)

        self.layout = BatchLayout(example_batch)
        self.dev_buffer = torch.zeros(self.layout.nbytes, dtype=torch.uint8, device=self.device)
        self.dev = self.layout.views(self.dev_buffer)
        self.h2d_bytes = self.layout.nbytes
        B, T, Pa, A = example_batch['action_mask'].shape
        P = example_batch['turn_mask'].shape[2]
        self.dims = (B, T, P, Pa, A)
        self.prio_state = None
        if self.priority is not None:
            self.prio_state = priority.PriorityState(self.priority, priority.ring_slots(args), B, self.device)
        self.prio_snap = None            # priorities of the epoch hand-off (_prio_views)
        if self.prio_state is not None and self.save_replay:
            self.prio_snap = self._prio_image(self.device)
            self._handoff.append(_Handoff('prio', self.prio_snap, self._prio_copies(self.prio_snap)))
        Bm = B // k                      # windows per micro-batch: what the net and the loss kernel see at once
        # micro-batch i: views of rows [i*Bm, (i+1)*Bm) of every (batch-major) tensor of the packed batch and of the window
        # weights (k = 1: the whole batch); its loss pass writes its sums to row i of loss_rows (the tail's columns, then the
        # zeros of the optimiser's diagnostics entries) and its rows of the advantage tap (_build_loss_buffers)
        self._micro = [tree_map(lambda t, i=i: t[i * Bm:(i + 1) * Bm], self.dev) for i in range(k)]
        self._win_weight = [self.prio_state.win_weight[i * Bm:(i + 1) * Bm] if self.prio_state is not None else None
                            for i in range(k)]
        self.loss_rows = torch.zeros((k, NUM_LOSS + NUM_DISTILL + NUM_DIAG), dtype=torch.float32, device=self.device)
        self.advantage = torch.zeros((B, T, P, 1), dtype=torch.float32, device=self.device) if self.prio_state is not None else None
        self.hidden0 = self.teacher_hidden0 = None
        if hasattr(self.model, 'init_hidden'):
            self.hidden0 = tree_map(lambda h: h.to(self.device), self.model.init_hidden([Bm, P]))
        if self.teacher is not None and hasattr(self.teacher, 'init_hidden'):
            self.teacher_hidden0 = tree_map(lambda h: h.to(self.device), self.teacher.init_hidden([Bm, P]))
        from . import tower
        if fused_tower and small_boards and self.hidden0 is None and tower.supports(self.model) and \
                torch.is_tensor(example_batch['observation']) and example_batch['observation'].shape[-2] * example_batch['observation'].shape[-1] <= 16:
            self.engine = tower.FusedBoardNet(self.model, Bm * T * Pa, self.device, bf16=tensor_cores == 'bf16')
        self.loss_buf = self._loss_bufs = None      # built by the first forward (_build_loss_buffers)
        self.last_losses = torch.zeros(NUM_LOSS, device=self.device)
        self.accum = torch.zeros(self.slots.n, dtype=torch.float64, device=self.device)
        self._mutable.append(self.accum)
        self.loss_accum = self.accum[self.slots.loss]
        self.diag_accum = self.distill_accum = None
        if self.slots.distill is not None:
            self.distill_accum = self.accum[self.slots.distill]
        if diagnostics:
            self.diag_accum = self.accum[self.slots.diag]
            self.opt.diag = self.diag_accum[NUM_LOSS_DIAG:]        # the optimiser's entries: accumulated by its own kernel
        # guard against non-finite steps: the count of rejected steps is the accumulator's last slot; the buffers the forward
        # moves (StateStore bytes [f_off, nbytes)) are saved at the start of every step and put back when it is rejected
        self.skipped = self.guard_saved = None
        if self.skip_nonfinite:
            self.skipped = self.accum[self.slots.skipped]
            self.opt.skip = torch.zeros(1, dtype=torch.int32, device=self.device)
            self.opt.guard_tail = NUM_LOSS
            self._mutable.append(self.opt.skip)
            if self.state.nbytes > self.state.f_off:
                self.guard_saved = torch.empty(self.state.nbytes - self.state.f_off, dtype=torch.uint8, device=self.device)
                self._mutable.append(self.guard_saved)
        self.host_slots = torch.zeros((8, NUM_LOSS)).pin_memory()
        self._slot = 0
        self.graph = self.graph_fwd = self.graph_bwd = None
        self.use_graph = use_graph
        self.steps = 0
        self.stream = torch.cuda.Stream(device=self.device)
        self._warm = PackedBatch(self.layout).fill(example_batch)

    def _probe_outputs(self, example_batch):
        """The net's outputs on one observation (eval mode, no gradient): which heads it has."""
        obs = tree_map(lambda o: o[:1, :1, :1].flatten(0, 2).to(self.device), example_batch['observation'])
        hidden = None
        if hasattr(self.model, 'init_hidden'):
            hidden = tree_map(lambda h: h.to(self.device), self.model.init_hidden([obs_rows(obs)]))
        was_training = self.model.training
        self.model.eval()
        with torch.no_grad():
            outs = self.model(obs, hidden)
        self.model.train(was_training)
        return {k: v for k, v in outs.items() if k != 'hidden' and v is not None}

    def _uses_dense_convs(self, example_batch, model=None):
        """One no-grad probe call of the net (or of `model`, the teacher) on a two-sample slice: do its convolutions take the
        dense small-board path (then activations stay NCHW) or cuDNN (then NHWC, whose implicit-GEMM kernels are the fast
        ones)?"""
        model = self.model if model is None else model
        before = fastnet.BoardConv2d.dense_calls
        obs = tree_map(lambda o: o[:1, :1].flatten(0, 2).to(self.device), example_batch['observation'])
        hidden = None
        if hasattr(model, 'init_hidden'):
            hidden = tree_map(lambda h: h.to(self.device), model.init_hidden([obs_rows(obs)]))
        was_training = model.training
        model.eval()
        with torch.no_grad():
            model(obs, hidden)
        model.train(was_training)
        return fastnet.BoardConv2d.dense_calls > before

    # -- the device work of one step, on the current stream (inputs already in self.dev)
    def _begin_step(self):
        if self.guard_saved is not None:        # one device-to-device copy: what a rejected step puts back
            self.guard_saved.copy_(self._guarded_buffers())
        fastnet.new_step()          # adjoint-weight copies of the previous step are stale: the optimiser has run
        self.opt.zero_grad()

    def _forward(self, dev):
        """The net's raw outputs (B', T, Pa, ...) on the windows of `dev` (the batch, or one micro-batch of it)."""
        if self.engine is not None:
            B, T, Pa = dev['action'].shape[:3]
            flat = self.engine.forward(dev['observation'].flatten(0, 2))
            return {k: v.unflatten(0, (B, T, Pa)) for k, v in flat.items()}
        return forward_raw(self.model, self.hidden0, dev, self.args, self.memory_format)

    def _build_loss_buffers(self, outs):
        """The loss passes' buffers, built on the first forward because the heads come from the net's outputs.  One
        LossBuffers per micro-batch: all share the output gradients and workspaces of B/k windows (the micro-batches run in
        order), and micro-batch i's sums go to row i of loss_rows and its advantage tap to its rows of `advantage`.
        loss_buf is micro-batch 0's; val_buf takes the validation passes' forward-only outputs."""
        B, T, P, Pa, A = self.dims
        Bm = B // self.micro_batches
        value_bins_mod.check_net_heads(self.value_bins, outs)
        heads = ('value' in outs, 'return' in outs)
        base = ops.LossBuffers(Bm, T, P, Pa, A, *heads, self.device, diagnostics=self.diagnostics, value_bins=self.value_bins)
        self._loss_bufs = []
        for i in range(self.micro_batches):
            buf = copy.copy(base)
            buf.losses = self.loss_rows[i, self.slots.loss]
            if self.diagnostics:
                buf.diagnostics = self.loss_rows[i, self.slots.diag]
            if self.advantage is not None:
                buf.advantage = self.advantage[i * Bm:(i + 1) * Bm]
            self._loss_bufs.append(buf)
        self.loss_buf = self._loss_bufs[0]
        if self.validation:
            self.val_buf = ops.LossBuffers(Bm, T, P, Pa, A, *heads, self.device, grads=False, value_bins=self.value_bins)

    def _net_backward(self, outs, buf, accumulate=False):
        """The net's backward from the loss kernel's output gradients in `buf`, into the gradient bucket (added to it when
        `accumulate`; the module path's autograd always adds)."""
        if self.engine is not None:
            self.engine.backward(buf.dpolicy.flatten(0, 2), buf.dvalue.flatten(0, 2),
                                 buf.dreturn.flatten(0, 2) if buf.dreturn is not None else None, accumulate=accumulate)
        else:
            heads, grads = [outs['policy']], [buf.dpolicy]
            for h, g in (('value', buf.dvalue), ('return', buf.dreturn)):
                if h in outs:
                    heads.append(outs[h])
                    grads.append(buf.dlogits[h] if h in buf.value_bins else g)      # a categorical head: its logit gradient
            with ops.deferred_weight_gradients():       # shared (recurrent) convolution weights: one product per weight, at the end
                torch.autograd.backward(heads, grads)

    def _step_parts(self):
        """The device work of one step, on the current stream (inputs already in self.dev): begin, then for each micro-batch
        in order net forward -> fused loss kernel -> net backward into the bucket, then the loss-pass sums into the bucket
        tail and _finish_step.  A generator that pauses once, yielding the last micro-batch's loss kernel launch (a
        callable) for the caller to run: _device_step runs it in place, time_loss_kernel between two graphs."""
        self._begin_step()          # (guard_saved is taken before micro-batch 0: a rejected step restores all k forwards)
        for i, (dev, weight) in enumerate(zip(self._micro, self._win_weight)):
            teacher = self._teacher_policy(dev) if self.teacher is not None else None
            outs = self._forward(dev)
            if self.loss_buf is None:
                self._build_loss_buffers(outs)
            buf = self._loss_bufs[i]
            loss = functools.partial(ops.loss_fwd_bwd, self._loss_heads(outs, buf), dev,
                                     self.args, buffers=buf, diagnostics=self.diagnostics, window_weight=weight)
            if i == len(self._micro) - 1:
                yield loss
            else:
                loss()
            for h, spec in buf.value_bins.items():      # the categorical heads' cross-entropy, from the targets the loss left
                ops.value_bins_fwd_bwd(outs[h].contiguous(), h, spec, dev, self.args, buf, window_weight=weight)
            if teacher is not None:
                ops.distill_fwd_bwd(outs['policy'], teacher, dev, self.args, buf, self.opt.step_count, self.distill['coef'],
                                    self.distill['anneal_steps'], window_weight=weight,
                                    sums=self.loss_rows[i, self.slots.distill])
            self._net_backward(outs, buf, accumulate=i > 0)
            del outs, loss, teacher     # this micro-batch's activations and autograd graph go back to the pool before the next forward
        # the tail (loss sums [+ distillation] [+ the loss pass's diagnostics]) rides the gradient bucket: one row is copied,
        # k rows are summed
        n = self.slots.n_tail
        if self.micro_batches == 1:
            self.opt.extra_slots[:n].copy_(self.loss_rows[0, :n])
        else:
            ops.sum_rows(self.loss_rows, n, self.opt.extra_slots)
        self._finish_step()

    def _loss_heads(self, outs, buf):
        """The heads the fused loss reads: the net's raw outputs, each categorical head replaced by its expectation (one
        ops.value_bins_expect launch per head, into buf.expect)."""
        heads = {k: outs[k] for k in ('policy', 'value', 'return') if k in outs}
        for h, spec in buf.value_bins.items():
            heads[h] = ops.value_bins_expect(outs[h].contiguous(), spec, h, out=buf.expect[h], P=self.dims[2])
        return heads

    def _finish_step(self):
        """The step's tail, once per step: the (all-reduced) bucket -> the optimiser and what follows it."""
        if self.peer is not None:
            reduced = self.peer(self.opt.n_pad, self.opt.partials)      # all-reduce + norm partials, one kernel
            self.opt.step_reduced(reduced)
            tail = reduced[self.opt.n_pad:]
        else:
            if self.world > 1:
                torch.distributed.all_reduce(self.opt.flat_grad, op=torch.distributed.ReduceOp.SUM, group=self.pg)
            self.opt.step()
            tail = self.opt.extra_slots
        self.last_losses.copy_(tail[:NUM_LOSS])
        n = self.slots.n_tail
        if self.skip_nonfinite:         # one launch: accumulate an accepted step, or count a rejected one and restore its buffers
            ops.step_commit(self.opt.skip, tail[:n], self.accum[:n], self.skipped,
                            self._guarded_buffers() if self.guard_saved is not None else None, self.guard_saved)
        else:
            self.accum[:n].add_(tail[:n])
        if self.avg is not None:        # after the optimiser: step_count already counts this step
            ops.weight_ema_update(self.avg, self.state.bytes[:self.state.i_off].view(torch.float32), self.opt.step_count,
                                  self.weight_ema, self.avg_seeded, skip=self.opt.skip)
        if self.prio_state is not None:     # after the optimiser: a rejected step stores no priority
            ops.priority_update(self.prio_state, self.advantage, self.dev['turn_mask'], self.args.get('burn_in_steps', 0),
                                skip=self.opt.skip)

    def _teacher_policy(self, dev):
        """The teacher's raw policy (B', T, Pa, A) on the windows of `dev`: eval mode, no gradient, the module path."""
        before = ops.LAUNCHES['n']
        with torch.no_grad():
            outs = forward_raw(self.teacher, self.teacher_hidden0, dev, self.args, self.teacher_format, train=False)
        self.launches_per_teacher = ops.LAUNCHES['n'] - before
        return outs['policy'].float().contiguous()

    def _guarded_buffers(self):
        """The buffers a step's forward moves (BatchNorm running statistics, num_batches_tracked): StateStore bytes
        [f_off, nbytes)."""
        return self.state.bytes[self.state.f_off:self.state.nbytes]

    def _device_step(self):
        for loss in self._step_parts():
            loss()

    def _device_validate(self, averaged):
        """The device work of one validation pass, on the current stream (inputs already in self.dev)."""
        store = self.state
        self.val_saved.copy_(store.bytes)          # the train-mode forward moves the BatchNorm running statistics
        if averaged:
            store.bytes[:store.i_off].copy_(self.avg_bytes)
        fastnet.new_step()          # the weights differ from those the cached convolution images were packed from
        for dev in self._micro:         # the same micro-batches as the step
            with torch.no_grad():
                outs = self._forward(dev)
            if self.loss_buf is None:
                self._build_loss_buffers(outs)
            sums = ops.loss_fwd(self._loss_heads(outs, self.val_buf), dev, self.args, buffers=self.val_buf)
            for h, spec in self.val_buf.value_bins.items():
                ops.value_bins_fwd_bwd(outs[h].contiguous(), h, spec, dev, self.args, self.val_buf, forward_only=True)
            (self.val_ema_accum if averaged else self.val_accum).add_(sums)
            del outs
        store.bytes.copy_(self.val_saved)

    def _validation_forms(self):
        return [False, True] if self.val_ema_accum is not None else [False]

    def _capture(self):
        # warm-up on the step stream (cuDNN heuristics, lazy inits, NCCL communicator), then capture
        self.stream.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(self.stream):
            self.dev_buffer.copy_(self._warm.buffer, non_blocking=True)
            state = self._snapshot()
            for i in range(3):
                before = ops.LAUNCHES['n']
                self._device_step()
                self.launches_per_step = ops.LAUNCHES['n'] - before      # this library's kernels in one step
            if self.validation:
                for averaged in self._validation_forms():
                    for i in range(2):
                        before = ops.LAUNCHES['n']
                        self._device_validate(averaged)
                        self.launches_per_validation = ops.LAUNCHES['n'] - before
            self.stream.synchronize()
            self._restore(state)
            if self.use_graph and not self.time_loss_kernel:
                self.graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(self.graph, stream=self.stream):
                    self._device_step()
                self._capture_validation(self.graph.pool())
                self._restore(state)
            elif self.use_graph:
                # the (last micro-batch's) loss kernel is launched between two graphs so that CUDA events can bracket it
                parts = self._step_parts()
                self.graph_fwd = torch.cuda.CUDAGraph()
                with torch.cuda.graph(self.graph_fwd, stream=self.stream):
                    self._timed_loss = next(parts)
                self._timed_loss()
                self.graph_bwd = torch.cuda.CUDAGraph()
                with torch.cuda.graph(self.graph_bwd, pool=self.graph_fwd.pool(), stream=self.stream):
                    next(parts, None)
                self._capture_validation(self.graph_fwd.pool())
                self._restore(state)
            self.stream.synchronize()
        self._captured = True

    def _capture_validation(self, pool):
        """One CUDA graph per validation form, after the step graph and in its memory pool: the graphs never run concurrently,
        so the pass reuses the step's activation memory instead of doubling it."""
        if not self.validation:
            return
        for averaged in self._validation_forms():
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, pool=pool, stream=self.stream):
                self._device_validate(averaged)
            self.val_graphs[averaged] = g

    def _snapshot(self):
        return [t.clone() for t in self._mutable]

    def _restore(self, saved):
        """Put back what _snapshot saved, into the same tensors, and zero the sums of the warm-up's validation passes."""
        for t, s in zip(self._mutable, saved):
            t.copy_(s)
        for t in self._zeroed:
            t.zero_()

    def new_packed(self):
        return PackedBatch(self.layout)

    def warm_up(self):
        """Run the warm-up steps and capture the graphs now (otherwise done lazily by the first step)."""
        if not self._captured:
            self._capture()

    def step(self, packed):
        """Enqueue H2D + one learner step for a PackedBatch; returns without waiting for the GPU.
        `packed.in_flight` tells when its host buffer may be refilled."""
        self._enqueue(packed.buffer, packed)

    def step_in_place(self):
        """Same step when the inputs were written directly into self.dev (GPU replay gather) on the step stream."""
        self._enqueue(None, None)

    def step_resident(self, dev_bytes):
        """Same step with the packed batch already in HBM (e.g. produced by the replay gather kernel)."""
        self._enqueue(dev_bytes, None)

    def _enqueue(self, src_bytes, packed):
        if not self._captured:
            self._capture()
        if packed is not None:
            # host batch: the H2D copy runs on the copy stream into one of two staging buffers, i.e. while the previous
            # step still computes; the step stream only waits for it and moves the bytes device-to-device (~1 us)
            if self._staging is None:
                self._staging = [torch.empty_like(self.dev_buffer) for _ in range(2)]
                self._staging_free = [None, None]
            k = self._staging_i % 2
            self._staging_i += 1
            with torch.cuda.stream(self.copy_stream):
                if self._staging_free[k] is not None:
                    self.copy_stream.wait_event(self._staging_free[k])
                self._staging[k].copy_(src_bytes, non_blocking=True)
                arrived = torch.cuda.Event()
                arrived.record(self.copy_stream)
            packed.in_flight = arrived
            with torch.cuda.stream(self.stream):
                self.stream.wait_event(arrived)
                self.dev_buffer.copy_(self._staging[k], non_blocking=True)
                freed = torch.cuda.Event()
                freed.record(self.stream)
                self._staging_free[k] = freed
            src_bytes = None
        with torch.cuda.stream(self.stream):
            if src_bytes is not None:
                self.dev_buffer.copy_(src_bytes, non_blocking=True)
            if not self.use_graph:
                self._device_step()
            elif not self.time_loss_kernel:
                self.graph.replay()
            else:
                self.graph_fwd.replay()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(self.stream)
                self._timed_loss()
                e1.record(self.stream)
                self.kernel_events.append((e0, e1))
                self.graph_bwd.replay()
        self.steps += 1

    def validate_in_place(self, averaged=False):
        """Enqueue one validation pass on the batch in self.dev (written there by GpuBatcher.fill_validation on the step
        stream): the six loss sums of the current weights -- or of their moving average when `averaged` -- are added to
        val_accum (val_ema_accum).  Returns without waiting for the GPU; the learner's state is left as it was.  The first step
        (or warm_up) runs the capture, which uses self.dev: write the batch after it."""
        if not self.validation:
            raise RuntimeError('LearnerStep was built without validation (train_args["validation_rate"] / validation=True)')
        if averaged:
            self._require_average()
        if not self._captured:
            self._capture()
        with torch.cuda.stream(self.stream):
            if self.use_graph:
                self.val_graphs[averaged].replay()
            else:
                self._device_validate(averaged)

    def validation_sums(self, values):
        """{'validation': {LOSS_KEYS: sum}[, 'validation_ema': ...]} of a host list in val_accum_all's layout."""
        out = {'validation': dict(zip(LOSS_KEYS, values[:NUM_LOSS]))}
        if self.val_ema_accum is not None:
            out['validation_ema'] = dict(zip(LOSS_KEYS, values[NUM_LOSS:2 * NUM_LOSS]))
        return out

    def pop_validation(self):
        """Validation sums accumulated since the last call or epoch boundary (one host sync): {'validation': {p, v, r, ent,
        total, dcnt}} and, with a moving average of the weights, 'validation_ema'; divide by dcnt for the printed means."""
        if not self.validation:
            raise RuntimeError('LearnerStep was built without validation (train_args["validation_rate"] / validation=True)')
        self.stream.synchronize()
        vals = self.val_accum_all.cpu().tolist()
        self.val_accum_all.zero_()
        return self.validation_sums(vals)

    def loss_kernel_ms(self):
        """Average device time of the fused loss kernel over the steps since the last call
        (needs time_loss_kernel=True)."""
        self.stream.synchronize()
        ts = [a.elapsed_time(b) for a, b in self.kernel_events]
        self.kernel_events = []
        return sum(ts) / max(1, len(ts)), len(ts)

    def fetch_losses_async(self):
        """Enqueue the D2H copy of the last step's six loss sums (24 bytes) behind that step and
        return a handle; handle() waits for just that copy and returns the dict."""
        slot = self.host_slots[self._slot % self.host_slots.shape[0]]
        self._slot += 1
        with torch.cuda.stream(self.stream):
            slot.copy_(self.last_losses, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self.stream)

        def get():
            ev.synchronize()
            return dict(zip(LOSS_KEYS, slot.tolist()))
        return get

    def read_losses(self):
        """Blocking read of the last step's six loss sums."""
        return self.fetch_losses_async()()

    def pop_accumulated(self):
        """Loss sums accumulated since the last call (ONE host sync per epoch)."""
        self.stream.synchronize()
        vals = self.loss_accum.cpu().tolist()
        self.loss_accum.zero_()
        return dict(zip(LOSS_KEYS, vals))

    def pop_diagnostics(self):
        """Diagnostics sums (ops.DIAG_KEYS -> float) accumulated since the last call or epoch boundary (one host sync);
        ops.summarize_diagnostics turns them into means."""
        if self.diag_accum is None:
            raise RuntimeError('LearnerStep was built without diagnostics (train_args["diagnostics"] / diagnostics=True)')
        self.stream.synchronize()
        vals = self.diag_accum.cpu().tolist()
        self.diag_accum.zero_()
        return dict(zip(DIAG_KEYS, vals))

    def close(self):
        """Release the captured graphs (they pin NCCL kernels: destroy them before the process group)."""
        self.stream.synchronize()
        self.graph = self.graph_fwd = self.graph_bwd = None
        self.val_graphs = {}
        self._timed_loss = None
        self._captured = False
        import gc
        gc.collect()
        torch.cuda.synchronize(self.device)

    def cpu_state_dict(self):
        """Blocking copy of the model's state_dict to the host (tests, checkpoints)."""
        self.stream.synchronize()
        return self._state_dict_of(self.state.bytes.cpu())

    def _state_dict_of(self, host):
        keys = [k for k in self.model.state_dict().keys() if not k.endswith('_sel_cache')]
        out = self.state.state_dict_from(host, keys)
        for k, b in self.state.loose:
            out[k] = b.detach().cpu().clone()
        return {k: out[k] for k in keys}

    def _require_average(self):
        if self.avg is None:
            raise RuntimeError('LearnerStep was built without a weight average (train_args["weight_ema"] / weight_ema=decay)')

    def ema_state_dict(self):
        """Blocking copy of the moving average of the weights to the host, keyed like cpu_state_dict(); the int64 buffers
        and the buffers StateStore keeps outside its allocation are the live model's."""
        self._require_average()
        self.stream.synchronize()
        host_avg = torch.empty_like(self.state.bytes, device='cpu')       # as end_epoch hands it over: an image of `bytes`
        host_avg[:self.state.i_off] = self.avg_bytes.cpu()
        return self._state_dict_of(self.state.averaged_bytes(host_avg, self.state.bytes.cpu()))

    def seed_weight_ema(self, state_dict):
        """Start the average from a saved one (a CPU state_dict keyed like the model's, e.g. a <epoch>.ema.pth file): its fp32
        entries replace the average, and every later step weighs the live weights with 1 - decay.  Call it before the first
        step (or warm_up), which fixes the captured launch."""
        self._require_average()
        if self._captured:
            raise RuntimeError('seed_weight_ema must come before the first step / warm_up()')
        store = self.state
        views = {'p': self.avg[:store.n_pad], 'f': self.avg[store.f_off // 4:]}
        fp32 = [k for k, (tag, _, _) in store.where.items() if tag in views]
        missing = [k for k in fp32 if k not in state_dict]
        if missing:
            raise KeyError('seed_weight_ema: the state_dict lacks %s' % ', '.join(missing))
        with torch.no_grad():
            for k in fp32:
                tag, off, shape = store.where[k]
                src = torch.as_tensor(state_dict[k])
                if tuple(src.shape) != shape:
                    raise ValueError('seed_weight_ema: %s has shape %s, the model %s' % (k, tuple(src.shape), shape))
                n = src.numel()
                views[tag][off:off + n].copy_(src.reshape(-1).to(torch.float32))
        self.avg_seeded = True

    def _optim_views(self, buf):
        """(exp_avg, exp_avg_sq, step_count, lr, ema) views of a byte buffer in the optim_snap layout:
        [exp_avg | exp_avg_sq (n_pad fp32 each) | step_count (int64) | lr | ema (fp32)]."""
        n4 = 4 * self.opt.n_pad
        return (buf[:n4].view(torch.float32), buf[n4:2 * n4].view(torch.float32), buf[2 * n4:2 * n4 + 8].view(torch.int64),
                buf[2 * n4 + 8:2 * n4 + 12].view(torch.float32), buf[2 * n4 + 12:2 * n4 + 16].view(torch.float32))

    def _optim_image(self, device):
        return torch.empty(8 * self.opt.n_pad + 16, dtype=torch.uint8, device=device)

    def _optim_copies(self, image):
        """The (view of image, live tensor) copies that fill a buffer in the optim_snap layout."""
        return list(zip(self._optim_views(image),
                        (self.opt.exp_avg, self.opt.exp_avg_sq, self.opt.step_count, self.opt.lr, self.ema)))

    def optimizer_state_from(self, host_optim, steps):
        """The OptimizerStateFormat dict of a host copy of optim_snap, scheduled at step count `steps`."""
        m, v, sc, lr, ema = self._optim_views(host_optim)
        return self.optim_format.to_dict(m, v, int(sc[0]), float(lr[0]), float(ema[0]), steps)

    def optimizer_state_dict(self):
        """Blocking copy of the optimiser state the next step uses, in the OptimizerStateFormat dict (what end_epoch hands
        over as PendingModel.optim_state)."""
        self.stream.synchronize()
        image = self._optim_image('cpu')
        for dst, src in self._optim_copies(image):
            dst.copy_(src)
        return self.optimizer_state_from(image, self.schedule_steps)

    def load_optimizer_state(self, d):
        """Resume from an OptimizerStateFormat dict (e.g. a <epoch>.optim.pth file): Adam's moments and step count, the
        learning rate and the data-count average.  Call it before the first step (or warm_up), which snapshots the state
        around the capture's warm-up steps.  A dict whose parameter names or shapes differ from the net's, or whose betas,
        eps, weight_decay or max_norm differ from this learner's, or that another optimiser wrote (Adam / LAMB,
        OptimizerStateFormat.check_algorithm), raises KeyError / ValueError and changes nothing."""
        if self._captured:
            raise RuntimeError('load_optimizer_state must come before the first step / warm_up()')
        m, v, step, lr, data_cnt_ema, steps = self.optim_format.unpack(d)
        with torch.no_grad():
            self.opt.exp_avg.copy_(m)
            self.opt.exp_avg_sq.copy_(v)
            self.opt.step_count.fill_(step)
            self.opt.lr.fill_(lr)
            self.ema.fill_(data_cnt_ema)
        self.schedule_steps = steps

    def _prio_views(self, buf):
        """(prio_serial, prio, max_prio) views of a byte buffer in the prio_snap layout:
        [prio_serial (ring int64) | prio (ring fp32) | max_prio (fp32)], padded to 8 bytes."""
        r = self.prio_state.ring
        return buf[:8 * r].view(torch.int64), buf[8 * r:12 * r].view(torch.float32), buf[12 * r:12 * r + 4].view(torch.float32)

    def _prio_image(self, device):
        return torch.empty((12 * self.prio_state.ring + 4 + 7) // 8 * 8, dtype=torch.uint8, device=device)

    def _prio_copies(self, image):
        ps = self.prio_state
        return list(zip(self._prio_views(image), (ps.prio_serial, ps.prio, ps.max_prio)))

    def _require_priorities(self):
        if self.prio_state is None:
            raise RuntimeError('LearnerStep was built without prioritised replay (train_args["prioritized_replay"])')

    def priority_state_from(self, host_prio):
        """{'slot_serial': int64 [ring], 'priority': float32 [ring], 'max_prio': float} of a host copy of prio_snap: per slot of
        the replay directory, the serial of the episode the priority belongs to (-1: none yet) and the priority."""
        serial, prio, mx = self._prio_views(host_prio)
        return {'slot_serial': serial.clone(), 'priority': prio.clone(), 'max_prio': float(mx[0])}

    def priority_state_dict(self):
        """Blocking copy of the priorities as the next batch's sampler finds them (what end_epoch hands over as
        PendingModel.priority_state under save_replay)."""
        self._require_priorities()
        self.stream.synchronize()
        image = self._prio_image('cpu')
        for dst, src in self._prio_copies(image):
            dst.copy_(src)
        return self.priority_state_from(image)

    def load_priority_state(self, slots, serials, priorities, max_prio):
        """Give the episodes in directory slots `slots`, which hold serials `serials`, the priorities `priorities`, and set
        max_prio: ordinary indexed copies on the step stream, outside the captured step.  Every other slot is left alone, so
        its episode starts at max_prio when the sampler first sees it.  The capture's warm-up steps run with serial -1 and
        write no priority, so this may come before or after warm_up(); it must come before the first prioritised batch."""
        self._require_priorities()
        ps = self.prio_state
        idx = torch.as_tensor(np.asarray(slots, np.int64))
        ser = torch.as_tensor(np.asarray(serials, np.int64))
        pri = torch.as_tensor(np.asarray(priorities, np.float32))
        if not (idx.shape == ser.shape == pri.shape and idx.dim() == 1):
            raise ValueError('load_priority_state: slots, serials and priorities must be 1-d and of one length')
        if idx.numel() and (int(idx.min()) < 0 or int(idx.max()) >= ps.ring or idx.unique().numel() != idx.numel()):
            raise ValueError('load_priority_state: slots outside [0, %d) or repeated' % ps.ring)
        if not (np.isfinite(float(max_prio)) and float(max_prio) > 0 and bool(torch.isfinite(pri).all()) and bool((pri > 0).all())):
            raise ValueError('load_priority_state: priorities and max_prio must be finite and positive')
        with torch.cuda.stream(self.stream):
            dev = idx.to(self.device)
            ps.prio.index_copy_(0, dev, pri.to(self.device))
            ps.prio_serial.index_copy_(0, dev, ser.to(self.device))
            ps.max_prio.fill_(float(max_prio))

    def epoch_schedule(self, batch_cnt, steps, default_lr):
        """Device half of the epoch boundary, on the current stream: move the epoch's loss sums aside and apply the
        learning-rate schedule from the (all-reduced, hence global) data count.  Every rank of a sharded learner
        enqueues this at the same step, so all ranks keep identical learning rates without a broadcast."""
        self.acc_snap.copy_(self.accum)
        self.accum.zero_()
        dcnt = self.acc_snap[self.slots.loss][-1:].float()     # dcnt: the last of the loss sums
        fresh = self.ema * 0.8 + dcnt * (0.2 / (1e-2 + batch_cnt))
        self.ema.copy_(torch.where(dcnt > 0, fresh, self.ema))
        self.opt.lr.copy_(self.ema * (default_lr / (1 + steps * 1e-5)))
        self.schedule_steps = int(steps)

    def end_epoch(self, batch_cnt, steps, default_lr, template, heads):
        """Epoch boundary without a host synchronisation (train.py:378-387): on the step stream, snapshot the loss
        sums and the whole model state device-to-device, apply the learning-rate schedule ON THE DEVICE
        (data_cnt_ema <- 0.8 ema + 0.2 dcnt/(0.01+batch_cnt); lr <- 3e-8 ema/(1+steps 1e-5), train.py:382-384 -- dcnt is
        the all-reduced global count) and let a side stream carry the snapshot to pinned host memory while the
        next epoch's steps already run.  Returns a PendingModel (with the moving average of the weights and the optimiser
        state, when they are kept, snapshot and copied the same way; the optimiser state is taken after the schedule, i.e.
        as the next step uses it)."""
        if self._handoff_slots is None:
            self._handoff_slots = [{e.name: torch.empty(e.room or e.snap.numel(), dtype=e.snap.dtype).pin_memory()
                                    for e in self._handoff} for _ in range(2)]
        host = self._handoff_slots[self._handoff_i % 2]
        self._handoff_i += 1
        with torch.cuda.stream(self.stream):
            self.epoch_schedule(batch_cnt, steps, default_lr)
            if self._last_done is not None:
                self.stream.wait_event(self._last_done)          # the previous snapshot has left the device buffer
            for e in self._handoff:
                for dst, src in e.copies:
                    dst.copy_(src)
                if e.after:
                    e.after()
            ready = torch.cuda.Event()
            ready.record(self.stream)
        with torch.cuda.stream(self.copy_stream):
            self.copy_stream.wait_event(ready)
            for e in self._handoff:
                host[e.name][:e.snap.numel()].copy_(e.snap, non_blocking=True)
            done = torch.cuda.Event()
            done.record(self.copy_stream)
        self._last_done = done
        return PendingModel(self, done, host['state'], host['losses'], heads, template, host=host, steps=int(steps),
                            diagnostics=self.diagnostics, skip_nonfinite=self.skip_nonfinite, batch_cnt=batch_cnt,
                            distill=self.teacher is not None)


# --------------------------------------------------------------------------- batcher + trainer

class _FlatCache:
    """Decoded episodes for the host batcher, least-recently-used first, bounded in bytes (the reference keeps only
    the bz2 blocks, train.py:54; an unbounded cache of decoded arrays would grow to tens of GB at
    maximum_episodes = 100000 and trip the Learner's memory guard)."""

    def __init__(self, budget_bytes):
        self.budget, self.used = int(budget_bytes), 0
        self.items = collections.OrderedDict()       # id(episode) -> (episode, FlatEpisode, bytes)
        self.lock = threading.Lock()

    @staticmethod
    def _size(fe):
        return sum(a.nbytes for a in tree_leaves(fe.obs)) + fe.amask.nbytes + fe.value.nbytes + 24 * fe.prob.size

    def get(self, ep):
        from .wire import episode_to_flat
        key = id(ep)
        with self.lock:
            hit = self.items.get(key)
            if hit is not None and hit[0] is ep:
                self.items.move_to_end(key)
                return hit[1]
        fe = episode_to_flat(ep)          # flat wire format if the worker sent it, else decode the moments
        size = self._size(fe)
        with self.lock:
            self.items[key] = (ep, fe, size)
            self.used += size
            while self.used > self.budget and len(self.items) > 1:
                _, (_, _, sz) = self.items.popitem(last=False)
                self.used -= sz
        return fe


class Batcher:
    """Feeds the trainer: recency-biased window sampling (train.py:291-315) and collation.

    Unlike the reference there is no process pool shipping pickled batches through pipes
    (train.py:274, connection.py:133-173): episodes are decoded once into FlatEpisode arrays
    (a byte-bounded LRU cache) and batches are built by `num_batchers` threads with numpy
    gathers that release the GIL.
    """

    def __init__(self, args, episodes):
        self.args = args
        self.episodes = episodes
        self.out = queue.Queue(maxsize=8)
        self.threads = []
        self.started = False
        self.stop_event = threading.Event()
        self.cache = _FlatCache(args.get('host_cache_bytes', 2 << 30))

    def _fetch(self, idx):
        ep = self.episodes[idx]           # ONE read: the deque may shift under us (train.py:298-302)
        return ep['steps'], ep

    def select_episode(self):
        idx, st, ed, tst, ep = sample_window(lambda: len(self.episodes), self._fetch, self.args)
        cs = self.args['compress_steps']
        b0, b1 = st // cs, (ed - 1) // cs + 1
        return {'args': ep['args'], 'outcome': ep['outcome'], 'moment': ep['moment'][b0:b1], 'base': b0 * cs,
                'start': st, 'end': ed, 'train_start': tst, 'total': ep['steps'], '_episode': ep}

    def _make(self):
        windows = []
        for _ in range(self.args['batch_size']):
            sel = self.select_episode()
            fe = self.cache.get(sel['_episode'])
            windows.append((fe, sel['start'], sel['end'], sel['start'], sel['train_start'], sel['total']))
        nb = gather_windows(windows, self.args)
        return tree_map(lambda a: torch.from_numpy(a), nb)

    def _worker(self, bid):
        print('started batcher %d' % bid)
        while not self.stop_event.is_set():
            try:
                item = self._make()
            except Exception:              # a batcher thread must never die silently: Batcher.batch() would spin forever
                traceback.print_exc()
                time.sleep(0.05)
                continue
            while not self.stop_event.is_set():
                try:
                    self.out.put(item, timeout=0.2)
                    break
                except queue.Full:
                    continue
        print('finished batcher %d' % bid)

    def run(self):
        if self.started:
            return
        self.started = True
        for i in range(self.args['num_batchers']):
            th = threading.Thread(target=self._worker, args=(i,), daemon=True)
            th.start()
            self.threads.append(th)

    def batch(self):
        while True:
            try:
                return self.out.get(timeout=0.2)
            except queue.Empty:
                if self.stop_event.is_set():
                    return None

    def stop(self):
        self.stop_event.set()
        for th in self.threads:
            th.join(timeout=5)


class EpisodeDeque(deque):
    """The `Trainer.episodes` deque the Learner appends to (train.py:472, 482-483), with a tap: every appended
    episode is also handed to a listener (the GPU replay feeder) exactly once."""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.listener = None

    def append(self, ep):
        super().append(ep)
        if self.listener is not None:
            self.listener(ep)

    def extend(self, eps):
        for ep in eps:
            self.append(ep)


def sample_batch(replay, B, args, rng, sym_rng=None, K=0):
    """The draws of one GPU-replay batch: B window descriptors from `rng` (DeviceReplay.sample_windows) and, with sym_rng,
    the transform of each window, uniform in [0, K), from that generator alone -- so the descriptors are the same with and
    without augmentation.  Returns (windows, transforms or None); the transforms are checked here, on the host, because
    the gather kernel trusts them."""
    win = replay.sample_windows(B, args, rng)
    if sym_rng is None:
        return win, None
    sym = symmetry.draw(sym_rng, B, K)
    if sym.size and (sym.min() < 0 or sym.max() >= K):
        raise ValueError('sample_batch: transform outside [0, %d)' % K)
    return win, sym


class GpuBatcher:
    """Batcher on the GPU-resident replay (replay.py + the gather/pad kernel): arriving episodes are decoded once
    by a feeder thread and uploaded into the device ring; a batch is B window descriptors (drawn with array
    operations, same sampling law as Batcher.select_episode) + ONE kernel that writes straight into the learner
    step's input buffer.

    Feeder and learner never wait for each other's GPU work on the host: the upload stream waits (on the device) for
    the last gather that may read rows it overwrites, the step stream waits for the last upload; the only shared
    host lock covers "sample + enqueue gather" on one side and "update directory + enqueue copies" on the other
    (microseconds each: staging into pinned memory happens outside it).

    With train_args['validation_rate'] = r, the episodes replay.held_out() picks (a fraction r, decided from their content)
    never enter the training ring: they go to a second DeviceReplay, `val_replay`, of r times the ring's steps and
    r * maximum_episodes episodes, that fill_validation() samples from -- or, with keep_validation=False (helper ranks, which
    do not validate), nowhere.

    With train_args['symmetry'] set (symmetry.py), fill() gathers every window through a transform drawn uniformly from the
    group by its own generator (symmetry.sampler_rng(seed)): the window descriptors are those drawn without the key.  The
    tables are built once from the first episode's leaf shapes and uploaded once; the transforms ride in the pinned
    descriptor slot behind the descriptors, in the same copy.  fill_validation() never augments.

    With train_args['prioritized_replay'] set (priority.py), fill() draws the windows on the device instead: the replay keeps a
    device mirror of its directory, and hrl_replay_sample reads it with the stepper's priority state (LearnerStep.prio_state)
    and writes the descriptors and the importance weights straight into the buffers the gather and the step read.  The host
    only snapshots (head, count) under the locks, as it does to sample; the Philox key comes from the seed
    (priority.sampler_key) and the counter is the number of batches drawn.  Symmetry transforms are still drawn on the host.
    fill_validation() keeps the host sampler.

    With train_args['value_bins'] listing the value head (value_bins.py), the feeder reduces each arriving episode's stored
    K-vector values (the categorical head's logits) to their expectation before staging, so the ring keeps one value per
    player.

    With a `limiter` (a ReplayRatioLimiter, train_args['replay_ratio']), the feeder adds the steps of the episodes it committed
    to the training ring after each commit; held-out episodes add nothing.

    With train_args['save_replay'] set (or track_resident=True), both rings keep the episodes they hold as they arrived
    (DeviceReplay.resident, references only) and snapshot() returns them with the sampler's state; restore_sampler() puts that
    state back.  `restore`: the dict of a replay file whose episodes are this batcher's backlog; the ring is then sized to hold
    at least the file's capacity_steps where memory allows."""

    DESC_SLOTS = 4        # pinned descriptor buffers in rotation: bounds how far the host runs ahead of the GPU

    def __init__(self, args, episodes, device, seed=None, forward=None, keep_validation=True, limiter=None,
                 track_resident=None, restore=None):
        from .replay import DeviceReplay
        from .wire import episode_to_flat
        self.args = args
        self.validation = validation_rate(args)
        self.device = device
        self.forward = forward              # multi-GPU: callable(list of episodes) that ships them to the other ranks
        self.limiter = limiter
        self.pending = queue.Queue()
        self.upload_stream = torch.cuda.Stream(device=device)
        self.last_upload = None
        self.last_gather = None
        self.order_lock = threading.Lock()
        self.stop_event = threading.Event()
        seed = seed if seed is not None else args.get('seed', 0) * 7919 + 17
        self.rng = np.random.default_rng(seed)
        self.val_rng = np.random.default_rng(seed + 1)      # validation draws leave the training stream alone
        self.symmetry = symmetry.config(args)
        self.sym_rng = symmetry.sampler_rng(seed) if self.symmetry is not None else None
        self.sym_tables = None
        self.priority = priority.config(args)
        self.value_bins = value_bins_mod.config(args)
        self.prio_key = priority.sampler_key(seed)
        self.prio_batches = 0               # the Philox counter of the next prioritised batch
        self.fed = 0
        self._slots = None
        self._slot_i = 0
        self.track_resident = bool(_save_replay_spec(args) is not None if track_resident is None else track_resident)
        self._arrivals = 0                  # episodes the feeder has split so far: orders the two rings' episodes in a snapshot

        # tap first, then the backlog: nothing is missed; what the tap saw meanwhile is not enqueued twice, and the
        # backlog keeps its (recency) order ahead of it
        tapped, tap_lock = [], threading.Lock()

        def tap(ep):
            with tap_lock:
                if tapped is not None and self._backlog_open:
                    tapped.append(ep)
                    return
            self.pending.put(ep)

        self._backlog_open = True
        episodes.listener = tap
        backlog = list(episodes)
        with tap_lock:
            seen = {id(e) for e in tapped}
            backlog = [e for e in backlog if id(e) not in seen] + tapped
            self._backlog_open = False
        for ep in backlog:
            self.pending.put(ep)
        self.backlog_n = len(backlog)

        # ring capacity from the observed episode lengths and the free HBM (the reference bounds episodes, not steps)
        fe0 = episode_to_flat(backlog[0]) if backlog else None
        if self.symmetry is not None and fe0 is not None:      # malformed tables raise here, before any upload
            self.sym_tables = symmetry.build_tables(self.symmetry, [l.shape[2:] for l in tree_leaves(fe0.obs)],
                                                    fe0.amask.shape[-1])
        cap = int(args.get('replay_capacity_steps', 0))
        lens = [e['steps'] for e in backlog] or [64]
        mean_len, max_len = sum(lens) / len(lens), max(lens)
        if not cap:
            want = int(args['maximum_episodes'] * mean_len * 1.25) + 4 * max_len
            budget = want
            if fe0 is not None and torch.device(device).type == 'cuda':
                free, _ = torch.cuda.mem_get_info(device)
                budget = int(args.get('replay_memory_fraction', 0.5) * free / DeviceReplay.bytes_per_step(fe0))
            cap = max(4 * max_len, min(want, budget))
            est = int(cap / max(mean_len, 1))
            if est < args['maximum_episodes']:
                print('handyrl_b200: the GPU replay holds about %d episodes (%d steps), fewer than maximum_episodes=%d'
                      % (est, cap, args['maximum_episodes']))
        saved = int(restore['capacity_steps']) if restore is not None else 0
        if saved > cap:                     # a restored backlog filled a ring of `saved` steps: hold all of it where memory allows
            room = saved
            if fe0 is not None and torch.device(device).type == 'cuda':
                free, _ = torch.cuda.mem_get_info(device)
                room = int(args.get('replay_memory_fraction', 0.5) * free / DeviceReplay.bytes_per_step(fe0))
            if room < saved:
                print('handyrl_b200: the GPU replay holds about %d episodes (%d steps), fewer than maximum_episodes=%d'
                      % (int(max(cap, room) / max(mean_len, 1)), max(cap, room), args['maximum_episodes']))
            cap = max(cap, min(saved, room))
        self.replay = DeviceReplay(cap, args['maximum_episodes'], device=device, mirror=self.priority is not None,
                                   track=self.track_resident)
        self.val_replay = None
        if self.validation is not None and keep_validation:
            r = self.validation
            self.val_replay = DeviceReplay(max(int(r * cap), 2 * max_len), max(1, int(round(r * args['maximum_episodes']))),
                                           device=device, track=self.track_resident)
        self.thread = threading.Thread(target=self._feed, daemon=True)

    def run(self):
        if not self.thread.is_alive():
            self.thread.start()

    def _feed(self):
        from .replay import held_out
        from .wire import episode_to_flat
        while not self.stop_event.is_set():
            try:
                eps = [self.pending.get(timeout=0.2)]
            except queue.Empty:
                continue
            while len(eps) < 256:            # everything that has queued up goes in one upload
                try:
                    eps.append(self.pending.get_nowait())
                except queue.Empty:
                    break
            try:
                if self.forward is not None:
                    self.forward(eps)
                fes = [reduce_values(episode_to_flat(ep), self.value_bins) for ep in eps]
                held = [held_out(fe, self.validation) for fe in fes]
                train = [fe for fe, h in zip(fes, held) if not h]
                val = [fe for fe, h in zip(fes, held) if h] if self.val_replay is not None else []
                items = val_items = ()      # without resident lists the rings are staged exactly as before
                if self.track_resident:     # (arrival number, the episode as it arrived) rides with each directory entry
                    tagged = list(zip(range(self._arrivals, self._arrivals + len(eps)), eps))
                    self._arrivals += len(eps)
                    items = ([it for it, h in zip(tagged, held) if not h],)
                    val_items = ([it for it, h in zip(tagged, held) if h],)
                staged = self.replay.stage(train, *items) if train else None
                val_staged = self.val_replay.stage(val, *val_items) if val else None
                with self.order_lock:
                    if self.last_gather is not None:   # device-side: never overwrite rows an enqueued gather reads
                        self.upload_stream.wait_event(self.last_gather)
                    with torch.cuda.stream(self.upload_stream):
                        if staged is not None:
                            self.replay.commit(staged)
                        if val_staged is not None:
                            self.val_replay.commit(val_staged)
                        ev = torch.cuda.Event()
                        ev.record(self.upload_stream)
                        self.last_upload = ev
                if self.limiter is not None and train:       # before `fed` moves: a ready() replay has its credit
                    self.limiter.store(sum(fe.steps for fe in train))
            except Exception:
                traceback.print_exc()
            self.fed += len(eps)

    def snapshot(self):
        """What a replay file stores of this batcher, as of one instant (taken under the lock that orders sampling and
        uploads): {'episodes': the episodes resident in the training and held-out rings, oldest arrival first, as they arrived;
        'serials': int64 tensor, the training ring's serial of each, -1 for a held-out one; 'capacity_steps';
        'maximum_episodes'; 'sampler': {'rng', 'val_rng', 'sym_rng' (None without symmetry): bit_generator.state dicts,
        'prio_batches': the Philox counter of the next prioritised batch}}.  References and small arrays only."""
        if not self.track_resident:
            raise RuntimeError("GpuBatcher keeps no resident lists (train_args['save_replay'] / track_resident=True)")
        with self.order_lock:
            with self.replay.lock:
                items = list(self.replay.resident)
                serials = self.replay.positions()[1]
            val_items = []
            if self.val_replay is not None:
                with self.val_replay.lock:
                    val_items = list(self.val_replay.resident)
            sampler = {'rng': copy.deepcopy(self.rng.bit_generator.state),
                       'val_rng': copy.deepcopy(self.val_rng.bit_generator.state),
                       'sym_rng': copy.deepcopy(self.sym_rng.bit_generator.state) if self.sym_rng is not None else None,
                       'prio_batches': int(self.prio_batches)}
        if val_items:                       # two runs sorted by arrival: one stable merge
            serials = np.concatenate([serials, np.full(len(val_items), -1, np.int64)])
            items = items + val_items
            order = np.argsort(np.fromiter((a for a, _ in items), np.int64, len(items)), kind='stable')
            items, serials = [items[i] for i in order], serials[order]
        return {'episodes': [ep for _, ep in items], 'serials': torch.from_numpy(np.ascontiguousarray(serials)),
                'capacity_steps': int(self.replay.capacity), 'maximum_episodes': int(self.args['maximum_episodes']),
                'sampler': sampler}

    def restore_sampler(self, sampler):
        """Put back the sampler state of a snapshot(): the generators of the training, validation and transform draws and the
        prioritised sampler's batch counter.  A generator the snapshot lacks (symmetry was off) keeps its seed."""
        with self.order_lock:
            for name in ('rng', 'val_rng', 'sym_rng'):
                gen, state = getattr(self, name), sampler.get(name)
                if gen is not None and state is not None:
                    gen.bit_generator.state = state
            self.prio_batches = int(sampler['prio_batches'])

    def ready(self):
        """True once the whole backlog the trainer started with is resident (the reference samples from at least
        `minimum_episodes` episodes from its first step on)."""
        return self.fed >= self.backlog_n and len(self.replay) > 0

    def _descriptor_slot(self, B):
        from .replay import WINDOW_DTYPE
        if self._slots is None:
            nb = B * WINDOW_DTYPE.itemsize
            if self.symmetry is None:
                self._slots = [{'host': torch.empty(nb, dtype=torch.uint8).pin_memory(),
                                'dev': torch.empty((B, WINDOW_DTYPE.itemsize), dtype=torch.uint8, device=self.device),
                                'event': None} for _ in range(self.DESC_SLOTS)]
            else:       # descriptors, then B int32 transforms: one buffer, one copy
                self._slots = []
                for _ in range(self.DESC_SLOTS):
                    host = torch.empty(nb + 4 * B, dtype=torch.uint8).pin_memory()
                    dev = torch.empty(nb + 4 * B, dtype=torch.uint8, device=self.device)
                    self._slots.append({'host': host, 'host_sym': host[nb:].view(torch.int32),
                                        'dev': dev[:nb].view(B, WINDOW_DTYPE.itemsize), 'dev_all': dev,
                                        'sym': dev[nb:].view(torch.int32), 'event': None})
        slot = self._slots[self._slot_i % self.DESC_SLOTS]
        self._slot_i += 1
        if slot['event'] is not None:
            slot['event'].synchronize()      # the gather that read this slot DESC_SLOTS steps ago
        return slot

    def validation_ready(self):
        """True once the held-out ring holds an episode."""
        return self.val_replay is not None and len(self.val_replay) > 0

    def fill(self, stepper):
        """Sample a batch and gather it into stepper.dev (on the step stream); augmented under train_args['symmetry'], drawn by
        the device sampler under train_args['prioritized_replay']."""
        self._fill(stepper, self.replay, self.rng, self.symmetry is not None, self.priority is not None)

    def fill_validation(self, stepper):
        """Sample a batch of held-out windows (the same sampling law) and gather it into stepper.dev (on the step stream), for
        LearnerStep.validate_in_place.  Never augmented: validation measures the real data."""
        self._fill(stepper, self.val_replay, self.val_rng, False)

    def _tables(self):
        if self.sym_tables is None:         # no backlog at construction: the first stored episode fixes the shapes
            self.sym_tables = symmetry.build_tables(self.symmetry, self.replay.leaf_shapes, self.replay.A)
        return self.sym_tables

    def _fill(self, stepper, replay, rng, augment, prioritized=False):
        B = stepper.dims[0]
        if prioritized and stepper.prio_state is None:
            raise ValueError("GpuBatcher: train_args['prioritized_replay'] needs a LearnerStep built with the key")
        slot = self._descriptor_slot(B)
        with self.order_lock:
            if prioritized:         # the device draws the windows: the host takes the directory snapshot only
                with replay.lock:
                    head, count = replay.snapshot(self.args['maximum_episodes'])
                if count <= 0:
                    raise IndexError('the replay is empty')
                sym = None
                if augment:
                    K = self._tables().K
                    sym = symmetry.draw(self.sym_rng, B, K)
                    self._tables().check_sym(sym)
            else:
                win, sym = sample_batch(replay, B, self.args, rng, self.sym_rng if augment else None,
                                        self._tables().K if augment else 0)
                slot['host'][:win.nbytes].numpy()[:] = win.view(np.uint8)
            if sym is not None:
                slot['host_sym'].numpy()[:] = sym
            with torch.cuda.stream(stepper.stream):
                if self.last_upload is not None:
                    stepper.stream.wait_event(self.last_upload)
                if not prioritized:
                    slot.get('dev_all', slot['dev']).view(-1).copy_(slot['host'], non_blocking=True)
                else:
                    if sym is not None:
                        slot['sym'].copy_(slot['host_sym'], non_blocking=True)
                    ops.replay_sample(stepper.prio_state, replay, head, count, self.args, slot['dev'], self.prio_key,
                                      self.prio_batches, solo=not self.args['turn_based_training'])
                    self.prio_batches += 1
                out = dict(stepper.dev)
                single_leaf = torch.is_tensor(stepper.dev['observation'])
                if single_leaf:
                    out['observation'] = stepper.dev['observation'].view(*stepper.dev['observation'].shape[:3], -1)
                else:
                    out['observation'] = self._flat_obs(stepper)
                out['value'] = self._value_sink(stepper)
                if sym is not None:
                    replay.gather(slot['dev'], self.args, out=out, sym=slot['sym'], tables=self.sym_tables)
                else:
                    replay.gather(slot['dev'], self.args, out=out)
                if not single_leaf:
                    nested = replay.split_observation(out['observation'])
                    for d, s_ in zip(tree_leaves(stepper.dev['observation']), tree_leaves(nested)):
                        d.copy_(s_)
                ev = torch.cuda.Event()
                ev.record(stepper.stream)
                self.last_gather = ev
                slot['event'] = ev

    def _flat_obs(self, stepper):
        if not hasattr(self, '_obs_buf'):
            B, T, Pa = stepper.dev['action'].shape[:3]
            self._obs_buf = torch.empty((B, T, Pa, self.replay.OE), device=self.device)   # both rings hold one kind of episode
        return self._obs_buf

    def _value_sink(self, stepper):
        if not hasattr(self, '_val_buf'):
            B, T, P = stepper.dev['turn_mask'].shape[:3]
            self._val_buf = torch.empty((B, T, P, 1), device=self.device)    # behaviour value: unused by the loss
        return self._val_buf

    def stop(self):
        self.stop_event.set()
        if self.thread.is_alive():
            self.thread.join(timeout=5)


def restore_priorities(stepper, batcher, d):
    """Give the episodes of the replay file dict `d` that are resident in `batcher` (a GpuBatcher fed the very objects of
    d['episodes']) their saved priorities in `stepper`, and set max_prio.  An episode is found by its object, since the
    restored ring hands out new slots and serials.  Returns how many got one (0 when either side has no priorities)."""
    if d['priorities'] is None or stepper.prio_state is None:
        return 0
    index = {id(ep): i for i, ep in enumerate(d['episodes'])}
    with batcher.replay.lock:
        items = list(batcher.replay.resident)
        slots, serials = batcher.replay.positions()
    positions = np.fromiter((index.get(id(ep), -1) for _, ep in items), np.int64, len(items))
    saved = {k: np.asarray(d['priorities'][k]) for k in ('serial', 'priority')}
    slots, serials, prio = priority.restore_entries(saved, np.asarray(d['serials']), positions, slots, serials)
    stepper.load_priority_state(slots, serials, prio, d['priorities']['max_prio'])
    return len(slots)


class Trainer:
    """Drop-in for handyrl.train.Trainer (train.py:321-400): same constructor, attributes
    (`episodes`, `steps`), `run()` thread body and `update()` hand-off, same printed lines.

    Multi-GPU (the reference wraps its model in nn.DataParallel when it sees several GPUs, train.py:325, 339-340):
    with train_args['num_gpus'] > 1 (default: every visible GPU, as the reference) this process is rank 0 and spawns
    one helper process per further GPU (multigpu.py); every rank holds the whole replay, samples batch_size/num_gpus
    windows per step and the gradient bucket is all-reduced (SUM) inside the captured step.

    train_args['weight_ema'] = d in (0, 1): the learner also keeps a moving average of the weights (LearnerStep), and
    update() writes it to models/<epoch>.ema.pth and models/latest.ema.pth (AveragedCheckpoints) beside the Learner's
    checkpoints; a run restarted at restart_epoch resumes from models/<restart_epoch>.ema.pth when that file exists.  The
    returned model is the live one either way.

    train_args['save_optimizer'] = True: update() also writes the optimiser state and learning-rate schedule the next step
    uses to models/<epoch>.optim.pth and models/latest.optim.pth (OptimizerStateFormat), numbered by the same
    AveragedCheckpoints as the averages; a run restarted at restart_epoch resumes Adam's moments and step count, the
    learning rate, the data-count average and `steps` from models/<restart_epoch>.optim.pth when that file exists.

    train_args['validation_rate'] = r in (0, 1): a fraction r of the episodes (replay.held_out) is held out of training, and
    after every round(1 / r)-th step one batch of held-out windows is evaluated with the live weights (and with their moving
    average under weight_ema) without an update (LearnerStep.validate_in_place).  Each epoch prints 'validation = ...' (and
    'validation_ema = ...') after the loss line, in its format, once the held-out ring holds an episode.  Only rank 0
    validates; every rank leaves the held-out episodes out of its training ring.

    train_args['skip_nonfinite'] = True: a step whose loss or gradient is not finite (a NaN or Inf from an environment's
    observation, reward or outcome) is rejected on the device and leaves the learner as it was (LearnerStep).  Each epoch
    that rejected a step prints 'skipped = <n> of <steps> steps: non-finite loss or gradient' after the loss (and
    diagnostics) line, even when update() drops the epoch.  `steps` keeps counting batches drawn.  Every rank sees the same
    all-reduced bucket, so all ranks reject alike.

    train_args['symmetry'] = {'group': ..., 'board': [H, W]} or {'tables': 'module:function'} (symmetry.py): every training
    window is gathered through a board transform drawn uniformly per window (GpuBatcher); the printed lines, the step and
    the validation batches are unchanged.  Needs gpu_replay.

    train_args['prioritized_replay'] = True or {'alpha': a, 'beta': b, 'epsilon': e} (priority.py): training windows are drawn
    on the device with probability proportional to the recency law times a per-episode priority from the fused loss's
    advantages, and weighted to correct the bias (LearnerStep, GpuBatcher).  The printed lines keep their format; the loss
    line reports the weighted objective.  Validation batches use the host sampler and no weights.  Each rank keeps the
    priorities of its own shard.  Priorities are saved with the replay under save_replay; without it every episode starts at
    max_prio after a restart.  Needs gpu_replay.

    train_args['replay_ratio'] = r > 0: before each batch (each chunk with several GPUs) the trainer thread waits until the
    samples trained since this Trainer started, that batch included, are at most r times the steps stored in the training
    replay since then (ReplayRatioLimiter; the backlog counts, held-out episodes and validation batches do not).  So that
    update() cannot deadlock the Learner, an epoch that has not taken a step yet when update() waits lets one step (chunk)
    through: each epoch exceeds the limit by at most that.  Each epoch prints 'replay_ratio = <ratio> limit:<r>
    waited:<fraction>' after the loss, diagnostics and skipped lines; replay_ratio_stats() returns the counts.

    train_args['save_replay'] = True, n or {'every': n, 'keep': k}: with every n-th numbered epoch, update() hands the episodes
    resident in the GPU replay (training and held-out rings), the sampler's random state, the priorities and the limiter's
    counts -- all as of the epoch boundary the checkpoint's weights belong to -- to a writer thread that writes
    models/<epoch>.replay.pth (replay_file, ReplayCheckpoints; numbered like .ema.pth and .optim.pth) and keeps the newest k
    files this run wrote.  A run restarted at restart_epoch with models/<restart_epoch>.replay.pth present starts with those
    episodes in `episodes`, trains at once, and restores the sampler state and priorities before its first batch; it prints
    'restored replay: <n> episodes (<m> held out), <s> steps, priorities: <yes|no>'.  Needs gpu_replay.

    train_args['gradient_accumulation'] = k: each batch of batch_size windows is trained as k micro-batches of batch_size / k
    with one optimiser step (LearnerStep), so the net's activations take 1/k of the memory.  k must divide batch_size
    (ValueError otherwise); with several GPUs each rank runs k micro-batches of its batch_size / num_gpus windows, and when
    batch_size % (num_gpus * k) != 0 the trainer prints one line and uses one GPU.  Steps, the learning-rate law and the
    printed lines are unchanged; BatchNorm normalises each micro-batch with its own statistics.

    train_args['distill'] = {'teacher': path, 'net': 'module:function', 'coef': c0, 'anneal_steps': N} (distill.py): the
    teacher is built and loaded here (ValueError for a bad key, file or net), and every step adds the annealed term
    c_n * KL(teacher || student) on the trained policy rows (LearnerStep).  Each epoch prints 'distill = kl:<kl> term:<c_n kl>'
    (both over dcnt) after the loss and diagnostics lines.  Helper ranks build their teacher from the same key.

    train_args['optimizer'] = 'lamb' or {'name': 'lamb', 'lr_scale': s} (optimizer_config; ValueError for anything but these,
    'adam' and None): every rank's LearnerStep runs clip + LAMB instead of clip + Adam on the same all-reduced bucket, with
    the learning rate of the same schedule times s.  The .optim.pth files carry 'algorithm': 'lamb', and a restart refuses a
    file the other optimiser wrote.

    train_args['value_bins'] = {'value': {'bins': K, 'low': lo, 'high': hi, 'symlog': bool, 'sigma': s}, 'return': {...}}
    (value_bins.py; ValueError here for a malformed key): the listed heads output K logits and train by cross-entropy against
    two-hot (sigma 0) or HL-Gauss targets (LearnerStep).  The GPU replay reduces the K logits the workers stored as each
    moment's value to their expectation when the episode arrives, so the replay and its files hold one value per player as
    before.  The epoch line's v: / r: is then the mean cross-entropy per dcnt."""

    def __init__(self, args, model):
        self.optimizer = optimizer_config(args.get('optimizer'))
        ratio = replay_ratio(args)
        self.micro_batches = gradient_accumulation(args)
        if args['batch_size'] % self.micro_batches:
            raise ValueError("train_args['gradient_accumulation'] = %d does not divide batch_size = %d"
                             % (self.micro_batches, args['batch_size']))
        self.save_replay = save_replay(args)
        self.weight_ema = weight_ema_decay(args.get('weight_ema'))
        self.validation = validation_rate(args)
        self.symmetry = symmetry.config(args)
        self.priority = priority.config(args)
        self.distill = distill_mod.config(args)
        self.value_bins = value_bins_mod.config(args)      # malformed train_args['value_bins'] fails here
        # the teacher of train_args['distill'], built now (a deep copy of the net as received, before the learner rewrites it)
        self.teacher = distill_mod.teacher_net(self.distill, model) if self.distill is not None else None
        self.validate_every = max(1, int(round(1.0 / self.validation))) if self.validation is not None else 0
        self.save_optimizer = bool(args.get('save_optimizer', False))
        self.checkpoint_files = None         # numbers the .ema.pth and .optim.pth files of one epoch alike
        if self.weight_ema is not None or self.save_optimizer or self.save_replay is not None:
            self.checkpoint_files = AveragedCheckpoints(args.get('restart_epoch', 0))
        self.ema_files = self.checkpoint_files if self.weight_ema is not None else None
        self.optim_files = self.checkpoint_files if self.save_optimizer else None
        self.episodes = EpisodeDeque()
        self.args = args
        self.model = model
        self.gpu_replay = bool(args.get('gpu_replay', True))
        self.gpu_batcher = None
        self.default_lr = 3e-8
        self.data_cnt_ema = self.args['batch_size'] * self.args['forward_steps']
        self.limiter = None
        self.replay_ratio_epoch = None       # the figures of the last epoch update() handed over
        if ratio is not None:
            self.limiter = ReplayRatioLimiter(ratio, self.data_cnt_ema)
            if not self.gpu_replay:          # the host batcher samples this deque: what it appends is stored
                self.episodes.listener = lambda ep: self.limiter.store(ep['steps'])
        self.params = list(self.model.parameters())
        self.lr = self.default_lr * self.data_cnt_ema
        self.steps = 0
        self.batcher = Batcher(self.args, self.episodes)
        self.update_flag = False
        self.update_queue = queue.Queue(maxsize=1)
        self.stepper = None
        self.fleet = None
        self.stop_event = threading.Event()
        if len(self.params) > 0 and not torch.cuda.is_available():
            raise RuntimeError('handyrl_b200.Trainer needs a CUDA device; there is no CPU learner in this package')
        self.world = 1
        if len(self.params) > 0:
            want = args.get('num_gpus')
            self.world = max(1, min(int(want), torch.cuda.device_count()) if want else torch.cuda.device_count())
            if self.world > 1 and (not self.gpu_replay or args['batch_size'] % self.world != 0):
                print('handyrl_b200: multi-GPU needs gpu_replay and batch_size %% num_gpus == 0; using one GPU')
                self.world = 1
            elif self.world > 1 and args['batch_size'] % (self.world * self.micro_batches) != 0:
                print('handyrl_b200: multi-GPU with gradient_accumulation needs batch_size %% (num_gpus * gradient_accumulation) == 0 '
                      '(num_gpus %d, gradient_accumulation %d, batch_size %d); using one GPU'
                      % (self.world, self.micro_batches, args['batch_size']))
                self.world = 1
        self.replay_files = None             # the writer of the .replay.pth files
        self.restored = None                 # the replay file this run resumed from, until its sampler state is put back
        self.restored_limiter = None         # the limiter counts that file held
        if self.save_replay is not None:
            self.replay_files = ReplayCheckpoints(self.checkpoint_files.directory, keep=self.save_replay['keep'])
            if self.checkpoint_files.restart_epoch > 0:
                self._restore_replay()

    def _restore_replay(self):
        """Start from models/<restart_epoch>.replay.pth: its episodes go into `episodes`, oldest first, before the Learner
        appends any; the sampler state and the priorities follow once they are resident (_finish_restore)."""
        path = self.checkpoint_files.seed_path('replay')
        if path is None:
            print('handyrl_b200: no %s, the replay starts empty'
                  % self.checkpoint_files.path(self.checkpoint_files.restart_epoch, 'replay'))
            return
        d = load_replay_file(path)
        if d['episodes'] and len(self.params) > 0:
            self._check_fits_net(d['episodes'][0], path)
        self.episodes.extend(d['episodes'])
        self.restored = d
        self.restored_limiter = d.get('limiter')
        held = int((d['serials'] < 0).sum())
        print('restored replay: %d episodes (%d held out), %d steps, priorities: %s'
              % (len(d['episodes']), held, sum(ep['steps'] for ep in d['episodes']),
                 'yes' if d['priorities'] is not None and self.priority is not None else 'no'))

    def _check_fits_net(self, episode, path):
        """A saved episode must be one this run's net can train on: the net takes its observation and answers with one
        logit per saved action.  Raises ValueError naming the file."""
        from .wire import episode_to_flat
        fe = episode_to_flat(episode)
        obs = tree_map(lambda a: torch.from_numpy(np.ascontiguousarray(a[0, :1], dtype=np.float32)).to(self.params[0].device), fe.obs)
        was_training = self.model.training
        self.model.eval()
        try:
            with torch.no_grad():
                hidden = self.model.init_hidden([1]) if hasattr(self.model, 'init_hidden') else None
                policy = self.model(obs, hidden)['policy']
        except Exception as e:
            raise ValueError('%s: the net does not take its observations of shape %s (%s: %s)'
                             % (path, [tuple(l.shape[2:]) for l in tree_leaves(fe.obs)], type(e).__name__, e))
        finally:
            self.model.train(was_training)
        if policy.shape[-1] != fe.amask.shape[-1]:
            raise ValueError('%s: %d actions, the net has %d' % (path, fe.amask.shape[-1], policy.shape[-1]))

    def _finish_restore(self):
        """The restored backlog is resident: put back the sampler state and the priorities (rank 0's; helper ranks start
        theirs afresh)."""
        d, self.restored = self.restored, None
        self.gpu_batcher.restore_sampler(d['sampler'])
        restore_priorities(self.stepper, self.gpu_batcher, d)

    def update(self):
        """Called by the Learner (train.py:342-345, 533): ends the running epoch and returns (CPU model in eval
        mode, steps).  The trainer thread only enqueues the hand-off; the wait for the side-stream copy, the
        state_dict rebuild and the pickling happen here, on the caller's thread."""
        while True:
            self.update_flag = True
            if self.limiter is not None:
                self.limiter.wake()          # a trainer waiting for credit ends its epoch now
            item, steps = self.update_queue.get()
            if not isinstance(item, PendingModel):
                return item, steps
            model, sums = item.resolve()
            if self.limiter is not None:
                self.replay_ratio_epoch = item.replay_ratio
            if sums['dcnt'] > 0:           # train.py:357: an epoch needs at least one sample with a turn in it
                break
        if self.checkpoint_files is not None:
            files = {}
            if self.ema_files is not None and item.ema_state is not None:
                files['ema'] = item.ema_state
            if self.optim_files is not None and item.optim_state is not None:
                files['optim'] = item.optim_state
            self.checkpoint_files.save_epoch(files)
            epoch = self.checkpoint_files.epoch
            if self.replay_files is not None and item.replay is not None and epoch % self.save_replay['every'] == 0:
                self.replay_files.submit(epoch, replay_file(
                    item.replay, item.priority_state, self.limiter.snapshot() if self.limiter is not None else None,
                    item.steps, epoch))
        # host mirrors of the schedule the device applied (train.py:382-384), for inspection / logging
        self.data_cnt_ema = self.data_cnt_ema * 0.8 + sums['dcnt'] / (1e-2 + item.batch_cnt) * 0.2
        self.lr = self.default_lr * self.data_cnt_ema / (1 + steps * 1e-5)
        return model, steps

    def replay_ratio_stats(self):
        """None without train_args['replay_ratio']; otherwise the limiter's counts since this Trainer started: {'limit': r,
        'trained': samples trained, 'stored': steps stored in the training replay, 'waited': seconds the trainer thread spent
        waiting for credit, 'waiting': whether it waits now, 'epoch': the figures of the last epoch update() handed over (what
        its replay_ratio line printed: ReplayRatioLimiter.end_epoch), or None before the first}."""
        if self.limiter is None:
            return None
        stats = dict(self.limiter.snapshot(), epoch=self.replay_ratio_epoch)
        if self.save_replay is not None:     # what the replay file this run resumed from recorded; not applied to the limiter
            stats['restored'] = self.restored_limiter
        return stats

    def _start_stepper(self):
        # the first batch is built on the host: it fixes every shape of the captured step
        batch = self._first_host_batch()
        self.cpu_template = copy.deepcopy(self.model)
        self.cpu_template.eval()
        optim_state = None
        if self.optim_files is not None and self.optim_files.restart_epoch > 0:
            path = self.optim_files.seed_path('optim')
            if path is not None:
                optim_state = torch.load(path, map_location='cpu')
                OptimizerStateFormat((), optimizer=self.optimizer).check_algorithm(optim_state)
                sched = optim_state['schedule']         # before the helper ranks spawn: they start at self.lr
                self.steps, self.data_cnt_ema, self.lr = int(sched['steps']), float(sched['data_cnt_ema']), float(sched['lr'])
            else:
                print('handyrl_b200: no %s, the optimiser state starts fresh'
                      % self.optim_files.path(self.optim_files.restart_epoch, 'optim'))
        pg = None
        if self.world > 1:
            from . import multigpu
            batch = tree_map(lambda t: t[:t.shape[0] // self.world].contiguous(), batch)
            self.fleet = multigpu.Fleet(self.world, self.args, self.cpu_template, list(self.episodes), self.lr,
                                        optim_state=optim_state)
            pg = self.fleet.process_group
        self.stepper = LearnerStep(self.model, self.args, batch, self.lr, process_group=pg, teacher=self.teacher)
        if optim_state is not None:
            self.stepper.load_optimizer_state(optim_state)
        seed = self.ema_files.seed_path() if self.ema_files is not None else None
        if seed is not None:
            self.stepper.seed_weight_ema(torch.load(seed, map_location='cpu'))
        self.stepper.warm_up()
        self.batcher.pool = [self.stepper.new_packed() for _ in range(4)]
        if self.gpu_replay:
            self.gpu_batcher = GpuBatcher(self.args, self.episodes, self.stepper.device,
                                          forward=self.fleet.send_episodes if self.fleet is not None else None,
                                          limiter=self.limiter, restore=self.restored)
            self.gpu_batcher.run()
        loss_buf = self.stepper.loss_buf
        self.heads = ['p'] + (['v'] if loss_buf.has_value else []) + (['r'] if loss_buf.has_return else []) + ['ent', 'total']

    def train(self):
        if len(self.params) == 0:          # non-parametric model (train.py:348-350)
            time.sleep(0.1)
            return self.model
        batch_cnt = 0
        chunk = int(self.args.get('multi_gpu_chunk', 8))
        if self.limiter is not None:
            self.limiter.start_epoch()
        while True:
            if self.stop_event.is_set() and (self.fleet is None or batch_cnt % chunk == 0):
                return None                 # (sharded: only between chunks -- the other ranks run whole chunks)
            if self.stepper is None:
                self._start_stepper()
            if self.gpu_batcher is not None:
                while not (self.gpu_batcher.ready() and (self.fleet is None or self.fleet.all_ready())):
                    if self.stop_event.is_set():
                        return None
                    time.sleep(0.01)
                if self.restored is not None:
                    self._finish_restore()
            if self.limiter is not None and (self.fleet is None or batch_cnt % chunk == 0):
                if not self.limiter.acquire(1 if self.fleet is None else chunk,
                                            lambda: self.stop_event.is_set() or self.update_flag):
                    if self.stop_event.is_set():
                        return None
                    if batch_cnt > 0:
                        break               # update() waits: end the epoch without another step
                    # update() waits for an epoch that has no step yet: this step (chunk) goes through over the limit
            if self.gpu_batcher is not None:
                if self.fleet is not None and batch_cnt % chunk == 0:
                    self.fleet.run_steps(chunk)          # every rank runs exactly the steps rank 0 runs
                self.gpu_batcher.fill(self.stepper)
                self.stepper.step_in_place()
                if self.validate_every and (batch_cnt + 1) % self.validate_every == 0 and self.gpu_batcher.validation_ready():
                    self.gpu_batcher.fill_validation(self.stepper)
                    self.stepper.validate_in_place()
                    if self.stepper.avg is not None:
                        self.stepper.validate_in_place(averaged=True)
            else:
                batch = self.batcher.batch()
                if batch is None:           # stop() was called
                    return None
                packed = self.batcher.pool[batch_cnt % len(self.batcher.pool)]
                packed.wait_reusable()
                packed.fill(batch)
                self.stepper.step(packed)
            batch_cnt += 1
            self.steps += 1
            if self.limiter is not None:
                self.limiter.drew()
            if self.update_flag and (self.fleet is None or batch_cnt % chunk == 0):
                break
        # epoch boundary: nothing here waits for the GPU (LearnerStep.end_epoch)
        if self.fleet is not None:
            self.fleet.end_epoch(batch_cnt, self.steps, self.default_lr)
        pending = self.stepper.end_epoch(batch_cnt, self.steps, self.default_lr, self.cpu_template, self.heads)
        pending.batch_cnt = batch_cnt
        if self.limiter is not None:
            pending.replay_ratio = self.limiter.end_epoch()
        if self.replay_files is not None and self.gpu_batcher is not None:
            # on this thread, between two batches: the sampler state is the one the boundary's weights and priorities go with
            pending.replay = self.gpu_batcher.snapshot()
        return pending

    def _first_host_batch(self):
        return self.batcher._make()

    def run(self):
        print('waiting training')
        while len(self.episodes) < self.args['minimum_episodes']:
            if self.stop_event.is_set():
                return
            time.sleep(1)
        if len(self.params) > 0:
            if not self.gpu_replay:
                self.batcher.run()
            print('started training')
        while not self.stop_event.is_set():
            model = self.train()
            if model is None:
                break
            self.update_flag = False
            while not self.stop_event.is_set():
                try:
                    self.update_queue.put((model, self.steps), timeout=0.2)
                    break
                except queue.Full:
                    continue
        print('finished training')

    def stop(self):
        """Not in the reference (its threads die with the process): lets tests and embedders shut the
        trainer down cleanly -- stops the batcher threads, the helper ranks, and ends run()."""
        self.stop_event.set()
        if self.limiter is not None:
            self.limiter.wake()
        self.batcher.stop()
        if self.gpu_batcher is not None:
            self.gpu_batcher.stop()
        if self.replay_files is not None:
            self.replay_files.close()
        if self.stepper is not None:
            self.stepper.stream.synchronize()
        if self.fleet is not None:
            self.fleet.stop()
            self.stepper.close()
            self.fleet.destroy()


def install(flat_episodes=False):
    """Swap the reference's learner hot path for this one in an importable `handyrl` package
    (flat_episodes=True additionally makes workers forked afterwards ship the flat wire format of wire.py):
    after `handyrl_b200.train.install()`, `python main.py --train` runs the reference's Learner,
    workers and server unchanged on top of this Trainer (see INTEGRATION.md)."""
    import handyrl.train as ref
    ref.Trainer = Trainer
    ref.Batcher = Batcher
    ref.make_batch = make_batch
    ref.forward_prediction = forward_prediction
    ref.compute_loss = compute_loss
    import handyrl.losses as ref_losses
    ref_losses.compute_target = ops.compute_target
    if flat_episodes:
        from .wire import install_worker_hook
        install_worker_hook()
    return ref
