"""Thin Python front end of the C ABI: torch tensors in, torch tensors out.

torch is used for device memory and streams only; every computation happens in the
CUDA library (handyrl_b200/libhrl_b200.so, sources in handyrl_b200/csrc/).  There is no
fallback path: a CPU tensor or a missing library raises.
"""
import ctypes as C

import torch

from . import _capi
from ._capi import ALGO_ID, DIAG_KEYS, GEMM_EPILOGUES, LOSS_KEYS, NUM_DIAG, NUM_LOSS, HrlLossArgs, check, lib

# kernels of THIS library launched through the wrappers below (bench.py reports them as `gpu_launches`; a CUDA graph
# replays the launches counted while it was captured)
LAUNCHES = {'n': 0}


def _count(n=1):
    LAUNCHES['n'] += n


_BATCH_KEYS = ('action_mask', 'action', 'selected_prob', 'reward', 'return', 'turn_mask', 'observation_mask',
               'episode_mask', 'progress', 'outcome')


def _stream_ptr():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _dev_f32(t, name):
    if t is None:
        return None
    if not t.is_cuda:
        raise _capi.HrlError('handyrl_b200: %s must be a CUDA tensor (no CPU path exists)' % name)
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def algo_id(name):
    try:
        return ALGO_ID[name]
    except KeyError:
        # the reference prints 'No algorithm named ...' and returns None (losses.py:79-80)
        raise ValueError('No algorithm named %s' % name)


class LossBuffers:
    """Pre-allocated outputs of one fused loss launch (re-used across steps / graph replays).  grads=False: the outputs of the
    forward-only pass (loss_fwd), without gradient buffers."""

    def __init__(self, B, T, P, Pa, A, has_value, has_return, device, taps=False, policy_dtype=torch.float32, diagnostics=False,
                 grads=True, advantage=False, value_bins=None):
        f = dict(dtype=torch.float32, device=device)
        self.dims = (B, T, P, Pa, A)
        self.policy_dtype = policy_dtype
        self.has_value, self.has_return = bool(has_value), bool(has_return)
        # value_bins (value_bins.config): the categorical heads.  Such a head has no scalar gradient here: the fused loss
        # reads its expectation (`expect`, (B, T, Pa, 1)), writes its targets to `bins_target` (B, T, P, 1), and the
        # cross-entropy kernel writes its logit gradient to `dlogits` (B, T, Pa, K)
        self.value_bins = dict(value_bins or {})
        cat = {h for h in self.value_bins if (has_value if h == 'value' else has_return)}
        self.value_bins = {h: s for h, s in self.value_bins.items() if h in cat}
        self.dpolicy = torch.empty((B, T, Pa, A), dtype=policy_dtype, device=device) if grads else None   # bf16 logits: bf16 gradients
        self.dvalue = torch.empty((B, T, Pa, 1), **f) if has_value and grads and 'value' not in cat else None
        self.dreturn = torch.empty((B, T, Pa, 1), **f) if has_return and grads and 'return' not in cat else None
        self.expect = {h: torch.zeros((B, T, Pa, 1), **f) for h in cat}
        self.dlogits = {h: torch.empty((B, T, Pa, s['bins']), **f) for h, s in self.value_bins.items()} if grads else {}
        self.bins_target = {h: torch.zeros((B, T, P, 1), **f) for h in cat}
        self.bins_workspace = torch.zeros(max([lib().hrl_value_bins_workspace_bytes(B, T, P, Pa, s['bins'])
                                               for s in self.value_bins.values()] or [0]), dtype=torch.uint8, device=device) \
            if cat else None
        self.losses = torch.zeros(NUM_LOSS, **f)
        self.taps = None
        if taps:
            self.taps = {
                'target_value': torch.zeros((B, T, P, 1), **f), 'target_return': torch.zeros((B, T, P, 1), **f),
                'advantage': torch.zeros((B, T, P, 1), **f), 'logp': torch.zeros((B, T, Pa, 1), **f),
                'rho': torch.zeros((B, T, Pa, 1), **f), 'entropy': torch.zeros((B, T, Pa), **f),
            }
        # advantage=True: the advantage tap alone (B, T, P, 1), which the priority update of prioritised replay reduces
        self.advantage = torch.zeros((B, T, P, 1), **f) if advantage and not taps else None
        self.workspace = torch.zeros(lib().hrl_loss_workspace_bytes(B, T, P, Pa, A), dtype=torch.uint8, device=device)
        self.diagnostics = self.diag_workspace = None
        if diagnostics:
            self.enable_diagnostics()

    def enable_diagnostics(self):
        """Allocate the outputs of the diagnostics form of the pass: `diagnostics` (NUM_DIAG sums in DIAG_KEYS order) and its
        own, larger workspace."""
        if self.diagnostics is None:
            device = self.losses.device
            self.diagnostics = torch.zeros(NUM_DIAG, dtype=torch.float32, device=device)
            self.diag_workspace = torch.zeros(lib().hrl_loss_diag_workspace_bytes(*self.dims), dtype=torch.uint8, device=device)


def loss_fwd_bwd(outputs, batch, args, buffers=None, taps=False, tuning=None, diagnostics=False, window_weight=None):
    """Fused mask epilogue + compute_loss + closed-form backward (reference train.py:176-267).

    outputs: raw net outputs {'policy': (B,T,Pa,A), 'value': (B,T,Pa,1)?, 'return': (B,T,Pa,1)?}
    batch:   the make_batch dict (device tensors)
    args:    train_args (lambda, gamma, entropy_regularization[_decay], policy_target, value_target,
             turn_based_training, burn_in_steps)
    tuning:  None (the library chooses), or a dict for tests / profiling with any of
             variant ('rows-direct'|'rows-staged'|'bulk'|'element'|'group'), recurrence ('serial'|'scan'),
             cluster, consumers, threads, unstaged, trace (an int64 CUDA tensor of >= 32 elements)
    diagnostics: also accumulate the learner diagnostics sums (hrl_loss_fwd_bwd_diag) into .diagnostics, in DIAG_KEYS order;
             losses and gradients are bit-identical to the plain pass
    window_weight: None, or a (B,) float32 CUDA tensor of importance weights (prioritised replay): every per-cell loss term of
             window b and its gradients are scaled by window_weight[b]; dcnt and the diagnostics are not.  Weights of exactly 1
             give the bits of window_weight=None.
    returns  LossBuffers with .losses = [p, v, r, ent, total, dcnt] and the gradients.
    """
    return _loss_call(outputs, batch, args, buffers, taps, tuning, 'diag' if diagnostics else 'fwd_bwd', window_weight)


def loss_fwd(outputs, batch, args, buffers=None, taps=False, tuning=None):
    """The forward half of loss_fwd_bwd (hrl_loss_fwd): the same kernel choice with the gradient phase compiled out, for losses
    on data the optimiser does not see.  Same arguments (buffers: LossBuffers(..., grads=False), or any LossBuffers -- its
    gradient buffers are left untouched); returns the (6,) device tensor of sums [p, v, r, ent, total, dcnt], bit-identical
    to loss_fwd_bwd(...).losses on the same inputs."""
    return _loss_call(outputs, batch, args, buffers, taps, tuning, 'fwd').losses


def _loss_call(outputs, batch, args, buffers, taps, tuning, form, window_weight=None):
    diagnostics = form == 'diag'
    policy = outputs['policy']
    io_bf16 = policy.dtype == torch.bfloat16       # wide rows only: 8 instead of 12 bytes per action through HBM (include/hrl_b200.h)
    if io_bf16:
        if not (policy.is_cuda and policy.is_contiguous()):
            raise _capi.HrlError('handyrl_b200: bf16 policy logits must be a contiguous CUDA tensor')
    else:
        policy = _dev_f32(policy, 'policy')
    B, T, Pa, A = policy.shape
    P = batch['turn_mask'].shape[2]
    value = _dev_f32(outputs.get('value'), 'value')
    ret_head = _dev_f32(outputs.get('return'), 'return')
    if buffers is None:
        buffers = LossBuffers(B, T, P, Pa, A, value is not None, ret_head is not None, policy.device, taps=taps, policy_dtype=policy.dtype,
                              grads=form != 'fwd')
    assert buffers.dims == (B, T, P, Pa, A) and buffers.policy_dtype == policy.dtype
    if form != 'fwd' and buffers.dpolicy is None:
        raise ValueError('loss_fwd_bwd: these LossBuffers were built without gradient buffers (grads=False)')
    if diagnostics:
        buffers.enable_diagnostics()
    if window_weight is not None and not (window_weight.is_cuda and window_weight.dtype == torch.float32 and
                                          window_weight.is_contiguous() and window_weight.numel() == B):
        raise _capi.HrlError('handyrl_b200: window_weight must be a contiguous float32 CUDA tensor of B=%d weights' % B)

    # static buffers (CUDA-graph replays): the argument block of the previous call is still valid
    key = (policy.data_ptr(), 0 if value is None else value.data_ptr(), 0 if ret_head is None else ret_head.data_ptr(),
           args['value_target'], args['policy_target'], bool(args['turn_based_training']), args.get('burn_in_steps', 0),
           args['lambda'], args['gamma'], args['entropy_regularization'], args['entropy_regularization_decay'],
           buffers.taps is not None, 0 if window_weight is None else window_weight.data_ptr(), None if tuning is None else tuple(sorted((k, v if not torch.is_tensor(v) else v.data_ptr())
                                                                                 for k, v in tuning.items()))) + \
        tuple(batch[k].data_ptr() for k in _BATCH_KEYS)
    slot = '_cached_' + form      # one argument block per form
    cached = getattr(buffers, slot, None)
    if cached is not None and cached[0] == key:
        _launch(cached[1], buffers, form)
        return buffers

    a = HrlLossArgs()
    a.B, a.T, a.P, a.Pa, a.A = B, T, P, Pa, A
    a.burn_in = int(args.get('burn_in_steps', 0))
    a.value_target = algo_id(args['value_target'])
    a.policy_target = algo_id(args['policy_target'])
    a.two_player_zero_sum = int(bool(args['turn_based_training']) and P == 2)
    a.lambda_ = float(args['lambda'])
    a.gamma = float(args['gamma'])
    a.entropy_regularization = float(args['entropy_regularization'])
    a.entropy_regularization_decay = float(args['entropy_regularization_decay'])

    action = batch['action']
    if not action.is_cuda:
        raise _capi.HrlError('handyrl_b200: the batch must live on the GPU')
    keep = [policy, value, ret_head,
            _dev_f32(batch['action_mask'], 'action_mask'), action.long().contiguous(),
            _dev_f32(batch['selected_prob'], 'selected_prob'), _dev_f32(batch['reward'], 'reward'),
            _dev_f32(batch['return'], 'return'), _dev_f32(batch['turn_mask'], 'turn_mask'),
            _dev_f32(batch['observation_mask'], 'observation_mask'), _dev_f32(batch['episode_mask'], 'episode_mask'),
            _dev_f32(batch['progress'], 'progress'), _dev_f32(batch['outcome'], 'outcome')]
    (a.policy_raw, a.value_raw, a.return_raw, a.action_mask, a.action, a.selected_prob, a.reward, a.ret,
     a.turn_mask, a.observation_mask, a.episode_mask, a.progress, a.outcome) = [_ptr(t) for t in keep]
    if form != 'fwd':
        a.dpolicy_raw, a.dvalue_raw, a.dreturn_raw = _ptr(buffers.dpolicy), _ptr(buffers.dvalue), _ptr(buffers.dreturn)
    a.losses = _ptr(buffers.losses)
    if buffers.taps is not None:
        t = buffers.taps
        a.tap_target_value, a.tap_target_return, a.tap_advantage = _ptr(t['target_value']), _ptr(t['target_return']), _ptr(t['advantage'])
        a.tap_logp, a.tap_rho, a.tap_entropy = _ptr(t['logp']), _ptr(t['rho']), _ptr(t['entropy'])
    elif getattr(buffers, 'advantage', None) is not None:
        a.tap_advantage = _ptr(buffers.advantage)
    for bit, head, tap in ((1, 'value', 'tap_target_value'), (2, 'return', 'tap_target_return')):
        if head in buffers.value_bins:      # a categorical head: its loss is the cross-entropy kernel's (value_bins_fwd_bwd)
            a.external_heads |= bit
            setattr(a, tap, _ptr(bins_targets(buffers)[head]))
    a.window_weight = _ptr(window_weight)
    a.io_bf16 = int(io_bf16)
    ws = buffers.diag_workspace if diagnostics else buffers.workspace
    a.workspace = _ptr(ws)
    a.workspace_bytes = ws.numel()
    if tuning:
        t = dict(tuning)
        a.tuning.variant = _capi.LOSS_VARIANTS[t.pop('variant', 'auto')]
        a.tuning.recurrence = _capi.LOSS_RECURRENCES[t.pop('recurrence', 'auto')]
        trace = t.pop('trace', None)
        if trace is not None:
            assert trace.is_cuda and trace.dtype == torch.int64 and trace.numel() >= 32
            a.tuning.trace = trace.data_ptr()
        for k in ('cluster', 'consumers', 'threads', 'unstaged'):
            setattr(a.tuning, k, int(t.pop(k, 0)))
        if t:
            raise ValueError('unknown loss tuning keys: %s' % sorted(t))
    _launch(a, buffers, form)
    buffers._keep = keep  # the launch is asynchronous: keep temporaries alive
    if all(k is None or k is o for k, o in zip(keep[3:], (batch['action_mask'], batch['action'], batch['selected_prob'],
                                                          batch['reward'], batch['return'], batch['turn_mask'],
                                                          batch['observation_mask'], batch['episode_mask'],
                                                          batch['progress'], batch['outcome']))):
        setattr(buffers, slot, (key, a))   # only when no temporary copies were made
    return buffers


def _launch(a, buffers, form):
    if form == 'diag':
        check(lib().hrl_loss_fwd_bwd_diag(C.byref(a), _ptr(buffers.diagnostics), _stream_ptr()))
    elif form == 'fwd':
        check(lib().hrl_loss_fwd(C.byref(a), _stream_ptr()))
    else:
        check(lib().hrl_loss_fwd_bwd(C.byref(a), _stream_ptr()))
    _count()


def bins_targets(buffers):
    """Where the loss pass writes the targets of each categorical head: the taps' tensors when the buffers keep taps."""
    if buffers.taps is not None:
        return {h: buffers.taps['target_' + h] for h in buffers.value_bins}
    return buffers.bins_target


def _bins_args(spec, head, logits, batch_dims, burn_in):
    B, T, Pa, K = logits.shape
    if K != spec['bins']:
        raise ValueError("value_bins: the %s head has %d logits per row, the key %d bins" % (head, K, spec['bins']))
    a = _capi.HrlValueBinsArgs()
    a.B, a.T, a.P, a.Pa, a.K = B, T, batch_dims, Pa, K
    a.burn_in = int(burn_in)
    a.low, a.high, a.symlog, a.sigma = spec['low'], spec['high'], int(spec['symlog']), spec['sigma']
    a.head = 0 if head == 'value' else 1
    a.logits = _ptr(logits)
    return a


def _bins_logits(logits, head):
    if not (logits.is_cuda and logits.dtype == torch.float32 and logits.is_contiguous() and logits.dim() == 4):
        raise _capi.HrlError('handyrl_b200: the %s logits must be a contiguous (B, T, Pa, K) float32 CUDA tensor' % head)
    return logits


def value_bins_expect(logits, spec, head='value', out=None, P=None):
    """The expectation v = s^-1(sum_k softmax(z)_k c_k) of a categorical head (hrl_value_bins_expect; the law in
    value_bins.py): (B, T, Pa, K) float32 logits -> out (B, T, Pa, 1), allocated when None.  P: the batch's players (Pa when
    None).  Returns out."""
    logits = _bins_logits(logits, head)
    B, T, Pa, K = logits.shape
    if out is None:
        out = torch.empty((B, T, Pa, 1), dtype=torch.float32, device=logits.device)
    assert out.is_contiguous() and out.dtype == torch.float32 and out.numel() == B * T * Pa
    a = _bins_args(spec, head, logits, Pa if P is None else P, 0)
    a.expect = _ptr(out)
    check(lib().hrl_value_bins_expect(C.byref(a), _stream_ptr()))
    _count()
    return out


def value_bins_fwd_bwd(logits, head, spec, batch, args, buffers, window_weight=None, forward_only=False):
    """The cross-entropy of a categorical head (hrl_value_bins_fwd_bwd; the law in value_bins.py), launched after the fused
    loss pass that wrote `buffers` (LossBuffers with value_bins) on the same batch, from the targets that pass left in
    bins_targets(buffers)[head].  Writes buffers.losses[v|r] = L and adds L to the total; writes dL/dz to
    buffers.dlogits[head] unless forward_only (the held-out form: no gradient, window_weight ignored).  Returns the
    (B, T, Pa, K) gradient, or None when forward_only."""
    logits = _bins_logits(logits, head)
    B, T, Pa, K = logits.shape
    P = batch['observation_mask'].shape[2]
    assert buffers.dims[:4] == (B, T, P, Pa) and head in buffers.value_bins
    om = batch['observation_mask']
    grad = None if forward_only else buffers.dlogits[head]
    if window_weight is not None and not (window_weight.is_cuda and window_weight.dtype == torch.float32 and
                                          window_weight.is_contiguous() and window_weight.numel() == B):
        raise _capi.HrlError('handyrl_b200: window_weight must be a contiguous float32 CUDA tensor of B=%d weights' % B)
    target = bins_targets(buffers)[head]
    burn_in = int(args.get('burn_in_steps', 0))
    key = (logits.data_ptr(), om.data_ptr(), target.data_ptr(), 0 if window_weight is None else window_weight.data_ptr(),
           0 if grad is None else grad.data_ptr(), buffers.losses.data_ptr(), burn_in, tuple(sorted(spec.items())))
    slot = '_cached_bins_%s_%d' % (head, int(forward_only))     # static buffers (CUDA-graph replays): the same argument block
    cached = getattr(buffers, slot, None)
    if cached is None or cached[0] != key:
        keep = [_dev_f32(om, 'observation_mask')]
        a = _bins_args(spec, head, logits, P, burn_in)
        a.target, a.observation_mask = _ptr(target), _ptr(keep[0])
        a.window_weight = None if forward_only else _ptr(window_weight)
        a.dlogits, a.losses = _ptr(grad), _ptr(buffers.losses)
        a.workspace, a.workspace_bytes = _ptr(buffers.bins_workspace), buffers.bins_workspace.numel()
        cached = (key, a, keep)
        if keep[0] is om:
            setattr(buffers, slot, cached)
    check(lib().hrl_value_bins_fwd_bwd(C.byref(cached[1]), _stream_ptr()))
    setattr(buffers, '_bins_keep_' + head, cached[2])       # the launch is asynchronous: keep temporaries alive
    _count()
    return grad


def distill_fwd_bwd(policy, teacher, batch, args, buffers, step_count, coef, anneal_steps=0, window_weight=None, sums=None):
    """The policy distillation term (hrl_distill_fwd_bwd, csrc/distill_kernel.cu; the law in distill.py), launched after the
    fused loss pass that wrote `buffers` (LossBuffers with gradients) on the same batch: adds c_n * d kl / d policy to
    buffers.dpolicy and, when c_n > 0, c_n * kl to buffers.losses' total.  policy / teacher: the student's and the teacher's
    raw (B, T, Pa, A) float32 logits; step_count: FlatAdam.step_count (n, read on the device); coef, anneal_steps: c0 and N.
    sums: a (2,) float32 CUDA tensor that receives [kl, c_n * kl] (allocated on `buffers` when None).  Returns sums."""
    if policy.dtype != torch.float32 or teacher.dtype != torch.float32:
        raise _capi.HrlError('handyrl_b200: distillation takes float32 logits (bf16 logit I/O is not supported)')
    for t, name in ((policy, 'policy'), (teacher, 'teacher')):
        if not (t.is_cuda and t.is_contiguous()):
            raise _capi.HrlError('handyrl_b200: %s logits must be a contiguous CUDA tensor' % name)
    if teacher.shape != policy.shape:
        raise ValueError('distillation: the teacher policy is shaped %s, the student\'s %s' % (tuple(teacher.shape), tuple(policy.shape)))
    B, T, Pa, A = policy.shape
    P = batch['turn_mask'].shape[2]
    assert buffers.dims == (B, T, P, Pa, A) and buffers.dpolicy is not None and buffers.policy_dtype == torch.float32
    if not (step_count.is_cuda and step_count.dtype == torch.int64 and step_count.numel() == 1):
        raise _capi.HrlError('handyrl_b200: step_count must be a one-element int64 CUDA tensor')
    if window_weight is not None and not (window_weight.is_cuda and window_weight.dtype == torch.float32 and
                                          window_weight.is_contiguous() and window_weight.numel() == B):
        raise _capi.HrlError('handyrl_b200: window_weight must be a contiguous float32 CUDA tensor of B=%d weights' % B)
    if sums is None:
        if getattr(buffers, 'distill_sums', None) is None:
            buffers.distill_sums = torch.zeros(2, dtype=torch.float32, device=policy.device)
        sums = buffers.distill_sums
    if not (sums.is_cuda and sums.dtype == torch.float32 and sums.is_contiguous() and sums.numel() == 2):
        raise _capi.HrlError('handyrl_b200: sums must be a contiguous float32 CUDA tensor of 2')
    if getattr(buffers, 'distill_workspace', None) is None:
        buffers.distill_workspace = torch.zeros(lib().hrl_distill_workspace_bytes(B, T, P, Pa, A), dtype=torch.uint8,
                                                device=policy.device)
    amask, tmask = batch['action_mask'], batch['turn_mask']
    burn_in = int(args.get('burn_in_steps', 0))
    key = (policy.data_ptr(), teacher.data_ptr(), amask.data_ptr(), tmask.data_ptr(), 0 if window_weight is None else window_weight.data_ptr(),
           step_count.data_ptr(), float(coef), int(anneal_steps), burn_in, buffers.dpolicy.data_ptr(), buffers.losses.data_ptr(),
           sums.data_ptr())
    cached = getattr(buffers, '_cached_distill', None)      # static buffers (CUDA-graph replays): the same argument block
    if cached is None or cached[0] != key:
        keep = [_dev_f32(amask, 'action_mask'), _dev_f32(tmask, 'turn_mask')]
        a = _capi.HrlDistillArgs()
        a.B, a.T, a.P, a.Pa, a.A, a.burn_in = B, T, P, Pa, A, burn_in
        a.policy_raw, a.teacher_raw, a.action_mask, a.turn_mask = _ptr(policy), _ptr(teacher), _ptr(keep[0]), _ptr(keep[1])
        a.window_weight, a.step_count = _ptr(window_weight), _ptr(step_count)
        a.coef, a.anneal_steps = float(coef), int(anneal_steps)
        a.dpolicy_raw, a.losses, a.sums = _ptr(buffers.dpolicy), _ptr(buffers.losses), _ptr(sums)
        a.workspace, a.workspace_bytes = _ptr(buffers.distill_workspace), buffers.distill_workspace.numel()
        cached = (key, a, keep)
        if keep[0] is amask and keep[1] is tmask:
            buffers._cached_distill = cached
    check(lib().hrl_distill_fwd_bwd(C.byref(cached[1]), _stream_ptr()))
    buffers._distill_keep = cached[2]       # the launch is asynchronous: keep temporaries alive
    _count()
    return sums


def summarize_diagnostics(sums):
    """Diagnostics sums (a sequence in DIAG_KEYS order, or a dict keyed by DIAG_KEYS; missing entries count as 0) -> means:
      rho     mean unclipped importance ratio pi(a)/mu(a)        clip    fraction of samples with rho > 1 (clipped at 1)
      kl      -mean log ratio, the sample estimate of KL(mu||pi)  logr_sd spread of the log ratio
      adv     mean advantage                                      adv_sd  its standard deviation
      ev_v    explained variance of the value target, 1 - Var(target - value) / Var(target); ev_r: the return head's
      gnorm   mean pre-clip global gradient norm                  gclip   fraction of steps whose norm exceeded max_norm
    A field whose count (or target variance) is zero is left out: nothing is ever divided by zero."""
    if isinstance(sums, dict):
        s = {k: float(sums.get(k, 0.0)) for k in DIAG_KEYS}
    else:
        vals = [float(x) for x in (sums.tolist() if hasattr(sums, 'tolist') else sums)]
        s = dict(zip(DIAG_KEYS, vals + [0.0] * (NUM_DIAG - len(vals))))

    def sd(total, total2, n):
        return max(total2 / n - (total / n) ** 2, 0.0) ** 0.5

    out = {}
    n = s['n_pol']
    if n > 0:
        out['rho'] = s['rho'] / n
        out['clip'] = s['rho_clip'] / n
        out['kl'] = -s['logr'] / n
        out['logr_sd'] = sd(s['logr'], s['logr2'], n)
        out['adv'] = s['adv'] / n
        out['adv_sd'] = sd(s['adv'], s['adv2'], n)
    n = s['n_val']
    if n > 0:
        for key, t, t2, e, e2 in (('ev_v', 'tv', 'tv2', 'ev', 'ev2'), ('ev_r', 'tr', 'tr2', 'er', 'er2')):
            var_t = s[t2] / n - (s[t] / n) ** 2      # (0 without the head)
            if var_t > 0:
                out[key] = 1.0 - max(s[e2] / n - (s[e] / n) ** 2, 0.0) / var_t
    n = s['steps']
    if n > 0:
        out['gnorm'] = s['gnorm'] / n
        out['gnorm_sd'] = sd(s['gnorm'], s['gnorm2'], n)
        out['gclip'] = s['gclip'] / n
    return out


_DIAG_FORMAT = (('rho', '%.3f'), ('clip', '%.3f'), ('kl', '%.4g'), ('logr_sd', '%.4g'), ('adv', '%.4g'), ('adv_sd', '%.4g'),
                ('ev_v', '%.3f'), ('ev_r', '%.3f'), ('gnorm', '%.4g'), ('gnorm_sd', '%.4g'), ('gclip', '%.3f'))


def format_diagnostics(summary):
    """The Trainer's per-epoch line: 'diagnostics = rho:1.024 clip:0.318 kl:0.041 ...' -- `key:value` pairs in a fixed
    order, fields absent from `summary` left out."""
    return 'diagnostics = %s' % ' '.join(k + ':' + (f % summary[k]) for k, f in _DIAG_FORMAT if k in summary)


def compute_target(algorithm, values, returns, rewards, lmb, gamma, rhos, cs, masks):
    """Drop-in for handyrl.losses.compute_target on CUDA tensors of shape (B,T,P,1)."""
    aid = algo_id(algorithm)
    returns = _dev_f32(returns, 'returns')
    if values is None:  # losses.py:64-66
        return returns, returns
    values = _dev_f32(values, 'values')
    B, T, P = values.shape[:3]
    rewards, rhos, cs, masks = (_dev_f32(x, n) for x, n in ((rewards, 'rewards'), (rhos, 'rhos'), (cs, 'cs'), (masks, 'masks')))
    if masks is not None and masks.shape[2] != P:
        masks = masks.expand(B, T, P, 1).contiguous()
    Tr = returns.shape[1]
    if returns.shape[2] != P:
        returns = returns.expand(B, Tr, P, 1).contiguous()
    Pr = rhos.shape[2] if rhos is not None else 1
    targets = torch.empty_like(values)
    advantages = torch.empty_like(values)
    check(lib().hrl_compute_target(aid, B, T, P, Tr, Pr, _ptr(values), _ptr(returns), _ptr(rewards), float(lmb),
                                   float(gamma), _ptr(rhos), _ptr(cs), _ptr(masks), _ptr(targets), _ptr(advantages),
                                   _stream_ptr()))
    _count()
    return targets, advantages


class FlatAdam:
    """clip_grad_norm_(max_norm) + Adam(weight_decay) on one flat fp32 bucket (train.py:331, 370-371).

    The model's parameters are re-pointed into one contiguous buffer and their .grad into a
    second one, so that (a) the multi-GPU gradient exchange is ONE all-reduce(SUM) and
    (b) the whole optimiser step is two kernel launches.  `extra` floats are appended to the
    gradient bucket (the learner puts the six loss scalars there so they ride the same
    all-reduce).
    """

    def __init__(self, params, lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-5, max_norm=4.0, extra=0, grad_alloc=None,
                 param_storage=None):
        params = [p for p in params]
        assert len(params) > 0 and all(p.is_cuda and p.dtype == torch.float32 for p in params)
        self.params = params
        device = params[0].device
        self.n = sum(p.numel() for p in params)
        n_pad = (self.n + 3) // 4 * 4
        self.extra = extra
        # param_storage lets the caller place the weights inside a larger state buffer (LearnerStep: weights + BatchNorm
        # buffers in one allocation, so the per-epoch model hand-off is ONE device-to-host copy)
        if param_storage is not None:
            assert param_storage.numel() == n_pad and param_storage.dtype == torch.float32 and param_storage.data_ptr() % 16 == 0
        self.flat_param = param_storage if param_storage is not None else torch.zeros(n_pad, dtype=torch.float32, device=device)
        extra = (extra + 3) // 4 * 4
        self.extra = extra
        # grad_alloc(numel) lets the caller place the bucket in NVLink-symmetric memory (peer all-reduce)
        self.grad_storage = grad_alloc(n_pad + extra) if grad_alloc is not None else None
        self.flat_grad = (self.grad_storage[:n_pad + extra] if self.grad_storage is not None
                          else torch.zeros(n_pad + extra, dtype=torch.float32, device=device))
        off = 0
        with torch.no_grad():
            for p in params:
                k = p.numel()
                self.flat_param[off:off + k].copy_(p.reshape(-1))
                p.data = self.flat_param[off:off + k].view_as(p)
                p.grad = self.flat_grad[off:off + k].view_as(p)
                off += k
        self.n_pad = n_pad
        self.exp_avg = torch.zeros(n_pad, dtype=torch.float32, device=device)
        self.exp_avg_sq = torch.zeros(n_pad, dtype=torch.float32, device=device)
        self.partials = torch.zeros(lib().hrl_sumsq_num_partials(), dtype=torch.float32, device=device)
        self.lr = torch.full((1,), float(lr), dtype=torch.float32, device=device)
        self.step_count = torch.zeros(1, dtype=torch.int64, device=device)
        self.grad_norm = torch.zeros(1, dtype=torch.float32, device=device)
        self.betas, self.eps, self.weight_decay, self.max_norm = betas, eps, weight_decay, max_norm
        # diagnostics: a float64 CUDA tensor of 4 (the gnorm, gnorm2, gclip, steps entries of a DIAG_KEYS accumulator) that
        # every step adds its pre-clip norm statistics to, in the step's own launch; None = off
        self.diag = None
        # guard against non-finite steps: a one-element int32 CUDA tensor the step sets to 1 when it rejected itself (the
        # pre-clip norm or one of the first `guard_tail` extra slots of the bucket not finite; hrl_clip_adam_step),
        # else 0; None = off
        self.skip = None
        self.guard_tail = 0

    @property
    def extra_slots(self):
        return self.flat_grad[self.n_pad:]

    def set_lr(self, lr):
        self.lr.fill_(float(lr))

    def zero_grad(self):
        self.flat_grad.zero_()

    def step_reduced(self, reduced):
        """clip + Adam on an already all-reduced bucket whose sum-of-squares partials are in self.partials
        (hrl_peer_allreduce_sumsq)."""
        self._clip_adam(reduced, _stream_ptr())
        _count(2)

    def _clip_adam(self, grad, s):
        fixed = (_ptr(self.flat_param), _ptr(grad), _ptr(self.exp_avg), _ptr(self.exp_avg_sq), self.n_pad, _ptr(self.partials),
                 _ptr(self.lr), _ptr(self.step_count), self.max_norm, self.betas[0], self.betas[1], self.eps, self.weight_decay,
                 _ptr(self.grad_norm))
        if self.diag is not None:
            assert self.diag.is_cuda and self.diag.dtype == torch.float64 and self.diag.numel() == 4 and self.diag.is_contiguous()
        if self.skip is not None:
            assert self.skip.is_cuda and self.skip.dtype == torch.int32 and self.skip.numel() == 1
            assert 0 <= self.guard_tail <= self.extra and grad.numel() >= self.n_pad + self.extra
        check(lib().hrl_clip_adam_step(*fixed, _ptr(self.diag), _ptr(grad[self.n_pad:]), self.guard_tail, _ptr(self.skip), s))

    def step(self):
        s = _stream_ptr()
        check(lib().hrl_grad_sumsq(_ptr(self.flat_grad), self.n_pad, _ptr(self.partials), s))
        self._clip_adam(self.flat_grad, s)
        _count(3)
        from . import fastnet
        fastnet.new_step()          # cached adjoint weights of the convolutions are stale now


def lamb_plan(numels):
    """hrl_lamb_plan on the host: the (chunks, 5) int64 CPU tensor of the chunks a bucket of tensors of `numels` words (back to
    back from word 0) is cut into -- per chunk its first word, its length, its tensor's index, and that tensor's first chunk
    and chunk count."""
    sizes = torch.tensor([int(k) for k in numels], dtype=torch.int64)
    n_chunks = lib().hrl_lamb_plan(_ptr(sizes), sizes.numel(), None)
    check(min(0, n_chunks))
    plan = torch.empty((n_chunks, 5), dtype=torch.int64)
    check(min(0, lib().hrl_lamb_plan(_ptr(sizes), sizes.numel(), _ptr(plan))))
    return plan


class FlatLamb(FlatAdam):
    """clip_grad_norm_(max_norm) + LAMB (You et al., 2020, Algorithm 2) on FlatAdam's bucket: Adam's moments, the decay
    added to the update direction u instead of the gradient, and one trust ratio r_i = |w_i| / |u_i| per parameter (1 when
    either norm is 0), so w_i <- w_i - lr * lr_scale * r_i * u_i (hrl_clip_lamb_step).  The parameters' spans of the bucket
    are cut into chunks (`plan`, lamb_plan) whose fp64 partial norms (`chunk_sums`) fold in a fixed order; `update` is the
    scratch bucket for u.  `ratio`: None, or a float32 CUDA tensor of one entry per parameter that every step fills with the
    r_i it applied.  Everything else -- buffers, guard, diagnostics, the peer all-reduce path -- is FlatAdam's."""

    def __init__(self, params, lr, lr_scale=1.0, **kw):
        super().__init__(params, lr, **kw)
        device = self.flat_param.device
        self.lr_scale = float(lr_scale)
        self.plan = lamb_plan([p.numel() for p in self.params]).to(device)
        self.update = torch.zeros(self.n_pad, dtype=torch.float32, device=device)
        self.chunk_sums = torch.zeros(2 * self.plan.shape[0], dtype=torch.float64, device=device)
        self.ratio = None

    def step_reduced(self, reduced):
        """clip + LAMB on an already all-reduced bucket whose sum-of-squares partials are in self.partials."""
        self._clip_lamb(reduced, _stream_ptr())
        _count(3)

    def _clip_lamb(self, grad, s):
        if self.diag is not None:
            assert self.diag.is_cuda and self.diag.dtype == torch.float64 and self.diag.numel() == 4 and self.diag.is_contiguous()
        if self.skip is not None:
            assert self.skip.is_cuda and self.skip.dtype == torch.int32 and self.skip.numel() == 1
            assert 0 <= self.guard_tail <= self.extra and grad.numel() >= self.n_pad + self.extra
        if self.ratio is not None:
            assert self.ratio.is_cuda and self.ratio.dtype == torch.float32 and self.ratio.numel() == len(self.params)
        check(lib().hrl_clip_lamb_step(
            _ptr(self.flat_param), _ptr(grad), _ptr(self.exp_avg), _ptr(self.exp_avg_sq), _ptr(self.update), self.n_pad,
            _ptr(self.plan), self.plan.shape[0], _ptr(self.chunk_sums), _ptr(self.partials), _ptr(self.lr), _ptr(self.step_count),
            self.max_norm, self.betas[0], self.betas[1], self.eps, self.weight_decay, self.lr_scale, _ptr(self.grad_norm),
            _ptr(self.diag), _ptr(grad[self.n_pad:]), self.guard_tail, _ptr(self.skip), _ptr(self.ratio), s))

    def step(self):
        s = _stream_ptr()
        check(lib().hrl_grad_sumsq(_ptr(self.flat_grad), self.n_pad, _ptr(self.partials), s))
        self._clip_lamb(self.flat_grad, s)
        _count(4)
        from . import fastnet
        fastnet.new_step()          # cached adjoint weights of the convolutions are stale now


MUON_KINDS = ('adam', 'matrix', 'too_large')     # HrlMuonKind


def muon_plan(shapes):
    """hrl_muon_plan on the host for parameters of `shapes` laid out back to back from word 0: (kinds, mats, spans) with
    kinds[i] in MUON_KINDS -- 'matrix' for a Muon-owned tensor, 'too_large' for a matrix outside the kernel's envelope
    (Adam-owned), 'adam' for the rest -- mats the (matrices, 4) int64 CPU tensor {first word, r, k, transposed} and spans the
    (spans, 2) int64 CPU tensor {first word, words} of the Adam-owned words."""
    shapes = [tuple(int(d) for d in s) for s in shapes]
    dims = torch.tensor([d for s in shapes for d in s] or [0], dtype=torch.int64)
    ndim = torch.tensor([len(s) for s in shapes], dtype=torch.int32)
    kind = torch.zeros(len(shapes), dtype=torch.int32)
    counts = torch.zeros(2, dtype=torch.int32)
    check(lib().hrl_muon_plan(_ptr(dims), _ptr(ndim), len(shapes), _ptr(kind), _ptr(counts), None, None))
    mats = torch.zeros((int(counts[0]), 4), dtype=torch.int64)
    spans = torch.zeros((int(counts[1]), 2), dtype=torch.int64)
    check(lib().hrl_muon_plan(_ptr(dims), _ptr(ndim), len(shapes), _ptr(kind), _ptr(counts), _ptr(mats), _ptr(spans)))
    return [MUON_KINDS[int(k)] for k in kind], mats, spans


class FlatMuon(FlatAdam):
    """clip_grad_norm_(max_norm) + Muon on FlatAdam's bucket (hrl_clip_muon_step): each Muon-owned weight matrix (muon_plan)
    takes its Nesterov momentum (mu = 0.95, kept in exp_avg; its exp_avg_sq stays zero) orthogonalised by five Newton-Schulz
    iterations on bf16 tensor-core products, scaled by lr_scale * 0.2 * sqrt(max(r, k)), with decoupled weight decay; every
    other word takes FlatAdam's update bit for bit.  `names` (optional, one per parameter) name the parameters; `muon_params`
    lists the names (or indices) of the Muon-owned ones.  `ortho`: None, or a float32 CUDA tensor of n_pad words that every
    step fills with O at the matrices' words.  Everything else -- buffers, guard, diagnostics, the peer all-reduce path -- is
    FlatAdam's, and a step takes as many launches as FlatAdam's."""

    def __init__(self, params, lr, lr_scale=1.0, names=None, **kw):
        params = list(params)
        super().__init__(params, lr, **kw)
        device = self.flat_param.device
        self.lr_scale = float(lr_scale)
        names = list(range(len(params))) if names is None else list(names)
        assert len(names) == len(params)
        self.kinds, mats, spans = muon_plan([tuple(p.shape) for p in params])
        self.muon_params = [k for k, kind in zip(names, self.kinds) if kind == 'matrix']
        self.mats, self.spans = mats.to(device), spans.to(device)
        self.ortho = None

    def step_reduced(self, reduced):
        """clip + Muon on an already all-reduced bucket whose sum-of-squares partials are in self.partials."""
        self._clip_muon(reduced, _stream_ptr())
        _count(2)

    def _clip_muon(self, grad, s):
        if self.diag is not None:
            assert self.diag.is_cuda and self.diag.dtype == torch.float64 and self.diag.numel() == 4 and self.diag.is_contiguous()
        if self.skip is not None:
            assert self.skip.is_cuda and self.skip.dtype == torch.int32 and self.skip.numel() == 1
            assert 0 <= self.guard_tail <= self.extra and grad.numel() >= self.n_pad + self.extra
        if self.ortho is not None:
            assert self.ortho.is_cuda and self.ortho.dtype == torch.float32 and self.ortho.numel() >= self.n_pad
        check(lib().hrl_clip_muon_step(
            _ptr(self.flat_param), _ptr(grad), _ptr(self.exp_avg), _ptr(self.exp_avg_sq), self.n_pad,
            _ptr(self.mats), self.mats.shape[0], _ptr(self.spans), self.spans.shape[0], _ptr(self.partials), _ptr(self.lr),
            _ptr(self.step_count), self.max_norm, self.betas[0], self.betas[1], self.eps, self.weight_decay, self.lr_scale,
            _ptr(self.grad_norm), _ptr(self.diag), _ptr(grad[self.n_pad:]), self.guard_tail, _ptr(self.skip), _ptr(self.ortho), s))

    def step(self):
        s = _stream_ptr()
        check(lib().hrl_grad_sumsq(_ptr(self.flat_grad), self.n_pad, _ptr(self.partials), s))
        self._clip_muon(self.flat_grad, s)
        _count(3)
        from . import fastnet
        fastnet.new_step()          # cached adjoint weights of the convolutions are stale now


def _check_skip(skip):
    if not (skip.is_cuda and skip.dtype == torch.int32 and skip.numel() == 1):
        raise _capi.HrlError('handyrl_b200: skip must be a one-element int32 CUDA tensor')


def weight_ema_update(avg, state_f32, step_count, decay, seeded, skip=None):
    """avg <- fmaf(w, state_f32 - avg, avg) in place, w = max(1 - decay, 1 / t) (1 - decay when `seeded`), t = the int64 device
    counter `step_count` as it stands when the launch runs (hrl_weight_ema, csrc/optim_kernel.cu).  One launch, graph-capturable.
    `skip` (FlatAdam.skip of a guarded optimiser, or None): the launch changes nothing when that step was rejected."""
    for t, name in ((avg, 'avg'), (state_f32, 'state_f32')):
        if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()):
            raise _capi.HrlError('handyrl_b200: %s must be a contiguous float32 CUDA tensor' % name)
    if avg.numel() != state_f32.numel():
        raise _capi.HrlError('handyrl_b200: avg (%d) and state_f32 (%d) differ in size' % (avg.numel(), state_f32.numel()))
    if not (step_count.is_cuda and step_count.dtype == torch.int64 and step_count.numel() == 1):
        raise _capi.HrlError('handyrl_b200: step_count must be a one-element int64 CUDA tensor')
    if skip is not None:
        _check_skip(skip)
    check(lib().hrl_weight_ema(_ptr(avg), _ptr(state_f32), avg.numel(), _ptr(step_count), float(decay), int(bool(seeded)),
                               _ptr(skip), _stream_ptr()))
    _count()


def sum_rows(rows, n, out):
    """out[:n] = the sum of the rows of the (k, ld) float32 CUDA tensor `rows` over their first n columns, in row order in
    float64 and rounded once (hrl_sum_rows: the loss-pass sums of a gradient-accumulation step into the bucket tail).  One
    launch, bit-reproducible."""
    for t, name in ((rows, 'rows'), (out, 'out')):
        if not (t.is_cuda and t.dtype == torch.float32 and t.stride(-1) == 1):
            raise _capi.HrlError('handyrl_b200: %s must be a float32 CUDA tensor with unit column stride' % name)
    if rows.dim() != 2 or not 1 <= n <= rows.shape[1] or out.numel() < n:
        raise _capi.HrlError('handyrl_b200: sum_rows needs (k, ld) rows with ld >= n and n <= out.numel()')
    check(lib().hrl_sum_rows(_ptr(rows), rows.shape[0], rows.stride(0), int(n), _ptr(out), _stream_ptr()))
    _count()


def step_commit(skip, tail, accum, skip_count, state=None, saved=None):
    """What follows a guarded optimiser step (hrl_step_commit, one launch reading the device flag `skip`): when the step was
    accepted, accum[:tail.numel()] += tail (float32 sums into the float64 accumulator, as ATen's add_ does); when it was
    rejected, skip_count += 1 and the bytes of `saved` go back to `state` (both uint8 CUDA tensors of one size, or None)."""
    _check_skip(skip)
    if not (tail.is_cuda and tail.dtype == torch.float32 and tail.is_contiguous()):
        raise _capi.HrlError('handyrl_b200: tail must be a contiguous float32 CUDA tensor')
    for t, name in ((accum, 'accum'), (skip_count, 'skip_count')):
        if not (t.is_cuda and t.dtype == torch.float64 and t.is_contiguous()):
            raise _capi.HrlError('handyrl_b200: %s must be a contiguous float64 CUDA tensor' % name)
    if accum.numel() < tail.numel() or skip_count.numel() != 1:
        raise _capi.HrlError('handyrl_b200: accum holds %d of the %d tail sums, or skip_count is not one element'
                             % (accum.numel(), tail.numel()))
    lo, hi = skip_count.data_ptr(), skip_count.data_ptr() + 8
    if tail.numel() and lo < accum.data_ptr() + 8 * tail.numel() and accum.data_ptr() < hi:
        raise _capi.HrlError('handyrl_b200: skip_count lies inside the accumulated sums')
    nbytes = 0
    if state is not None or saved is not None:
        if state is None or saved is None:
            raise _capi.HrlError('handyrl_b200: state and saved come in pairs')
        for t, name in ((state, 'state'), (saved, 'saved')):
            if not (t.is_cuda and t.dtype == torch.uint8 and t.is_contiguous()):
                raise _capi.HrlError('handyrl_b200: %s must be a contiguous uint8 CUDA tensor' % name)
        if state.numel() != saved.numel():
            raise _capi.HrlError('handyrl_b200: state (%d) and saved (%d) differ in size' % (state.numel(), saved.numel()))
        nbytes = state.numel()
    check(lib().hrl_step_commit(_ptr(skip), _ptr(tail), tail.numel(), _ptr(accum), _ptr(skip_count),
                                _ptr(state) if nbytes else None, _ptr(saved) if nbytes else None, nbytes, _stream_ptr()))
    _count()


def replay_sample(state, replay, head, count, args, windows, seed, counter, solo):
    """Launch hrl_replay_sample (one kernel on the current stream): draw state.B windows of the replay `replay` (a
    DeviceReplay keeping its directory mirror) by prioritised replay, into `windows` (a (B, 32) uint8 CUDA tensor, the
    gather's descriptor buffer) and state.win_slot / win_serial / win_weight.  head, count: the directory snapshot the host
    took under the replay lock; seed, counter: the Philox key and this batch's counter."""
    if replay.dir_dev is None:
        raise _capi.HrlError('handyrl_b200: the replay keeps no device directory (DeviceReplay(..., mirror=True))')
    if replay.dir_dev.shape[0] != state.ring:
        raise _capi.HrlError('handyrl_b200: the replay directory has %d slots, the priorities %d' % (replay.dir_dev.shape[0], state.ring))
    if not (windows.is_cuda and windows.dtype == torch.uint8 and windows.is_contiguous() and windows.numel() == 32 * state.B):
        raise _capi.HrlError('handyrl_b200: windows must be a contiguous uint8 CUDA buffer of %d descriptors' % state.B)
    g = _capi.HrlReplaySampleArgs()
    g.B, g.ring, g.head, g.count = state.B, state.ring, int(head), int(count)
    g.burn_in, g.forward_steps = int(args.get('burn_in_steps', 0)), int(args['forward_steps'])
    g.Ps, g.solo = int(replay.Ps), int(bool(solo))
    g.alpha, g.beta = state.alpha, state.beta
    g.seed, g.counter = int(seed) % (1 << 64), int(counter) % (1 << 64)
    g.dir, g.prio, g.prio_serial, g.max_prio = _ptr(replay.dir_dev), _ptr(state.prio), _ptr(state.prio_serial), _ptr(state.max_prio)
    g.workspace, g.windows = _ptr(state.cdf), _ptr(windows)
    g.win_slot, g.win_serial, g.win_weight = _ptr(state.win_slot), _ptr(state.win_serial), _ptr(state.win_weight)
    check(lib().hrl_replay_sample(C.byref(g), _stream_ptr()))
    _count()


def priority_update(state, advantage, turn_mask, burn_in, skip=None):
    """Launch hrl_replay_priority_update (one kernel on the current stream): the window priorities of this step's
    advantage tap and turn mask ((B, T, P[, 1]) float32 CUDA tensors) go to state.prio where the windows' serials still
    match, and raise state.max_prio.  skip: the guarded optimiser's flag (nothing is written when it is set), or None."""
    for t, name in ((advantage, 'advantage'), (turn_mask, 'turn_mask')):
        if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and t.shape[0] == state.B):
            raise _capi.HrlError('handyrl_b200: %s must be a contiguous float32 CUDA tensor of %d windows' % (name, state.B))
    if advantage.shape[:3] != turn_mask.shape[:3]:
        raise _capi.HrlError('handyrl_b200: advantage %s and turn_mask %s differ in shape' % (tuple(advantage.shape), tuple(turn_mask.shape)))
    if skip is not None:
        _check_skip(skip)
    B, T, P = turn_mask.shape[:3]
    check(lib().hrl_replay_priority_update(B, T, P, int(burn_in), _ptr(advantage), _ptr(turn_mask), float(state.epsilon),
                                           _ptr(state.win_slot), _ptr(state.win_serial), _ptr(state.prio), _ptr(state.prio_serial),
                                           _ptr(state.max_prio), _ptr(skip), _stream_ptr()))
    _count()


# K slices of a product: one CTA computes one output tile (_TILE_ROWS x _TILE_COLS) over one K slice, and a product is split over
# as many slices as keep the _SMS SMs of an H100 busy, with at least _MIN_SLICE_K elements of K per slice
_TILE_ROWS, _TILE_COLS, _SMS, _MIN_SLICE_K = 128, 288, 132, 64


def k_splits(rows, cols, K, segments=1):
    """K slices for a product of rows x cols outputs reducing over K (each of `segments` pairs of a segmented product getting its
    own), counted as the library produces them (hrl_gemm_effective_splits: whole 32-element chunks, no empty slice)."""
    tiles = -(-rows // _TILE_ROWS) * -(-cols // _TILE_COLS)
    return lib().hrl_gemm_effective_splits(K, max(1, min(K // _MIN_SLICE_K, _SMS // (tiles * segments))))


def _operand(o, t, t2=None, consts=None, relu=False, kmajor=True, by_row=False, packed=False):
    o.ptr, o.ptr2 = _ptr(t), _ptr(t2)
    o.ld = 0 if packed else t.stride(0)
    o.kmajor, o.relu, o.feature_is_row, o.packed = int(kmajor), int(relu), int(by_row), int(packed)
    if consts is not None:
        o.p, o.r = _ptr(consts[0]), _ptr(consts[-1])
        o.q = _ptr(consts[1]) if len(consts) == 3 else None


def gemm_fused(a, b, M, N, K, out=None, ws=None, splits=1, bias=None, epilogue='store', ep=None, col_partials=None, bf16=False,
               conv=None, ones_row=False, segments=None):
    """One hrl_gemm_fused launch (csrc/gemm_kernel.cu): C[M x N] = A_op @ B_op^T with the operands' transforms and the epilogue.

    a, b: keyword arguments of _operand (the tensor `t` and its layout / transform).  out: C, or None to leave the product in
    `ws` as its K-slice partials, M*N floats apart (one slice: the product itself).  ws: the workspace of a split or segmented
    product (hrl_gemm_workspace_floats floats).  ep: the epilogue's tensors by name (y, scale, shift, mean, rstd).
    conv: (conv_mode, neighbour table, cells, taps, channels) of an implicit convolution product; ones_row: its bias-gradient
    column.  segments: the (dy, x) pairs of a segmented weight gradient.
    Counts the launch, and the library's sum of the slice partials into `out`."""
    g = _capi.HrlGemmArgs()
    _operand(g.a, **a)
    _operand(g.b, **b)
    g.M, g.N, g.K, g.splits, g.bf16 = M, N, K, splits, int(bf16)
    g.bias, g.epilogue, g.col_partials = _ptr(bias), GEMM_EPILOGUES[epilogue], _ptr(col_partials)
    split = splits > 1 or segments is not None
    if out is not None:
        g.C, g.ldc = _ptr(out), out.stride(0)
    else:
        g.C, g.ldc = (None if split else _ptr(ws)), N
    g.workspace = _ptr(ws) if split else None
    if ep is not None:
        if 'y' in ep:
            g.ep_y, g.ep_ldy = _ptr(ep['y']), ep['y'].stride(0)
        g.ep_scale, g.ep_shift = _ptr(ep.get('scale')), _ptr(ep.get('shift'))
        g.ep_mean, g.ep_rstd = _ptr(ep.get('mean')), _ptr(ep.get('rstd'))
    if conv is not None:
        g.conv_mode, g.conv_off, g.conv_hw, g.conv_taps, g.conv_cin = conv[0], _ptr(conv[1]), *conv[2:]
        g.conv_ones_row = int(ones_row)
    if segments is not None:
        seg_a = (C.c_void_p * len(segments))(*[dy.data_ptr() for dy, _ in segments])
        seg_b = (C.c_void_p * len(segments))(*[x.data_ptr() for _, x in segments])
        g.seg_a, g.seg_b, g.segments = C.cast(seg_a, C.c_void_p), C.cast(seg_b, C.c_void_p), len(segments)
    check(lib().hrl_gemm_fused(C.byref(g), _stream_ptr()))
    _count(2 if out is not None and splits > 1 and lib().hrl_gemm_effective_splits(K, splits) > 1 else 1)


def _gemm_dense(a, b, bias, a_kmajor, b_kmajor, splits, out, partials, bf16):
    assert a.is_cuda and b.is_cuda and a.dtype == torch.float32 and b.dtype == torch.float32
    assert a.dim() == 2 and b.dim() == 2 and a.stride(1) == 1 and b.stride(1) == 1
    M, K = (a.shape[0], a.shape[1]) if a_kmajor else (a.shape[1], a.shape[0])
    N, Kb = (b.shape[0], b.shape[1]) if b_kmajor else (b.shape[1], b.shape[0])
    assert K == Kb, (a.shape, b.shape, a_kmajor, b_kmajor)
    ws = partials
    if partials is not None:
        out = None
    else:
        if out is None:
            out = torch.empty((M, N), dtype=torch.float32, device=a.device)
        if splits > 1:
            ws = torch.empty(lib().hrl_gemm_workspace_floats(M, N, K, splits), dtype=torch.float32, device=a.device)
    gemm_fused(dict(t=a, kmajor=a_kmajor), dict(t=b, kmajor=b_kmajor), M, N, K, out=out, ws=ws, splits=splits, bias=bias, bf16=bf16)
    return out


def gemm_tf32x3(a, b, bias=None, a_kmajor=True, b_kmajor=True, splits=1, out=None):
    """C = A_op @ B_op^T (+ bias) on the tensor cores with fp32-class accuracy (3xTF32, hrl_gemm_fused).

    a: (M, K) if a_kmajor else (K, M) -- the operand as it lies in memory; b likewise (N, K) / (K, N).
    """
    return _gemm_dense(a, b, bias, a_kmajor, b_kmajor, splits, out, None, False)


def gemm_bf16(a, b, bias=None, a_kmajor=True, b_kmajor=True, splits=1, out=None, partials=None):
    """C = A_op @ B_op^T on the tensor cores with bf16 operands (hrl_gemm_fused with HrlGemmArgs.bf16): both operands rounded to
    the nearest bf16, products accumulated in fp32.  Layouts as gemm_tf32x3.  partials: a workspace of
    hrl_gemm_workspace_floats floats that receives the K-slice partials instead of C (no sum, nothing returned)."""
    return _gemm_dense(a, b, bias, a_kmajor, b_kmajor, splits, out, partials, True)


class _LinearTC(torch.autograd.Function):
    """y = x @ w^T with all three products (forward, input gradient, weight gradient) on the tensor cores at fp32-class
    accuracy (gemm_tf32x3).  The weight gradient reduces over the rows of x (samples): both operands are read
    transposed on the fly and the reduction is split over enough K slices to fill the GPU."""

    @staticmethod
    def forward(ctx, x, w):
        x, w = x.contiguous(), w.contiguous()
        ctx.save_for_backward(x, w)
        return gemm_tf32x3(x, w)

    @staticmethod
    def backward(ctx, dy):
        x, w = ctx.saved_tensors
        dy = dy.contiguous()
        dx = dw = None
        if ctx.needs_input_grad[0]:
            dx = gemm_tf32x3(dy, w, b_kmajor=False)                       # (M,N) x (N,K): w is read as stored
        if ctx.needs_input_grad[1]:
            dw = gemm_tf32x3(dy, x, a_kmajor=False, b_kmajor=False, splits=k_splits(w.shape[0], w.shape[1], x.shape[0]))
        return dx, dw


def linear_tc(x, w):
    return _LinearTC.apply(x, w)


class _BoardDense(torch.autograd.Function):
    """Dense matrix of a small-board convolution from its weight (hrl_board_expand) and the adjoint (hrl_board_fold)."""

    @staticmethod
    def forward(ctx, weight, H, W):
        weight = weight.contiguous()
        Cout, Cin, kh, kw = weight.shape
        ctx.dims = (Cout, Cin, kh, kw, H, W)
        dense = torch.empty((Cout * H * W, Cin * H * W), dtype=torch.float32, device=weight.device)
        check(lib().hrl_board_expand(_ptr(weight), _ptr(dense), Cout, Cin, kh, kw, H, W, _stream_ptr()))
        _count()
        return dense

    @staticmethod
    def backward(ctx, ddense):
        Cout, Cin, kh, kw, H, W = ctx.dims
        ddense = ddense.contiguous()
        dw = torch.empty((Cout, Cin, kh, kw), dtype=torch.float32, device=ddense.device)
        check(lib().hrl_board_fold(_ptr(ddense), 1, 0, _ptr(dw), Cout, Cin, kh, kw, H, W, _stream_ptr()))
        _count()
        return dw, None, None


def board_dense(weight, H, W):
    return _BoardDense.apply(weight, H, W)


class _BoardConv(torch.autograd.Function):
    """A stride-1 "same" convolution over a tiny board, NCHW in and out, as dense products on the tensor cores:
    forward   y = x2d @ dense(w)^T            (hrl_board_expand + hrl_gemm_fused)
    backward  dx = dy2d @ dense(w)            (hrl_gemm_fused, the dense matrix read as stored)
              dw = fold(sum_s dy2d_s^T x2d_s) (split-K hrl_gemm_fused leaving its slice partials, folded AND summed by
                                               one hrl_board_fold launch: no dense gradient is ever materialised)
    The products are 3xTF32 (gemm_tf32x3), or with bf16 on bf16 operands (gemm_bf16); the dense matrix and the fold stay fp32."""

    @staticmethod
    def forward(ctx, x, weight, bf16=False):
        x = x.contiguous()
        weight = weight.contiguous()
        N, Cin, H, W = x.shape
        Cout, _, kh, kw = weight.shape
        dense = torch.empty((Cout * H * W, Cin * H * W), dtype=torch.float32, device=x.device)
        check(lib().hrl_board_expand(_ptr(weight), _ptr(dense), Cout, Cin, kh, kw, H, W, _stream_ptr()))
        _count()
        y = (gemm_bf16 if bf16 else gemm_tf32x3)(x.view(N, Cin * H * W), dense)
        ctx.save_for_backward(x, dense)
        ctx.dims = (N, Cin, H, W, Cout, kh, kw)
        ctx.bf16 = bf16
        return y.view(N, Cout, H, W)

    @staticmethod
    def backward(ctx, dy):
        x, dense = ctx.saved_tensors
        N, Cin, H, W, Cout, kh, kw = ctx.dims
        dy2 = dy.contiguous().view(N, Cout * H * W)
        x2 = x.view(N, Cin * H * W)
        dx = dw = None
        gemm = gemm_bf16 if ctx.bf16 else gemm_tf32x3
        if ctx.needs_input_grad[0]:
            dx = gemm(dy2, dense, b_kmajor=False).view(N, Cin, H, W)
        if ctx.needs_input_grad[1]:
            rows, cols = Cout * H * W, Cin * H * W
            splits = k_splits(rows, cols, N)
            dw = torch.empty((Cout, Cin, kh, kw), dtype=torch.float32, device=dy.device)
            ws = torch.empty(splits * rows * cols, dtype=torch.float32, device=dy.device)
            gemm_fused(dict(t=dy2, kmajor=False), dict(t=x2, kmajor=False), rows, cols, N, ws=ws, splits=splits, bf16=ctx.bf16)
            check(lib().hrl_board_fold(_ptr(ws), splits, rows * cols, _ptr(dw), Cout, Cin, kh, kw, H, W, _stream_ptr()))
            _count()
        return dx, dw, None


def board_conv(x, weight, bf16=False):
    """bf16: the products on bf16 operands (fastnet.optimize_small_boards(model, tensor_cores='bf16'))."""
    return _BoardConv.apply(x, weight, bool(bf16))


# ---- stride-1 "same" / wrap-around convolutions as implicit tensor-core products (hrl_gemm_fused conv_mode 1 / 2) -----------
_CONV_TABLES = {}        # (H, W, kh, kw, wrap, device) -> int16 neighbour-offset table on the device
_CONV_IMAGES = {}        # (weight ptr, shape, bf16) -> [forward image, adjoint image, generation they were packed in, weight ref]
_CONV_GENERATION = [0]   # bumped whenever the parameters may have changed (fastnet.new_step)


def conv_weights_changed():
    _CONV_GENERATION[0] += 1


def _conv_table(H, W, kh, kw, wrap, device):
    key = (H, W, kh, kw, bool(wrap), str(device))
    t = _CONV_TABLES.get(key)
    if t is None:
        import numpy as np
        host = np.empty(H * W * kh * kw, dtype=np.int16)
        check(lib().hrl_conv_geometry(H, W, kh, kw, int(bool(wrap)), host.ctypes.data))
        t = _CONV_TABLES[key] = torch.from_numpy(host).to(device)
    return t


def _conv_images(w, bf16=False):
    """The weight's packed forward / adjoint operand images, re-packed once per parameter generation.  (Keyed by address AND
    identity: a freed model's weight address can be handed to another tensor of the same shape; and by precision: bf16 images
    (hrl_conv_pack_bf16, a quarter of the size) for the bf16 products.)"""
    import weakref
    Cout, Cin, kh, kw = w.shape
    key = (w.data_ptr(), tuple(w.shape), bool(bf16))
    ent = _CONV_IMAGES.get(key)
    if ent is None or ent[3]() is not w:
        if ent is None:
            z = lambda rows, ch: torch.zeros(lib().hrl_conv_pack_floats(rows, ch, kh * kw) // (4 if bf16 else 1), dtype=torch.float32,
                                             device=w.device)
            ent = _CONV_IMAGES[key] = [z(Cout, Cin), z(Cin, Cout), None, None]
        ent[2], ent[3] = None, weakref.ref(w)
    gen = (_CONV_GENERATION[0], w._version)
    if ent[2] != gen:
        pack = lib().hrl_conv_pack_bf16 if bf16 else lib().hrl_conv_pack
        check(pack(_ptr(w), Cout, Cin, kh, kw, _ptr(ent[0]), _ptr(ent[1]), _stream_ptr()))
        _count()
        ent[2] = gen
    return ent[0], ent[1]


def conv_implicit_supported(x, w):
    """Shapes the implicit products cover: fp32 CUDA, at most 256 cells and 9 taps, channel counts that are multiples of 4 (16-byte
    pixel rows) and at most 288 (one operand tile)."""
    if not (x.is_cuda and x.dtype == torch.float32 and w.dtype == torch.float32 and x.dim() == 4):
        return False
    Cout, Cin, kh, kw = w.shape
    return (x.shape[2] * x.shape[3] <= 256 and kh * kw <= 9 and kh % 2 == 1 and kw % 2 == 1 and Cin % 4 == 0 and Cout % 4 == 0
            and Cin <= 288 and Cout <= 288 and x.shape[1] == Cin)


def _pixels(t):
    """(N, C, H, W) tensor -> its channels-last (N*H*W, C) view (copying only if it is not channels-last already)."""
    t = t.contiguous(memory_format=torch.channels_last)
    return t, t.permute(0, 2, 3, 1).reshape(-1, t.shape[1])


def _conv_product(pix, image, rows, cin, taps, table, hw, bias=None, bf16=False):
    """out[pixel][row] = sum over (tap, channel) of pix[neighbour(pixel, tap)][channel] * image[row][tap, channel]"""
    M = pix.shape[0]
    out = torch.empty((M, rows), dtype=torch.float32, device=pix.device)
    gemm_fused(dict(t=pix), dict(t=image, packed=True), M, rows, taps * ((cin + 31) // 32 * 32), out=out, bias=bias,
               conv=(1, table, hw, taps, cin), bf16=bf16)
    return out


# Deferred weight gradients.  A recurrent net applies the same convolution at every time step (and DRC cells several times per step):
# computing its weight gradient per application means T x repeats small products, slice reductions and gradient accumulations --
# ~1,000 launches of a 4,400-launch Geister step, in a chain that is launch-bound.  Inside `deferred_weight_gradients()` the backward of
# conv_implicit only records its (dy, x) pair; on exit ONE segmented product per weight and board geometry reduces over all its pairs
# (hrl_gemm_fused with `segments`), its ones row yields the bias gradient, and hrl_conv_wgrad_reduce2 adds the result into
# weight.grad / bias.grad.
_DEFER = {'on': False, 'pending': {}}


class deferred_weight_gradients:
    def __enter__(self):
        assert not _DEFER['on']
        _DEFER['on'], _DEFER['pending'] = True, {}
        return self

    def __exit__(self, exc_type, exc, tb):
        pending, _DEFER['pending'], _DEFER['on'] = _DEFER['pending'], {}, False
        if exc_type is None:
            for job in pending.values():
                _flush_weight_gradient(job)
        return False


def _flush_weight_gradient(job):
    w, b, pairs = job['w'], job['b'], job['pairs']
    Cout, Cin, kh, kw = w.shape
    taps, (table, hw) = kh * kw, job['geom']
    # the ones row (bias gradient as one more column) is free unless that column opens a new 288-wide tile AND the extra tile's CTAs
    # take K slices away from the others (a weight used once: 1 tile x 132 slices vs 2 tiles x 66): then a column sum does it
    cols, pixels = taps * Cin, pairs[0][0].shape[0]
    n0 = min(len(pairs), 64)
    ones = b is not None and k_splits(Cout, cols + 1, pixels, n0) >= k_splits(Cout, cols, pixels, n0)
    if b is not None and not ones:
        if b.grad is None:
            b.grad = torch.zeros_like(b)
        for dy2, _ in pairs:
            b.grad.add_(dy2.sum(0))
    ncols = cols + (1 if ones else 0)
    for start in range(0, len(pairs), 64):
        chunk = pairs[start:start + 64]
        n = len(chunk)
        per = k_splits(Cout, ncols, pixels, n)
        ws = torch.empty((n * per, Cout, ncols), dtype=torch.float32, device=w.device)
        gemm_fused(dict(t=chunk[0][0], kmajor=False), dict(t=chunk[0][1], kmajor=False), Cout, ncols, pixels, ws=ws, splits=per,
                   conv=(2, table, hw, taps, Cin), ones_row=ones, segments=chunk, bf16=job['bf16'])
        for t, shape in ((w, w.shape), (b, None)):
            if t is not None and t.grad is None:
                t.grad = torch.zeros_like(t, memory_format=torch.contiguous_format)
        assert w.grad.is_contiguous()
        check(lib().hrl_conv_wgrad_reduce2(_ptr(ws), n * per, ncols, _ptr(w.grad), _ptr(b.grad) if ones else None, Cout, Cin, taps, 1,
                                           _stream_ptr()))
        _count()


class _ConvImplicit(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b, wrap, bf16=False):
        N, Cin, H, W = x.shape
        Cout, _, kh, kw = w.shape
        table = _conv_table(H, W, kh, kw, wrap, x.device)
        fwd, _ = _conv_images(w, bf16)
        xl, x2 = _pixels(x)
        y2 = _conv_product(x2, fwd, Cout, Cin, kh * kw, table, H * W, bias=b, bf16=bf16)
        ctx.save_for_backward(xl, w)
        ctx.wrap, ctx.has_bias, ctx.bf16 = wrap, b is not None, bf16
        ctx.params = (w, b)             # the Parameter objects themselves (their .grad is what a deferred flush accumulates into)
        return y2.view(N, H, W, Cout).permute(0, 3, 1, 2)           # logical NCHW, channels-last in memory

    @staticmethod
    def backward(ctx, dy):
        xl, w = ctx.saved_tensors
        N, Cin, H, W = xl.shape
        Cout, _, kh, kw = w.shape
        taps = kh * kw
        table = _conv_table(H, W, kh, kw, ctx.wrap, xl.device)
        dyl, dy2 = _pixels(dy)
        dx = dw = db = None
        pw, pb = ctx.params
        if ctx.needs_input_grad[0]:
            _, adj = _conv_images(pw, ctx.bf16)           # (the object forward saw: the image cache checks identity)
            dx = _conv_product(dy2, adj, Cin, Cout, taps, table, H * W, bf16=ctx.bf16).view(N, H, W, Cin).permute(0, 3, 1, 2)
        if (ctx.needs_input_grad[1] and _DEFER['on'] and pw.is_leaf and (pb is None or (pb.is_leaf and ctx.needs_input_grad[2]))
                and (pw.grad is None or pw.grad.is_contiguous())):
            # one job per board geometry: its product reads every pair through the job's neighbour table (a weight applied to
            # two board shapes, or with both paddings, gets one flush per geometry, each adding into the same .grad)
            job = _DEFER['pending'].setdefault((pw.data_ptr(), ctx.bf16, H, W, ctx.wrap),
                                               {'w': pw, 'b': pb, 'pairs': [], 'geom': (table, H * W), 'bf16': ctx.bf16})
            if not job['pairs'] or job['pairs'][0][0].shape[0] == dy2.shape[0]:      # (pairs of one product cover the same pixels)
                job['pairs'].append((dy2, xl.permute(0, 2, 3, 1).reshape(-1, Cin)))
                return dx, None, None, None, None
        if ctx.needs_input_grad[1]:
            x2 = xl.permute(0, 2, 3, 1).reshape(-1, Cin)
            pixels, cols = x2.shape[0], taps * Cin
            s = k_splits(Cout, cols, pixels)
            ws = torch.empty((s, Cout, cols), dtype=torch.float32, device=xl.device)
            gemm_fused(dict(t=dy2, kmajor=False), dict(t=x2, kmajor=False), Cout, cols, pixels, ws=ws, splits=s,
                       conv=(2, table, H * W, taps, Cin), bf16=ctx.bf16)
            dw = torch.empty_like(w, memory_format=torch.contiguous_format)
            check(lib().hrl_conv_wgrad_reduce(_ptr(ws), s, _ptr(dw), Cout, Cin, taps, _stream_ptr()))
            _count()
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = dy2.sum(0)
        return dx, dw, db, None, None


def conv_implicit(x, w, b=None, wrap=False, bf16=False):
    """Stride-1 convolution with `same` zero padding (wrap=False) or wrap-around padding on both axes (wrap=True) of a board of at most
    256 cells, forward / input gradient / weight gradient on the tensor cores at fp32-class accuracy (3xTF32), or with bf16=True on
    bf16 operands (rounded to nearest even, fp32 accumulation; bias and bias gradient stay fp32)."""
    return _ConvImplicit.apply(x, w, b, bool(wrap), bool(bf16))


def _is_channels_last(t):
    return t.dim() == 4 and t.is_contiguous(memory_format=torch.channels_last) and not t.is_contiguous()


class _LstmGates(torch.autograd.Function):
    """The kernels index (sample, 4 gates x CS, ...) blocks.  A channels-last tensor is exactly that with sample := pixel and
    CS := C (the gate maps of one pixel are contiguous), so channels-last gates (what the tensor-core convolution produces) are
    processed in place, no layout copy, and h', c' come out channels-last for the next convolution."""

    @staticmethod
    def forward(ctx, gates, c_prev):
        cl = _is_channels_last(gates)
        fmt = torch.channels_last if cl else torch.contiguous_format
        gates, c_prev = gates.contiguous(memory_format=fmt), c_prev.contiguous(memory_format=fmt)
        N, C4 = gates.shape[:2]
        S = gates[0, 0].numel()
        h, c = torch.empty_like(c_prev), torch.empty_like(c_prev)          # (preserve_format: channels-last stays channels-last)
        dims = (N * S, C4 // 4, 1) if cl else (N, C4 // 4, S)
        check(lib().hrl_lstm_gates_fwd(_ptr(gates), _ptr(c_prev), _ptr(h), _ptr(c), *dims, _stream_ptr()))
        _count()
        ctx.save_for_backward(gates, c_prev)
        ctx.dims, ctx.fmt = dims, fmt
        return h, c

    @staticmethod
    def backward(ctx, dh, dc):
        gates, c_prev = ctx.saved_tensors
        dgates, dc_prev = torch.empty_like(gates), torch.empty_like(c_prev)
        # (named, not temporaries: a converted copy freed before the launch is enqueued could be handed to the next conversion)
        dh_ = None if dh is None else dh.contiguous(memory_format=ctx.fmt)
        dc_ = None if dc is None else dc.contiguous(memory_format=ctx.fmt)
        check(lib().hrl_lstm_gates_bwd(_ptr(gates), _ptr(c_prev), _ptr(dh_), _ptr(dc_), _ptr(dgates), _ptr(dc_prev), *ctx.dims,
                                       _stream_ptr()))
        _count()
        return dgates, dc_prev


def lstm_gates(gates, c_prev):
    """(h', c') of a convolutional LSTM cell from its gate pre-activations (N,4C,...) in the order i, f, o, g."""
    return _LstmGates.apply(gates, c_prev)


def _mask_view(om):
    """observation_mask[:, t] (B,P,1) as (pointer tensor, batch stride): element (b,p) at base + b*stride + p."""
    assert om.dim() == 3 and om.shape[2] == 1 and (om.stride(1) == 1 or om.shape[1] == 1) and om.dtype == torch.float32
    return om, om.stride(0)


# The hidden-state kernels treat a leaf as (B, P, R) blocks and are elementwise inside a block, so any dense ordering of the
# R elements works as long as every operand of a call shares it.  A leaf (B, P, C, H, W) whose (C, H, W) block is channels-last
# (what a net built on the tensor-core convolutions hands back) is therefore used as it lies: no layout copies in the time loop.
def _block_layout(t):
    if t.is_contiguous():
        return 'std'
    if t.dim() == 5 and t.stride(0) == t.shape[1] * t.stride(1) and _is_channels_last(t.flatten(0, 1)):
        return 'cl'
    if _is_channels_last(t):
        return 'cl'
    return None


def _as_block_layout(t, layout):
    if layout == 'cl' and t.dim() in (4, 5):
        if _block_layout(t) == 'cl':
            return t
        lead = t.shape[:-3]
        return t.reshape(-1, *t.shape[-3:]).contiguous(memory_format=torch.channels_last).view(*lead, *t.shape[-3:])
    return t.contiguous()


def _empty_block_layout(shape, layout, device):
    if layout == 'cl' and len(shape) in (4, 5):
        lead = tuple(shape[:-3])
        n = 1
        for d in lead:
            n *= d
        return torch.empty((n,) + tuple(shape[-3:]), dtype=torch.float32, device=device,
                           memory_format=torch.channels_last).view(*lead, *shape[-3:])
    return torch.empty(tuple(shape), dtype=torch.float32, device=device)


class _HiddenVisible(torch.autograd.Function):
    @staticmethod
    def forward(ctx, h, om, sum_players):
        layout = _block_layout(h) or 'std'
        h = _as_block_layout(h, layout)
        B, P = h.shape[:2]
        R = h[0, 0].numel()
        om, stride = _mask_view(om)
        out = _empty_block_layout((B,) + tuple(h.shape[2:]) if sum_players else tuple(h.shape), layout, h.device)
        check(lib().hrl_hidden_visible_fwd(_ptr(h), _ptr(om), stride, _ptr(out), B, P, R, int(sum_players), _stream_ptr()))
        _count()
        ctx.save_for_backward(om)
        ctx.meta = (B, P, R, stride, bool(sum_players), tuple(h.shape), layout)
        return out

    @staticmethod
    def backward(ctx, dout):
        om, = ctx.saved_tensors
        B, P, R, stride, sum_players, shape, layout = ctx.meta
        dh = _empty_block_layout(shape, layout, dout.device)
        dout = _as_block_layout(dout, layout)
        check(lib().hrl_hidden_visible_bwd(_ptr(dout), _ptr(om), stride, _ptr(dh), B, P, R, int(sum_players), _stream_ptr()))
        _count()
        return dh, None, None


class _HiddenBlend(torch.autograd.Function):
    @staticmethod
    def forward(ctx, h, nh, om):
        layout = _block_layout(nh) or 'std'          # the net's output decides: it keeps coming back in that layout
        h, nh = _as_block_layout(h, layout), _as_block_layout(nh, layout)
        B, P = h.shape[:2]
        Pn = nh.shape[1]
        R = h[0, 0].numel()
        om, stride = _mask_view(om)
        out = _empty_block_layout(tuple(h.shape), layout, h.device)
        check(lib().hrl_hidden_blend_fwd(_ptr(h), _ptr(nh), _ptr(om), stride, _ptr(out), B, P, Pn, R, _stream_ptr()))
        _count()
        ctx.save_for_backward(om)
        ctx.meta = (B, P, Pn, R, stride, tuple(h.shape), tuple(nh.shape), layout)
        return out

    @staticmethod
    def backward(ctx, dout):
        om, = ctx.saved_tensors
        B, P, Pn, R, stride, hshape, nshape, layout = ctx.meta
        dh = _empty_block_layout(hshape, layout, dout.device) if ctx.needs_input_grad[0] else None
        dnh = _empty_block_layout(nshape, layout, dout.device)
        dout = _as_block_layout(dout, layout)
        check(lib().hrl_hidden_blend_bwd(_ptr(dout), _ptr(om), stride, _ptr(dh), _ptr(dnh), B, P, Pn, R, _stream_ptr()))
        _count()
        return dh, dnh, None


def hidden_visible(h, om, sum_players):
    """The hidden leaf a recurrent net sees at one step (train.py:152-158): h (B,P,...) masked by om (B,P,1), summed
    over players when sum_players (turn-alternating batches) -- one kernel instead of mul + sum."""
    return _HiddenVisible.apply(h, om, sum_players)


def hidden_blend(h, nh, om):
    """h (1 - om) + nh om (train.py:173), nh (B,Pa,...) broadcast over players when Pa == 1 -- one kernel."""
    return _HiddenBlend.apply(h, nh, om)


def _nchw_or_nhwc(x):
    """(tensor in one of the two dense layouts, channels_last flag)"""
    if x.is_contiguous():
        return x, 0
    if x.is_contiguous(memory_format=torch.channels_last):
        return x, 1
    return x.contiguous(), 0


class _BatchNormTrain(torch.autograd.Function):
    """nn.BatchNorm2d (training mode) on (N, C, H, W) activations in NCHW or channels-last memory, through hrl_bn_train_fwd / _bwd."""

    @staticmethod
    def forward(ctx, x, weight, bias, running_mean, running_var, eps, momentum):
        x, cl = _nchw_or_nhwc(x)
        N, Cn, H, W = x.shape
        y = torch.empty_like(x)          # keeps the memory format
        mean = torch.empty(Cn, dtype=torch.float32, device=x.device)
        rstd = torch.empty_like(mean)
        ws = torch.empty(lib().hrl_bn_workspace_floats(N, Cn, H * W, cl), dtype=torch.float32, device=x.device)
        check(lib().hrl_bn_train_fwd(_ptr(x), _ptr(weight), _ptr(bias), _ptr(y), _ptr(mean), _ptr(rstd), _ptr(running_mean),
                                     _ptr(running_var), N, Cn, H * W, cl, float(eps), float(momentum), _ptr(ws), _stream_ptr()))
        _count(3)
        ctx.save_for_backward(x, weight, mean, rstd)
        ctx.cl = cl
        return y

    @staticmethod
    def backward(ctx, dy):
        x, weight, mean, rstd = ctx.saved_tensors
        cl = ctx.cl
        dy = dy.contiguous(memory_format=torch.channels_last) if cl else dy.contiguous()
        N, Cn, H, W = x.shape
        dx = torch.empty_like(x)
        dgamma = torch.empty(Cn, dtype=torch.float32, device=x.device)
        dbeta = torch.empty_like(dgamma)
        ws = torch.empty(lib().hrl_bn_workspace_floats(N, Cn, H * W, cl), dtype=torch.float32, device=x.device)
        check(lib().hrl_bn_train_bwd(_ptr(x), _ptr(dy), _ptr(weight), _ptr(mean), _ptr(rstd), _ptr(dx), _ptr(dgamma), _ptr(dbeta),
                                     N, Cn, H * W, cl, _ptr(ws), _stream_ptr()))
        _count(3)
        return dx, (dgamma if weight is not None else None), (dbeta if ctx.needs_input_grad[2] else None), None, None, None, None


def batch_norm_train(x, weight, bias, running_mean, running_var, eps, momentum):
    """Fused train-mode BatchNorm for small boards (updates the running statistics in place)."""
    return _BatchNormTrain.apply(x, weight, bias, running_mean, running_var, eps, momentum)


class PeerAllReduce:
    """One-shot all-reduce(SUM) of the flat gradient bucket over NVLink peer memory, fused with the gradient-norm
    partials (hrl_peer_allreduce_sumsq).  The bucket lives in torch symmetric memory so that every rank holds a
    mapping of every other rank's bucket; ranks synchronise inside the kernel with system-scope flags stored
    behind the bucket.  Bit-identical results on all ranks (fixed summation order), CUDA-graph capturable,
    no NCCL call on the step."""

    def __init__(self, group, device):
        import torch.distributed as dist
        self.group, self.device = group, device
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        self.numel = None

    def alloc(self, numel):
        """Bucket of `numel` floats (+ 2*world flag words) in symmetric memory; rendezvous with the peers."""
        import torch.distributed._symmetric_memory as symm
        self.numel = numel
        words = numel + 2 * self.world + 64
        self.storage = symm.empty(words, dtype=torch.float32, device=self.device)
        self.storage.zero_()
        try:
            self.handle = symm.rendezvous(self.storage, self.group)
        except Exception:
            symm.enable_symm_mem_for_group(self.group.group_name)
            self.handle = symm.rendezvous(self.storage, self.group.group_name)
        torch.cuda.synchronize(self.device)
        self.handle.barrier()
        ptrs = [int(p) for p in self.handle.buffer_ptrs]
        assert len(ptrs) == self.world and ptrs[self.rank] == self.storage.data_ptr()
        self.peer_ptrs = torch.tensor(ptrs, dtype=torch.int64, device=self.device)
        self.reduced = torch.zeros(numel, dtype=torch.float32, device=self.device)
        self.epoch = torch.zeros(1, dtype=torch.int32, device=self.device)
        self.ticket = torch.zeros(1, dtype=torch.int32, device=self.device)
        self.status = torch.zeros(1, dtype=torch.int32, device=self.device)
        return self.storage

    def check(self):
        """Raise if a rank ever failed to arrive in the in-kernel rendezvous (the kernel gives up after 20 s instead of
        spinning forever; its sums are then garbage).  Synchronises the current stream."""
        if int(self.status.item()) != 0:
            raise _capi.HrlError('hrl_peer_allreduce_sumsq: a peer rank did not arrive within the timeout')

    def __call__(self, n_norm, partials):
        """Enqueue the fused reduce on the current stream; returns the reduced bucket."""
        check(lib().hrl_peer_allreduce_sumsq(_ptr(self.reduced), _ptr(self.peer_ptrs), self.numel, self.world, self.rank,
                                             self.numel, n_norm, _ptr(partials), _ptr(self.epoch), _ptr(self.ticket),
                                             _ptr(self.status), _stream_ptr()))
        _count(1)
        return self.reduced
