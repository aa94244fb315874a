"""ctypes binding of include/hrl_b200.h (the C ABI of the CUDA library).

The library is built in-tree by `__graft_entry__.build()` / `handyrl_b200/csrc/build.py`
into handyrl_b200/libhrl_b200.so.  There is NO fallback: if the library is missing or a
symbol is absent, importing `lib()` raises.
"""
import ctypes as C
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libhrl_b200.so')

HRL_ABI_VERSION = 3
ALGO_ID = {'MC': 0, 'TD': 1, 'UPGO': 2, 'VTRACE': 3}
LOSS_KEYS = ('p', 'v', 'r', 'ent', 'total', 'dcnt')
NUM_LOSS = 6
# learner diagnostics sums, in the order of the HRL_DIAG_* indices of include/hrl_b200.h: the loss pass's first
# (HRL_NUM_LOSS_DIAG of them), then the optimiser's
DIAG_KEYS = ('n_pol', 'rho', 'rho_clip', 'logr', 'logr2', 'adv', 'adv2', 'n_val', 'tv', 'tv2', 'ev', 'ev2', 'tr', 'tr2', 'er', 'er2',
             'gnorm', 'gnorm2', 'gclip', 'steps')
NUM_LOSS_DIAG = 16
NUM_DIAG = 20

_f32p = C.POINTER(C.c_float)
_i64p = C.POINTER(C.c_int64)


class HrlLossTuning(C.Structure):
    _fields_ = [('variant', C.c_int32), ('recurrence', C.c_int32), ('cluster', C.c_int32), ('consumers', C.c_int32),
                ('threads', C.c_int32), ('unstaged', C.c_int32), ('trace', C.c_void_p)]


LOSS_VARIANTS = {'auto': 0, 'rows-direct': 1, 'rows-staged': 2, 'bulk': 3, 'element': 4, 'group': 5}
LOSS_RECURRENCES = {'auto': 0, 'serial': 1, 'scan': 2}


class HrlLossArgs(C.Structure):
    _fields_ = [
        ('B', C.c_int32), ('T', C.c_int32), ('P', C.c_int32), ('Pa', C.c_int32), ('A', C.c_int32),
        ('burn_in', C.c_int32), ('value_target', C.c_int32), ('policy_target', C.c_int32),
        ('two_player_zero_sum', C.c_int32),
        ('lambda_', C.c_float), ('gamma', C.c_float),
        ('entropy_regularization', C.c_float), ('entropy_regularization_decay', C.c_float),
        ('policy_raw', C.c_void_p), ('value_raw', C.c_void_p), ('return_raw', C.c_void_p),
        ('action_mask', C.c_void_p), ('action', C.c_void_p), ('selected_prob', C.c_void_p),
        ('reward', C.c_void_p), ('ret', C.c_void_p), ('turn_mask', C.c_void_p),
        ('observation_mask', C.c_void_p), ('episode_mask', C.c_void_p), ('progress', C.c_void_p),
        ('outcome', C.c_void_p),
        ('dpolicy_raw', C.c_void_p), ('dvalue_raw', C.c_void_p), ('dreturn_raw', C.c_void_p),
        ('losses', C.c_void_p),
        ('tap_target_value', C.c_void_p), ('tap_target_return', C.c_void_p), ('tap_advantage', C.c_void_p),
        ('tap_logp', C.c_void_p), ('tap_rho', C.c_void_p), ('tap_entropy', C.c_void_p),
        ('workspace', C.c_void_p), ('workspace_bytes', C.c_size_t),
        ('tuning', HrlLossTuning), ('io_bf16', C.c_int32), ('external_heads', C.c_int32), ('window_weight', C.c_void_p),
    ]


class HrlGemmOperand(C.Structure):
    _fields_ = [('ptr', C.c_void_p), ('ptr2', C.c_void_p), ('p', C.c_void_p), ('q', C.c_void_p), ('r', C.c_void_p),
                ('ld', C.c_int64), ('kmajor', C.c_int32), ('relu', C.c_int32), ('feature_is_row', C.c_int32), ('packed', C.c_int32)]


GEMM_EPILOGUES = {'store': 0, 'relu': 1, 'stats': 2, 'mask_stats': 3}


class HrlGemmArgs(C.Structure):
    _fields_ = [('a', HrlGemmOperand), ('b', HrlGemmOperand), ('bias', C.c_void_p), ('C', C.c_void_p),
                ('ldc', C.c_int64), ('M', C.c_int64), ('N', C.c_int64), ('K', C.c_int64),
                ('splits', C.c_int32), ('epilogue', C.c_int32), ('workspace', C.c_void_p),
                ('ep_y', C.c_void_p), ('ep_ldy', C.c_int64), ('ep_scale', C.c_void_p), ('ep_shift', C.c_void_p),
                ('ep_mean', C.c_void_p), ('ep_rstd', C.c_void_p), ('col_partials', C.c_void_p),
                ('conv_off', C.c_void_p), ('conv_mode', C.c_int32), ('conv_hw', C.c_int32), ('conv_taps', C.c_int32),
                ('conv_cin', C.c_int32), ('seg_a', C.c_void_p), ('seg_b', C.c_void_p), ('segments', C.c_int32),
                ('conv_ones_row', C.c_int32), ('bf16', C.c_int32)]


MAX_BOARD_JOBS = 8
# rows of a packed board-convolution image (hrl_board_pack_many, hrl_gemm_fused's packed B operand): features x cells
MAX_BOARD_ROWS = 288


class HrlPackJob(C.Structure):
    _fields_ = [('w', C.c_void_p), ('Cout', C.c_int32), ('Cin', C.c_int32), ('kh', C.c_int32), ('kw', C.c_int32), ('H', C.c_int32),
                ('W', C.c_int32), ('image_fwd', C.c_void_p), ('fwd_rows', C.c_int32), ('fwd_row0', C.c_int32),
                ('image_bwd', C.c_void_p), ('bwd_rows', C.c_int32), ('bwd_k0', C.c_int32), ('bias', C.c_void_p),
                ('bias_cells', C.c_void_p), ('bf16', C.c_int32)]


class HrlFoldJob(C.Structure):
    _fields_ = [('ddense', C.c_void_p), ('splits', C.c_int32), ('split_stride', C.c_int64), ('dw', C.c_void_p),
                ('Cout', C.c_int32), ('Cin', C.c_int32), ('kh', C.c_int32), ('kw', C.c_int32), ('H', C.c_int32), ('W', C.c_int32),
                ('accumulate', C.c_int32)]


class HrlWindow(C.Structure):
    _fields_ = [('first_step', C.c_int64), ('start', C.c_int32), ('end', C.c_int32),
                ('train_start', C.c_int32), ('total', C.c_int32), ('outcome_row', C.c_int32),
                ('player', C.c_int32)]


class HrlGatherArgs(C.Structure):
    _fields_ = [
        ('B', C.c_int32), ('T', C.c_int32), ('P', C.c_int32), ('Pa', C.c_int32), ('A', C.c_int32),
        ('Ps', C.c_int32), ('burn_in', C.c_int32), ('obs_elems', C.c_int32), ('turn_alternating', C.c_int32),
        ('windows', C.c_void_p),
        ('st_obs', C.c_void_p), ('st_prob', C.c_void_p), ('st_action', C.c_void_p), ('st_amask', C.c_void_p),
        ('st_value', C.c_void_p), ('st_reward', C.c_void_p), ('st_return', C.c_void_p),
        ('st_flags', C.c_void_p), ('st_turn', C.c_void_p), ('st_outcome', C.c_void_p),
        ('observation', C.c_void_p), ('selected_prob', C.c_void_p), ('value', C.c_void_p),
        ('action', C.c_void_p), ('outcome', C.c_void_p), ('reward', C.c_void_p), ('ret', C.c_void_p),
        ('episode_mask', C.c_void_p), ('turn_mask', C.c_void_p), ('observation_mask', C.c_void_p),
        ('action_mask', C.c_void_p), ('progress', C.c_void_p),
    ]


class HrlReplaySampleArgs(C.Structure):
    _fields_ = [
        ('B', C.c_int32), ('ring', C.c_int32), ('head', C.c_int32), ('count', C.c_int32),
        ('burn_in', C.c_int32), ('forward_steps', C.c_int32), ('Ps', C.c_int32), ('solo', C.c_int32),
        ('alpha', C.c_float), ('beta', C.c_float), ('seed', C.c_uint64), ('counter', C.c_uint64),
        ('dir', C.c_void_p), ('prio', C.c_void_p), ('prio_serial', C.c_void_p), ('max_prio', C.c_void_p),
        ('workspace', C.c_void_p), ('windows', C.c_void_p), ('win_slot', C.c_void_p), ('win_serial', C.c_void_p),
        ('win_weight', C.c_void_p),
    ]


class HrlDistillArgs(C.Structure):
    _fields_ = [
        ('B', C.c_int32), ('T', C.c_int32), ('P', C.c_int32), ('Pa', C.c_int32), ('A', C.c_int32), ('burn_in', C.c_int32),
        ('policy_raw', C.c_void_p), ('teacher_raw', C.c_void_p), ('action_mask', C.c_void_p), ('turn_mask', C.c_void_p),
        ('window_weight', C.c_void_p), ('step_count', C.c_void_p), ('coef', C.c_float), ('anneal_steps', C.c_int64),
        ('dpolicy_raw', C.c_void_p), ('losses', C.c_void_p), ('sums', C.c_void_p),
        ('workspace', C.c_void_p), ('workspace_bytes', C.c_size_t), ('io_bf16', C.c_int32),
    ]


class HrlValueBinsArgs(C.Structure):
    _fields_ = [
        ('B', C.c_int32), ('T', C.c_int32), ('P', C.c_int32), ('Pa', C.c_int32), ('K', C.c_int32), ('burn_in', C.c_int32),
        ('low', C.c_float), ('high', C.c_float), ('symlog', C.c_int32), ('sigma', C.c_float), ('head', C.c_int32),
        ('logits', C.c_void_p), ('expect', C.c_void_p), ('target', C.c_void_p), ('observation_mask', C.c_void_p),
        ('window_weight', C.c_void_p), ('dlogits', C.c_void_p), ('losses', C.c_void_p),
        ('workspace', C.c_void_p), ('workspace_bytes', C.c_size_t),
    ]


# every symbol include/hrl_b200.h declares: name -> (restype, argtypes)
SYMBOLS = {
    'hrl_loss_workspace_bytes': (C.c_size_t, [C.c_int32] * 5),
    'hrl_loss_fwd_bwd': (C.c_int, [C.POINTER(HrlLossArgs), C.c_void_p]),
    'hrl_loss_fwd': (C.c_int, [C.POINTER(HrlLossArgs), C.c_void_p]),
    'hrl_loss_diag_workspace_bytes': (C.c_size_t, [C.c_int32] * 5),
    'hrl_loss_fwd_bwd_diag': (C.c_int, [C.POINTER(HrlLossArgs), C.c_void_p, C.c_void_p]),
    'hrl_compute_target': (C.c_int, [C.c_int32] * 6 + [C.c_void_p] * 3 + [C.c_float, C.c_float] +
                           [C.c_void_p] * 5 + [C.c_void_p]),
    'hrl_sumsq_num_partials': (C.c_int32, []),
    'hrl_grad_sumsq': (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    'hrl_clip_adam_step': (C.c_int, [C.c_void_p] * 4 + [C.c_int64] + [C.c_void_p] * 3 + [C.c_double] * 5 +
                           [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    'hrl_lamb_plan': (C.c_int64, [C.c_void_p, C.c_int32, C.c_void_p]),
    'hrl_clip_lamb_step': (C.c_int, [C.c_void_p] * 5 + [C.c_int64, C.c_void_p, C.c_int32] + [C.c_void_p] * 4 + [C.c_double] * 6 +
                           [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    'hrl_step_commit': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                  C.c_void_p]),
    'hrl_weight_ema': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_float, C.c_int32, C.c_void_p, C.c_void_p]),
    'hrl_sum_rows': (C.c_int, [C.c_void_p, C.c_int32, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p]),
    'hrl_peer_allreduce_sumsq': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int64, C.c_int64,
                                           C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    'hrl_bn_workspace_floats': (C.c_size_t, [C.c_int64, C.c_int32, C.c_int32, C.c_int32]),
    'hrl_bn_train_fwd': (C.c_int, [C.c_void_p] * 8 + [C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_float, C.c_void_p, C.c_void_p]),
    'hrl_bn_train_bwd': (C.c_int, [C.c_void_p] * 8 + [C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    'hrl_gather_pad': (C.c_int, [C.POINTER(HrlGatherArgs), C.c_void_p]),
    'hrl_gather_pad_sym': (C.c_int, [C.POINTER(HrlGatherArgs)] + [C.c_void_p] * 4 + [C.c_int32, C.c_void_p]),
    'hrl_replay_sample': (C.c_int, [C.POINTER(HrlReplaySampleArgs), C.c_void_p]),
    'hrl_replay_priority_update': (C.c_int, [C.c_int32] * 4 + [C.c_void_p] * 2 + [C.c_float] + [C.c_void_p] * 7),
    'hrl_gemm_workspace_floats': (C.c_size_t, [C.c_int64, C.c_int64, C.c_int64, C.c_int32]),
    'hrl_gemm_tf32x3': (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_int64,
                                   C.c_int64, C.c_int64, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p]),
    'hrl_gemm_fused': (C.c_int, [C.POINTER(HrlGemmArgs), C.c_void_p]),
    'hrl_bn_finalize_fwd': (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p, C.c_float, C.c_float] +
                            [C.c_void_p] * 8),
    'hrl_bn_finalize_bwd': (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int64] + [C.c_void_p] * 8 +
                            [C.c_int32, C.c_void_p]),
    'hrl_heads_num_blocks': (C.c_int32, [C.c_int64]),
    'hrl_heads_fwd': (C.c_int, [C.c_void_p, C.c_int64, C.c_int64] + [C.c_int32] * 5 + [C.c_float] + [C.c_void_p] * 7),
    'hrl_heads_bwd': (C.c_int, [C.c_void_p, C.c_int64, C.c_int64] + [C.c_int32] * 5 + [C.c_float] + [C.c_void_p] * 15 +
                      [C.c_int32, C.c_void_p]),
    'hrl_gemm_set_debug': (None, [C.c_int]),
    'hrl_gemm_padded_rows': (C.c_int32, [C.c_int64]),
    'hrl_board_pack_floats': (C.c_size_t, [C.c_int64, C.c_int64]),
    'hrl_board_pack': (C.c_int, [C.c_void_p] + [C.c_int32] * 6 + [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]),
    'hrl_board_expand': (C.c_int, [C.c_void_p, C.c_void_p] + [C.c_int32] * 6 + [C.c_void_p]),
    'hrl_conv_geometry': (C.c_int, [C.c_int32] * 5 + [C.c_void_p]),
    'hrl_conv_pack_floats': (C.c_size_t, [C.c_int32] * 3),
    'hrl_conv_pack': (C.c_int, [C.c_void_p] + [C.c_int32] * 4 + [C.c_void_p] * 3),
    'hrl_conv_pack_bf16': (C.c_int, [C.c_void_p] + [C.c_int32] * 4 + [C.c_void_p] * 3),
    'hrl_conv_wgrad_reduce2': (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p] + [C.c_int32] * 4 + [C.c_void_p]),
    'hrl_conv_wgrad_reduce': (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    'hrl_board_pack_many': (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p]),
    'hrl_board_pack_many_pivot': (C.c_int, [C.c_void_p, C.c_int32] + [C.c_void_p] * 3 + [C.c_int32] * 3 + [C.c_void_p]),
    'hrl_board_fold_many': (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p]),
    'hrl_board_fold': (C.c_int, [C.c_void_p, C.c_int32, C.c_int64, C.c_void_p] + [C.c_int32] * 6 + [C.c_void_p]),
    'hrl_gemm_effective_splits': (C.c_int32, [C.c_int64, C.c_int32]),
    'hrl_lstm_gates_fwd': (C.c_int, [C.c_void_p] * 4 + [C.c_int64, C.c_int32, C.c_int32, C.c_void_p]),
    'hrl_lstm_gates_bwd': (C.c_int, [C.c_void_p] * 6 + [C.c_int64, C.c_int32, C.c_int32, C.c_void_p]),
    'hrl_hidden_visible_fwd': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    'hrl_hidden_visible_bwd': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    'hrl_hidden_blend_fwd': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    'hrl_hidden_blend_bwd': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    'hrl_distill_workspace_bytes': (C.c_size_t, [C.c_int32] * 5),
    'hrl_distill_fwd_bwd': (C.c_int, [C.POINTER(HrlDistillArgs), C.c_void_p]),
    'hrl_value_bins_workspace_bytes': (C.c_size_t, [C.c_int32] * 5),
    'hrl_value_bins_expect': (C.c_int, [C.POINTER(HrlValueBinsArgs), C.c_void_p]),
    'hrl_value_bins_fwd_bwd': (C.c_int, [C.POINTER(HrlValueBinsArgs), C.c_void_p]),
    'hrl_last_error': (C.c_char_p, []),
    'hrl_abi_version': (C.c_int32, []),
}

_lib = None
_lock = threading.Lock()


class HrlError(RuntimeError):
    pass


def lib():
    """Load (once) and return the CUDA library; raises if it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise HrlError('handyrl_b200: %s is missing -- run `python -c "import __graft_entry__ as g; g.build()"` '
                           '(there is no CPU or PyTorch fallback for the learner hot path)' % LIB_PATH)
        h = C.CDLL(LIB_PATH)
        for name, (res, argt) in SYMBOLS.items():
            fn = getattr(h, name)  # AttributeError if the symbol is not exported
            fn.restype = res
            fn.argtypes = argt
        if h.hrl_abi_version() != HRL_ABI_VERSION:
            raise HrlError('handyrl_b200: ABI mismatch (library %d, binding %d)' % (h.hrl_abi_version(), HRL_ABI_VERSION))
        _lib = h
    return _lib


def check(status):
    if status != 0:
        raise HrlError('hrl_b200 error %d: %s' % (status, lib().hrl_last_error().decode()))
