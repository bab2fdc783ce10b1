"""ctypes binding of libgantts_b200.so (the C ABI declared in include/gantts_b200.h).

There is NO CPU fallback: if the shared library is missing the import of any op fails loudly, and
every op rejects non-CUDA tensors.
"""
import ctypes
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libgantts_b200.so")

MAX_STREAMS = 8
MAX_WINDOWS = 4
MAX_TAPS = 5
MLPG_HALF_TAPS = 24
MLPG_NTAPS = 2 * MLPG_HALF_TAPS + 1
MLPG_TABLE_COLS = 60      # GANTTS_MLPG_TABLE_COLS: FIR taps + banded-Cholesky rows

ENGINE_SIMT = 0
ENGINE_TC = 1
ACT_NONE = 0
ACT_LEAKY_DROPOUT = 1
ACT_SIGMOID = 2


class StreamsT(ctypes.Structure):
    _fields_ = [("n", ctypes.c_int),
                ("in_start", ctypes.c_int * MAX_STREAMS),
                ("sd", ctypes.c_int * MAX_STREAMS),
                ("dyn", ctypes.c_int * MAX_STREAMS),
                ("out_start", ctypes.c_int * MAX_STREAMS)]


class WindowsT(ctypes.Structure):
    _fields_ = [("n", ctypes.c_int),
                ("l", ctypes.c_int * MAX_WINDOWS),
                ("u", ctypes.c_int * MAX_WINDOWS),
                ("coef", (ctypes.c_float * MAX_TAPS) * MAX_WINDOWS)]


class DistortionColsT(ctypes.Structure):
    _fields_ = [("mcd_start", ctypes.c_int), ("mcd_count", ctypes.c_int),
                ("bap_start", ctypes.c_int), ("bap_count", ctypes.c_int),
                ("lf0_col", ctypes.c_int), ("vuv_col", ctypes.c_int),
                ("lf0_linear", ctypes.c_int),
                ("mse_start", ctypes.c_int), ("mse_count", ctypes.c_int)]


METRIC_ACOUSTIC, METRIC_DURATION, METRIC_VC = 0, 1, 2
LOG_UPDATE_D, LOG_UPDATE_G, LOG_SPOOF = 1, 2, 4
LOG_N, LOG_FRAMES, LOG_LOSSES, LOG_SPOOFED, LOG_METRICS, LOG_SLOTS = 0, 1, 2, 14, 15, 20

MAX_LAYERS = 8


class MlpT(ctypes.Structure):
    _fields_ = [("num_layers", ctypes.c_int),
                ("dims", ctypes.c_int * (MAX_LAYERS + 1)),
                ("W", ctypes.c_void_p * MAX_LAYERS),
                ("b", ctypes.c_void_p * MAX_LAYERS),
                ("slope", ctypes.c_float),
                ("dropout_p", ctypes.c_float),
                ("last_act", ctypes.c_int),
                ("seed", ctypes.c_uint64)]


MAX_COLS = 256


class HighwayT(ctypes.Structure):
    _fields_ = [("static_dim", ctypes.c_int)]


MAX_SRU_LAYERS = 8


class SruStackT(ctypes.Structure):
    _fields_ = [("num_layers", ctypes.c_int),
                ("in_dim", ctypes.c_int), ("hidden", ctypes.c_int), ("bidirectional", ctypes.c_int),
                ("act", ctypes.c_int),
                ("dropout", ctypes.c_float), ("rnn_dropout", ctypes.c_float)]


MAX_LSTM_LAYERS = 3


class LstmStackT(ctypes.Structure):
    _fields_ = [("num_layers", ctypes.c_int),
                ("in_dim", ctypes.c_int), ("hidden", ctypes.c_int), ("bidirectional", ctypes.c_int),
                ("dropout", ctypes.c_float)]


MAX_STEP_TENSORS = 32


class StepTensorsT(ctypes.Structure):
    _fields_ = [("n", ctypes.c_int),
                ("param", ctypes.c_void_p * MAX_STEP_TENSORS),
                ("state", ctypes.c_void_p * MAX_STEP_TENSORS),
                ("state2", ctypes.c_void_p * MAX_STEP_TENSORS)]


class OptimizerT(ctypes.Structure):
    _fields_ = [("own", ctypes.c_int), ("optimizer", ctypes.c_int),
                ("beta1", ctypes.c_float), ("beta2", ctypes.c_float), ("eps", ctypes.c_float),
                ("opt_step", ctypes.c_int64)]


class GanStepT(ctypes.Structure):
    _fields_ = [("B", ctypes.c_int), ("T", ctypes.c_int),
                ("g", MlpT), ("highway", HighwayT), ("sru", SruStackT), ("lstm", LstmStackT), ("d", MlpT),
                ("g_tensors", StepTensorsT), ("d_tensors", StepTensorsT),
                ("streams", StreamsT), ("windows", WindowsT),
                ("mlpg_table", ctypes.c_void_p),
                ("n_static", ctypes.c_int), ("n_static_cols", ctypes.c_int),
                ("static_cols", ctypes.c_int * MAX_COLS),
                ("n_adv", ctypes.c_int), ("adv_cols", ctypes.c_int * MAX_COLS),
                ("d_conditioned", ctypes.c_int),
                ("lr_g", ctypes.c_float), ("lr_d", ctypes.c_float), ("wd_g", ctypes.c_float),
                ("wd_d", ctypes.c_float), ("eps", ctypes.c_float), ("max_norm", ctypes.c_float),
                ("w_d", ctypes.c_float), ("mse_w", ctypes.c_float), ("mge_w", ctypes.c_float),
                ("adv_w", ctypes.c_float),
                ("optimizer", ctypes.c_int), ("beta1", ctypes.c_float), ("beta2", ctypes.c_float),
                ("d_opt", OptimizerT),
                ("opt_step", ctypes.c_int64),
                ("d_lstm", LstmStackT)]


class EpochLogT(ctypes.Structure):
    _fields_ = [("kind", ctypes.c_int), ("n_static", ctypes.c_int),
                ("static_cols", ctypes.c_int * MAX_COLS),
                ("cols", DistortionColsT)]


OPT_ADAGRAD, OPT_ADAM = 0, 1
MCEP_R0, MCEP_SP = 0, 1     # GANTTS_MCEP_*: merlin_post_filter's energy operator, mc2sp's
SUBPHONE_FEATURES = 9       # GANTTS_SUBPHONE_FEATURES: Merlin's "full" frame-position columns
FRAMES_BAD_DURATION, FRAMES_TOO_LONG = 1, 2     # GANTTS_FRAMES_*: gantts_state_frame_offsets' status bits
MAX_FRAMES = 1 << 24        # per state duration and per row
CORPUS_BAD_ROW = 1          # GANTTS_CORPUS_BAD_ROW: gantts_corpus_gather's status bit
GANTTS_E_BADARG = 1

_lib = None

_vp, _i, _i64, _f, _u64, _sz = (ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float,
                                ctypes.c_uint64, ctypes.c_size_t)

# name -> (restype, argtypes); every symbol include/gantts_b200.h declares.
SIGNATURES = {
    "gantts_version": (_i, []),
    "gantts_last_error_string": (ctypes.c_char_p, []),
    "gantts_device_supported": (_i, []),
    "gantts_launch_count": (ctypes.c_longlong, []),
    "gantts_profile_enable": (_i, [_i]),
    "gantts_profile_collect": (_i, [_vp, _vp, _vp]),
    "gantts_mlpg_table": (_i, [ctypes.POINTER(WindowsT), _i, _vp]),
    "gantts_mlpg_table_device": (_i, [ctypes.POINTER(WindowsT), _i, _vp, _vp]),
    "gantts_mlpg_fwd": (_i, [_vp, _i64, _i64, _vp, _i64, _i64, _vp, ctypes.POINTER(StreamsT),
                             ctypes.POINTER(WindowsT), _i, _i, _vp]),
    "gantts_mlpg_bwd": (_i, [_vp, _i64, _i64, _vp, _i64, _i64, _vp, ctypes.POINTER(StreamsT),
                             ctypes.POINTER(WindowsT), _i, _i, _i, _vp]),
    "gantts_gather_cols": (_i, [_vp, _i64, _vp, _i64, _vp, _i, _i64, _vp]),
    "gantts_scatter_cols_add": (_i, [_vp, _i64, _vp, _i64, _vp, _i, _i64, _vp]),
    "gantts_sequence_mask": (_i, [_vp, _vp, _i, _i, _vp]),
    "gantts_masked_sse_workspace_bytes": (_sz, []),
    "gantts_masked_sse_fwd": (_i, [_vp, _i64, _vp, _i64, _vp, _i64, _i, _vp, _vp, _sz, _vp]),
    "gantts_masked_sse_bwd": (_i, [_vp, _i64, _vp, _i64, _vp, _i64, _i, _vp, _vp, _i64, _i, _vp]),
    "gantts_mlpg_var_workspace_bytes": (_sz, [ctypes.POINTER(WindowsT), _i, _i, _i]),
    "gantts_mlpg_var": (_i, [_vp, _i64, _i64, _vp, _i64, _i64, _vp, _i64, _i64, ctypes.POINTER(WindowsT),
                             _i, _i, _i, _vp, _sz, _vp]),
    "gantts_mlpg_ragged_workspace_bytes": (_sz, [ctypes.POINTER(StreamsT), ctypes.POINTER(WindowsT), _vp, _i, _i]),
    "gantts_mlpg_ragged": (_i, [_vp, _i64, _i64, _vp, _vp, _vp, _vp, _i64, _i64, _vp, _vp, ctypes.POINTER(StreamsT),
                                ctypes.POINTER(WindowsT), _vp, _i, _i, _vp, _sz, _vp]),
    "gantts_mcep_operator": (_i, [ctypes.c_double, _i, _i, _i, _vp]),
    "gantts_mcep_postfilter": (_i, [_vp, _i64, _i64, _vp, _i64, _i64, _vp, ctypes.c_double, _vp, _i, _i, _i, _i, _vp]),
    "gantts_mcep_to_sp": (_i, [_vp, _i64, _i64, _vp, _i64, _i64, _vp, _vp, _i, _i, _i, _i, _vp]),
    "gantts_modspec": (_i, [_vp, _i64, _i64, _vp, _i, _i, _i, _i, _vp, _vp, _vp]),
    "gantts_global_variance": (_i, [_vp, _i64, _i64, _vp, _i, _i, _i, _vp, _vp]),
    "gantts_state_frame_offsets": (_i, [_vp, _i64, _i64, _vp, _i, _i, _i, _vp, _vp, _vp, _vp]),
    "gantts_expand_state_frames": (_i, [_vp, _i64, _i64, _vp, _i64, _i64, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp,
                                        _vp]),
    "gantts_corpus_gather": (_i, [_vp, _vp, _i64, _i, _i, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp]),
    "gantts_distortions_workspace_bytes": (_sz, []),
    "gantts_distortions": (_i, [_vp, _i64, _i64, _vp, _i64, _i64, _vp, _i, _i, _i, _vp, _vp,
                                ctypes.POINTER(DistortionColsT), _vp, _vp, _sz, _vp]),
    "gantts_epoch_log_workspace_bytes": (_sz, [ctypes.POINTER(EpochLogT)]),
    "gantts_epoch_log_reset": (_i, [_vp, _vp]),
    "gantts_epoch_log_add": (_i, [ctypes.POINTER(EpochLogT), _i, _vp, _vp, _vp, _i64, _i64, _i, _vp, _i64, _i64, _vp,
                                  _i, _i, _vp, _vp, _vp, _vp, _sz, _vp]),
    "gantts_masked_bce_fwd": (_i, [_vp, _vp, _i64, _i, _vp, _vp, _sz, _vp]),
    "gantts_masked_bce_bwd": (_i, [_vp, _vp, _i64, _i, _vp, _vp, _vp]),
    "gantts_linear_workspace_bytes": (_sz, [_i64, _i, _i, _i]),
    "gantts_linear_fwd": (_i, [_vp, _i64, _vp, _vp, _vp, _i64, _i64, _i, _i, _i, _f, _f, _u64, _i,
                               _vp, _sz, _vp]),
    "gantts_linear_bwd": (_i, [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _vp, _vp, _i64, _vp, _vp, _i64,
                               _i, _i, _i, _f, _f, _i, _i, _vp, _sz, _vp]),
    "gantts_mlp_tape_bytes": (_sz, [ctypes.POINTER(MlpT), _i64]),
    "gantts_mlp_workspace_bytes": (_sz, [ctypes.POINTER(MlpT), _i64]),
    "gantts_mlp_fwd": (_i, [ctypes.POINTER(MlpT), _vp, _i64, _i64, _vp, _i64, _vp, _sz, _vp]),
    "gantts_mlp_bwd": (_i, [ctypes.POINTER(MlpT), _vp, _i64, _vp, _i64, _i64, _vp, _sz, _vp, _i64, _vp, _vp,
                            _i, _vp, _sz, _vp]),
    "gantts_gan_step_workspace_bytes": (_sz, [ctypes.POINTER(GanStepT)]),
    "gantts_gan_step_grad_buffer": (_i, [ctypes.POINTER(GanStepT), _vp, _i, ctypes.POINTER(ctypes.c_void_p),
                                         ctypes.POINTER(ctypes.c_int64)]),
    "gantts_gan_step": (_i, [ctypes.POINTER(GanStepT), _i, _vp, _vp, _vp, _f, _u64, _vp, _vp, _vp, _vp, _sz, _vp]),
    "gantts_gan_step_shaped": (_i, [ctypes.POINTER(GanStepT), _i, _i, _vp, _i, _vp, _vp, _vp, _f, _u64, _vp, _vp, _vp,
                                    _vp, _sz, _vp]),
    "gantts_spoof_count_workspace_bytes": (_sz, [ctypes.POINTER(MlpT), _i64]),
    "gantts_spoof_count": (_i, [ctypes.POINTER(MlpT), _vp, _i, ctypes.POINTER(ctypes.c_int), _i, _vp, _i, _i, _vp, _vp,
                                _sz, _vp]),
    "gantts_spoof_count_lstm_workspace_bytes": (_sz, [ctypes.POINTER(LstmStackT), ctypes.POINTER(MlpT), _i, _i]),
    "gantts_spoof_count_lstm": (_i, [ctypes.POINTER(LstmStackT), _vp, _i, ctypes.POINTER(MlpT), _vp, _i,
                                     ctypes.POINTER(ctypes.c_int), _i, _vp, _i, _i, _vp, _vp, _sz, _vp]),
    "gantts_lstm_workspace_bytes": (_sz, []),
    "gantts_lstm_layer_supported": (_i, [_i, _i, _i]),
    "gantts_lstm_layer_fwd": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp, _sz, _vp]),
    "gantts_lstm_layer_bwd": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp, _sz, _vp]),
    "gantts_lstm_hprev": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "gantts_dropout": (_i, [_vp, _vp, _i64, _i, _f, _u64, _vp]),
    "gantts_sru_fwd": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "gantts_sru_bwd": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "gantts_sru_fwd_lengths": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "gantts_optim_workspace_bytes": (_sz, []),
    "gantts_grad_sumsq": (_i, [_vp, _vp, _i, _vp, _vp, _sz, _vp]),
    "gantts_clip_adagrad_step": (_i, [_vp, _vp, _vp, _vp, _i, _vp, _f, _f, _f, _f, _vp]),
    "gantts_clip_adam_step": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _vp, _f, _f, _f, _f, _f, _f, _i64, _vp]),
    "gantts_gan_step_seed": (_u64, [_u64, _i]),
    "gantts_mlp_layer_seed": (_u64, [_u64, _i]),
    "gantts_sru_mask_seed": (_u64, [_u64, _i, _i]),
    "gantts_lstm_mask_seed": (_u64, [_u64, _i]),
    "gantts_d_lstm_mask_seed": (_u64, [_u64, _i, _i]),
}

STEP_D, STEP_G, STEP_FINISH, STEP_EVAL, STEP_D_ONLY = 1, 2, 4, 8, 16


def load():
    """Load the shared library (once).  Raises RuntimeError when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            "gantts_b200: %s is missing -- build it with `python -m gantts_b200.build` "
            "(or __graft_entry__.build()).  There is no CPU fallback." % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc):
    if rc != 0:
        msg = load().gantts_last_error_string()
        raise RuntimeError("gantts_b200 error %d: %s" % (rc, msg.decode() if msg else "?"))


def make_windows(windows):
    """windows: list of (l, u, coef array) as in reference hparams.py:22-26."""
    w = WindowsT()
    if not 1 <= len(windows) <= MAX_WINDOWS:
        raise RuntimeError("gantts_b200: between 1 and %d windows are supported" % MAX_WINDOWS)
    w.n = len(windows)
    for i, (l, u, coef) in enumerate(windows):
        coef = [float(c) for c in coef]
        if len(coef) != l + u + 1 or len(coef) > MAX_TAPS:
            raise RuntimeError("gantts_b200: bad window %d" % i)
        w.l[i], w.u[i] = int(l), int(u)
        for k, c in enumerate(coef):
            w.coef[i][k] = c
    return w


def make_streams(entries):
    """entries: list of (in_start, sd, dyn, out_start)."""
    s = StreamsT()
    if not 1 <= len(entries) <= MAX_STREAMS:
        raise RuntimeError("gantts_b200: between 1 and %d streams are supported" % MAX_STREAMS)
    s.n = len(entries)
    for i, (a, sd, dyn, o) in enumerate(entries):
        s.in_start[i], s.sd[i], s.dyn[i], s.out_start[i] = int(a), int(sd), int(bool(dyn)), int(o)
    return s
