"""Fused GAN step: ONE C call (gantts_gan_step) per mini-batch for an MLP, In2OutHighwayNet, In2OutRNNHighwayNet or
SRURNN generator + MLP, LSTMRNN or GRURNN discriminator -- the whole of reference train.py:528-580 enqueued on the current stream without a
single host synchronisation (SURVEY.md 8f row 3).  Not drop-in for train.py (which owns its step
functions); offered next to the compatible modular path (gantts_b200.step.GanTrainer), which also runs
the LSTMRNN / GRURNN generators.

The step is built for a (B, T) that is its capacity: each call trains on its own mini-batch shape (b, t), b <= B and
t <= T, with exactly the arithmetic of a step built for (b, t) -- so the batches of train.py's collate_fn, padded to their
own max_len with a short last batch, map onto it one by one.

Data parallel: utterance shards, the two flat gradient buffers are SUM all-reduced (NCCL via
torch.distributed on the same stream) between the phases of the step; losses are normalised by the
GLOBAL number of valid frames.  Every rank pads its shard to the GLOBAL max_len of the mini-batch (the same t on every
rank; b may differ), as the MLPG and the SRU's reverse direction depend on the padded length.
"""
import collections
import ctypes

import numpy as np
import torch

from . import _lib
from . import models
from . import multistream
from . import ops
from . import parallel

LOSS_NAMES = ("loss_d", "loss_fake_d", "loss_real_d", "loss_mse", "loss_mge", "loss_adv", "loss_g",
              "real_correct", "fake_correct", "frames", "d_grad_norm", "g_grad_norm")


def _generator_parts(model_g):
    """(highway gate Linear or None, [SRUCell...] (empty unless SRURNN), nn.LSTM or None (In2OutRNNHighwayNet),
    [MLP layers..., last layer]) of a generator the fused step runs."""
    if isinstance(model_g, models.In2OutHighwayNet):
        return model_g.T, [], None, list(model_g.H) + [model_g.last_linear]
    if isinstance(model_g, models.In2OutRNNHighwayNet):
        return model_g.T, [], _check_lstm(model_g.lstm), [model_g.hidden2out]
    if isinstance(model_g, models.SRURNN):
        return None, list(model_g.gru.rnn_lst), None, [model_g.hidden2out]
    if hasattr(model_g, "layers") and hasattr(model_g, "last_linear"):
        return None, [], None, list(model_g.layers) + [model_g.last_linear]
    raise RuntimeError("FusedGanStep: generator %s is not supported (MLP, In2OutHighwayNet, In2OutRNNHighwayNet and SRURNN "
                       "are); train it with gantts_b200.step.GanTrainer" % type(model_g).__name__)


def _discriminator_parts(model_d):
    """(nn.LSTM or None, [MLP layers..., last layer]) of a discriminator the fused step runs: an MLP, or an LSTMRNN / GRURNN
    (reference train.py:774 builds the class hp.discriminator names; GRURNN keeps its nn.LSTM as .gru) whose last layer is
    hidden2out."""
    if isinstance(model_d, models._LSTMNet):
        return _check_lstm(getattr(model_d, model_d._rnn_attr)), [model_d.hidden2out]
    if hasattr(model_d, "layers") and hasattr(model_d, "last_linear"):
        return None, list(model_d.layers) + [model_d.last_linear]
    raise RuntimeError("FusedGanStep: discriminator %s is not supported (MLP, LSTMRNN and GRURNN are); train it with "
                       "gantts_b200.step.GanTrainer" % type(model_d).__name__)


def _check_lstm(lstm, who="FusedGanStep"):
    """An nn.LSTM of a generator or discriminator, if the fused step implements it."""
    why = None
    if getattr(lstm, "proj_size", 0) > 0:
        why = "proj_size > 0"
    elif not lstm.bias:
        why = "bias=False"
    elif not lstm.batch_first:
        why = "batch_first=False"
    elif lstm.num_layers > _lib.MAX_LSTM_LAYERS:
        why = "%d layers (at most %d)" % (lstm.num_layers, _lib.MAX_LSTM_LAYERS)
    if why is not None:
        raise RuntimeError("%s: an nn.LSTM with %s is not supported%s" % (
            who, why, "; train it with gantts_b200.step.GanTrainer" if who == "FusedGanStep" else ""))
    return lstm


def _fill_sru(desc, cells):
    """The shape block of gantts_sru_stack_t from an SRU stack (rnn.SRU.rnn_lst)."""
    if len(cells) > _lib.MAX_SRU_LAYERS:
        raise RuntimeError("gantts_b200: at most %d SRU layers" % _lib.MAX_SRU_LAYERS)
    c0 = cells[0]
    ncols = c0.n_out * (2 if c0.bidirectional else 1)
    for i, cell in enumerate(cells):
        same = (cell.n_out, cell.bidirectional, cell.activation_type, cell.rnn_dropout) == \
               (c0.n_out, c0.bidirectional, c0.activation_type, c0.rnn_dropout)
        # rnn.SRU: layer i > 0 reads the ncols outputs of the one below; every layer but the last has the stack's
        # output dropout
        if not same or (i > 0 and cell.n_in != ncols) or (i + 1 < len(cells) and cell.dropout != c0.dropout):
            raise RuntimeError("FusedGanStep: the SRU layers must form one rnn.SRU stack")
    desc.num_layers = len(cells)
    desc.in_dim, desc.hidden, desc.bidirectional = int(c0.n_in), int(c0.n_out), int(bool(c0.bidirectional))
    desc.act = int(c0.activation_type)
    desc.dropout = float(c0.dropout) if len(cells) > 1 else 0.0
    desc.rnn_dropout = float(c0.rnn_dropout)


def _fill_lstm(desc, lstm):
    """The shape block of gantts_lstm_stack_t from an nn.LSTM (its tensors go into the step's tensor tables)."""
    desc.num_layers, desc.in_dim, desc.hidden = lstm.num_layers, lstm.input_size, lstm.hidden_size
    desc.bidirectional = int(bool(lstm.bidirectional))
    desc.dropout = float(lstm.dropout) if lstm.num_layers > 1 else 0.0


def _fill_mlp(desc, layers, p, last_act):
    """The shape block of gantts_mlp_t (its tensors go into the step's tensor tables)."""
    if len(layers) > _lib.MAX_LAYERS:
        raise RuntimeError("gantts_b200: at most %d layers" % _lib.MAX_LAYERS)
    desc.num_layers = len(layers)
    desc.dims[0] = layers[0].weight.shape[1]
    for i, l in enumerate(layers):
        desc.dims[i + 1] = l.weight.shape[0]
    desc.slope, desc.dropout_p, desc.last_act, desc.seed = ops.LEAKY_SLOPE, float(p), int(last_act), 0


def adversarial_columns(hp):
    """Columns of y_hat_static the discriminator sees: get_selected_static_stream of reference train.py:232-242 (stream
    select, then the first mask_nth_mgc_for_adv_loss columns dropped)."""
    sizes = multistream.get_static_stream_sizes(hp.stream_sizes, hp.has_dynamic_features, len(hp.windows))
    acols = multistream.select_stream_columns(sizes, hp.adversarial_streams)
    if hp.mask_nth_mgc_for_adv_loss > 0:
        acols = acols[hp.mask_nth_mgc_for_adv_loss:]
    return [int(v) for v in acols]


def check_reference_discriminator(model_ref, n_adv, who):
    """The reference discriminator of the spoofing-rate count (train.py:549-558): an MLP, or an LSTMRNN / GRURNN
    (train.py:779-781 builds it from hp.discriminator like D), with one sigmoid output and whose input is the n_adv
    adversarial columns alone."""
    if isinstance(model_ref, models._LSTMNet):
        if not model_ref.last_sigmoid:
            raise RuntimeError("%s: the reference discriminator must have a sigmoid output (last_sigmoid=True)" % who)
        width = int(_check_lstm(getattr(model_ref, model_ref._rnn_attr), who).input_size)
    elif not (hasattr(model_ref, "layers") and hasattr(model_ref, "last_linear")) or not model_ref.last_sigmoid:
        raise RuntimeError("%s: the reference discriminator must be a sigmoid-output MLP, LSTMRNN or GRURNN" % who)
    else:
        width = int(model_ref.layers[0].weight.shape[1] if len(model_ref.layers) else model_ref.last_linear.weight.shape[1])
    if width != n_adv:
        raise RuntimeError("%s: the reference discriminator takes %d inputs, but train.py:549-555 feeds it the %d "
                           "adversarial columns alone (no linguistic conditioning)" % (who, width, n_adv))


class FusedGanStep(object):
    def __init__(self, model_g, model_d, hp, B, T, w_d=1.0, mse_w=0.0, mge_w=1.0, lr=0.01, weight_decay=1e-7,
                 max_norm=1.0, process_group=None, seed=None, optimizer="Adagrad", optimizer_params=None,
                 reference_discriminator=None):
        """``optimizer`` / ``optimizer_params`` mirror ``getattr(optim, hp.optimizer_g)(params, **hp.optimizer_g_params)``
        of reference train.py:784-789 (one setting for both models): "Adagrad" (lr, weight_decay, eps; the defaults
        are hparams.py:201-206) or "Adam" (lr, betas, eps, weight_decay; hparams.py:125-130).

        ``reference_discriminator``: the frozen discriminator of the adversarial stage (train.py --checkpoint-r); every
        step then counts the frames of the pre-update y_hat_static it takes for natural (train.py:549-558) into the
        device scalar ``spoof_count``.  It runs with dropout off, sees no linguistic conditioning and is never updated.
        It is an MLP, or an LSTMRNN / GRURNN (train.py:779-781 builds it from hp.discriminator like D) of at most 3 layers
        and a configured B of at most 128, whose stack runs over the call's packed sequences."""
        lib = _lib.load()
        if optimizer not in ("Adagrad", "Adam"):
            raise RuntimeError("FusedGanStep: no native optimiser %r (Adagrad and Adam are the ones hparams.py uses)" % optimizer)
        self.optimizer = optimizer
        okw = dict(optimizer_params or {})
        if optimizer == "Adam":
            lr, weight_decay = okw.get("lr", 1e-3), okw.get("weight_decay", 0.0)
        else:
            lr, weight_decay = okw.get("lr", lr), okw.get("weight_decay", weight_decay)
        self.g, self.d, self.hp, self.pg = model_g, model_d, hp, process_group
        self.B, self.T = int(B), int(T)
        dev = next(model_g.parameters()).device
        self.device = dev
        parallel.broadcast_parameters(model_g, group=process_group)
        parallel.broadcast_parameters(model_d, group=process_group)
        c = _lib.GanStepT()
        c.B, c.T = self.B, self.T
        gate, sru, lstm, g_layers = _generator_parts(model_g)
        d_lstm, d_layers = _discriminator_parts(model_d)
        _fill_mlp(c.g, g_layers, getattr(model_g, "dropout_p", 0.0), _lib.ACT_NONE)
        _fill_mlp(c.d, d_layers, getattr(model_d, "dropout_p", 0.0), _lib.ACT_SIGMOID)
        if getattr(model_g, "last_sigmoid", False) or not model_d.last_sigmoid:
            raise RuntimeError("FusedGanStep: generator must be linear-output, discriminator sigmoid-output")
        if gate is not None:
            c.highway.static_dim = int(model_g.static_dim)
        if sru:
            _fill_sru(c.sru, sru)
        if lstm is not None:
            _fill_lstm(c.lstm, lstm)
        if d_lstm is not None:
            _fill_lstm(c.d_lstm, d_lstm)
        # the tensor tables, in model.parameters() order; the C step binds them to its stages from the shapes above
        self._params = list(model_g.parameters()) + list(model_d.parameters())
        self._ng = len(list(model_g.parameters()))          # generator tensors: their optimiser state comes first
        ops.require_cuda(*self._params)
        if not all(t.is_contiguous() for t in self._params):
            raise RuntimeError("gantts_b200: parameters must be contiguous")
        # Adagrad: state_sum | Adam: exp_avg, exp_avg_sq
        self._sums = [torch.zeros_like(t) for t in self._params]
        self._sqs = [torch.zeros_like(t) for t in self._params] if optimizer == "Adam" else []
        for tab, lo, hi in ((c.g_tensors, 0, self._ng), (c.d_tensors, self._ng, len(self._params))):
            if hi - lo > _lib.MAX_STEP_TENSORS:
                raise RuntimeError("gantts_b200: a model of more than %d tensors" % _lib.MAX_STEP_TENSORS)
            tab.n = hi - lo
            for i in range(lo, hi):
                tab.state[i - lo] = self._sums[i].data_ptr()
                if self._sqs:
                    tab.state2[i - lo] = self._sqs[i].data_ptr()
        self._bind_params(c)
        nw = len(hp.windows)
        entries, n_static = multistream.mlpg_stream_entries(hp.stream_sizes, hp.has_dynamic_features,
                                                            [True] * len(hp.stream_sizes), nw)
        c.streams = _lib.make_streams(entries)
        c.windows = _lib.make_windows(hp.windows)
        # the host table of the configured T (it also validates the windows); other padded lengths get tables built on
        # the device (ops.mlpg_table_device, bit-identical), kept in a small LRU cache
        self._table = ops.mlpg_table(hp.windows, self.T, dev)
        c.mlpg_table = self._table.data_ptr()
        self._tables = collections.OrderedDict()
        scols = multistream.static_feature_columns(nw, hp.stream_sizes, hp.has_dynamic_features,
                                                   [True] * len(hp.stream_sizes))
        c.n_static, c.n_static_cols = n_static, len(scols)
        for i, v in enumerate(scols):
            c.static_cols[i] = v
        acols = adversarial_columns(hp)
        c.n_adv = len(acols)
        for i, v in enumerate(acols):
            c.adv_cols[i] = v
        c.d_conditioned = 1 if hp.discriminator_linguistic_condition else 0
        c.lr_g = c.lr_d = float(lr)
        c.wd_g = c.wd_d = float(weight_decay)
        c.max_norm = float(max_norm)
        if optimizer == "Adam":
            betas = okw.get("betas", (0.9, 0.999))
            self._betas = (float(betas[0]), float(betas[1]))          # as given (the C struct holds them as float32)
            c.optimizer, c.beta1, c.beta2, c.eps = _lib.OPT_ADAM, float(betas[0]), float(betas[1]), float(okw.get("eps", 1e-8))
        else:
            c.optimizer, c.eps = _lib.OPT_ADAGRAD, float(okw.get("eps", 1e-10))
        c.opt_step = 1
        c.w_d, c.mse_w, c.mge_w, c.adv_w = float(w_d), float(mse_w), float(mge_w), 1.0
        self.cfg = c
        nbytes = lib.gantts_gan_step_workspace_bytes(ctypes.byref(c))
        if nbytes == 0:
            raise RuntimeError("gantts_b200 gan_step config rejected: %s" % lib.gantts_last_error_string().decode())
        self._ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        self.losses = torch.zeros(len(LOSS_NAMES), dtype=torch.float32, device=dev)
        # y_hat / y_hat_static are (b, t, .) views of these buffers after a call of shape (b, t); the buffers themselves
        # at the configured shape
        self._y_hat_buf = torch.empty(self.B, self.T, c.g.dims[c.g.num_layers], dtype=torch.float32, device=dev)
        self._y_hat_static_buf = torch.empty(self.B, self.T, n_static, dtype=torch.float32, device=dev)
        self.y_hat, self.y_hat_static = self._y_hat_buf, self._y_hat_static_buf
        self._shape = (self.B, self.T, self._table.data_ptr())      # (b, t, MLPG table) of the next native call
        self._seed = int(seed) if seed is not None else ops.draw_seed() & ((1 << 60) - 1)
        self._step = 0                          # training calls: the seed stream
        self._opt_steps = {"g": 0, "d": 0}      # optimiser steps per model (they differ after D-only steps)
        self._grad_views = {}
        self.ref_d = reference_discriminator
        if reference_discriminator is not None:
            check_reference_discriminator(reference_discriminator, len(acols), "FusedGanStep")
            self._ref_lstm = None
            if isinstance(reference_discriminator, models._LSTMNet):
                # LSTMRNN / GRURNN: its nn.LSTM's tensors (model.parameters() order), then hidden2out as the head
                ref_rnn = getattr(reference_discriminator, reference_discriminator._rnn_attr)
                self._ref_lstm = _lib.LstmStackT()
                _fill_lstm(self._ref_lstm, ref_rnn)
                ref_layers = [reference_discriminator.hidden2out]
                self._ref_rnn_params = list(ref_rnn.parameters())
            else:
                ref_layers = list(reference_discriminator.layers) + [reference_discriminator.last_linear]
                self._ref_rnn_params = []
            self._ref_params = [t for l in ref_layers for t in (l.weight, l.bias)]
            ops.require_cuda(*(self._ref_rnn_params + self._ref_params))
            if not all(t.is_contiguous() for t in self._ref_rnn_params + self._ref_params):
                raise RuntimeError("gantts_b200: parameters must be contiguous")
            self._ref_desc = _lib.MlpT()
            _fill_mlp(self._ref_desc, ref_layers, 0.0, _lib.ACT_SIGMOID)
            self._adv_cols = (ctypes.c_int * len(acols))(*acols)
            if self._ref_lstm is not None:
                # laid out for the configured (B, T), which holds every call's (b, t); refuses B > 128
                rbytes = lib.gantts_spoof_count_lstm_workspace_bytes(ctypes.byref(self._ref_lstm),
                                                                     ctypes.byref(self._ref_desc), self.B, self.T)
            else:
                rbytes = lib.gantts_spoof_count_workspace_bytes(ctypes.byref(self._ref_desc), self.B * self.T)
            if rbytes == 0:
                raise RuntimeError("gantts_b200 spoof_count config rejected: %s" % lib.gantts_last_error_string().decode())
            self._ref_ws = torch.empty(rbytes, dtype=torch.uint8, device=dev)
            self.spoof_count = torch.zeros((), dtype=torch.float32, device=dev)

    def _bind_params(self, cfg):
        for tab, lo, hi in ((cfg.g_tensors, 0, self._ng), (cfg.d_tensors, self._ng, len(self._params))):
            for i in range(lo, hi):
                tab.param[i - lo] = self._params[i].data_ptr()

    def grad_buffer(self, which):
        """Flat fp32 gradient buffer (0 = generator, 1 = discriminator) as a tensor view."""
        if which not in self._grad_views:
            lib = _lib.load()
            ptr, cnt = ctypes.c_void_p(), ctypes.c_int64()
            _lib.check(lib.gantts_gan_step_grad_buffer(ctypes.byref(self.cfg), self._ws.data_ptr(), which,
                                                       ctypes.byref(ptr), ctypes.byref(cnt)))
            off = ptr.value - self._ws.data_ptr()
            self._grad_views[which] = self._ws[off:off + 4 * cnt.value].view(torch.float32)
        return self._grad_views[which]

    TABLE_CACHE = 64            # device-built MLPG tables kept (one per padded length t != T)

    def _mlpg_table(self, t):
        """The MLPG table of padded length t: the host one for the configured T, else built on the device once."""
        if t == self.T:
            return self._table
        tab = self._tables.get(t)
        if tab is None:
            tab = ops.mlpg_table_device(self.hp.windows, t, self.device)
            self._tables[t] = tab
            if len(self._tables) > self.TABLE_CACHE:
                self._tables.popitem(last=False)
        else:
            self._tables.move_to_end(t)
        return tab

    def _set_shape(self, b, t):
        """y_hat / y_hat_static as (b, t, .) views of their buffers (the buffers themselves at the configured shape)."""
        if (b, t) == (self.B, self.T):
            self.y_hat, self.y_hat_static = self._y_hat_buf, self._y_hat_static_buf
        elif tuple(self.y_hat.shape[:2]) != (b, t):
            self.y_hat, self.y_hat_static = (buf.view(-1)[:b * t * buf.shape[2]].view(b, t, buf.shape[2])
                                             for buf in (self._y_hat_buf, self._y_hat_static_buf))

    def _call(self, phases, x, y, lengths, inv_frames, seed):
        lib = _lib.load()
        b, t, table = self._shape
        _lib.check(lib.gantts_gan_step_shaped(ctypes.byref(self.cfg), b, t, table, phases,
                                              x.data_ptr(), y.data_ptr(), lengths.data_ptr(), inv_frames, seed,
                                              self.y_hat.data_ptr(), self.y_hat_static.data_ptr(), self.losses.data_ptr(),
                                              self._ws.data_ptr(), self._ws.numel(), ops._stream()))

    def step(self, x, y, lengths, frames=None, adv_w=1.0, train=None, update_g=True):
        """x (b,t,d_in), y (b,t,d_out) contiguous CUDA float32 with 1 <= b <= B and 1 <= t <= T of the configured (B, T);
        lengths CUDA int64 (b,); frames = GLOBAL number of valid frames (host number; checked against the device-side
        count when the losses are read, see loss_dict).  Returns the device tensor of 12 loss scalars; y_hat and
        y_hat_static are then (b, t, .) views.

        Each mini-batch may have its own shape, like the batches of train.py's collate_fn (padded to their own max_len,
        the last one shorter): the call computes exactly what a step built for (b, t) computes from the same state and
        seed.  MLPG solves over the padded length t, so padding a batch further changes its result.

        ``train=None`` follows the models like the reference's train_loop does (train.py:481-486): both models
        in ``.train()`` -> training step; both in ``.eval()`` -> the "test" phase (forwards and losses only,
        dropout off, parameters and Adagrad state untouched).

        ``update_g=False`` is the discriminator warm-up step (train.py --discriminator-warmup, :696): the generator runs
        forward in train mode, the discriminator is updated, the generator and its optimiser state are left alone.
        loss_adv and g_grad_norm are then 0 and loss_g = mse_w loss_mse + mge_w loss_mge of the forward.  Ignored in
        the test phase, which updates nothing."""
        ops.require_cuda(x, y)
        if not (x.is_contiguous() and y.is_contiguous()):
            raise RuntimeError("FusedGanStep: x and y must be contiguous")
        if x.dim() != 3 or y.dim() != 3 or tuple(x.shape[:2]) != tuple(y.shape[:2]):
            raise RuntimeError("FusedGanStep: x and y must be (b, t, .) batches of the same shape")
        b, t = int(x.shape[0]), int(x.shape[1])
        if not (1 <= b <= self.B and 1 <= t <= self.T):
            raise RuntimeError("FusedGanStep: batch shape (%d, %d) exceeds the configured (B, T) = (%d, %d)"
                               % (b, t, self.B, self.T))
        if not lengths.is_cuda or lengths.dtype != torch.int64:
            raise RuntimeError("FusedGanStep: lengths must be a CUDA int64 tensor")
        if tuple(lengths.shape) != (b,):
            raise RuntimeError("FusedGanStep: lengths must have shape (b,) = (%d,)" % b)
        self._set_shape(b, t)
        self._shape = (b, t, self._mlpg_table(t).data_ptr())
        self.cfg.adv_w = float(adv_w)
        self._bind_params(self.cfg)             # parameters may have been re-allocated (load_state_dict keeps them)
        if train is None:
            if self.g.training != self.d.training:
                raise RuntimeError("FusedGanStep: generator and discriminator disagree on train()/eval()")
            train = self.g.training
        world = torch.distributed.get_world_size(self.pg) if (torch.distributed.is_available()
                                                              and torch.distributed.is_initialized()) else 1
        if frames is None:
            # single process: the step derives 1 / mask.sum() on the device from `lengths` (no host number to trust)
            if world > 1:
                raise RuntimeError("FusedGanStep: data-parallel steps need frames = the GLOBAL number of valid frames")
            self._frames_claim, inv = None, 0.0
        else:
            self._frames_claim = float(frames)
            inv = 1.0 / float(frames)
        if not train:
            self._call(_lib.STEP_EVAL, x, y, lengths, inv, 0)
            self._count_spoofed(lengths)
            return self.losses
        if not update_g and not self.cfg.w_d > 0:
            raise RuntimeError("FusedGanStep: update_g=False trains the discriminator alone and needs w_d > 0")
        seed = (self._seed + self._step) & ((1 << 61) - 1)
        self.last_seed = seed
        self._step += 1
        # Adam's bias corrections: the number of the step each model is taking
        self._opt_steps["d"] += 1
        if update_g:
            self._opt_steps["g"] += 1
        n_g, n_d = self._opt_steps["g"], self._opt_steps["d"]
        d_only = 0 if update_g else _lib.STEP_D_ONLY
        if world == 1 and (n_g == n_d or d_only):
            self.cfg.opt_step = n_d
            self._call(7 | d_only, x, y, lengths, inv, seed)
        elif world == 1:
            self.cfg.opt_step = n_d
            self._call(1 | 2, x, y, lengths, inv, seed)
            self.cfg.opt_step = n_g
            self._call(4, x, y, lengths, inv, seed)
        else:
            self.cfg.opt_step = n_d
            self._call(1 | d_only, x, y, lengths, inv, seed)
            parallel.allreduce_sum_(self.grad_buffer(1), self.pg)
            self._call(2 | d_only, x, y, lengths, inv, seed)
            if update_g:
                parallel.allreduce_sum_(self.grad_buffer(0), self.pg)
            self.cfg.opt_step = n_g
            self._call(4 | d_only, x, y, lengths, inv, seed)
        self._count_spoofed(lengths)
        return self.losses

    def _count_spoofed(self, lengths):
        """spoof_count = frames of this step's y_hat_static (the pre-update generator's output) the reference
        discriminator takes for natural (train.py:549-558); local to the rank, like `frames`."""
        if self.ref_d is None:
            return
        lib = _lib.load()
        d = self._ref_desc
        for i, (w, b) in enumerate(zip(self._ref_params[0::2], self._ref_params[1::2])):
            d.W[i], d.b[i] = w.data_ptr(), b.data_ptr()
        ws = self._ref_ws
        b, t, n_static = self.y_hat_static.shape
        if self._ref_lstm is not None:
            tensors = (ctypes.c_void_p * len(self._ref_rnn_params))(*[p.data_ptr() for p in self._ref_rnn_params])
            _lib.check(lib.gantts_spoof_count_lstm(ctypes.byref(self._ref_lstm), tensors, len(self._ref_rnn_params),
                                                   ctypes.byref(d), self.y_hat_static.data_ptr(), n_static,
                                                   self._adv_cols, len(self._adv_cols), lengths.data_ptr(), b, t,
                                                   self.spoof_count.data_ptr(), ws.data_ptr(), ws.numel(),
                                                   ops._stream()))
            return
        _lib.check(lib.gantts_spoof_count(ctypes.byref(d), self.y_hat_static.data_ptr(), n_static,
                                          self._adv_cols, len(self._adv_cols), lengths.data_ptr(), b, t,
                                          self.spoof_count.data_ptr(), ws.data_ptr(), ws.numel(), ops._stream()))

    def loss_dict(self):
        """Host copy of the 12 loss scalars (one synchronising read).  Single process: also verifies the `frames`
        the caller passed to step() against the device-side sum of the mask -- a wrong value would silently
        rescale every loss and gradient.  With a reference discriminator the dict also holds "spoof_count"."""
        if self.ref_d is None:
            v = dict(zip(LOSS_NAMES, self.losses.tolist()))
        else:
            vals = torch.cat((self.losses, self.spoof_count.view(1))).tolist()
            v = dict(zip(LOSS_NAMES + ("spoof_count",), vals))
        world = torch.distributed.get_world_size(self.pg) if (torch.distributed.is_available()
                                                              and torch.distributed.is_initialized()) else 1
        claim = getattr(self, "_frames_claim", None)
        if world == 1 and claim is not None and v["frames"] != claim:
            raise RuntimeError("FusedGanStep: step() was told frames=%g but the lengths sum to %g valid frames"
                               % (claim, v["frames"]))
        return v

    # ---- checkpoint / resume (reference train.py:162-171 save_checkpoint, :174-199 load_checkpoint round-trip
    # optimizer.state_dict(); the layout below is torch.optim.Adagrad's, one entry per parameter in
    # model.parameters() order, so the files are interchangeable with the reference's)
    def _opt_state(self, lo, hi, lr, wd, nstep):
        n = hi - lo
        step = torch.tensor(float(nstep))
        if self.optimizer == "Adam":
            return {"state": {i: {"step": step.clone(), "exp_avg": self._sums[lo + i].detach().clone(),
                                  "exp_avg_sq": self._sqs[lo + i].detach().clone()} for i in range(n)},
                    "param_groups": [{"lr": lr, "betas": self._betas,
                                      "eps": float(self.cfg.eps), "weight_decay": wd, "amsgrad": False, "maximize": False,
                                      "foreach": None, "capturable": False, "differentiable": False, "fused": None,
                                      "params": list(range(n))}]}
        return {"state": {i: {"step": step.clone(), "sum": self._sums[lo + i].detach().clone()} for i in range(n)},
                "param_groups": [{"lr": lr, "lr_decay": 0, "eps": float(self.cfg.eps), "weight_decay": wd,
                                  "initial_accumulator_value": 0, "foreach": None, "maximize": False,
                                  "differentiable": False, "fused": None, "params": list(range(n))}]}

    def state_dict(self):
        ng, n = self._ng, len(self._sums)
        return {"optimizer_g": self._opt_state(0, ng, float(self.cfg.lr_g), float(self.cfg.wd_g), self._opt_steps["g"]),
                "optimizer_d": self._opt_state(ng, n, float(self.cfg.lr_d), float(self.cfg.wd_d), self._opt_steps["d"]),
                "step": self._step, "seed": self._seed}

    def load_state_dict(self, sd):
        ng, n = self._ng, len(self._sums)
        step = int(sd.get("step", self._step))
        for key, lo, hi in (("optimizer_g", 0, ng), ("optimizer_d", ng, n)):
            st = sd[key]["state"]
            for i in range(hi - lo):
                e = st.get(i, st.get(str(i)))
                if e is None:
                    raise RuntimeError("FusedGanStep.load_state_dict: %s has no state for parameter %d" % (key, i))
                if i == 0:              # each optimiser's own step count (the models differ after D-only steps)
                    self._opt_steps[key[-1]] = int(float(e["step"])) if "step" in e else step
                if self.optimizer == "Adam":
                    self._sums[lo + i].copy_(e["exp_avg"])
                    self._sqs[lo + i].copy_(e["exp_avg_sq"])
                else:
                    self._sums[lo + i].copy_(e["sum"])
            grp = (sd[key].get("param_groups") or [{}])[0]
            if self.optimizer == "Adam" and "betas" in grp:
                self._betas = (float(grp["betas"][0]), float(grp["betas"][1]))
                self.cfg.beta1, self.cfg.beta2 = self._betas
            if key == "optimizer_g":
                self.cfg.lr_g = float(grp.get("lr", self.cfg.lr_g))
                self.cfg.wd_g = float(grp.get("weight_decay", self.cfg.wd_g))
            else:
                self.cfg.lr_d = float(grp.get("lr", self.cfg.lr_d))
                self.cfg.wd_d = float(grp.get("weight_decay", self.cfg.wd_d))
        self._step = step
        self._seed = int(sd.get("seed", self._seed))
