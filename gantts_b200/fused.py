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
from .optim import OptimizerState

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


def _optimizer_hyper(kind, params, lr, weight_decay):
    """The hyper-parameters of one model's optimiser: ``params`` over the defaults of its kind (Adagrad: the step's
    ``lr`` / ``weight_decay`` arguments; Adam: lr 1e-3, weight_decay 0)."""
    hyper = dict(lr=lr, weight_decay=weight_decay) if kind == "Adagrad" else dict(lr=1e-3, weight_decay=0.0)
    hyper.update(params or {})
    return hyper


class FusedGanStep(object):
    def __init__(self, model_g, model_d, hp, B, T, w_d=1.0, mse_w=0.0, mge_w=1.0, lr=0.01, weight_decay=1e-7,
                 max_norm=1.0, process_group=None, seed=None, optimizer="Adagrad", optimizer_params=None,
                 reference_discriminator=None, optimizer_d=None, optimizer_d_params=None):
        """``optimizer`` / ``optimizer_params`` and ``optimizer_d`` / ``optimizer_d_params`` mirror
        ``getattr(optim, hp.optimizer_g)(model_g.parameters(), **hp.optimizer_g_params)`` and the same for ``_d`` of
        reference train.py:796-799: "Adagrad" (lr, weight_decay, eps; lr and weight_decay default to the ``lr`` /
        ``weight_decay`` arguments, hparams.py:201-206) or "Adam" (lr, betas, eps, weight_decay; lr 1e-3 and
        weight_decay 0 by default, hparams.py:125-130).  ``optimizer_d=None`` gives the discriminator the generator's
        kind; ``optimizer_d_params=None`` gives it the generator's parameters when the kinds agree, else its kind's
        defaults.  ``opt_g`` / ``opt_d`` hold each model's hyper-parameters and state with torch.optim's
        ``param_groups``, ``state_dict()`` and ``load_state_dict()``: every step reads lr, weight_decay, eps and betas
        from the groups, so train.py's exp_lr_scheduler (:323-333), save_checkpoint and load_checkpoint (:162-171,
        :651-658) work on them as written.

        ``reference_discriminator``: the frozen discriminator of the adversarial stage (train.py --checkpoint-r); every
        step then counts the frames of the pre-update y_hat_static it takes for natural (train.py:549-558) into the
        device scalar ``spoof_count``.  It runs with dropout off, sees no linguistic conditioning and is never updated.
        It is an MLP, or an LSTMRNN / GRURNN (train.py:779-781 builds it from hp.discriminator like D) of at most 3 layers
        and a configured B of at most 128, whose stack runs over the call's packed sequences."""
        lib = _lib.load()
        kind_d = optimizer if optimizer_d is None else optimizer_d
        for kind in (optimizer, kind_d):
            if kind not in ("Adagrad", "Adam"):
                raise RuntimeError("FusedGanStep: no native optimiser %r (Adagrad and Adam are the ones hparams.py uses)"
                                   % kind)
        if optimizer_d_params is None and kind_d == optimizer:
            optimizer_d_params = optimizer_params
        hyper_g = _optimizer_hyper(optimizer, optimizer_params, lr, weight_decay)
        hyper_d = _optimizer_hyper(kind_d, optimizer_d_params, lr, weight_decay)
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
        # each model's optimiser state -- Adagrad: state_sum | Adam: exp_avg, exp_avg_sq -- in model.parameters() order
        opts = []
        for tab, params, kind, hyper in ((c.g_tensors, self._params[:self._ng], optimizer, hyper_g),
                                         (c.d_tensors, self._params[self._ng:], kind_d, hyper_d)):
            if len(params) > _lib.MAX_STEP_TENSORS:
                raise RuntimeError("gantts_b200: a model of more than %d tensors" % _lib.MAX_STEP_TENSORS)
            state = [torch.zeros_like(t) for t in params]
            state2 = [torch.zeros_like(t) for t in params] if kind == "Adam" else []
            tab.n = len(params)
            for i, t in enumerate(state):
                tab.state[i] = t.data_ptr()
            for i, t in enumerate(state2):
                tab.state2[i] = t.data_ptr()
            opts.append(OptimizerState(kind, params, state, state2, **hyper))
        self.opt_g, self.opt_d = opts
        # the state tensors of both models (G's first); _sqs holds exp_avg_sq of the Adam models only
        self._sums = self.opt_g._state + self.opt_d._state
        self._sqs = self.opt_g._state2 + self.opt_d._state2
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
        c.max_norm = float(max_norm)
        self.cfg = c
        self._set_optimizers(1, 1)
        c.w_d, c.mse_w, c.mge_w, c.adv_w = float(w_d), float(mse_w), float(mge_w), 1.0
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

    @property
    def _opt_steps(self):
        """Optimiser steps per model (they differ after D-only steps)."""
        return {"g": self.opt_g.steps, "d": self.opt_d.steps}

    def _set_optimizers(self, n_g, n_d):
        """The optimiser fields of the C config from opt_g / opt_d's groups; n_g, n_d = the number of the step each
        model would take (Adam's bias corrections).  The discriminator always has its own block."""
        c = self.cfg
        for opt, n, d in ((self.opt_g, n_g, False), (self.opt_d, n_d, True)):
            grp = opt.param_groups[0]
            kind = _lib.OPT_ADAM if opt.kind == "Adam" else _lib.OPT_ADAGRAD
            b1, b2 = grp["betas"] if opt.kind == "Adam" else (0.0, 0.0)
            if d:
                c.lr_d, c.wd_d = float(grp["lr"]), float(grp["weight_decay"])
                o = c.d_opt
                o.own, o.optimizer, o.beta1, o.beta2, o.eps, o.opt_step = 1, kind, b1, b2, float(grp["eps"]), n
            else:
                c.lr_g, c.wd_g = float(grp["lr"]), float(grp["weight_decay"])
                c.optimizer, c.beta1, c.beta2, c.eps, c.opt_step = kind, b1, b2, float(grp["eps"]), n

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
        # the hyper-parameters as the groups hold them now, and the number of the step each model takes (Adam's bias
        # corrections; G's is not read by a D-only step)
        self._set_optimizers(self.opt_g.steps + 1, self.opt_d.steps + 1)
        d_only = 0 if update_g else _lib.STEP_D_ONLY
        if world == 1:
            self._call(7 | d_only, x, y, lengths, inv, seed)
        else:
            self._call(1 | d_only, x, y, lengths, inv, seed)
            parallel.allreduce_sum_(self.grad_buffer(1), self.pg)
            self._call(2 | d_only, x, y, lengths, inv, seed)
            if update_g:
                parallel.allreduce_sum_(self.grad_buffer(0), self.pg)
            self._call(4 | d_only, x, y, lengths, inv, seed)
        self.opt_d.steps += 1
        if update_g:
            self.opt_g.steps += 1
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
    # optimizer.state_dict()): one torch.optim layout per model, opt_g's and opt_d's own, so each entry is
    # interchangeable with a torch.optim.Adagrad / Adam over that model's parameters
    def state_dict(self):
        return {"optimizer_g": self.opt_g.state_dict(), "optimizer_d": self.opt_d.state_dict(),
                "step": self._step, "seed": self._seed}

    def load_state_dict(self, sd):
        step = int(sd.get("step", self._step))
        for key, opt in (("optimizer_g", self.opt_g), ("optimizer_d", self.opt_d)):
            opt.steps = step                    # an entry without "step" counts every training call
            opt.load_state_dict(sd[key])
        self._step = step
        self._seed = int(sd.get("seed", self._seed))
