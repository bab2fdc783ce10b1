"""CPU restatement (torch CPU fp32) of the reference GAN-step hot path.  TEST INFRASTRUCTURE.

Each function cites the reference file:line it follows (reference = r9y9/gantts @ fb1e75f).  The
reference itself is Python and cannot travel to the GPU box, so this port is what the ``-m gpu``
parity tests, ``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline / ``--impl reference``
leg run there.  It is PINNED: ``tests/golden/make_golden.py`` runs the unmodified reference
(``oracle.reference_loader``) and this port on the same seeded inputs in the build container and
commits the reference outputs under ``tests/golden/``; ``tests/test_oracle_golden.py`` checks the
port against those vectors (bit-exact for masks/indexing, <=1e-6 relative for float outputs: the
port issues the same torch CPU ops in the same order as the reference).

Written as plain functions over explicit weight lists (no nn.Module copies of the reference
classes): parameters are passed as ``[(W0, b0), (W1, b1), ...]`` with ``W`` laid out ``[out, in]``
exactly like the reference's ``nn.Linear`` state_dict entries.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from . import nnmnkwii_port as nn_port

LEAKY_SLOPE = 0.01          # nn.LeakyReLU() default, reference gantts/models.py:37,132
BCE_EPS = 1e-20             # reference train.py:246,285


# ----------------------------------------------------------------------------- seqloss.py
def sequence_mask(lengths, max_len=None):
    """reference gantts/seqloss.py:9-20 -- ``arange(max_len)[None] < len[:, None]`` as float."""
    lengths = torch.as_tensor(lengths).long().view(-1)
    if max_len is None:
        max_len = int(lengths.max())
    rng = torch.arange(0, int(max_len)).long().unsqueeze(0).expand(lengths.numel(), int(max_len))
    return (rng < lengths.unsqueeze(1)).float()


def masked_mse(inp, target, lengths=None, mask=None, max_len=None):
    """reference gantts/seqloss.py:27-43 -- sum(((in - tgt) * m)^2) / sum(m), m is (B,T,1)."""
    if lengths is None and mask is None:
        raise RuntimeError("Should provide either lengths or mask")
    if mask is None:
        mask = sequence_mask(lengths, max_len).unsqueeze(-1)
    m = mask.expand_as(inp)
    loss = F.mse_loss(inp * m, target * m, reduction="sum")
    return loss / mask.sum()


# ------------------------------------------------------------------------- multistream.py
def get_static_stream_sizes(stream_sizes, has_dynamic_features, num_windows):
    """reference gantts/multistream.py:46-53."""
    out = np.array(stream_sizes)
    sel = np.asarray(has_dynamic_features, dtype=bool)
    out[sel] = out[sel] / num_windows
    return out


def select_streams(inputs, stream_sizes=(60, 1, 1, 1), streams=(True, True, True, True)):
    """reference gantts/multistream.py:33-43 -- column gather of enabled streams."""
    starts = np.hstack(([0], np.cumsum(stream_sizes)[:-1]))
    parts = [inputs[:, :, int(s):int(s) + int(n)]
             for s, n, on in zip(starts, stream_sizes, streams) if on]
    return torch.cat(parts, dim=-1)


def get_static_features(inputs, num_windows, stream_sizes=(180, 3, 1, 3),
                        has_dynamic_features=(True, True, False, True),
                        streams=(True, True, True, True)):
    """reference gantts/multistream.py:56-79 -- static columns of a static+delta tensor."""
    D = inputs.size(-1)
    if stream_sizes is None or (len(stream_sizes) == 1 and has_dynamic_features[0]):
        return inputs[:, :, :D // num_windows]
    if len(stream_sizes) == 1 and not has_dynamic_features[0]:
        return inputs
    starts = np.hstack(([0], np.cumsum(stream_sizes)[:-1]))
    parts = []
    for s, n, dyn, on in zip(starts, stream_sizes, has_dynamic_features, streams):
        if not on:
            continue
        width = int(n) // num_windows if dyn else int(n)
        parts.append(inputs[:, :, int(s):int(s) + width])
    return torch.cat(parts, dim=-1)


def multi_stream_mlpg(inputs, R, stream_sizes=(180, 3, 1, 3),
                      has_dynamic_features=(True, True, False, True),
                      streams=(True, True, True, True)):
    """reference gantts/multistream.py:82-123 -- per-stream dense-R MLPG, static streams copied."""
    if inputs.size(-1) != sum(stream_sizes):
        raise RuntimeError("You probably have specified wrong dimention params.")
    starts = np.hstack(([0], np.cumsum(stream_sizes)[:-1]))
    ends = np.cumsum(stream_sizes)
    parts = []
    for s, e, dyn, on in zip(starts, ends, has_dynamic_features, streams):
        if not on:
            continue
        x = inputs[:, :, int(s):int(e)]
        parts.append(nn_port.unit_variance_mlpg(R, x) if dyn else x)
    return torch.cat(parts, dim=-1)


# ------------------------------------------------------------------------------ models.py
def mlp_forward(x, layers, dropout_p=0.0, training=False, last_sigmoid=False, masks=None):
    """reference gantts/models.py:137-141 -- x = Dropout(LeakyReLU(Linear(x))) per hidden
    layer, then last_linear (+ sigmoid).  ``layers`` = [(W, b), ...]; the last pair is
    ``last_linear``.

    ``masks`` (test hook, SURVEY.md 7 hard part 4): one tensor per hidden layer holding the dropout
    multiplier {0, 1/(1-p)} of every element; when given it REPLACES ``F.dropout`` (same place in
    the chain: Linear -> LeakyReLU -> Dropout), so a train-mode run of the product can be compared
    against this port with the product's own keep decisions injected (torch's Philox stream cannot
    be reproduced on the device)."""
    for l, (W, b) in enumerate(layers[:-1]):
        h = F.leaky_relu(F.linear(x, W, b), LEAKY_SLOPE)
        x = h * masks[l].view_as(h) if masks is not None else F.dropout(h, dropout_p, training)
    W, b = layers[-1]
    x = F.linear(x, W, b)
    return torch.sigmoid(x) if last_sigmoid else x


def in2out_highway_forward(x, R, gate, layers, static_dim, dropout_p=0.0, training=False, masks=None):
    """reference gantts/models.py:54-69 -- returns (y_hat, x_static + sigmoid(T x_static) * MLPG(y_hat))."""
    x = x.unsqueeze(0) if x.dim() == 2 else x
    x_static = x[:, :, :static_dim]
    Tx = torch.sigmoid(F.linear(x_static, gate[0], gate[1]))
    h = mlp_forward(x, layers, dropout_p, training, last_sigmoid=False, masks=masks)
    Gx = nn_port.unit_variance_mlpg(R, h)
    return h, x_static + Tx * Gx


def lstm_stack(x, lengths, layers, masks=None):
    """pack -> nn.LSTM -> pad (reference gantts/models.py:100-108,182-187,205-210) through a torch ``nn.LSTM``, or
    through each nn.LSTM of the list ``layers`` in turn, padded back to x's length (``lengths=None``: unpacked, as the
    reference runs it).  The oracle for the recurrent kernels is torch's own CPU LSTM, as in the reference;
    ``GeneratorOracle`` and ``DiscriminatorOracle`` run it one layer at a time so that ``masks[k]`` ([B * T][ndir H]
    multipliers, the product's own inter-layer dropout decisions) can scale the output of layer k < len(layers) - 1.
    Without masks, single-layer LSTMs in turn give on CPU exactly the bits of one multi-layer nn.LSTM without
    dropout."""
    if isinstance(layers, torch.nn.LSTM):
        layers = [layers]
    h = x
    for k, lstm in enumerate(layers):
        if lengths is None:
            h, _ = lstm(h)
        else:
            out, _ = lstm(torch.nn.utils.rnn.pack_padded_sequence(h, [int(l) for l in lengths], batch_first=True))
            h, _ = torch.nn.utils.rnn.pad_packed_sequence(out, batch_first=True, total_length=x.size(1))
        if masks is not None and k + 1 < len(layers):
            h = h * masks[k].view_as(h)
    return h


def in2out_rnn_highway_forward(x, R, lengths, gate, lstm, hidden2out, static_dim, masks=None):
    """reference gantts/models.py:92-118 -- ``lstm_stack`` -> hidden2out -> MLPG; returns
    ``(x, x_static + sigmoid(T x_static) * Gx)``: the FIRST output is the input itself (``:118``)."""
    x = x.unsqueeze(0) if x.dim() == 2 else x
    x_static = x[:, :, :static_dim]
    Tx = torch.sigmoid(F.linear(x_static, gate[0], gate[1]))
    out = F.linear(lstm_stack(x, lengths, lstm, masks), hidden2out[0], hidden2out[1])
    Gx = nn_port.unit_variance_mlpg(R, out)
    return x, x_static + Tx * Gx


def lstm_forward(x, lengths, lstm, hidden2out, last_sigmoid=False, masks=None):
    """reference gantts/models.py:204-213 (LSTMRNN) / :181-190 (GRURNN, also an nn.LSTM):
    ``lstm_stack`` -> Linear (-> sigmoid).  ``lstm``: a torch ``nn.LSTM`` or a list of them (see ``lstm_stack``)."""
    out = F.linear(lstm_stack(x, lengths, lstm, masks), hidden2out[0], hidden2out[1])
    return torch.sigmoid(out) if last_sigmoid else out


def sru_forward(x, layers, hidden2out, bidirectional, activation_type, masks=None):
    """SRURNN (reference gantts/models.py:144-167): ``sru_layer_forward`` per layer, then hidden2out.  ``layers`` holds
    each layer's (weight, bias) as the model stores them, the bias [f-bias | r-bias] over both directions;
    ``activation_type`` 0 / 1 / 2 is identity / tanh / ReLU.  ``masks`` = [(mask_x, mask_h or None)] per layer."""
    dirs = 2 if bidirectional else 1
    h = x
    for i, (W, b) in enumerate(layers):
        nc = b.numel() // 2
        bport = torch.stack([b[:nc].view(dirs, nc // dirs), b[nc:].view(dirs, nc // dirs)], 1).reshape(-1)
        mx, mh = masks[i] if masks is not None else (None, None)
        h = sru_layer_forward(h.transpose(0, 1), W, bport, bidirectional=bidirectional, use_tanh=activation_type == 1,
                              use_relu=activation_type == 2, mask_x=mx, mask_h=mh).transpose(0, 1)
    return F.linear(h, hidden2out[0], hidden2out[1])


# ------------------------------------------------------------------- train.py step functions
def get_selected_static_stream(y_static, hp):
    """reference train.py:232-242 -- adversarial streams, first ``mask_nth`` mgc columns dropped."""
    sizes = get_static_stream_sizes(hp["stream_sizes"], hp["has_dynamic_features"],
                                    hp["num_windows"])
    sel = select_streams(y_static, sizes, streams=hp["adversarial_streams"])
    if hp.get("mask_nth_mgc_for_adv_loss", 0) > 0:
        sel = sel[:, :, hp["mask_nth_mgc_for_adv_loss"]:]
    return sel


def bce_real(D, mask, T, eps=BCE_EPS):
    """reference train.py:269 -- -(log(D + eps) * m).sum() / T."""
    return -(torch.log(D + eps) * mask).sum() / T


def bce_fake(D, mask, T, eps=BCE_EPS):
    """reference train.py:270 -- -(log(1 - D + eps) * m).sum() / T."""
    return -(torch.log(1 - D + eps) * mask).sum() / T


def clip_grad_norm(grads, max_norm=1.0):
    """torch.nn.utils.clip_grad_norm_ semantics (reference train.py:275,317)."""
    total = torch.sqrt(sum((g.detach() ** 2).sum() for g in grads))
    coef = torch.clamp(max_norm / (total + 1e-6), max=1.0)
    for g in grads:
        g.mul_(coef)
    return total


def adagrad_step(params, grads, state_sums, lr=0.01, weight_decay=1e-7, eps=1e-10):
    """torch.optim.Adagrad (lr_decay=0, initial_accumulator_value=0) as configured in reference
    hparams.py:223-227,240-244 and stepped at train.py:276,318."""
    with torch.no_grad():
        for p, g, s in zip(params, grads, state_sums):
            g = g + weight_decay * p
            s.addcmul_(g, g, value=1.0)
            p.addcdiv_(g, s.sqrt() + eps, value=-lr)


class AdamStepper(object):
    """torch.optim.Adam (amsgrad off) as configured by reference hparams.py:125-130 for the duration model
    (lr 1e-3, betas (0.5, 0.9), weight_decay 0, eps 1e-8) and stepped at train.py:276,318:
    g' = g + wd p; m = b1 m + (1 - b1) g'; v = b2 v + (1 - b2) g'^2;
    p -= lr / (1 - b1^t) * m / (sqrt(v) / sqrt(1 - b2^t) + eps).  Callable as ``stepper(params, grads)``;
    pass it to ``gan_step(..., d_opt=..., g_opt=...)`` in place of the default Adagrad."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0):
        self.lr, self.b1, self.b2, self.eps, self.wd = float(lr), float(betas[0]), float(betas[1]), float(eps), float(weight_decay)
        self.m = [torch.zeros_like(p) for p in params]
        self.v = [torch.zeros_like(p) for p in params]
        self.t = 0

    def __call__(self, params, grads):
        self.t += 1
        c1, c2 = 1.0 - self.b1 ** self.t, 1.0 - self.b2 ** self.t
        with torch.no_grad():
            for p, g, m, v in zip(params, grads, self.m, self.v):
                g = g + self.wd * p
                m.mul_(self.b1).add_(g, alpha=1.0 - self.b1)
                v.mul_(self.b2).addcmul_(g, g, value=1.0 - self.b2)
                p.addcdiv_(m, v.sqrt() / math.sqrt(c2) + self.eps, value=-self.lr / c1)


class GanStepState(object):
    """Weights + Adagrad accumulators for one MLP-G / MLP-D pair (plain tensors)."""

    def __init__(self, g_layers, d_layers):
        self.g = [(W.clone().requires_grad_(True), b.clone().requires_grad_(True)) for W, b in g_layers]
        self.d = [(W.clone().requires_grad_(True), b.clone().requires_grad_(True)) for W, b in d_layers]
        self.g_sum = [torch.zeros_like(t) for pair in self.g for t in pair]
        self.d_sum = [torch.zeros_like(t) for pair in self.d for t in pair]

    def g_params(self):
        return [t for pair in self.g for t in pair]

    def d_params(self):
        return [t for pair in self.d for t in pair]


def apply_generator(model_out, x, R, hp, include_parameter_generation=False):
    """reference train.py:336-355 given the generator's raw output: models that include parameter
    generation return ``(y_hat, y_hat_static)`` themselves; generic models return ``y_hat`` which is
    (front-)padded to the input length if pad_packed_sequence shortened it (``:347-349``, a no-op
    whenever the longest utterance spans the padded length, as in train.py's own batches) and goes
    through ``multi_stream_mlpg``."""
    if include_parameter_generation:
        return model_out
    y_hat = model_out
    if y_hat.size(1) != x.size(1):
        y_hat = F.pad(y_hat.unsqueeze(0), (0, 0, x.size(1) - y_hat.size(-2), 0)).squeeze(0)
    return y_hat, multi_stream_mlpg(y_hat, R, hp["stream_sizes"], hp["has_dynamic_features"])


def gan_step(g_forward, g_params, g_sum, d, d_sum, x, y, lengths, R, hp, w_d=1.0, mse_w=0.0,
             mge_w=1.0, adv_w=1.0, dropout_d=0.0, training=True, lr=0.01, weight_decay=1e-7, update=True,
             update_g=True, d_masks=None, d_opt=None, g_opt=None):
    """One mini-batch of the reference train_loop body (train.py:528-580) for ANY generator:
    ``g_forward()`` -> ``(y_hat, y_hat_static)`` is the result of ``apply_generator`` (train.py:336-355)
    with autograd history on ``g_params``; ``d`` is a ``DiscriminatorOracle``, the MLP discriminator
    ``[(W, b), ...]`` or None.  ``d_masks`` = {"real": [...], "fake": [...], "adv": [...]} injects dropout
    multipliers into the three discriminator forwards (see ``DiscriminatorOracle.forward``).

    Order of operations and quirks preserved (SURVEY.md section 3.2): single zero_grad at the
    top; y_hat_static is NOT detached in the discriminator update, so ``loss_d.backward`` also
    deposits the fake-term gradient on the generator; the discriminator steps before the third
    D forward used by the adversarial loss; gradients of both backwards accumulate on G before
    its clip + Adagrad step.  ``training=False`` with ``update=False`` is the "test" phase of
    train.py:481-486 (forwards and losses only).  ``update_g=False`` is the discriminator warm-up step
    (train.py --discriminator-warmup, :696): the generator runs without a graph and update_generator is not
    called, so the step reports loss_adv = 0, g_grad_norm = 0 and loss_g = mse_w loss_mse + mge_w loss_mge.
    The discriminator steps in place with Adagrad (state ``d_sum``) or the stepper ``d_opt``, the generator
    with ``g_sum`` or ``g_opt``.  Returns a dict of python floats and the generator outputs."""
    if isinstance(d, list):
        d = DiscriminatorOracle.of_layers(d)
    nw = hp["num_windows"]
    y_static = get_static_features(y, nw, hp["stream_sizes"], hp["has_dynamic_features"])   # :528-529
    mask = sequence_mask(lengths, x.size(1)).unsqueeze(-1)                                   # :535
    d_params = d.params() if d is not None else []
    for p in list(g_params) + d_params:                                                      # :538-539
        p.grad = None
    with torch.set_grad_enabled(torch.is_grad_enabled() and update_g):
        y_hat, y_hat_static = g_forward()                                                    # :542
    out = {}
    T = mask.sum().item()
    cond = hp.get("discriminator_linguistic_condition", False)
    dm = d_masks or {}
    if w_d > 0 and d is not None:
        # update_discriminator, train.py:245-279
        real_in = get_selected_static_stream(y_static, hp)
        fake_in = get_selected_static_stream(y_hat_static, hp)
        if cond:
            real_in = torch.cat((x, real_in), -1)
            fake_in = torch.cat((x, fake_in), -1)
        D_real = d.forward(real_in, lengths, dm.get("real"), dropout_d, training)
        out["real_correct"] = ((D_real > 0.5).float() * mask).sum().item()
        D_fake = d.forward(fake_in, lengths, dm.get("fake"), dropout_d, training)
        out["fake_correct"] = ((D_fake < 0.5).float() * mask).sum().item()
        loss_real = bce_real(D_real, mask, T)
        loss_fake = bce_fake(D_fake, mask, T)
        loss_d = loss_real + loss_fake
        if update:
            loss_d.backward(retain_graph=True)
            dg = [p.grad for p in d_params]
            out["d_grad_norm"] = float(clip_grad_norm(dg, 1.0))
            if d_opt is not None:
                d_opt(d_params, dg)                      # e.g. AdamStepper (hparams.py:125-130)
            else:
                adagrad_step(d_params, dg, d_sum, lr, weight_decay)
        out.update(loss_d=loss_d.item(), loss_fake_d=loss_fake.item(), loss_real_d=loss_real.item())
    # update_generator, train.py:282-320
    loss_mge = masked_mse(y_hat_static, y_static, mask=mask)
    loss_mse = masked_mse(y_hat, y, mask=mask)
    if adv_w > 0 and w_d > 0 and d is not None and update_g:
        fake_in = get_selected_static_stream(y_hat_static, hp)
        if cond:
            fake_in = torch.cat((x, fake_in), -1)
        D_adv = d.forward(fake_in, lengths, dm.get("adv"), dropout_d, training)
        loss_adv = bce_real(D_adv, mask, T)
    else:
        loss_adv = y.new_zeros(1)
        adv_w = 0.0
    loss_g = (mse_w * loss_mse + mge_w * loss_mge) + adv_w * loss_adv
    if update and update_g:
        loss_g.backward()
        g_params = list(g_params)
        gg = [p.grad if p.grad is not None else torch.zeros_like(p) for p in g_params]
        out["g_grad_norm"] = float(clip_grad_norm(gg, 1.0))
        if g_opt is not None:
            g_opt(g_params, gg)
        else:
            adagrad_step(g_params, gg, g_sum, lr, weight_decay)
    elif update:
        out["g_grad_norm"] = 0.0
    out.update(loss_mse=loss_mse.item(), loss_mge=loss_mge.item(), loss_adv=float(loss_adv.detach()),
               loss_g=float(loss_g.detach()), frames=T)
    return out, y_hat.detach(), y_hat_static.detach()


def gan_step_mlp(state, x, y, lengths, R, hp, w_d=1.0, mse_w=0.0, mge_w=1.0, adv_w=1.0,
                 dropout_g=0.0, dropout_d=0.0, training=True, lr=0.01, weight_decay=1e-7,
                 update=True, masks=None, d_opt=None, g_opt=None):
    """``gan_step`` for an MLP generator (reference ``MLP`` class, models.py:121-141) held in a
    ``GanStepState``.  ``masks`` = {"g": [...], "real": [...], "fake": [...], "adv": [...]} injects the
    dropout multipliers of the generator forward and of the three discriminator forwards."""
    masks = masks or {}

    def g_forward():
        y_hat = mlp_forward(x, state.g, dropout_g, training, last_sigmoid=False, masks=masks.get("g"))
        return apply_generator(y_hat, x, R, hp)

    return gan_step(g_forward, state.g_params(), state.g_sum, state.d if w_d > 0 else None, state.d_sum,
                    x, y, lengths, R, hp, w_d=w_d, mse_w=mse_w, mge_w=mge_w, adv_w=adv_w, dropout_d=dropout_d,
                    training=training, lr=lr, weight_decay=weight_decay, update=update, d_masks=masks,
                    d_opt=d_opt, g_opt=g_opt)


def _pair(sd, k, named, dtype=torch.float32):
    """(``k``.weight, ``k``.bias) of a reference state_dict as ``dtype`` leaf tensors (requires_grad), recorded in
    ``named``."""
    pair = tuple(torch.as_tensor(np.asarray(sd[k + s])).clone().to(dtype).requires_grad_(True)
                 for s in (".weight", ".bias"))
    named[k + ".weight"], named[k + ".bias"] = pair
    return pair


def _count(sd, pre):
    return len([k for k in sd if k.startswith(pre) and k.endswith(".weight")])


def _linear_layers(sd, pre, named, dtype=torch.float32):
    """[(W, b), ...] of the ``pre``.i layers then last_linear of a reference state_dict, recorded in ``named``."""
    return [_pair(sd, k, named, dtype)
            for k in ["%s.%d" % (pre, i) for i in range(_count(sd, pre + "."))] + ["last_linear"]]


def _lstm_layers(sd, prefix, num_layers, hidden, bidirectional, named, dtype=torch.float32):
    """One single-layer ``dtype`` torch nn.LSTM per layer of the nn.LSTM stored under ``prefix`` in a reference
    state_dict (see ``lstm_stack``); their parameters are recorded in ``named`` under the stack's names, in its
    parameters() order."""
    layers = []
    for k in range(num_layers):
        n_in = np.asarray(sd["%s.weight_ih_l%d" % (prefix, k)]).shape[1]
        lstm = torch.nn.LSTM(n_in, hidden, 1, batch_first=True, bidirectional=bidirectional).to(dtype)
        with torch.no_grad():
            for s in ("", "_reverse")[:2 if bidirectional else 1]:
                for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"):
                    p = getattr(lstm, "%s_l0%s" % (n, s))
                    p.copy_(torch.as_tensor(np.asarray(sd["%s.%s_l%d%s" % (prefix, n, k, s)])))
                    named["%s.%s_l%d%s" % (prefix, n, k, s)] = p
        layers.append(lstm)
    return layers


class GeneratorOracle(object):
    """CPU generator + Adagrad state for ``gan_step`` built from a reference ``state_dict`` (same key
    names as the reference classes, models.py:40-48,84-86,128-131,153-158,198-200).  ``kind``:
    "mlp" (MLP), "highway" (In2OutHighwayNet), "rnn_highway" (In2OutRNNHighwayNet), "lstm" (LSTMRNN;
    GRURNN with ``rnn_attr="gru"``), "sru" (SRURNN, with ``bidirectional`` and the cells' ``activation_type``;
    parity unpinned, see ``sru_layer_forward``).  Recurrent LSTM kinds run torch's own CPU ``nn.LSTM`` on
    packed sequences like the reference (``lstm_stack``).  ``named`` / ``params()`` / ``sums`` follow the
    model's parameters() order.

    ``forward``'s ``masks`` injects the product's dropout decisions: the hidden-layer multipliers of "mlp" /
    "highway" (see ``mlp_forward``), the inter-layer multipliers of "rnn_highway" / "lstm" (see ``lstm_stack``)
    and [(mask_x, mask_h or None)] per layer of "sru" (see ``sru_layer_forward``).  ``dropout_p`` / ``training``
    apply to "mlp" / "highway" without masks; the recurrent kinds drop out nothing of their own.

    ``dtype`` is that of every parameter (float32 as the reference trains; float64 gives a reference for the product's
    fp32 gradients, fed float64 inputs and a float64 R)."""

    def __init__(self, kind, sd, static_dim=None, num_hidden=None, hidden_dim=None, bidirectional=False,
                 rnn_attr="lstm", activation_type=2, dtype=torch.float32):
        self.kind, self.static_dim = kind, static_dim
        self.bidirectional, self.activation_type = bidirectional, activation_type
        self.named = {}
        if kind in ("highway", "rnn_highway"):
            self.gate = _pair(sd, "T", self.named, dtype)
        if kind in ("mlp", "highway"):
            self.layers = _linear_layers(sd, "layers" if kind == "mlp" else "H", self.named, dtype)
        else:
            if kind == "sru":
                n = _count(sd, "gru.rnn_lst.")
                self.layers = [_pair(sd, "gru.rnn_lst.%d" % i, self.named, dtype) for i in range(n)]
            else:
                self.layers = _lstm_layers(sd, rnn_attr, num_hidden, hidden_dim, bidirectional, self.named, dtype)
            self.h2o = _pair(sd, "hidden2out", self.named, dtype)
        self.sums = [torch.zeros_like(p) for p in self.params()]

    def params(self):
        return list(self.named.values())

    def include_parameter_generation(self):
        return self.kind in ("highway", "rnn_highway")

    def forward(self, x, R, lengths, hp, dropout_p=0.0, training=False, masks=None):
        """(y_hat, y_hat_static) as reference apply_generator (train.py:336-355) returns them."""
        if self.kind == "mlp":
            out = mlp_forward(x, self.layers, dropout_p, training, last_sigmoid=False, masks=masks)
        elif self.kind == "highway":
            out = in2out_highway_forward(x, R, self.gate, self.layers, self.static_dim, dropout_p, training, masks)
        elif self.kind == "rnn_highway":
            out = in2out_rnn_highway_forward(x, R, lengths, self.gate, self.layers, self.h2o, self.static_dim, masks)
        elif self.kind == "sru":
            out = sru_forward(x, self.layers, self.h2o, self.bidirectional, self.activation_type, masks)
        else:
            out = lstm_forward(x, lengths, self.layers, self.h2o, masks=masks)
        return apply_generator(out, x, R, hp, self.include_parameter_generation())


def discriminator_layers(sd, dtype=torch.float32):
    """[(W, b), ...] (``dtype``, requires_grad) of a reference ``MLP`` state_dict (``layers.i``, ``last_linear``)."""
    return _linear_layers(sd, "layers", {}, dtype)


class DiscriminatorOracle(object):
    """CPU discriminator for ``gan_step`` and the spoofing-rate count, built from a reference ``state_dict`` whose keys
    give its kind and whose tensors give its shape: ``MLP`` (``layers.i.*``, ``last_linear.*``; models.py:121-141) or
    ``LSTMRNN`` / ``GRURNN`` (an nn.LSTM under ``lstm.`` or ``gru.``, then ``hidden2out.*``; models.py:170-213), with
    last_sigmoid=True as train.py:774 builds it.  ``named`` / ``params()`` follow the state_dict.  A recurrent one
    runs ``lstm_stack`` and drops out nothing but the injected masks.  ``dtype`` as for ``GeneratorOracle``."""

    def __init__(self, sd, dtype=torch.float32):
        self.named = {}
        if "last_linear.weight" in sd:
            self.mlp = _linear_layers(sd, "layers", self.named, dtype)
            return
        self.mlp = None
        pre = "lstm" if "lstm.weight_ih_l0" in sd else "gru"
        n = len([k for k in sd if k.startswith(pre + ".weight_ih_l") and not k.endswith("_reverse")])
        hidden = np.asarray(sd[pre + ".weight_hh_l0"]).shape[1]
        self.layers = _lstm_layers(sd, pre, n, hidden, pre + ".weight_ih_l0_reverse" in sd, self.named, dtype)
        self.h2o = _pair(sd, "hidden2out", self.named, dtype)

    @classmethod
    def of_layers(cls, layers):
        """The MLP discriminator ``[(W, b), ...]`` itself (stepped in place), as ``discriminator_layers`` gives it."""
        d = cls.__new__(cls)
        d.mlp = layers
        names = ["layers.%d" % i for i in range(len(layers) - 1)] + ["last_linear"]
        d.named = {k + s: t for k, pair in zip(names, layers) for s, t in zip((".weight", ".bias"), pair)}
        return d

    def params(self):
        return list(self.named.values())

    def forward(self, x, lengths, masks=None, dropout_p=0.0, training=False):
        """D(x) in (0, 1); ``masks`` as ``mlp_forward`` / ``lstm_stack`` take them.  ``dropout_p`` / ``training``
        apply to an MLP without masks; an MLP ignores ``lengths``."""
        if self.mlp is not None:
            return mlp_forward(x, self.mlp, dropout_p, training, last_sigmoid=True, masks=masks)
        return lstm_forward(x, lengths, self.layers, self.h2o, last_sigmoid=True, masks=masks)


def reference_output(ref_d, y_hat_static, lengths, hp):
    """The reference discriminator's output on the adversarial columns of y_hat_static (train.py:549-558): dropout off
    (D_ref in eval mode, :445), no linguistic conditioning (:554-555).  ``ref_d`` is a ``DiscriminatorOracle``."""
    with torch.no_grad():
        return ref_d.forward(get_selected_static_stream(y_hat_static, hp), lengths)


def spoof_count(ref_d, y_hat_static, lengths, mask, hp):
    """``((D_ref(get_selected_static_stream(y_hat_static), lengths) > 0.5).float() * mask).sum()`` (train.py:549-558)."""
    return ((reference_output(ref_d, y_hat_static, lengths, hp) > 0.5).float() * mask).sum().item()


# ------------------------------------------------------------------------------ SRU (unpinned)
def sru_layer_forward(x, W, b, bidirectional=False, use_tanh=False, use_relu=True, mask_x=None, mask_h=None):
    """SRU v1 layer (Lei et al. 2017, github.com/taolei87/sru ``cuda_functional.py``; NOT vendored
    in the reference tree -- restated from the published recurrence, **parity unpinned**):

        U = x W ; per direction and hidden unit j, with k = 3 (n_in == n_out) or 4 gates
        f_t = sigmoid(U_f + b_f) ; r_t = sigmoid(U_r + b_r)
        c_t = f_t * c_{t-1} + (1 - f_t) * U_x
        h_t = r_t * g(c_t) + (1 - r_t) * x'_t     (x' = x if k == 3 else U_x')

    ``x``: (T, B, n_in); ``W``: (n_in, dirs*k*d) laid out ``[..., dir, d, k]`` (k fastest) as in
    the upstream kernel; ``b``: (dirs*2*d,) = [f-bias | r-bias] per direction.

    Train mode of upstream ``SRUCell.forward``: ``mask_x`` (B, n_in) is the variational ``rnn_dropout``
    multiplier applied to the GEMM input ONLY (``u = (x * mask_x) @ W``; the highway term keeps the unmasked
    ``x``); ``mask_h`` (B, dirs*d) is the ``dropout`` multiplier on ``g(c_t)`` inside the recurrence
    (``h_t = r_t * g(c_t) * mask_h + (1 - r_t) * x'_t``)."""
    T, B, n_in = x.shape
    dirs = 2 if bidirectional else 1
    d = b.numel() // (2 * dirs)
    k = W.shape[1] // (d * dirs)
    xin = x * mask_x.unsqueeze(0) if mask_x is not None else x
    U = (xin.reshape(-1, n_in) @ W).view(T, B, dirs, d, k)
    bias = b.view(dirs, 2, d)
    act = torch.tanh if use_tanh else (torch.relu if use_relu else (lambda v: v))
    outs = []
    for di in range(dirs):
        c = x.new_zeros(B, d)
        hs = [None] * T
        order = range(T) if di == 0 else range(T - 1, -1, -1)
        for t in order:
            u = U[t, :, di]
            f = torch.sigmoid(u[..., 1] + bias[di, 0])
            r = torch.sigmoid(u[..., 2] + bias[di, 1])
            c = f * c + (1 - f) * u[..., 0]
            xp = x[t][:, di * d:(di + 1) * d] if k == 3 else u[..., 3]
            gc = act(c) * mask_h[:, di * d:(di + 1) * d] if mask_h is not None else act(c)
            hs[t] = r * gc + (1 - r) * xp
        outs.append(torch.stack(hs, 0))
    return torch.cat(outs, -1)


# ------------------------------------------------------------------------------------------------------------------
# Logging metrics of the step (reference train.py:358-432): inv_scale :358-381, split_streams :384-397,
# compute_distortions :399-432.  numpy float64; `hp` needs .name and, for "acoustic", .windows / .stream_sizes /
# .has_dynamic_features, for "vc" .order.  nnmnkwii.preprocessing.inv_scale(x, m, s) = x * s + m.
def inv_scale_streams(mgc, lf0, vuv, bap, Y_mean, Y_std, hp):
    nw = len(hp.windows)
    mgc_dim, lf0_dim, vuv_dim, bap_dim = hp.stream_sizes                     # static + dynamic domain (:360)
    lf0_0 = mgc_dim
    vuv_0 = lf0_0 + lf0_dim
    bap_0 = vuv_0 + vuv_dim
    mgc = mgc * Y_std[:mgc_dim // nw] + Y_mean[:mgc_dim // nw]               # :368
    lf0 = lf0 * Y_std[lf0_0:lf0_0 + lf0_dim // nw] + Y_mean[lf0_0:lf0_0 + lf0_dim // nw]
    bap = bap * Y_std[bap_0:bap_0 + bap_dim // nw] + Y_mean[bap_0:bap_0 + bap_dim // nw]
    vuv = vuv * Y_std[vuv_0] + Y_mean[vuv_0]
    return mgc, lf0, (vuv > 0.5).astype(np.int64), bap                       # :376-379


def split_streams_np(y_static, Y_mean, Y_std, hp):
    from . import nnmnkwii_port  # noqa: F401  (same package: the metrics live next to the MLPG port)
    sizes = get_static_stream_sizes(hp.stream_sizes, hp.has_dynamic_features, len(hp.windows))   # :386
    a = np.cumsum([0] + list(sizes))
    y = np.asarray(y_static, dtype=np.float64)
    return inv_scale_streams(y[:, :, a[0]:a[1]], y[:, :, a[1]:a[2]], y[:, :, a[2]], y[:, :, a[3]:], Y_mean, Y_std, hp)


def compute_distortions(y_static, y_hat_static, Y_mean, Y_std, lengths, hp):
    from . import nnmnkwii_port as M
    Y_mean, Y_std = np.asarray(Y_mean, dtype=np.float64), np.asarray(Y_std, dtype=np.float64)
    if hp.name == "acoustic":                                                 # :400-417
        mgc, lf0, vuv, bap = split_streams_np(y_static, Y_mean, Y_std, hp)
        mgc_h, lf0_h, vuv_h, bap_h = split_streams_np(y_hat_static, Y_mean, Y_std, hp)
        try:
            f0_mse = M.lf0_mean_squared_error(lf0, vuv, lf0_h, vuv_h, lengths=lengths, linear_domain=True)
        except ZeroDivisionError:
            f0_mse = float("nan")
        return {"mcd": M.melcd(mgc[:, :, 1:], mgc_h[:, :, 1:], lengths=lengths),
                "bap_mcd": M.melcd(bap, bap_h, lengths=lengths) / 10.0,
                "f0_rmse": float(np.sqrt(f0_mse)),
                "vuv_err": M.vuv_error(vuv, vuv_h, lengths=lengths)}
    if hp.name == "duration":                                                 # :418-422
        a = np.asarray(y_static, dtype=np.float64) * Y_std + Y_mean
        b = np.asarray(y_hat_static, dtype=np.float64) * Y_std + Y_mean
        return {"dur_rmse": float(np.sqrt(M.mean_squared_error(a, b, lengths=lengths)))}
    if hp.name == "vc":                                                       # :423-428
        d = hp.order
        a = np.asarray(y_static, dtype=np.float64) * Y_std[:d] + Y_mean[:d]
        b = np.asarray(y_hat_static, dtype=np.float64) * Y_std[:d] + Y_mean[:d]
        return {"mcd": M.melcd(a, b, lengths=lengths)}
    raise AssertionError("unknown hp.name %r" % (hp.name,))
