"""Helpers shared by the fused-step test modules: the product's models and their oracles, batches, the step's own dropout
masks regenerated from its seeds, the oracle's re-sync between steps, the comparisons, and host-only gantts_gan_step_t
configurations for the configuration-rule tests.  The mask helpers call the product's gantts_dropout, so they live here
and not in the oracle package."""
import numpy as np
import pytest
import torch

from conftest import TTS_HP, WINDOWS
from oracle import gantts_port as gp

FAKE = 1 << 20          # placeholder device pointer: the configuration check and the workspace layout never dereference it
ADAM = dict(lr=1e-3, betas=(0.5, 0.9), weight_decay=0.0, eps=1e-8)
TTS_STREAMS = [(0, 60, 1, 0), (180, 1, 1, 60), (183, 1, 0, 61), (184, 1, 1, 62)]


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__
    __graft_entry__.build()
    return torch.device("cuda:0")


def npy(t):
    return t.detach().cpu().numpy()


def step_hp(ohp):
    """gantts_b200.step.HParams of an oracle hparams dict."""
    from gantts_b200 import step as gstep
    return gstep.HParams(windows=WINDOWS[:ohp["num_windows"]], stream_sizes=ohp["stream_sizes"],
                         has_dynamic_features=ohp["has_dynamic_features"],
                         adversarial_streams=ohp["adversarial_streams"],
                         mask_nth_mgc_for_adv_loss=ohp["mask_nth_mgc_for_adv_loss"],
                         discriminator_linguistic_condition=ohp["discriminator_linguistic_condition"])


def ragged_lengths(B, T, seed):
    rng = np.random.RandomState(seed)
    return sorted([T] + [int(v) for v in rng.randint(T // 2, T, B - 1)], reverse=True)


def make_batch(B, T, d_in, d_out, lens, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, T, d_in, generator=g)
    y = torch.randn(B, T, d_out, generator=g)
    for b, n in enumerate(lens):
        x[b, n:] = 0
        y[b, n:] = 0
    return x, y


def sd_numpy(m):
    return {k: v.detach().cpu().numpy() for k, v in m.state_dict().items()}


def snapshot(*tensors):
    return [t.detach().clone() for t in tensors]


def assert_equal_lists(a, b, what):
    assert len(a) == len(b)
    for i, (u, v) in enumerate(zip(a, b)):
        assert torch.equal(u, v), (what, i)


# ---- the product's models and their oracles
def vc_ohp(width, cond=False):
    return dict(stream_sizes=[width], has_dynamic_features=[True], adversarial_streams=[True],
                mask_nth_mgc_for_adv_loss=0, num_windows=3, discriminator_linguistic_condition=cond)


def tts_ohp(cond=False):
    return dict(TTS_HP, discriminator_linguistic_condition=cond)


def sru_models(seed, in_dim, out_dim, layers, hidden, bidir, relu, p, rnn_p, d_hidden, d_layers, d_p, n_adv):
    import gantts_b200
    torch.manual_seed(seed)
    mg = gantts_b200.models.SRURNN(in_dim=in_dim, out_dim=out_dim, num_hidden=layers, hidden_dim=hidden,
                                   bidirectional=bidir, dropout=p, use_relu=int(relu), rnn_dropout=rnn_p)
    for cell in mg.gru.rnn_lst:                        # non-zero forget / reset biases
        cell.bias.data.uniform_(-0.5, 0.5)
    md = gantts_b200.models.MLP(in_dim + n_adv, 1, d_layers, d_hidden, dropout=d_p, last_sigmoid=True)
    return mg, md


def rhw_models(seed, S, layers, hidden, bidir, p, d_hidden, d_layers, p_d, cond=False):
    import gantts_b200
    torch.manual_seed(seed)
    mg = gantts_b200.models.In2OutRNNHighwayNet(in_dim=3 * S, out_dim=3 * S, static_dim=S, num_hidden=layers,
                                                hidden_dim=hidden, bidirectional=bidir, dropout=p)
    md = gantts_b200.models.MLP(S + (3 * S if cond else 0), 1, d_layers, d_hidden, dropout=p_d, last_sigmoid=True)
    return mg, md


def build(kind, seed):
    """(model_g, model_d, oracle hparams, d_in, d_out, G hidden widths (MLP / highway), D hidden width, D dropout) with
    an MLP discriminator."""
    import gantts_b200
    M = gantts_b200.models
    torch.manual_seed(seed)
    if kind == "mlp":
        mg = M.MLP(20, 187, 2, 32, dropout=0.5, last_sigmoid=False)
        md = M.MLP(58, 1, 2, 16, dropout=0.5, last_sigmoid=True)
        return mg, md, TTS_HP, 20, 187, [32, 32], 16, 0.5
    if kind == "highway":
        mg = M.In2OutHighwayNet(in_dim=27, out_dim=27, static_dim=9, num_hidden=2, hidden_dim=24, dropout=0.5)
        md = M.MLP(9, 1, 2, 16, dropout=0.5, last_sigmoid=True)
        return mg, md, vc_ohp(27), 27, 27, [24, 24], 16, 0.5
    if kind == "vc_full":
        mg = M.In2OutHighwayNet(in_dim=177, out_dim=177, static_dim=59, num_hidden=3, hidden_dim=512, dropout=0.5)
        md = M.MLP(59, 1, 2, 256, dropout=0.5, last_sigmoid=True)
        return mg, md, vc_ohp(177), 177, 177, [512] * 3, 256, 0.5
    if kind == "sru":
        mg, md = sru_models(seed, 20, 187, 2, 16, True, True, 0.2, 0.2, 32, 2, 0.5, 58)
        return mg, md, tts_ohp(True), 20, 187, None, 32, 0.5
    mg, md = rhw_models(seed, 8, 2, 12, True, 0.3, 32, 2, 0.5)
    return mg, md, vc_ohp(24), 24, 24, None, 32, 0.5


def make_models(kind, seed, cond, d_layers=2, d_hidden=12, bidir=True, p_d=0.5, gru=False, full=False):
    """(generator, recurrent discriminator, ohp, generator input width) with every generator dropout 0; the
    discriminator is an LSTMRNN (GRURNN with gru=True) with LSTM dropout p_d."""
    import gantts_b200
    M = gantts_b200.models
    torch.manual_seed(seed)
    if kind == "mlp":
        ohp, d_in = tts_ohp(cond), 20
        mg = M.MLP(d_in, 187, 2, 24, dropout=0.0, last_sigmoid=False)
    elif kind == "highway":
        S = 59 if full else 8
        ohp, d_in = vc_ohp(3 * S, cond), 3 * S
        mg = M.In2OutHighwayNet(in_dim=d_in, out_dim=d_in, static_dim=S, num_hidden=3 if full else 2,
                                hidden_dim=512 if full else 24, dropout=0.0)
    elif kind == "rnn_highway":
        ohp, d_in = vc_ohp(24, cond), 24
        mg = M.In2OutRNNHighwayNet(in_dim=24, out_dim=24, static_dim=8, num_hidden=2, hidden_dim=12, bidirectional=True,
                                   dropout=0.0)
    else:
        ohp, d_in = tts_ohp(cond), 425 if full else 20
        mg = M.SRURNN(in_dim=d_in, out_dim=187, num_hidden=6 if full else 2, hidden_dim=512 if full else 16,
                      bidirectional=True, dropout=0.0, use_relu=1, rnn_dropout=0.0)
        for cell in mg.gru.rnn_lst:
            cell.bias.data.uniform_(-0.5, 0.5)
    n_adv = 58 if ohp["stream_sizes"] == TTS_HP["stream_sizes"] else d_in // 3
    cls = M.GRURNN if gru else M.LSTMRNN
    md = cls(in_dim=n_adv + (d_in if cond else 0), out_dim=1, num_hidden=d_layers, hidden_dim=d_hidden,
             bidirectional=bidir, dropout=p_d, last_sigmoid=True)
    return mg, md, ohp, d_in


def generator_oracle(mg, dtype=torch.float32):
    """gp.GeneratorOracle of the product's generator mg (MLP, In2OutHighwayNet, In2OutRNNHighwayNet or SRURNN)."""
    sd, name = sd_numpy(mg), type(mg).__name__
    if name == "MLP":
        return gp.GeneratorOracle("mlp", sd, dtype=dtype)
    if name == "In2OutHighwayNet":
        return gp.GeneratorOracle("highway", sd, static_dim=mg.static_dim, dtype=dtype)
    if name == "SRURNN":
        cell = mg.gru.rnn_lst[0]
        return gp.GeneratorOracle("sru", sd, bidirectional=cell.bidirectional, activation_type=cell.activation_type,
                                  dtype=dtype)
    lm = mg.lstm
    return gp.GeneratorOracle("rnn_highway", sd, static_dim=mg.static_dim, num_hidden=lm.num_layers,
                              hidden_dim=lm.hidden_size, bidirectional=lm.bidirectional, dtype=dtype)


def fused(mg, md, hp, B, T, optimizer="Adagrad", **kw):
    from gantts_b200 import fused as F
    return F.FusedGanStep(mg, md, step_hp(hp), B, T, weight_decay=0.0, optimizer=optimizer,
                          optimizer_params=ADAM if optimizer == "Adam" else None, **kw)


def split_step(fs, x, y, lengths, update_g=True, phases=(1, 6), between=None, frames=None):
    """FusedGanStep.step's training call as one native call per entry of `phases` (GANTTS_STEP_D = 1, _G = 2, _FINISH =
    4; the default is the discriminator phase, then the generator and finishing phases), with between(phase) called after
    each of them but the last, where a data-parallel caller all-reduces the gradient buffers.  frames: the normaliser a
    caller passes (the GLOBAL count of valid frames); None lets the step count the mask."""
    from gantts_b200 import _lib
    b, t = int(x.shape[0]), int(x.shape[1])
    fs._set_shape(b, t)
    fs._shape = (b, t, fs._mlpg_table(t).data_ptr())
    fs.cfg.adv_w = 1.0
    fs._bind_params(fs.cfg)
    seed = (fs._seed + fs._step) & ((1 << 61) - 1)
    fs.last_seed = seed
    fs._step += 1
    fs._set_optimizers(fs.opt_g.steps + 1, fs.opt_d.steps + 1)
    d_only = 0 if update_g else _lib.STEP_D_ONLY
    inv = 0.0 if frames is None else 1.0 / float(frames)
    for i, ph in enumerate(phases):
        fs._call(ph | d_only, x, y, lengths, inv, seed)
        if between is not None and i + 1 < len(phases):
            between(ph)
    fs.opt_d.steps += 1
    if update_g:
        fs.opt_g.steps += 1


# ---- the dropout masks of the product's last training step, regenerated from its seeds
def d_masks(fs, M, d_hidden, p, dev):
    """The MLP discriminator's keep masks (gantts_gan_step_seed: 1 = stacked real|fake, 2 = adv)."""
    from gantts_b200 import ops, _lib
    lib = _lib.load()
    s = fs.last_seed
    stacked = ops.mlp_dropout_masks(2 * M, d_hidden, p, lib.gantts_gan_step_seed(s, 1), dev)
    return {"real": [m[:M].cpu() for m in stacked], "fake": [m[M:].cpu() for m in stacked],
            "adv": [m.cpu() for m in ops.mlp_dropout_masks(M, d_hidden, p, lib.gantts_gan_step_seed(s, 2), dev)]}


def d_lstm_masks(fs, md, M, dev):
    """The recurrent discriminator's inter-layer masks (gantts_d_lstm_mask_seed: 1 = stacked real|fake, 2 = adv)."""
    from gantts_b200 import ops, _lib
    lib = _lib.load()
    lstm = getattr(md, md._rnn_attr)
    nh = lstm.hidden_size * (2 if lstm.bidirectional else 1)
    mk = lambda rows, which: [ops.dropout_mask(rows, nh, lstm.dropout, lib.gantts_d_lstm_mask_seed(fs.last_seed, which, k),
                                               dev).cpu() for k in range(lstm.num_layers - 1)]
    stacked = mk(2 * M, 1)
    return {"real": [m[:M] for m in stacked], "fake": [m[M:] for m in stacked], "adv": mk(M, 2)}


def sru_masks(fs, mg, B, dev):
    """The SRURNN generator's masks: [(mask_x, mask_h or None)] per layer (gantts_sru_mask_seed)."""
    from gantts_b200 import ops, _lib
    lib = _lib.load()
    cells = list(mg.gru.rnn_lst)
    out = []
    for i, cell in enumerate(cells):
        nc = cell.n_out * (2 if cell.bidirectional else 1)
        mx = ops.dropout_mask(B, cell.n_in, cell.rnn_dropout, lib.gantts_sru_mask_seed(fs.last_seed, i, 0), dev).cpu()
        mh = ops.dropout_mask(B, nc, cell.dropout, lib.gantts_sru_mask_seed(fs.last_seed, i, 1), dev).cpu() \
            if i + 1 < len(cells) else None
        out.append((mx, mh))
    return out


def lstm_masks(fs, mg, B, T, dev):
    """The In2OutRNNHighwayNet generator's inter-layer masks (gantts_lstm_mask_seed)."""
    from gantts_b200 import ops, _lib
    lib = _lib.load()
    lm = mg.lstm
    nh = lm.hidden_size * (2 if lm.bidirectional else 1)
    return [ops.dropout_mask(B * T, nh, lm.dropout, lib.gantts_lstm_mask_seed(fs.last_seed, k), dev).cpu()
            for k in range(lm.num_layers - 1)]


def g_masks(kind, fs, mg, B, T, g_hidden, dev):
    """The generator's keep masks of a `build(kind, ...)` generator."""
    from gantts_b200 import ops, _lib
    if kind == "sru":
        return sru_masks(fs, mg, B, dev)
    if kind == "rnn_highway":
        return lstm_masks(fs, mg, B, T, dev)
    seed = _lib.load().gantts_gan_step_seed(fs.last_seed, 0)
    return [m.cpu() for m in ops.mlp_dropout_masks(B * T, g_hidden, mg.dropout_p, seed, dev)]


def adv_loss_with(d, x, ys_ref, lens, ohp, adv_masks):
    """loss_adv of the oracle's y_hat_static through `d`, the gp.DiscriminatorOracle of the PRODUCT's updated
    discriminator.  The adversarial forward runs after the discriminator's first Adagrad / Adam step, which moves every
    weight by about lr * sign(g): a weight whose gradient is within rounding of zero lands 2 lr apart in the two
    implementations, and at the conditioned D's 483 inputs those few weights move loss_adv by a few 1e-4.  With the
    product's D on both sides the comparison isolates the generator's output and the loss arithmetic."""
    fake_in = gp.get_selected_static_stream(ys_ref, ohp)
    if ohp["discriminator_linguistic_condition"]:
        fake_in = torch.cat((x, fake_in), -1)
    mask = gp.sequence_mask(lens, x.size(1)).unsqueeze(-1)
    with torch.no_grad():
        return float(gp.bce_real(d.forward(fake_in, lens, adv_masks), mask, mask.sum().item()))


def loss_errors(got, ref, keys):
    return {k: abs(float(got[k]) - ref[k]) / max(abs(ref[k]), 1e-12) for k in keys}


def check_weights(model, named, tag, median=5e-6):
    """Every parameter of `model` against the oracle tensor of the same name: median |delta| below `median` and max
    <= 0.0201 (a first Adagrad / Adam step moves a weight by lr * sign(g))."""
    for k, v in model.named_parameters():
        d = np.abs(npy(v) - named[k].detach().numpy())
        assert np.median(d) < median and d.max() <= 0.0201, (tag, k, np.median(d), d.max())


def resync_oracle(fs, mg, md, gen, d_params, d_sums, g_opt=None, d_opt=None):
    """Start the oracle's next step from the product's weights and optimiser state: gen.named (keyed like
    mg.named_parameters()) with gen.sums or the Adam stepper g_opt in gen.named's order; d_params with d_sums or d_opt."""
    sd = fs.state_dict()
    order = list(gen.named)
    names = [n for n, _ in mg.named_parameters()]
    with torch.no_grad():
        for n, q in mg.named_parameters():
            gen.named[n].copy_(q.detach().cpu())
        for r, q in zip(d_params, md.parameters()):
            r.copy_(q.detach().cpu())
        for key, idx, sums, opt in (("optimizer_g", [order.index(n) for n in names], gen.sums, g_opt),
                                    ("optimizer_d", range(len(d_params)), d_sums, d_opt)):
            st = sd[key]["state"]
            for i, j in enumerate(idx):
                if opt is None:
                    sums[j].copy_(st[i]["sum"].cpu())
                else:
                    opt.m[j].copy_(st[i]["exp_avg"].cpu())
                    opt.v[j].copy_(st[i]["exp_avg_sq"].cpu())


def step_config(g_dims, d_dims, streams, static_cols, adv_cols, conditioned=False):
    """A gantts_gan_step_t with an MLP generator g_dims and discriminator d_dims, Adagrad, w_d = 1, B = 2 x T = 16 and no
    tensor tables yet (fill_tables); the caller adds its generator's shape block."""
    from gantts_b200 import _lib
    c = _lib.GanStepT()
    c.B, c.T = 2, 16
    for m, dims, act in ((c.g, g_dims, _lib.ACT_NONE), (c.d, d_dims, _lib.ACT_SIGMOID)):
        m.num_layers = len(dims) - 1
        for i, v in enumerate(dims):
            m.dims[i] = v
        m.last_act = act
    c.streams = _lib.make_streams(streams)
    c.windows = _lib.make_windows(WINDOWS)
    c.mlpg_table = FAKE
    c.n_static = c.n_static_cols = len(static_cols)
    for i, v in enumerate(static_cols):
        c.static_cols[i] = v
    c.n_adv = len(adv_cols)
    for i, v in enumerate(adv_cols):
        c.adv_cols[i] = v
    c.d_conditioned = int(conditioned)
    c.w_d, c.mge_w, c.adv_w, c.max_norm, c.lr_g, c.lr_d, c.eps = 1.0, 1.0, 1.0, 1.0, 0.01, 0.01, 1e-10
    c.optimizer = _lib.OPT_ADAGRAD
    return c


def fill_tables(c, n_g):
    """Placeholder tensors and Adagrad state for n_g generator tensors and the discriminator's 2 per layer."""
    for tab, n in ((c.g_tensors, n_g), (c.d_tensors, 2 * c.d.num_layers)):
        tab.n = n
        for i in range(n):
            tab.param[i] = tab.state[i] = FAKE
    return c


def use_adam(c, missing=()):
    """Switch c to Adam with exp_avg_sq for every tensor but the generator tensors in `missing`."""
    from gantts_b200 import _lib
    c.optimizer, c.beta1, c.beta2 = _lib.OPT_ADAM, 0.5, 0.9
    for tab in (c.g_tensors, c.d_tensors):
        for i in range(tab.n):
            tab.state2[i] = FAKE
    for i in missing:
        c.g_tensors.state2[i] = None


def _vc_step_config():
    """A valid In2OutHighwayNet configuration of gantts_gan_step_t: G 177 -> 64 -> 3 S with the gate (S = 59), D S -> 32
    -> 1 (host pointers are placeholders: only the configuration check and the workspace layout run)."""
    S = 59
    c = step_config((177, 64, 3 * S), (S, 32, 1), [(0, S, True, 0)], range(S), range(S))
    c.highway.static_dim = S
    return fill_tables(c, 2 + 2 * 2)


def _sru_step_config():
    """A valid SRURNN configuration of gantts_gan_step_t on the tts_acoustic layout with a conditioned D: 3 bidirectional
    layers of 16 over in_dim 40, hidden2out 32 -> 187, D 40 + 58 -> 32 -> 1 (host pointers are placeholders: only the
    configuration check and the workspace layout run)."""
    from gantts_b200 import multistream, step as gstep
    in_dim, hidden, nl = 40, 16, 3
    hp = gstep.TTS_ACOUSTIC
    entries, n_static = multistream.mlpg_stream_entries(hp.stream_sizes, hp.has_dynamic_features, [True] * 4, 3)
    c = step_config((2 * hidden, 187), (in_dim + 58, 32, 1), entries, range(n_static), range(2, 60), conditioned=True)
    s = c.sru
    s.num_layers, s.in_dim, s.hidden, s.bidirectional, s.act = nl, in_dim, hidden, 1, 2
    s.dropout, s.rnn_dropout = 0.2, 0.2
    return fill_tables(c, 2 * nl + 2)


def _rhw_step_config():
    """A valid In2OutRNNHighwayNet configuration of gantts_gan_step_t on the cfg3 layout: the gate (S = 59), 3
    bidirectional LSTM layers of 16 over 3 S, hidden2out 32 -> 3 S, D S -> 32 -> 1 (host pointers are placeholders: only
    the configuration check and the workspace layout run)."""
    S, H, nl = 59, 16, 3
    c = step_config((2 * H, 3 * S), (S, 32, 1), [(0, S, True, 0)], range(S), range(S))
    c.highway.static_dim = S
    ls = c.lstm
    ls.num_layers, ls.in_dim, ls.hidden, ls.bidirectional, ls.dropout = nl, 3 * S, H, 1, 0.5
    return fill_tables(c, 2 + 8 * nl + 2)


def _rnn_d_config(bidir=1, layers=2, hidden=16, cond=False):
    """An MLP generator 20 -> 24 -> 27 on one dynamic stream of 9 static columns, and an LSTMRNN D over those 9 columns
    (plus the 20 conditioning columns when cond): `layers` LSTM layers of `hidden` units, then hidden2out -> 1."""
    nh = hidden * (2 if bidir else 1)
    c = step_config((20, 24, 27), (nh, 1), [(0, 9, True, 0)], range(9), range(9), conditioned=cond)
    dl = c.d_lstm
    dl.num_layers, dl.in_dim, dl.hidden, dl.bidirectional, dl.dropout = layers, 9 + (20 if cond else 0), hidden, bidir, 0.5
    fill_tables(c, 4)
    c.d_tensors.n = 4 * layers * (2 if bidir else 1) + 2
    for i in range(c.d_tensors.n):
        c.d_tensors.param[i] = c.d_tensors.state[i] = c.g_tensors.param[0]
    return c


def config_checker():
    """(ws, err, rejected): the workspace size gantts_gan_step_workspace_bytes gives a config (0 = rejected), the last
    error message, and rejected(make, mutate, needle) asserting that mutate(make()) is rejected with `needle` in it."""
    import ctypes
    import __graft_entry__
    __graft_entry__.build()
    from gantts_b200 import _lib
    lib = _lib.load()
    ws = lambda c: lib.gantts_gan_step_workspace_bytes(ctypes.byref(c))
    err = lambda: lib.gantts_last_error_string().decode()

    def rejected(make, mutate, needle):
        c = make()
        mutate(c)
        assert ws(c) == 0 and needle in err(), (needle, err())
    return ws, err, rejected
