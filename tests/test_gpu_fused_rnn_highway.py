"""The fused GAN step (gantts_gan_step / FusedGanStep) with the In2OutRNNHighwayNet generator (reference
gantts/models.py:72-118; bench.py cfg3): the sigmoid gate on x_static, the packed-sequence LSTM stack, hidden2out and the
highway combine around the MLPG, their backward and their optimiser step inside the one-call step.

The checker, GeneratorOracle("rnn_highway"), composes one-layer CPU torch nn.LSTMs on packed sequences and injects the
step's own inter-layer dropout masks between them (every mask is gantts_dropout(ones[B * T][ndir * H], p,
gantts_lstm_mask_seed(seed, layer))); with all-ones masks it equals the reference's one multi-layer nn.LSTM.  The
discriminator's masks come from gantts_gan_step_seed as in test_gpu_fused_highway.py.  Tolerances: losses, gradient norms
and y_hat_static 2e-4 relative (the cfg3 bound of test_gpu_train_mode.py); y_hat is the input, bit for bit; post-step
weights median |delta| < 5e-6 and max <= 0.0201 (a first Adagrad / Adam step moves a weight by lr * sign(g)).  The
configuration-rule test is host-only (no mark).
"""
import numpy as np
import pytest
import torch

from conftest import WINDOWS, rel_err
from fused_step_helpers import (_rhw_step_config, adv_loss_with, check_weights, config_checker, d_masks,  # noqa: F401
                                dev, generator_oracle, loss_errors, lstm_masks, make_batch, npy, ragged_lengths,
                                resync_oracle, rhw_models, sd_numpy, step_hp, use_adam, vc_ohp)
from oracle import gantts_port as gp
from oracle import nnmnkwii_port as nnp

LOSS_KEYS = ("loss_d", "loss_fake_d", "loss_real_d", "loss_mge", "loss_mse", "loss_adv", "loss_g")
GOLD_KEYS = ("loss_d", "loss_fake_d", "loss_real_d", "loss_mse", "loss_mge", "loss_adv", "loss_g",
             "real_correct", "fake_correct")
TOL = 2e-4


def run_vs_oracle(dev, mg, md, ohp, B, T, steps, mse_w, p_d, d_hidden, seed, tag, optimizer="Adagrad"):
    """`steps` training steps of FusedGanStep, each against the oracle started from the product's weights and optimiser
    state, with the step's own masks injected."""
    from gantts_b200 import fused
    S = mg.static_dim
    gen = generator_oracle(mg)
    d_layers = gp.discriminator_layers(sd_numpy(md))
    d_params = [t for pair in d_layers for t in pair]
    d_sum = [torch.zeros_like(t) for t in d_params]
    okw = dict(lr=1e-3, betas=(0.5, 0.9), weight_decay=0.0, eps=1e-8) if optimizer == "Adam" else None
    g_opt = gp.AdamStepper(gen.params(), **okw) if okw else None
    d_opt = gp.AdamStepper(d_params, **okw) if okw else None
    mg.to(dev).train(), md.to(dev).train()
    fs = fused.FusedGanStep(mg, md, step_hp(ohp), B, T, w_d=1.0, mse_w=mse_w, mge_w=1.0, weight_decay=0.0, seed=seed,
                            optimizer=optimizer, optimizer_params=okw)
    R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, T))
    in_dim = 3 * S
    for it in range(steps):
        lens = ragged_lengths(B, T, seed + 10 * it)
        x, y = make_batch(B, T, in_dim, in_dim, lens, seed + 10 * it + 1)
        xd = x.to(dev)
        fs.step(xd, y.to(dev), torch.LongTensor(lens).to(dev), frames=sum(lens))
        got = fs.loss_dict()
        gm = lstm_masks(fs, mg, B, T, dev)
        dm = d_masks(fs, B * T, [d_hidden] * (len(d_layers) - 1), p_d, dev)
        ref, yh_ref, ys_ref = gp.gan_step(lambda: gen.forward(x, R, lens, ohp, masks=gm), gen.params(), gen.sums,
                                          d_layers, d_sum, x, y, lens, R, ohp, w_d=1.0, mse_w=mse_w, mge_w=1.0,
                                          adv_w=1.0, dropout_d=p_d, training=True, weight_decay=0.0, d_masks=dm,
                                          d_opt=d_opt, g_opt=g_opt)
        ref = dict(ref, loss_adv=adv_loss_with(gp.DiscriminatorOracle(sd_numpy(md)), x, ys_ref, lens, ohp, dm["adv"]))
        errs = loss_errors(got, ref, LOSS_KEYS + ("d_grad_norm", "g_grad_norm"))
        errs["y_hat_static"] = rel_err(npy(fs.y_hat_static), ys_ref.numpy())
        assert max(errs.values()) < TOL, (tag, it, errs)
        assert torch.equal(fs.y_hat, xd)                                   # models.py:118: the input is y_hat
        assert abs(got["real_correct"] - ref["real_correct"]) <= 3 and abs(got["fake_correct"] - ref["fake_correct"]) <= 3
        check_weights(mg, gen.named, "%s step %d" % (tag, it))
        resync_oracle(fs, mg, md, gen, d_params, d_sum, g_opt, d_opt)        # the next step starts from the product's state
    return fs


@pytest.mark.gpu
def test_fused_rnn_highway_golden(dev, golden_step_models):
    """The `rhw_` vectors of the UNMODIFIED reference's train.py step functions (In2OutRNNHighwayNet 27 -> 27, S = 9,
    2 x 12 bidirectional LSTM, D 9 -> 16 -> 16 -> 1, B = 3, T = 24, two mini-batches, ragged lengths, Adagrad wd 1e-7)
    through FusedGanStep: every loss (the counts exactly), y_hat == x bit for bit, y_hat_static, and every post-step
    generator and discriminator tensor."""
    import gantts_b200
    from gantts_b200 import fused
    g = golden_step_models
    sub = lambda pre: {k[len(pre):]: torch.from_numpy(g[k]) for k in g.files if k.startswith(pre)}
    mg = gantts_b200.models.In2OutRNNHighwayNet(in_dim=27, out_dim=27, static_dim=9, num_hidden=2, hidden_dim=12,
                                                bidirectional=True, dropout=0.0)
    mg.load_state_dict(sub("rhw_g0_"))
    md = gantts_b200.models.MLP(9, 1, 2, 16, dropout=0.0, last_sigmoid=True)
    md.load_state_dict(sub("rhw_d0_"))
    mg.to(dev).train(), md.to(dev).train()
    w_d, mse_w, mge_w = [float(v) for v in g["rhw_cfg"]]
    fs = fused.FusedGanStep(mg, md, step_hp(vc_ohp(27)), 3, 24, w_d=w_d, mse_w=mse_w, mge_w=mge_w, seed=5)
    for it in range(2):
        p = "rhw_it%d_" % it
        lens = [int(v) for v in g[p + "lengths"]]
        xd = torch.from_numpy(g[p + "x"]).to(dev)
        fs.step(xd, torch.from_numpy(g[p + "y"]).to(dev), torch.LongTensor(lens).to(dev), adv_w=1.0 if w_d > 0 else 0.0)
        got = fs.loss_dict()
        for k, v in zip(GOLD_KEYS, g[p + "losses"]):
            if np.isnan(v):
                continue
            if k.endswith("correct"):
                assert got[k] == v, (it, k, got[k], v)
            else:
                assert abs(got[k] - v) <= 1e-4 * max(abs(v), 1e-3), (it, k, got[k], v)
        assert torch.equal(fs.y_hat, xd)
        assert np.array_equal(npy(fs.y_hat), g[p + "y_hat"])
        assert rel_err(npy(fs.y_hat_static), g[p + "y_hat_static"]) < 1e-4
        for pre, m in (("g_", mg), ("d_", md)):
            for k, v in m.state_dict().items():
                d = np.abs(npy(v) - g[p + pre + k])
                assert np.median(d) < 5e-6 and d.max() <= 0.0201, (it, pre + k, np.median(d), d.max())


@pytest.mark.gpu
def test_fused_rnn_highway_cfg3_widths_train_mode(dev):
    """cfg3 widths: In2OutRNNHighwayNet 177 -> 177 (S = 59, 3 x 512 bidirectional LSTM, LSTM dropout 0.5), D 59 -> 256 ->
    256 -> 1 with dropout 0.5, B = 4 x T = 300 ragged (max length T), train mode, Adagrad: one step against the oracle
    with the step's own masks -- the losses, both gradient norms, y_hat_static, and every post-step generator tensor
    (weight_ih, weight_hh and both biases of every layer and direction).  With all-ones masks the oracle equals the
    oracle port's In2OutRNNHighwayNet on the reference's one multi-layer nn.LSTM."""
    B, T = 4, 300
    mg, md = rhw_models(5, 59, 3, 512, True, 0.5, 256, 2, 0.5)
    lens = ragged_lengths(B, T, 7)
    x, _ = make_batch(B, T, 177, 177, lens, 8)
    R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, T))
    gen = generator_oracle(mg)
    lstm = torch.nn.LSTM(177, 512, 3, batch_first=True, bidirectional=True)
    lstm.load_state_dict({k[5:]: torch.from_numpy(v) for k, v in sd_numpy(mg).items() if k.startswith("lstm.")})
    with torch.no_grad():
        _, a = gp.in2out_rnn_highway_forward(x, R, lens, gen.gate, lstm, gen.h2o, 59)
        _, b = gen.forward(x, R, lens, vc_ohp(177), masks=[torch.ones(B * T, 1024)] * 2)
    assert rel_err(b.numpy(), a.numpy()) < 1e-5
    run_vs_oracle(dev, mg, md, vc_ohp(177), B, T, 1, 0.0, 0.5, 256, 300, "cfg3")


TOY_CASES = [  # (bidirectional, layers, mse_w, conditioned D, optimizer)
    (True, 1, 0.0, False, "Adagrad"),
    (False, 2, 0.5, False, "Adagrad"),
    (True, 3, 0.5, True, "Adagrad"),
    (True, 2, 0.0, True, "Adam"),
    (False, 3, 0.0, False, "Adam"),
    (True, 3, 0.5, False, "Adam"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("bidir,layers,mse_w,cond,optimizer", TOY_CASES)
def test_fused_rnn_highway_toy_vs_oracle(dev, bidir, layers, mse_w, cond, optimizer):
    """Small stacks (S = 8: 24 -> 24, 12 hidden units per direction, LSTM dropout 0.3, D dropout 0.5), B = 3 x T = 40
    ragged, two training steps against the oracle across uni/bi, 1-3 layers, mse_w 0 / 0.5, a conditioned D, Adagrad
    and Adam."""
    mg, md = rhw_models(40 + layers + 4 * bidir, 8, layers, 12, bidir, 0.3, 32, 2, 0.5, cond)
    run_vs_oracle(dev, mg, md, vc_ohp(24, cond), 3, 40, 2, mse_w, 0.5, 32, 500 + layers, "toy", optimizer)


@pytest.mark.gpu
def test_fused_rnn_highway_matches_gan_trainer(dev):
    """bench.py cfg3 shape (B = 16, T = 2000, ragged with max length T) with every dropout 0: two training steps of
    FusedGanStep and of the modular GanTrainer agree on the losses, y_hat, y_hat_static and the updated weights; so do
    their eval phases.  Each step starts both from the fused step's weights: a first Adagrad step moves a weight whose
    gradient is near zero by +-lr on either side, and through 2000 recurrent steps that alone moves y_hat_static by
    more than the tolerance (3e-3 measured; the losses still agree to 1e-5)."""
    from gantts_b200 import fused, step as gstep
    B, T = 16, 2000
    hp = step_hp(vc_ohp(177))
    mk = lambda: rhw_models(21, 59, 3, 512, True, 0.0, 256, 2, 0.0)
    (mg, md), (tg, td) = mk(), mk()
    for m in (mg, md, tg, td):
        m.to(dev).train()
    fs = fused.FusedGanStep(mg, md, hp, B, T, w_d=1.0, mse_w=0.0, mge_w=1.0, weight_decay=0.0, seed=22)
    tr = gstep.GanTrainer(tg, td, hp, w_d=1.0, mse_w=0.0, mge_w=1.0, weight_decay=0.0)
    R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, T)).to(dev)
    for it in range(3):
        train = it < 2
        with torch.no_grad():
            for a, b in zip(list(mg.parameters()) + list(md.parameters()), list(tg.parameters()) + list(td.parameters())):
                b.copy_(a)
        if not train:
            for m in (mg, md, tg, td):
                m.eval()
        lens = ragged_lengths(B, T, 23 + it)
        x, y = make_batch(B, T, 177, 177, lens, 24 + it)
        xd, yd = x.to(dev), y.to(dev)
        fs.step(xd, yd, torch.LongTensor(lens).to(dev))
        got = fs.loss_dict()
        out, yh, ys = tr.step(xd, yd, lens, R, train=train)
        errs = loss_errors(got, {k: float(out[k]) for k in LOSS_KEYS}, LOSS_KEYS)
        errs["y_hat_static"] = rel_err(npy(fs.y_hat_static), npy(ys))
        assert max(errs.values()) < TOL, (it, errs)
        assert torch.equal(fs.y_hat, yh) and torch.equal(fs.y_hat, xd)
        for i, (a, b) in enumerate(zip(list(mg.parameters()) + list(md.parameters()),
                                       list(tg.parameters()) + list(td.parameters()))):
            d = np.abs(npy(a) - npy(b))
            assert np.median(d) < 5e-6 and d.max() <= 0.0201, (it, i, np.median(d), d.max())


@pytest.mark.gpu
def test_fused_rnn_highway_invariants(dev):
    """Phases 1, 2 and 4 called one by one give exactly what one call gives, with grad_buffer(0) holding every generator
    tensor in model_g.parameters() order; mse_w moves no generator weight (the model returns its input); an eval-phase
    call leaves every parameter and all optimiser state bit-unchanged; state_dict()'s generator part loads into
    torch.optim.Adagrad(model_g.parameters())."""
    from gantts_b200 import fused
    B, T = 3, 60
    hp = step_hp(vc_ohp(24))
    lens = ragged_lengths(B, T, 31)
    x, y = make_batch(B, T, 24, 24, lens, 32)
    xd, yd, ld = x.to(dev), y.to(dev), torch.LongTensor(lens).to(dev)
    runs = []
    for split, mse_w in ((False, 0.5), (True, 0.5), (False, 0.0)):
        mg, md = rhw_models(33, 8, 3, 16, True, 0.3, 32, 2, 0.5)
        mg.to(dev).train(), md.to(dev).train()
        fs = fused.FusedGanStep(mg, md, hp, B, T, mse_w=mse_w, weight_decay=0.0, seed=34)
        if split:
            fs.cfg.adv_w, fs._step, fs.cfg.opt_step = 1.0, 1, 1
            for ph in (1, 2, 4):
                fs._call(ph, xd, yd, ld, 0.0, fs._seed)
        else:
            fs.step(xd, yd, ld)
            assert fs.last_seed == fs._seed
        gb = fs.grad_buffer(0)
        params = list(mg.parameters())
        assert gb.numel() == sum(q.numel() for q in params) and len(params) == 2 + 8 * 3 + 2
        off = 0
        for q, s in zip(params, fs._sums):                 # weight decay 0: Adagrad's first state_sum = g^2
            n = q.numel()
            assert torch.equal((gb[off:off + n] * gb[off:off + n]).view_as(q), s)
            off += n
        ng = len(params)
        assert torch.equal(fs._sums[4], fs._sums[5])       # bias_ih_l0 and bias_hh_l0 get the same gradient
        runs.append([fs.losses.clone(), fs.y_hat.clone(), fs.y_hat_static.clone(), gb.clone(), fs.grad_buffer(1).clone()]
                    + [q.detach().clone() for q in list(mg.parameters()) + list(md.parameters())]
                    + [s.clone() for s in fs._sums[:ng]])
    for a, b in zip(runs[0], runs[1]):
        assert torch.equal(a, b)
    assert runs[2][0][6] != runs[0][0][6]                  # loss_g carries the MSE term ...
    for a, b in zip(runs[0][3:], runs[2][3:]):             # ... which sends no gradient into G
        assert torch.equal(a, b)
    wsnap = [q.detach().clone() for q in list(mg.parameters()) + list(md.parameters())]
    ssnap = [s.clone() for s in fs._sums]
    mg.eval(), md.eval()
    fs.step(xd, yd, ld)
    assert fs.loss_dict()["g_grad_norm"] == 0.0 and torch.equal(fs.y_hat, xd)
    for a, b in zip(wsnap, list(mg.parameters()) + list(md.parameters())):
        assert torch.equal(a, b.detach())
    for a, b in zip(ssnap, fs._sums):
        assert torch.equal(a, b)
    sd = fs.state_dict()
    assert len(sd["optimizer_g"]["state"]) == ng and len(sd["optimizer_d"]["state"]) == len(list(md.parameters()))
    opt = torch.optim.Adagrad(mg.parameters(), lr=0.01, weight_decay=0.0)
    opt.load_state_dict(sd["optimizer_g"])
    assert torch.equal(opt.state[mg.T.weight]["sum"], fs._sums[0])
    assert torch.equal(opt.state[mg.lstm.weight_hh_l2_reverse]["sum"], fs._sums[2 + 8 * 2 + 4 + 1])
    assert torch.equal(opt.state[mg.hidden2out.bias]["sum"], fs._sums[ng - 1])


@pytest.mark.gpu
def test_fused_rnn_highway_adam_resume(dev):
    """Under Adam, a step resumed from state_dict() in a new FusedGanStep is bit-identical to the uninterrupted one."""
    from gantts_b200 import fused
    B, T = 3, 50
    hp = step_hp(vc_ohp(24))
    okw = dict(lr=1e-3, betas=(0.5, 0.9), weight_decay=0.0, eps=1e-8)
    build = lambda: rhw_models(51, 8, 2, 16, True, 0.3, 32, 2, 0.5)
    mg, md = build()
    mg.to(dev).train(), md.to(dev).train()
    fs = fused.FusedGanStep(mg, md, hp, B, T, seed=52, optimizer="Adam", optimizer_params=okw)
    lens = ragged_lengths(B, T, 53)
    x, y = make_batch(B, T, 24, 24, lens, 54)
    xd, yd, ld = x.to(dev), y.to(dev), torch.LongTensor(lens).to(dev)
    fs.step(xd, yd, ld)
    snap = [q.detach().clone() for q in list(mg.parameters()) + list(md.parameters())]
    sd = fs.state_dict()
    fs.step(xd, yd, ld)
    want = fs.loss_dict()
    after = [q.detach().clone() for q in list(mg.parameters()) + list(md.parameters())]
    g2, d2 = build()
    g2.to(dev).train(), d2.to(dev).train()
    with torch.no_grad():
        for q, v in zip(list(g2.parameters()) + list(d2.parameters()), snap):
            q.copy_(v)
    fs2 = fused.FusedGanStep(g2, d2, hp, B, T, seed=999, optimizer="Adam", optimizer_params=okw)
    fs2.load_state_dict(sd)
    fs2.step(xd, yd, ld)
    assert fs2.loss_dict() == want
    for q, v in zip(list(g2.parameters()) + list(d2.parameters()), after):
        assert torch.equal(q.detach(), v)


@pytest.mark.gpu
def test_fused_step_still_rejects_grurnn_and_unsupported_lstms(dev):
    """GRURNN (an LSTM stack without the gate) is refused with a message that points to GanTrainer, and so is an
    In2OutRNNHighwayNet whose nn.LSTM the fused step does not implement."""
    import gantts_b200
    from gantts_b200 import fused
    hp = step_hp(vc_ohp(24))
    md = gantts_b200.models.MLP(8, 1, 2, 16, dropout=0.0, last_sigmoid=True).to(dev)
    mg = gantts_b200.models.GRURNN(in_dim=24, out_dim=24, num_hidden=1, hidden_dim=16).to(dev)
    with pytest.raises(RuntimeError, match="GanTrainer"):
        fused.FusedGanStep(mg, md, hp, 2, 10)
    for kw in (dict(proj_size=4), dict(bias=False), dict(batch_first=False), dict(num_layers=4)):
        mg, _ = rhw_models(1, 8, 2, 16, True, 0.0, 16, 2, 0.0)
        a = dict(input_size=24, hidden_size=16, num_layers=2, batch_first=True, bidirectional=True)
        a.update(kw)
        mg.lstm = torch.nn.LSTM(**a)
        mg.hidden2out = torch.nn.Linear((4 if "proj_size" in kw else 16) * 2, 24)
        with pytest.raises(RuntimeError, match="GanTrainer"):
            fused.FusedGanStep(mg.to(dev), md, hp, 2, 10)


def lstm_tensor(layer, direction, kind):
    """Index in the generator's table of an LSTM tensor (kind 0..3: W_ih, W_hh, b_ih, b_hh), bidirectional stack."""
    return 2 + 4 * (2 * layer + direction) + kind


def test_rnn_highway_step_config_rules_on_tensor_tables():
    """gantts_gan_step_workspace_bytes (host-only) accepts the In2OutRNNHighwayNet layout and rejects, with a message
    naming the rule, every LSTM configuration the step does not implement; the LSTM mask seeds are a stream of their
    own."""
    from gantts_b200 import _lib
    ws, err, rejected = config_checker()
    lib = _lib.load()
    c = _rhw_step_config()
    assert ws(c) > 0, err()
    with_lstm = ws(c)
    c.lstm.num_layers = 0                         # the gate + a one-layer MLP on x: no LSTM workspace
    c.g.dims[0] = 3 * 59
    c.g_tensors.n = 4
    assert 0 < ws(c) < with_lstm, err()

    def rej(mutate, needle):
        rejected(_rhw_step_config, mutate, needle)
    rej(lambda c: setattr(c.highway, "static_dim", 0), "highway gate")
    rej(lambda c: setattr(c.sru, "num_layers", 1), "mutually exclusive")
    rej(lambda c: setattr(c.lstm, "num_layers", _lib.MAX_LSTM_LAYERS + 1), "LSTM layer count")
    rej(lambda c: setattr(c.lstm, "num_layers", -1), "LSTM layer count")
    rej(lambda c: setattr(c.lstm, "hidden", 18), "multiple of 4")
    rej(lambda c: setattr(c, "B", 129), "LSTM_MAX_B")
    rej(lambda c: setattr(c.lstm, "dropout", 1.0), "LSTM dropout")
    rej(lambda c: setattr(c.lstm, "dropout", -0.1), "LSTM dropout")
    rej(lambda c: c.g.dims.__setitem__(0, 16), "hidden2out")
    rej(lambda c: setattr(c.g, "num_layers", 2), "hidden2out")
    rej(lambda c: setattr(c.lstm, "in_dim", 3 * 59 - 1), "in_dim")

    def narrow(c):                                # in_dim < S (with a matching hidden2out)
        c.lstm.in_dim = c.g.dims[1] = 40
    rej(narrow, "static_dim")
    rej(lambda c: c.g_tensors.param.__setitem__(lstm_tensor(2, 1, 1), None), "null generator tensor 23")
    rej(lambda c: c.g_tensors.param.__setitem__(lstm_tensor(0, 0, 2), None), "null generator tensor 4")
    rej(lambda c: c.g_tensors.state.__setitem__(lstm_tensor(1, 0, 3), None), "null generator optimiser state of tensor 13")
    rej(lambda c: setattr(c.lstm, "num_layers", 2), "generator table has 28 tensors, its shapes give 20")
    rej(lambda c: use_adam(c, missing=(lstm_tensor(2, 1, 1),)), "exp_avg_sq for generator tensor 23")
    # the seeds of the LSTM masks are a stream of their own
    for seed in (0, 5, 12345):
        lstm_seeds = {lib.gantts_lstm_mask_seed(seed, l) for l in range(_lib.MAX_LSTM_LAYERS)}
        others = {lib.gantts_gan_step_seed(seed, w) for w in range(4)}
        others |= {lib.gantts_sru_mask_seed(seed, l, w) for l in range(_lib.MAX_SRU_LAYERS) for w in range(2)}
        assert len(lstm_seeds) == _lib.MAX_LSTM_LAYERS and not lstm_seeds & others
