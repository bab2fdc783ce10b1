"""The fused GAN step (gantts_gan_step / FusedGanStep) with a recurrent discriminator: LSTMRNN, or GRURNN (also an
nn.LSTM), with last_sigmoid=True, as train.py:774 builds it from hp.discriminator.  Every generator the fused step runs,
conditioned and unconditioned, Adagrad and Adam, against the oracle's gan_step with a DiscriminatorOracle and the step's
own inter-layer masks injected (each is gantts_dropout(ones[rows][ndir H], p, gantts_d_lstm_mask_seed(seed, which,
layer)), rows = 2 B T on the stacked forward, B T on the adversarial one).  Tolerances are those of
test_gpu_fused_rnn_highway.py: losses, gradient norms and y_hat_static 2e-4 relative, post-step weights median |delta| <
5e-6 and max <= 0.0201.  The phase split, D-only and eval steps, shaped calls, GRURNN vs LSTMRNN and resume are compared
bit for bit.
"""
import numpy as np
import pytest
import torch

from conftest import WINDOWS, rel_err
from fused_step_helpers import (ADAM, adv_loss_with, check_weights, d_lstm_masks, dev, generator_oracle,  # noqa: F401
                                loss_errors, make_batch, make_models, npy, ragged_lengths, resync_oracle, sd_numpy,
                                step_hp)
from oracle import gantts_port as gp
from oracle import nnmnkwii_port as nnp

LOSS_KEYS = ("loss_d", "loss_fake_d", "loss_real_d", "loss_mge", "loss_mse", "loss_adv", "loss_g")
TOL = 2e-4


def run_vs_restatement(dev, kind, mg, md, ohp, d_in, B, T, steps, seed, optimizer="Adagrad", mse_w=0.0):
    from gantts_b200 import fused
    gen = generator_oracle(mg)
    d = gp.DiscriminatorOracle(sd_numpy(md))
    d_sum = [torch.zeros_like(t) for t in d.params()]
    okw = ADAM if optimizer == "Adam" else None
    g_opt = gp.AdamStepper(gen.params(), **okw) if okw else None
    d_opt = gp.AdamStepper(d.params(), **okw) if okw else None
    mg.to(dev).train(), md.to(dev).train()
    fs = fused.FusedGanStep(mg, md, step_hp(ohp), B, T, w_d=1.0, mse_w=mse_w, mge_w=1.0, weight_decay=0.0, seed=seed,
                            optimizer=optimizer, optimizer_params=okw)
    R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, T))
    d_out = mg.hidden2out.weight.shape[0] if hasattr(mg, "hidden2out") else mg.last_linear.weight.shape[0]
    for it in range(steps):
        lens = ragged_lengths(B, T, seed + 10 * it)
        x, y = make_batch(B, T, d_in, d_out, lens, seed + 10 * it + 1)
        if kind in ("mlp", "sru"):
            x = x.abs()
        fs.step(x.to(dev), y.to(dev), torch.LongTensor(lens).to(dev), frames=sum(lens))
        got = fs.loss_dict()
        dm = d_lstm_masks(fs, md, B * T, dev)
        ref, yh_ref, ys_ref = gp.gan_step(lambda: gen.forward(x, R, lens, ohp), gen.params(), gen.sums, d, d_sum, x, y,
                                          lens, R, ohp, mse_w=mse_w, weight_decay=0.0, d_masks=dm, d_opt=d_opt,
                                          g_opt=g_opt)
        ref = dict(ref, loss_adv=adv_loss_with(gp.DiscriminatorOracle(sd_numpy(md)), x, ys_ref, lens, ohp, dm["adv"]))
        errs = loss_errors(got, ref, LOSS_KEYS + ("d_grad_norm", "g_grad_norm"))
        errs["y_hat_static"] = rel_err(npy(fs.y_hat_static), ys_ref.numpy())
        assert max(errs.values()) < TOL, (kind, it, errs)
        assert abs(got["real_correct"] - ref["real_correct"]) <= 3 and abs(got["fake_correct"] - ref["fake_correct"]) <= 3
        check_weights(mg, gen.named, "%s G step %d" % (kind, it))
        check_weights(md, d.named, "%s D step %d" % (kind, it))
        resync_oracle(fs, mg, md, gen, d.params(), d_sum, g_opt, d_opt)
    return fs


CASES = [  # (generator, conditioned D, bidirectional D, optimizer)
    ("mlp", False, True, "Adagrad"),
    ("mlp", True, False, "Adam"),
    ("highway", False, False, "Adagrad"),
    ("highway", True, True, "Adam"),
    ("rnn_highway", False, True, "Adam"),
    ("rnn_highway", True, False, "Adagrad"),
    ("sru", True, True, "Adagrad"),
    ("sru", False, False, "Adam"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,cond,bidir,optimizer", CASES)
def test_fused_rnn_d_vs_restatement(dev, kind, cond, bidir, optimizer):
    """Two training steps, B = 3 x T = 40 ragged, a 2-layer LSTMRNN D of 12 units with dropout 0.5."""
    mg, md, ohp, d_in = make_models(kind, 60 + len(kind) + 2 * cond + bidir, cond, bidir=bidir)
    run_vs_restatement(dev, kind, mg, md, ohp, d_in, 3, 40, 2, 700 + len(kind), optimizer)


@pytest.mark.gpu
def test_fused_rnn_d_vc_full_width(dev):
    """vc: In2OutHighwayNet 177 -> 512 x 3 -> 177 with LSTMRNN(59, 1, 2, 256, bidirectional, dropout 0.5), B = 20 x
    T = 400."""
    mg, md, ohp, d_in = make_models("highway", 3, False, d_hidden=256, full=True)
    run_vs_restatement(dev, "highway", mg, md, ohp, d_in, 20, 400, 1, 31)


@pytest.mark.gpu
def test_fused_rnn_d_tts_acoustic_full_width(dev):
    """tts_acoustic: SRURNN 425 -> 6 x 512 bidirectional -> 187 with a conditioned LSTMRNN D (483 inputs, 2 x 64
    bidirectional, dropout 0.5), B = 4 x T = 200."""
    mg, md, ohp, d_in = make_models("sru", 4, True, d_hidden=64, full=True)
    run_vs_restatement(dev, "sru", mg, md, ohp, d_in, 4, 200, 1, 41)


def _snapshot(fs, mg, md):
    return ([fs.losses.clone(), fs.y_hat.clone(), fs.y_hat_static.clone(), fs.grad_buffer(0).clone(),
             fs.grad_buffer(1).clone()] + [q.detach().clone() for q in list(mg.parameters()) + list(md.parameters())]
            + [s.clone() for s in fs._sums + fs._sqs])


def _equal(a, b):
    assert len(a) == len(b)
    for i, (u, v) in enumerate(zip(a, b)):
        assert torch.equal(u, v), i


def _batch(B, T, d_in, d_out, seed, dev):
    lens = ragged_lengths(B, T, seed)
    x, y = make_batch(B, T, d_in, d_out, lens, seed + 1)
    return x.abs().to(dev), y.to(dev), torch.LongTensor(lens).to(dev)


@pytest.mark.gpu
def test_grurnn_d_equals_lstmrnn_d_bit_for_bit(dev):
    """A GRURNN discriminator trains exactly like an LSTMRNN one with the same weights: GRURNN is an nn.LSTM too."""
    from gantts_b200 import fused
    runs = []
    for gru in (False, True):
        mg, md, ohp, d_in = make_models("mlp", 5, False, gru=gru)
        mg.to(dev).train(), md.to(dev).train()
        fs = fused.FusedGanStep(mg, md, step_hp(ohp), 3, 30, seed=6)
        for it in range(2):
            fs.step(*_batch(3, 30, d_in, 187, 7 + it, dev))
        runs.append(_snapshot(fs, mg, md))
    _equal(*runs)


@pytest.mark.gpu
@pytest.mark.parametrize("cond", [False, True])
def test_fused_rnn_d_phase_split_d_only_and_eval(dev, cond):
    """Phases 1|2 then 4 equal one call bit for bit; a D-only step updates D exactly like the full step does (same seed)
    and leaves G and its state untouched; an eval call leaves every parameter and all optimiser state unchanged."""
    from gantts_b200 import fused
    B, T = 3, 36
    runs = {}
    for mode in ("one", "split", "d_only"):
        mg, md, ohp, d_in = make_models("rnn_highway", 8, cond)
        mg.to(dev).train(), md.to(dev).train()
        fs = fused.FusedGanStep(mg, md, step_hp(ohp), B, T, seed=9)
        x, y, ld = _batch(B, T, d_in, 24, 10, dev)
        g0 = [q.detach().clone() for q in mg.parameters()]
        if mode == "split":
            fs.cfg.adv_w, fs._step, fs.cfg.opt_step = 1.0, 1, 1
            for ph in (1 | 2, 4):
                fs._call(ph, x, y, ld, 0.0, fs._seed)
        else:
            fs.step(x, y, ld, update_g=mode != "d_only")
        runs[mode] = (fs, mg, md, _snapshot(fs, mg, md), g0)
    _equal(runs["one"][3], runs["split"][3])
    fs, mg, md, snap, g0 = runs["d_only"]
    ref_md = runs["one"][2]
    for a, b in zip(md.parameters(), ref_md.parameters()):
        assert torch.equal(a, b)
    assert torch.equal(fs.grad_buffer(1), runs["one"][0].grad_buffer(1))
    for a, b in zip(mg.parameters(), g0):
        assert torch.equal(a.detach(), b)
    got = fs.loss_dict()
    want = runs["one"][0].loss_dict()
    for k in ("loss_d", "loss_fake_d", "loss_real_d", "real_correct", "fake_correct", "d_grad_norm"):
        assert got[k] == want[k], k
    assert got["loss_adv"] == 0.0 and got["g_grad_norm"] == 0.0
    # eval: forwards and losses only
    fs, mg, md = runs["one"][:3]
    before = _snapshot(fs, mg, md)[5:]
    mg.eval(), md.eval()
    x, y, ld = _batch(B, T, 24, 24, 12, dev)
    fs.step(x, y, ld)
    _equal(before, _snapshot(fs, mg, md)[5:])
    ev = fs.loss_dict()
    assert ev["loss_adv"] > 0.0 and ev["d_grad_norm"] == 0.0 and ev["g_grad_norm"] == 0.0


@pytest.mark.gpu
def test_fused_rnn_d_shaped_calls_equal_exactly_sized_steps(dev):
    """A step built for (B, T) = (4, 40) runs a chain of shapes (train, D-only and eval calls) with exactly the results of
    steps built for each shape, bit for bit."""
    from gantts_b200 import fused
    shapes = [((4, 40), True, True), ((3, 29), True, True), ((2, 40), False, True), ((4, 17), True, False)]
    mg, md, ohp, d_in = make_models("highway", 11, False)
    mg.to(dev).train(), md.to(dev).train()
    cap = fused.FusedGanStep(mg, md, step_hp(ohp), 4, 40, seed=12)
    for i, ((b, t), update_g, train) in enumerate(shapes):
        tg, td, _, _ = make_models("highway", 11, False)
        tg.to(dev), td.to(dev)
        with torch.no_grad():
            for p, q in zip(list(tg.parameters()) + list(td.parameters()), list(mg.parameters()) + list(md.parameters())):
                p.copy_(q)
        ex = fused.FusedGanStep(tg, td, step_hp(ohp), b, t, seed=12)
        ex.load_state_dict(cap.state_dict())
        for m in (mg, md, tg, td):
            m.train(train)
        x, y, ld = _batch(b, t, d_in, d_in, 13 + i, dev)
        cap.step(x, y, ld, update_g=update_g)
        ex.step(x, y, ld, update_g=update_g)
        assert torch.equal(cap.losses, ex.losses), i
        assert torch.equal(cap.y_hat_static, ex.y_hat_static) and torch.equal(cap.y_hat, ex.y_hat), i
        for p, q in zip(list(tg.parameters()) + list(td.parameters()), list(mg.parameters()) + list(md.parameters())):
            assert torch.equal(p, q), i
        for s, r in zip(ex._sums, cap._sums):
            assert torch.equal(s, r), i


@pytest.mark.gpu
def test_fused_rnn_d_adam_resume_with_per_model_counts(dev):
    """Under Adam, after a D-only step (the models' step counts differ) a step resumed from state_dict() in a new
    FusedGanStep is bit-identical to the uninterrupted one."""
    from gantts_b200 import fused
    B, T = 3, 30
    build = lambda: make_models("sru", 14, True)
    mg, md, ohp, d_in = build()
    mg.to(dev).train(), md.to(dev).train()
    fs = fused.FusedGanStep(mg, md, step_hp(ohp), B, T, seed=15, optimizer="Adam", optimizer_params=ADAM)
    x, y, ld = _batch(B, T, d_in, 187, 16, dev)
    fs.step(x, y, ld, update_g=False)
    fs.step(x, y, ld)
    snap = [q.detach().clone() for q in list(mg.parameters()) + list(md.parameters())]
    sd = fs.state_dict()
    assert sd["optimizer_d"]["state"][0]["step"] == 2 and sd["optimizer_g"]["state"][0]["step"] == 1
    fs.step(x, y, ld)
    want = fs.loss_dict()
    after = [q.detach().clone() for q in list(mg.parameters()) + list(md.parameters())]
    g2, d2, _, _ = build()
    g2.to(dev).train(), d2.to(dev).train()
    with torch.no_grad():
        for q, v in zip(list(g2.parameters()) + list(d2.parameters()), snap):
            q.copy_(v)
    fs2 = fused.FusedGanStep(g2, d2, step_hp(ohp), B, T, seed=999, optimizer="Adam", optimizer_params=ADAM)
    fs2.load_state_dict(sd)
    fs2.step(x, y, ld)
    assert fs2.loss_dict() == want
    for q, v in zip(list(g2.parameters()) + list(d2.parameters()), after):
        assert torch.equal(q.detach(), v)


@pytest.mark.gpu
@pytest.mark.parametrize("cond", [False, True])
def test_gan_trainer_rnn_d_vs_restatement_and_fused(dev, cond):
    """GanTrainer with an LSTMRNN D (dropout 0) against the restatement, and against FusedGanStep within the same
    tolerance: two training steps then an eval step, each started from the fused step's weights (stacking real and fake
    changes split-K plans, so the two native paths are not bitwise equal)."""
    from gantts_b200 import fused, step as gstep
    B, T = 3, 40
    mk = lambda: make_models("highway", 17, cond, p_d=0.0)
    (mg, md, ohp, d_in), (tg, td, _, _) = mk(), mk()
    for m in (mg, md, tg, td):
        m.to(dev).train()
    hp = step_hp(ohp)
    fs = fused.FusedGanStep(mg, md, hp, B, T, weight_decay=0.0, seed=18)
    tr = gstep.GanTrainer(tg, td, hp, weight_decay=0.0)
    R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, T))
    for it in range(3):
        train = it < 2
        with torch.no_grad():
            for a, b in zip(list(mg.parameters()) + list(md.parameters()), list(tg.parameters()) + list(td.parameters())):
                b.copy_(a)
        gen = generator_oracle(tg)
        d = gp.DiscriminatorOracle(sd_numpy(td))
        if not train:
            for m in (mg, md, tg, td):
                m.eval()
        lens = ragged_lengths(B, T, 19 + it)
        x, y = make_batch(B, T, d_in, d_in, lens, 20 + it)
        out, yh, ys = tr.step(x.to(dev), y.to(dev), lens, R.to(dev), train=train)
        fs.step(x.to(dev), y.to(dev), torch.LongTensor(lens).to(dev))
        got = fs.loss_dict()
        ref, _, ys_ref = gp.gan_step(lambda: gen.forward(x, R, lens, ohp), gen.params(), gen.sums, d,
                                     [torch.zeros_like(t) for t in d.params()], x, y, lens, R, ohp, weight_decay=0.0,
                                     training=train, update=train)
        trained = {k: float(out[k]) for k in LOSS_KEYS}
        # loss_adv (and loss_g = loss_mge + loss_adv) through each side's own updated D on the other side's y_hat_static
        # (see adv_loss_with); from the second step on the optimiser states of the two sides differ as well
        ref["loss_adv"] = adv_loss_with(gp.DiscriminatorOracle(sd_numpy(td)), x, ys_ref, lens, ohp, None)
        ref["loss_g"] = ref["loss_mge"] + ref["loss_adv"]
        errs = loss_errors(trained, ref, LOSS_KEYS)
        errs["y_hat_static"] = rel_err(npy(ys), ys_ref.numpy())
        assert max(errs.values()) < TOL, ("GanTrainer vs restatement", it, errs)
        trained["loss_adv"] = adv_loss_with(gp.DiscriminatorOracle(sd_numpy(md)), x, ys.detach().cpu(), lens, ohp, None)
        trained["loss_g"] = trained["loss_mge"] + trained["loss_adv"]
        errs = loss_errors(got, trained, LOSS_KEYS)
        errs["y_hat_static"] = rel_err(npy(fs.y_hat_static), npy(ys))
        assert max(errs.values()) < TOL, ("FusedGanStep vs GanTrainer", it, errs)
        if it == 0:                 # the restatement's optimiser state starts at zero like GanTrainer's
            check_weights(td, d.named, "GanTrainer D step %d" % it)
        if train:
            for a, b in zip(list(mg.parameters()) + list(md.parameters()), list(tg.parameters()) + list(td.parameters())):
                dd = np.abs(npy(a) - npy(b))
                assert np.median(dd) < 5e-6 and dd.max() <= 0.0201, (it, np.median(dd), dd.max())
