"""One optimiser per model (reference train.py:796-799: optimizer_g and optimizer_d from their own hparams) in
FusedGanStep and GanTrainer, on the GPU.

Checkers: the oracle's gan_step (update_g=False for the D-only step) with a stepper per model and the step's own
dropout masks injected (tolerances of the fused-generator modules: losses 2e-4 relative, weights through check_weights); the
reference's per-batch logic (tests/trainpy_mirror.py) with torch.optim.Adam for G and torch.optim.Adagrad for D; and bit
for bit against the same step built another way (optimizer_d=None, the former two-call sequence, the data-parallel phase
calls, a step built with the decayed lr, a resumed step).
"""
import os

import numpy as np
import pytest
import torch

from conftest import ROOT, WINDOWS, rel_err
from fused_step_helpers import (ADAM, assert_equal_lists, build, check_weights, d_masks, dev, g_masks,  # noqa: F401
                                generator_oracle, make_batch, npy, ragged_lengths, resync_oracle, sd_numpy, snapshot,
                                step_hp)
from oracle import gantts_port as gp
from oracle import nnmnkwii_port as nnp

TOL = 2e-4
# (G kind, G params, D kind, D params): Adam G with an Adagrad D of its own lr, and Adagrad on both with different lrs
SETTINGS = {"adam_g_adagrad_d": ("Adam", ADAM, "Adagrad", dict(lr=1e-3, weight_decay=0.0)),
            "adagrad_two_lrs": ("Adagrad", dict(lr=0.01, weight_decay=0.0), "Adagrad", dict(lr=0.003, weight_decay=0.0))}
PRE_UPDATE_KEYS = ("loss_d", "loss_fake_d", "loss_real_d", "loss_mse", "loss_mge", "d_grad_norm")


def exp_lr_scheduler(optimizer, epoch, nepoch, init_lr=0.0001, lr_decay_epoch=100):
    """Reference train.py:323-333 (the print left out)."""
    lr = init_lr * (0.1 ** (epoch // lr_decay_epoch))
    for param_group in optimizer.param_groups:
        param_group['lr'] = lr
    return optimizer


def save_checkpoint(model, optimizer, epoch, checkpoint_dir, name):
    """Reference train.py:162-171 (the print left out)."""
    checkpoint_path = os.path.join(checkpoint_dir, "checkpoint_epoch{}_{}.pth".format(epoch, name))
    torch.save({"state_dict": model.state_dict(), "optimizer": optimizer.state_dict(), "global_epoch": epoch},
               checkpoint_path)
    return checkpoint_path


def load_checkpoint(model, optimizer, checkpoint_path):
    """Reference train.py:651-658 (returns global_epoch instead of setting the global)."""
    checkpoint = torch.load(checkpoint_path)
    model.load_state_dict(checkpoint["state_dict"])
    if optimizer is not None:
        optimizer.load_state_dict(checkpoint["optimizer"])
    return checkpoint["global_epoch"]


def fused(mg, md, hp, B, T, setting, **kw):
    from gantts_b200 import fused as F
    kg, pg, kd, pd = SETTINGS[setting]
    return F.FusedGanStep(mg, md, step_hp(hp), B, T, weight_decay=0.0, optimizer=kg, optimizer_params=pg,
                          optimizer_d=kd, optimizer_d_params=pd, **kw)


def stepper(kind, params, hyper, sums):
    """The oracle's optimiser of one model: AdamStepper, or Adagrad over `sums` with the model's own lr."""
    if kind == "Adam":
        return gp.AdamStepper(params, **hyper)
    return lambda ps, gs: gp.adagrad_step(ps, gs, sums, lr=hyper["lr"], weight_decay=hyper["weight_decay"])


def batches(n, B, T, d_in, d_out, seed):
    out = []
    for it in range(n):
        lens = ragged_lengths(B, T, seed + it)
        out.append((lens,) + make_batch(B, T, d_in, d_out, lens, seed + 10 + it))
    return out


def on(dev, lens, x, y):
    return x.to(dev), y.to(dev), torch.LongTensor(lens).to(dev)


@pytest.mark.gpu
@pytest.mark.parametrize("setting", sorted(SETTINGS))
@pytest.mark.parametrize("kind", ["mlp", "sru"])
def test_fused_step_with_an_optimiser_per_model_vs_oracle(dev, kind, setting):
    """One D-only step, then two full steps, against the oracle stepping each model with its own optimiser: the losses
    computed before D's update, y_hat_static, D's weights after every step and G's after the full steps.  The oracle's
    next step starts from the product's weights and optimiser state."""
    B, T = 3, 40
    kg, pg, kd, pd = SETTINGS[setting]
    mg, md, hp, d_in, d_out, g_hidden, d_hidden, p_d = build(kind, 80)
    gen = generator_oracle(mg)
    d_layers = gp.discriminator_layers(sd_numpy(md))
    d_params = [t for pair in d_layers for t in pair]
    d_sum = [torch.zeros_like(t) for t in d_params]
    g_opt, d_opt = stepper(kg, gen.params(), pg, gen.sums), stepper(kd, d_params, pd, d_sum)
    mg.to(dev).train(), md.to(dev).train()
    fs = fused(mg, md, hp, B, T, setting, seed=81)
    assert (fs.opt_g.kind, fs.opt_d.kind, fs.opt_g.lr, fs.opt_d.lr) == (kg, kd, pg["lr"], pd["lr"])
    R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, T))
    for it, (lens, x, y) in enumerate(batches(3, B, T, d_in, d_out, 82)):
        update_g = it > 0
        fs.step(*on(dev, lens, x, y), update_g=update_g)
        got = fs.loss_dict()
        gm = g_masks(kind, fs, mg, B, T, g_hidden, dev)
        dm = d_masks(fs, B * T, [d_hidden] * (len(d_layers) - 1), p_d, dev)
        ref, _, ys_ref = gp.gan_step(lambda: gen.forward(x, R, lens, hp, masks=gm), gen.params(), gen.sums, d_layers,
                                     d_sum, x, y, lens, R, hp, w_d=1.0, mse_w=0.0, mge_w=1.0, adv_w=1.0, dropout_d=p_d,
                                     training=True, weight_decay=0.0, update_g=update_g, d_masks=dm, d_opt=d_opt,
                                     g_opt=g_opt)
        errs = {k: abs(got[k] - ref[k]) / max(abs(ref[k]), 1e-12) for k in PRE_UPDATE_KEYS}
        errs["y_hat_static"] = rel_err(npy(fs.y_hat_static), ys_ref.numpy())
        assert max(errs.values()) < TOL, (kind, setting, it, errs)
        for q, r in zip(md.parameters(), d_params):
            dd = np.abs(npy(q) - r.detach().numpy())
            assert np.median(dd) < 5e-6 and dd.max() <= 0.0201, (kind, setting, it, np.median(dd), dd.max())
        if update_g:
            check_weights(mg, gen.named, "%s %s G after step %d" % (kind, setting, it))
        resync_oracle(fs, mg, md, gen, d_params, d_sum, g_opt if kg == "Adam" else None, d_opt if kd == "Adam" else None)
    assert (fs.opt_g.steps, fs.opt_d.steps) == (2, 3)
    if kg == "Adam":
        assert g_opt.t == 2


def _dropin_models(kind, seed, dev):
    """Generator and MLP discriminator without dropout (the reference's logic cannot be given the step's masks)."""
    import gantts_b200
    M = gantts_b200.models
    torch.manual_seed(seed)
    if kind == "mlp":
        mg = M.MLP(20, 187, 2, 32, dropout=0.0, last_sigmoid=False)
    else:
        mg = M.SRURNN(in_dim=20, out_dim=187, num_hidden=2, hidden_dim=16, bidirectional=True, dropout=0.0, use_relu=1,
                      rnn_dropout=0.0)
    md = M.MLP(58, 1, 2, 16, dropout=0.0, last_sigmoid=True)
    return mg.to(dev).train(), md.to(dev).train()


def _mirror_d_only(model_g, model_d, opt_d, x, y, lengths, R, hp, eps=1e-20):
    """tests/trainpy_mirror.train_step up to opt_d.step(): the discriminator warm-up step (train.py:696, update_g =
    False: train_loop :541-566 without update_generator)."""
    from gantts.multistream import get_static_features, multi_stream_mlpg
    from gantts.seqloss import sequence_mask
    from trainpy_mirror import selected_static_stream
    y_static = get_static_features(y, len(hp.windows), hp.stream_sizes, hp.has_dynamic_features)
    mask = sequence_mask(lengths).unsqueeze(-1)
    opt_d.zero_grad()
    y_hat = model_g(x, lengths=lengths)
    y_hat_static = multi_stream_mlpg(y_hat, R, hp.stream_sizes, hp.has_dynamic_features)
    real_in, fake_in = selected_static_stream(y_static, hp), selected_static_stream(y_hat_static, hp)
    T = mask.sum().item()
    loss_real_d = -(torch.log(model_d(real_in, lengths=lengths) + eps) * mask).sum() / T
    loss_fake_d = -(torch.log(1 - model_d(fake_in, lengths=lengths) + eps) * mask).sum() / T
    loss_d = loss_real_d + loss_fake_d
    loss_d.backward()
    torch.nn.utils.clip_grad_norm_(model_d.parameters(), 1.0)
    opt_d.step()
    return [loss_d.item(), loss_fake_d.item(), loss_real_d.item()]


@pytest.mark.gpu
@pytest.mark.parametrize("setting", sorted(SETTINGS))
@pytest.mark.parametrize("kind", ["mlp", "sru"])
def test_gan_trainer_with_an_optimiser_per_model_vs_trainpy_mirror(dev, kind, setting):
    """GanTrainer with optimizer_d / optimizer_d_params: a D-only step and two full steps against the reference's
    per-batch logic on the same modules with torch.optim.<G kind> for G and torch.optim.<D kind> for D.  Between steps
    the torch optimisers load GanTrainer's opt_g / opt_d state_dicts (the checkpoint layout, train.py:162-171)."""
    import sys
    sys.path.insert(1, os.path.join(ROOT, "compat"))
    import trainpy_mirror
    from gantts_b200 import step as gstep
    B, T = 4, 40
    kg, pg, kd, pd = SETTINGS[setting]
    hp = gstep.TTS_ACOUSTIC
    mg, md = _dropin_models(kind, 90, dev)
    rg, rd = _dropin_models(kind, 90, dev)
    tr = gstep.GanTrainer(mg, md, hp, w_d=1.0, mse_w=0.0, mge_w=1.0, optimizer=kg, optimizer_params=pg,
                          optimizer_d=kd, optimizer_d_params=pd)
    assert (type(tr.opt_g).__name__, type(tr.opt_d).__name__) == ("Clip" + kg, "Clip" + kd)
    og, od = getattr(torch.optim, kg)(rg.parameters(), **pg), getattr(torch.optim, kd)(rd.parameters(), **pd)
    R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, T)).to(dev)
    for it, (lens, x, y) in enumerate(batches(3, B, T, 20, 187, 91)):
        xd, yd, ld = on(dev, lens, x, y)
        update_g = it > 0
        out, _, _ = tr.step(xd, yd, lens, R, update_g=update_g)
        if update_g:
            losses = trainpy_mirror.train_step(rg, rd, og, od, xd, yd, ld, R, hp)[0]
            keys = ("loss_d", "loss_fake_d", "loss_real_d", "loss_mse", "loss_mge")
        else:
            losses = _mirror_d_only(rg, rd, od, xd, yd, ld, R, hp)
            keys = ("loss_d", "loss_fake_d", "loss_real_d")
        for k, v in zip(keys, losses):
            assert abs(float(out[k]) - v) <= 1e-4 * abs(v), (kind, setting, it, k, float(out[k]), v)
        for m, r in ((md, rd), (mg, rg)) if update_g else ((md, rd),):
            for q, w in zip(m.parameters(), r.parameters()):
                dd = np.abs(npy(q) - npy(w))
                assert np.median(dd) < 5e-6 and dd.max() <= 0.0201, (kind, setting, it, np.median(dd), dd.max())
        with torch.no_grad():                                    # the mirror's next step starts from GanTrainer's state
            for m, r in ((mg, rg), (md, rd)):
                for q, w in zip(m.parameters(), r.parameters()):
                    w.copy_(q)
        og.load_state_dict(tr.opt_g.state_dict())
        od.load_state_dict(tr.opt_d.state_dict())
    assert (tr.opt_g.steps, tr.opt_d.steps) == (2, 3)
    assert float(og.state_dict()["state"][0]["step"]) == 2.0 and float(od.state_dict()["state"][0]["step"]) == 3.0


def _run(fs, mg, md):
    """Snapshot of everything a step leaves: losses, outputs, both models' weights and optimiser state."""
    return [fs.losses.clone(), fs.y_hat.clone(), fs.y_hat_static.clone()] + snapshot(*mg.parameters(), *md.parameters()) \
        + [s.clone() for s in fs._sums + fs._sqs]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["Adagrad", "Adam"])
def test_optimizer_d_none_equals_an_explicit_identical_one(dev, kind):
    """optimizer_d=None (D takes G's setting) and optimizer_d / optimizer_d_params spelled out give the same steps bit for
    bit: a D-only step then two full steps."""
    from gantts_b200 import fused as F
    B, T = 3, 40
    params = ADAM if kind == "Adam" else dict(lr=0.01, weight_decay=1e-7)
    runs = []
    for explicit in (False, True):
        mg, md, hp, d_in, d_out = build("mlp", 100)[:5]
        mg.to(dev).train(), md.to(dev).train()
        kw = dict(optimizer_d=kind, optimizer_d_params=dict(params)) if explicit else {}
        fs = F.FusedGanStep(mg, md, step_hp(hp), B, T, optimizer=kind, optimizer_params=params, seed=101, **kw)
        snaps = []
        for it, (lens, x, y) in enumerate(batches(3, B, T, d_in, d_out, 102)):
            fs.step(*on(dev, lens, x, y), update_g=it > 0)
            snaps += _run(fs, mg, md)
        runs.append(snaps)
    assert_equal_lists(runs[0], runs[1], "optimizer_d=None vs explicit")


@pytest.mark.gpu
def test_one_call_after_d_only_steps_equals_the_two_call_sequence(dev):
    """Adam on both models after two D-only steps (D takes step 3, G step 1): the one call FusedGanStep makes equals the
    sequence it used to make -- phases 1|2 with D's step number, then 4 with G's, with a zero d_opt block."""
    from gantts_b200 import _lib
    B, T = 3, 40
    runs = []
    for split in (False, True):
        mg, md, hp, d_in, d_out = build("mlp", 110)[:5]
        mg.to(dev).train(), md.to(dev).train()
        from gantts_b200 import fused as F
        fs = F.FusedGanStep(mg, md, step_hp(hp), B, T, optimizer="Adam", optimizer_params=ADAM, seed=111)
        bs = batches(3, B, T, d_in, d_out, 112)
        for lens, x, y in bs[:2]:
            fs.step(*on(dev, lens, x, y), update_g=False)
        lens, x, y = bs[2]
        xd, yd, ld = on(dev, lens, x, y)
        if not split:
            fs.step(xd, yd, ld)
        else:
            seed = fs._seed + fs._step
            n_g, n_d = fs.opt_g.steps + 1, fs.opt_d.steps + 1
            assert (n_g, n_d) == (1, 3)
            fs._set_optimizers(n_g, n_d)
            fs.cfg.d_opt = _lib.OptimizerT()
            fs.cfg.opt_step = n_d
            fs._call(1 | 2, xd, yd, ld, 0.0, seed)
            fs.cfg.opt_step = n_g
            fs._call(4, xd, yd, ld, 0.0, seed)
        runs.append(_run(fs, mg, md))
    assert_equal_lists(runs[0], runs[1], "one call vs phases 1|2 then 4")


@pytest.mark.gpu
@pytest.mark.parametrize("update_g", [True, False])
def test_phase_calls_equal_the_single_call_with_mixed_optimisers(dev, update_g):
    """Adam G + Adagrad D after a D-only step: phases 1, 2 and 4 called one by one (the data-parallel schedule without
    the all-reduces) give exactly what the single call gives."""
    from gantts_b200 import _lib
    B, T = 3, 40
    runs = []
    for split in (False, True):
        mg, md, hp, d_in, d_out = build("sru", 120)[:5]
        mg.to(dev).train(), md.to(dev).train()
        fs = fused(mg, md, hp, B, T, "adam_g_adagrad_d", seed=121)
        bs = batches(2, B, T, d_in, d_out, 122)
        fs.step(*on(dev, *bs[0]), update_g=False)
        xd, yd, ld = on(dev, *bs[1])
        if not split:
            fs.step(xd, yd, ld, update_g=update_g)
        else:
            seed = fs._seed + fs._step
            fs._set_optimizers(fs.opt_g.steps + 1, fs.opt_d.steps + 1)
            d_only = 0 if update_g else _lib.STEP_D_ONLY
            for ph in (1, 2, 4):
                fs._call(ph | d_only, xd, yd, ld, 0.0, seed)
        runs.append(_run(fs, mg, md) + [fs.grad_buffer(0).clone(), fs.grad_buffer(1).clone()])
    assert_equal_lists(runs[0], runs[1], "phase calls vs one call")


@pytest.mark.gpu
def test_exp_lr_scheduler_on_fused_step_and_gan_trainer(dev):
    """train.py's exp_lr_scheduler on fs.opt_g / fs.opt_d and trainer.opt_g / trainer.opt_d over epoch boundaries (one
    mini-batch per epoch, lr_decay_epoch = 2): the groups hold the decayed lr, and the step after a decay equals, bit for
    bit, a step built with that lr from the same weights and optimiser state."""
    from gantts_b200 import fused as F
    from gantts_b200 import step as gstep
    B, T = 3, 40
    kg, pg, kd, pd = SETTINGS["adam_g_adagrad_d"]
    pd = dict(pd, lr=0.01)
    hp = gstep.TTS_ACOUSTIC
    bs = batches(4, B, T, 20, 187, 131)
    R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, T)).to(dev)
    for path in ("fused", "trainer"):
        mg, md = _dropin_models("mlp", 130, dev)
        if path == "fused":
            obj = F.FusedGanStep(mg, md, hp, B, T, optimizer=kg, optimizer_params=pg, optimizer_d=kd, optimizer_d_params=pd,
                                 seed=132)
        else:
            obj = gstep.GanTrainer(mg, md, hp, optimizer=kg, optimizer_params=pg, optimizer_d=kd, optimizer_d_params=pd)

        def step(o, lens, x, y):
            xd, yd, ld = on(dev, lens, x, y)
            if path == "fused":
                o.step(xd, yd, ld)
                return [o.losses.clone()]
            out, _, _ = o.step(xd, yd, lens, R)
            return [out[k].clone() for k in sorted(out)]
        for global_epoch in range(1, 5):
            for opt, init in ((obj.opt_g, pg["lr"]), (obj.opt_d, pd["lr"])):
                exp_lr_scheduler(opt, global_epoch - 1, 4, init_lr=init, lr_decay_epoch=2)
                assert opt.param_groups[0]["lr"] == init * (0.1 ** ((global_epoch - 1) // 2)) == opt.lr
            lens, x, y = bs[global_epoch - 1]
            if global_epoch != 3:
                step(obj, lens, x, y)
                continue
            # the first step after the decay, against one built with the decayed lr from the same state
            opt_sd = {k: {"state": o.state_dict()["state"]} for k, o in (("g", obj.opt_g), ("d", obj.opt_d))}
            w = snapshot(*mg.parameters(), *md.parameters())
            got = step(obj, lens, x, y) + snapshot(*mg.parameters(), *md.parameters())
            g2, d2 = _dropin_models("mlp", 130, dev)
            with torch.no_grad():
                for q, v in zip(list(g2.parameters()) + list(d2.parameters()), w):
                    q.copy_(v)
            kw = dict(optimizer=kg, optimizer_params=dict(pg, lr=obj.opt_g.lr), optimizer_d=kd,
                      optimizer_d_params=dict(pd, lr=obj.opt_d.lr))
            if path == "fused":
                o2 = F.FusedGanStep(g2, d2, hp, B, T, seed=132, **kw)
                o2._step = obj._step - 1
            else:
                o2 = gstep.GanTrainer(g2, d2, hp, **kw)
            o2.opt_g.load_state_dict(opt_sd["g"])
            o2.opt_d.load_state_dict(opt_sd["d"])
            assert (o2.opt_g.lr, o2.opt_d.lr) == (pg["lr"] * 0.1, pd["lr"] * 0.1)
            want = step(o2, lens, x, y) + snapshot(*g2.parameters(), *d2.parameters())
            assert_equal_lists(got, want, "%s: scheduled vs built with the decayed lr" % path)
            if path == "fused":
                assert obj.cfg.lr_d == np.float32(pd["lr"] * 0.1) and obj.cfg.lr_g == np.float32(pg["lr"] * 0.1)


@pytest.mark.gpu
def test_per_model_checkpoints(dev, tmp_path):
    """save_checkpoint(model, fs.opt_*, ...) of a mixed-optimiser FusedGanStep (Adam G, Adagrad D): the files load into
    torch.optim.Adam / torch.optim.Adagrad through load_checkpoint and come back; a FusedGanStep resumed from them
    continues bit for bit; a --reset_optimizers load (train.py:802-811: the model alone) starts from fresh optimiser
    state, like a new FusedGanStep over the same weights."""
    from gantts_b200 import fused as F
    from gantts_b200 import step as gstep
    B, T = 3, 40
    kg, pg, kd, pd = SETTINGS["adam_g_adagrad_d"]
    hp = gstep.TTS_ACOUSTIC
    kw = dict(optimizer=kg, optimizer_params=pg, optimizer_d=kd, optimizer_d_params=pd)
    bs = batches(3, B, T, 20, 187, 141)
    mg, md = _dropin_models("mlp", 140, dev)
    fs = F.FusedGanStep(mg, md, hp, B, T, seed=142, **kw)
    fs.step(*on(dev, *bs[0]), update_g=False)
    fs.step(*on(dev, *bs[1]))
    paths = {n: save_checkpoint(m, o, 7, str(tmp_path), n)
             for n, m, o in (("Generator", mg, fs.opt_g), ("Discriminator", md, fs.opt_d))}
    # into torch.optim and back
    for name, model, opt, tkind, keys in (("Generator", mg, fs.opt_g, "Adam", ("exp_avg", "exp_avg_sq")),
                                          ("Discriminator", md, fs.opt_d, "Adagrad", ("sum",))):
        tm = _dropin_models("mlp", 0, dev)[0 if name == "Generator" else 1]
        topt = getattr(torch.optim, tkind)(tm.parameters(), lr=0.5)
        assert load_checkpoint(tm, topt, paths[name]) == 7
        assert topt.param_groups[0]["lr"] == opt.lr
        for i, p in enumerate(tm.parameters()):
            assert float(topt.state[p]["step"]) == opt.steps
            for k, ts in zip(keys, (opt._state, opt._state2)):
                assert torch.equal(topt.state[p][k], ts[i])
        back = F.FusedGanStep(*_dropin_models("mlp", 0, dev), hp, B, T, **kw)
        bopt = back.opt_g if name == "Generator" else back.opt_d
        bopt.load_state_dict(topt.state_dict())
        fields = lambda o: {k: v for k, v in o.param_groups[0].items() if k != "params"}
        assert bopt.steps == opt.steps and fields(bopt) == fields(opt)
        assert_equal_lists(bopt._state + bopt._state2, opt._state + opt._state2, "%s state back from torch" % name)
    # resume from the two per-model files
    g2, d2 = _dropin_models("mlp", 0, dev)
    fs2 = F.FusedGanStep(g2, d2, hp, B, T, seed=142, **kw)
    load_checkpoint(g2, fs2.opt_g, paths["Generator"])
    load_checkpoint(d2, fs2.opt_d, paths["Discriminator"])
    assert fs2._opt_steps == {"g": 1, "d": 2}
    # --reset_optimizers: the models alone
    g3, d3 = _dropin_models("mlp", 0, dev)
    fs3 = F.FusedGanStep(g3, d3, hp, B, T, seed=142, **kw)
    load_checkpoint(g3, None, paths["Generator"])
    load_checkpoint(d3, None, paths["Discriminator"])
    assert fs3._opt_steps == {"g": 0, "d": 0} and all(not s.any() for s in fs3._sums + fs3._sqs)
    g4, d4 = _dropin_models("mlp", 0, dev)
    with torch.no_grad():
        for q, v in zip(list(g4.parameters()) + list(d4.parameters()), list(g3.parameters()) + list(d3.parameters())):
            q.copy_(v)
    fs4 = F.FusedGanStep(g4, d4, hp, B, T, seed=142, **kw)
    xd, yd, ld = on(dev, *bs[2])
    for f in (fs, fs2, fs3, fs4):
        f.step(xd, yd, ld)
    assert_equal_lists(_run(fs, mg, md), _run(fs2, g2, d2), "resumed from the per-model checkpoints")
    assert_equal_lists(_run(fs3, g3, d3), _run(fs4, g4, d4), "--reset_optimizers vs a new step")
    assert fs3._opt_steps == {"g": 1, "d": 1}


@pytest.mark.gpu
def test_clip_optimizers_restore_every_group_field(dev):
    """ClipAdam and ClipAdagrad read their hyper-parameters from param_groups at step() and load every group field
    (lr, betas, weight_decay, eps) from a state_dict: a step after load_state_dict equals torch.optim's with those
    fields."""
    from gantts_b200 import optim
    for kind, hyper in (("Adam", dict(lr=2e-3, betas=(0.6, 0.95), weight_decay=0.01, eps=1e-6)),
                        ("Adagrad", dict(lr=0.02, weight_decay=0.01, eps=1e-6))):
        torch.manual_seed(150)
        net = torch.nn.Linear(12, 5).to(dev)
        ref = [p.detach().clone().requires_grad_(True) for p in net.parameters()]
        ours = optim.make_optimizer(kind, net.parameters())
        topt = getattr(torch.optim, kind)(ref, **hyper)
        ours.load_state_dict(topt.state_dict())
        g = ours.param_groups[0]
        assert all(g[k] == v for k, v in hyper.items()) and ours.lr == hyper["lr"] and ours.eps == hyper["eps"]
        assert ours.weight_decay == hyper["weight_decay"]
        for it in range(2):
            ours.zero_grad()
            topt.zero_grad()
            for p, r in zip(net.parameters(), ref):
                gr = torch.randn_like(p) * 0.1
                p.grad.copy_(gr)
                r.grad = gr.clone()
            ours.step()
            torch.nn.utils.clip_grad_norm_(ref, 1.0)
            topt.step()
            for p, r in zip(net.parameters(), ref):
                assert rel_err(npy(p), npy(r)) < 2e-6, (kind, it)
