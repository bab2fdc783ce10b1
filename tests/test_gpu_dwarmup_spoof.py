"""The discriminator warm-up step (train.py --discriminator-warmup, :696 update_g = False) and the spoofing-rate count
(train.py:549-558) on the GPU: FusedGanStep(update_g=False) / GANTTS_STEP_D_ONLY, gantts_spoof_count, and the same two
features of GanTrainer.

Checkers: the full fused step from the same weights and seed (bit for bit), and the oracle's gan_step(update_g=False)
and spoof_count (pinned to the reference by test_dwarmup_host.py) with the step's own dropout masks injected.
Tolerances as in the fused-generator modules: losses, gradient norm and y_hat_static 2e-4 relative; post-step weights
median |delta| < 5e-6 and max <= 0.0201 (a first Adagrad / Adam step moves a weight by lr * sign(g)).
"""
import numpy as np
import pytest
import torch

from conftest import TTS_HP, WINDOWS, rel_err
from fused_step_helpers import (ADAM, assert_equal_lists, build, check_weights, d_masks, dev, fused,  # noqa: F401
                                g_masks, generator_oracle, make_batch, npy, ragged_lengths, sd_numpy, snapshot, step_hp)
from oracle import gantts_port as gp
from oracle import nnmnkwii_port as nnp

TOL = 2e-4
D_KEYS = ("loss_d", "loss_fake_d", "loss_real_d", "loss_mse", "loss_mge", "d_grad_norm")


@pytest.mark.gpu
@pytest.mark.parametrize("kind,optimizer", [("mlp", "Adagrad"), ("mlp", "Adam"), ("highway", "Adagrad"),
                                            ("sru", "Adagrad"), ("rnn_highway", "Adam")])
def test_d_only_step_equals_full_step_on_the_discriminator(dev, kind, optimizer):
    """From the same weights and seed, a D-only step and a full step agree bit for bit on y_hat, y_hat_static, the D
    losses, counts, frames, MSE / MGE, d_grad_norm, D's parameters and D's optimiser state; the D-only step leaves G's
    parameters and optimiser state untouched and reports g_grad_norm = loss_adv = 0, loss_g = mse_w mse + mge_w mge."""
    B, T = 3, 40
    runs = []
    for update_g in (False, True):
        mg, md, hp, d_in, d_out, _, _, _ = build(kind, 7)
        mg.to(dev).train(), md.to(dev).train()
        lens = ragged_lengths(B, T, 8)
        x, y = make_batch(B, T, d_in, d_out, lens, 9)
        fs = fused(mg, md, hp, B, T, optimizer, mse_w=0.5, seed=10)
        g0 = snapshot(*mg.parameters())
        ng = len(g0)
        fs.step(x.to(dev), y.to(dev), torch.LongTensor(lens).to(dev), update_g=update_g)
        got = fs.loss_dict()
        if not update_g:
            assert_equal_lists(g0, snapshot(*mg.parameters()), "G parameters")
            for s in fs._sums[:ng] + fs._sqs[:ng]:
                assert not s.any()
            assert got["g_grad_norm"] == 0.0 and got["loss_adv"] == 0.0
            assert got["loss_g"] == np.float32(np.float32(0.5 * got["loss_mse"]) + np.float32(got["loss_mge"]))
            sd = fs.state_dict()
            assert float(sd["optimizer_g"]["state"][0]["step"]) == 0.0 and float(sd["optimizer_d"]["state"][0]["step"]) == 1.0
        runs.append((got, [fs.y_hat.clone(), fs.y_hat_static.clone()] + snapshot(*md.parameters()) +
                     [s.clone() for s in fs._sums[ng:] + fs._sqs[ng:]]))
    (a, ta), (b, tb) = runs
    for k in D_KEYS + ("real_correct", "fake_correct", "frames"):
        assert a[k] == b[k], (k, a[k], b[k])
    assert_equal_lists(ta, tb, "outputs, D parameters and D optimiser state")


@pytest.mark.gpu
@pytest.mark.parametrize("optimizer", ["Adagrad", "Adam"])
@pytest.mark.parametrize("kind", ["mlp", "highway", "sru", "rnn_highway", "vc_full"])
def test_d_only_step_vs_oracle(dev, kind, optimizer):
    """Two D-only steps of every generator the fused step runs (toy sizes, and the `vc` models at full width) against the
    CPU restatement with the step's own G and D keep masks: D losses, counts, d_grad_norm, MSE / MGE, y_hat_static and
    D's post-step weights; G bit-unchanged.  The oracle's next step starts from the product's D and optimiser state."""
    B, T = (4, 100) if kind == "vc_full" else (3, 40)
    mg, md, hp, d_in, d_out, g_hidden, d_hidden, p_d = build(kind, 20)
    gen = generator_oracle(mg)
    d_layers = gp.discriminator_layers(sd_numpy(md))
    d_params = [t for pair in d_layers for t in pair]
    d_sum = [torch.zeros_like(t) for t in d_params]
    d_opt = gp.AdamStepper(d_params, **ADAM) if optimizer == "Adam" else None
    mg.to(dev).train(), md.to(dev).train()
    g0 = snapshot(*mg.parameters())
    fs = fused(mg, md, hp, B, T, optimizer, mse_w=0.5, seed=21)
    R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, T))
    for it in range(2):
        lens = ragged_lengths(B, T, 22 + it)
        x, y = make_batch(B, T, d_in, d_out, lens, 24 + it)
        fs.step(x.to(dev), y.to(dev), torch.LongTensor(lens).to(dev), frames=sum(lens), update_g=False)
        got = fs.loss_dict()
        gm = g_masks(kind, fs, mg, B, T, g_hidden, dev)
        dm = d_masks(fs, B * T, [d_hidden] * (len(d_layers) - 1), p_d, dev)
        ref, _, ys_ref = gp.gan_step(lambda: gen.forward(x, R, lens, hp, masks=gm), gen.params(), None, d_layers,
                                     d_sum, x, y, lens, R, hp, mse_w=0.5, dropout_d=p_d, weight_decay=0.0,
                                     update_g=False, d_masks=dm, d_opt=d_opt)
        errs = {k: abs(got[k] - ref[k]) / max(abs(ref[k]), 1e-12) for k in D_KEYS + ("loss_g",)}
        errs["y_hat_static"] = rel_err(npy(fs.y_hat_static), ys_ref.numpy())
        assert max(errs.values()) < TOL, (kind, it, errs)
        assert abs(got["real_correct"] - ref["real_correct"]) <= 3 and abs(got["fake_correct"] - ref["fake_correct"]) <= 3
        assert got["loss_adv"] == 0.0 and got["g_grad_norm"] == 0.0 and got["frames"] == float(sum(lens))
        for q, r in zip(md.parameters(), d_params):
            dd = np.abs(npy(q) - r.detach().numpy())
            assert np.median(dd) < 5e-6 and dd.max() <= 0.0201, (kind, it, np.median(dd), dd.max())
        assert_equal_lists(g0, snapshot(*mg.parameters()), "G parameters")
        sd = fs.state_dict()["optimizer_d"]["state"]
        with torch.no_grad():
            for i, (q, r) in enumerate(zip(md.parameters(), d_params)):
                r.copy_(q.detach().cpu())
                if d_opt is None:
                    d_sum[i].copy_(sd[i]["sum"].cpu())
                else:
                    d_opt.m[i].copy_(sd[i]["exp_avg"].cpu())
                    d_opt.v[i].copy_(sd[i]["exp_avg_sq"].cpu())


@pytest.mark.gpu
def test_d_only_phase_split_is_bitwise_equal(dev):
    """Phases 1|D_ONLY, 2|D_ONLY and 4|D_ONLY called one by one (the data-parallel schedule, without the all-reduce of
    the discriminator's buffer) give exactly what one 7|D_ONLY call gives."""
    from gantts_b200 import _lib
    B, T = 4, 60
    lens = ragged_lengths(B, T, 30)
    runs = []
    for split in (False, True):
        mg, md, hp, d_in, d_out, _, _, _ = build("highway", 31)
        mg.to(dev).train(), md.to(dev).train()
        x, y = make_batch(B, T, d_in, d_out, lens, 32)
        xd, yd, ld = x.to(dev), y.to(dev), torch.LongTensor(lens).to(dev)
        fs = fused(mg, md, hp, B, T, mse_w=0.5, seed=33)
        fs.cfg.adv_w, fs.cfg.opt_step = 1.0, 1
        for ph in ((1, 2, 4) if split else (7,)):
            fs._call(ph | _lib.STEP_D_ONLY, xd, yd, ld, 0.0, fs._seed)
        runs.append([fs.losses.clone(), fs.y_hat.clone(), fs.y_hat_static.clone(), fs.grad_buffer(1).clone()]
                    + snapshot(*mg.parameters(), *md.parameters()) + [s.clone() for s in fs._sums])
    assert_equal_lists(runs[0], runs[1], "split vs one call")


@pytest.mark.gpu
def test_adam_step_counts_per_model_and_resume(dev):
    """Two D-only steps then one full step under Adam: D's bias corrections use step 3 and G's step 1, as the oracle's
    steppers do (every weight of both models agrees with the oracle); state_dict reports each optimiser's own step and a
    FusedGanStep resumed from it takes the next step bit-identically."""
    B, T = 3, 40
    mg, md, hp, d_in, d_out, g_hidden, d_hidden, p_d = build("mlp", 40)
    gen = generator_oracle(mg)
    d_layers = gp.discriminator_layers(sd_numpy(md))
    d_params = [t for pair in d_layers for t in pair]
    g_opt, d_opt = gp.AdamStepper(gen.params(), **ADAM), gp.AdamStepper(d_params, **ADAM)
    mg.to(dev).train(), md.to(dev).train()
    fs = fused(mg, md, hp, B, T, "Adam", seed=41)
    R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, T))
    batches = []
    for it in range(4):
        lens = ragged_lengths(B, T, 42 + it)
        batches.append((lens,) + make_batch(B, T, d_in, d_out, lens, 46 + it))
    for it, update_g in enumerate((False, False, True)):
        lens, x, y = batches[it]
        fs.step(x.to(dev), y.to(dev), torch.LongTensor(lens).to(dev), update_g=update_g)
        gm = g_masks("mlp", fs, mg, B, T, g_hidden, dev)
        dm = d_masks(fs, B * T, [d_hidden] * (len(d_layers) - 1), p_d, dev)
        gp.gan_step(lambda: gen.forward(x, R, lens, hp, masks=gm), gen.params(), None, d_layers, None,
                    x, y, lens, R, hp, w_d=1.0, mse_w=0.0, mge_w=1.0, adv_w=1.0, dropout_d=p_d, training=True,
                    weight_decay=0.0, update_g=update_g, d_masks=dm, d_opt=d_opt, g_opt=g_opt)
        for q, r in zip(md.parameters(), d_params):
            dd = np.abs(npy(q) - r.detach().numpy())
            assert np.median(dd) < 5e-6 and dd.max() <= 0.0201, (it, np.median(dd), dd.max())
        with torch.no_grad():                    # the oracle's next step starts from the product's D
            for r, q in zip(d_params, md.parameters()):
                r.copy_(q.detach().cpu())
    assert (d_opt.t, g_opt.t) == (3, 1)
    sd = fs.state_dict()
    assert float(sd["optimizer_d"]["state"][0]["step"]) == 3.0 and float(sd["optimizer_g"]["state"][0]["step"]) == 1.0
    assert sd["step"] == 3
    check_weights(mg, gen.named, "G after one Adam step")
    # resume: the next (full) step from state_dict() equals the uninterrupted one
    wsnap = snapshot(*mg.parameters(), *md.parameters())
    lens, x, y = batches[3]
    xd, yd, ld = x.to(dev), y.to(dev), torch.LongTensor(lens).to(dev)
    fs.step(xd, yd, ld)
    want, wfinal = fs.loss_dict(), snapshot(*mg.parameters(), *md.parameters())
    mg2, md2 = build("mlp", 40)[:2]
    mg2.to(dev).train(), md2.to(dev).train()
    with torch.no_grad():
        for q, w in zip(list(mg2.parameters()) + list(md2.parameters()), wsnap):
            q.copy_(w)
    fs2 = fused(mg2, md2, hp, B, T, "Adam", seed=999)
    fs2.load_state_dict(sd)
    assert fs2._opt_steps == {"g": 1, "d": 3} and fs2._step == 3
    fs2.step(xd, yd, ld)
    assert fs2.loss_dict() == want
    assert_equal_lists(wfinal, snapshot(*mg2.parameters(), *md2.parameters()), "resumed step")
    sd2 = fs2.state_dict()
    assert float(sd2["optimizer_d"]["state"][0]["step"]) == 4.0 and float(sd2["optimizer_g"]["state"][0]["step"]) == 2.0


@pytest.mark.gpu
def test_gan_trainer_d_only_matches_oracle_and_fused_step(dev):
    """GanTrainer.step(update_g=False) with dropout 0 agrees with the CPU restatement and with the fused D-only step on
    every reported slot and on D's post-step weights; it leaves G and its optimiser untouched."""
    import gantts_b200
    from gantts_b200 import step as gstep
    B, T = 4, 50
    lens = ragged_lengths(B, T, 50)
    x, y = make_batch(B, T, 20, 187, lens, 51)
    xd, yd = x.to(dev), y.to(dev)
    R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, T))

    def models():
        torch.manual_seed(52)
        return (gantts_b200.models.MLP(20, 187, 2, 32, dropout=0.0, last_sigmoid=False).to(dev).train(),
                gantts_b200.models.MLP(58, 1, 2, 16, dropout=0.0, last_sigmoid=True).to(dev).train())
    mg, md = models()
    gen = generator_oracle(mg)
    d_layers = gp.discriminator_layers(sd_numpy(md))
    d_sum = [torch.zeros_like(t) for pair in d_layers for t in pair]
    ref, _, ys_ref = gp.gan_step(lambda: gen.forward(x, R, lens, TTS_HP, mg.dropout_p, True), gen.params(), None,
                                 d_layers, d_sum, x, y, lens, R, TTS_HP, mse_w=0.5, weight_decay=0.0, update_g=False)
    g0 = snapshot(*mg.parameters())
    tr = gstep.GanTrainer(mg, md, gstep.TTS_ACOUSTIC, w_d=1.0, mse_w=0.5, weight_decay=0.0)
    out, _, ys = tr.step(xd, yd, lens, R.to(dev), update_g=False)
    mg_f, md_f = models()
    fs = fused(mg_f, md_f, TTS_HP, B, T, mse_w=0.5, seed=53)
    fs.step(xd, yd, torch.LongTensor(lens).to(dev), update_g=False)
    got_f = fs.loss_dict()
    keys = ("loss_d", "loss_fake_d", "loss_real_d", "loss_mse", "loss_mge", "loss_g")
    for k in keys:
        assert abs(float(out[k]) - ref[k]) <= 1e-4 * abs(ref[k]), (k, float(out[k]), ref[k])
        assert abs(float(out[k]) - got_f[k]) <= 1e-4 * abs(got_f[k]), (k, float(out[k]), got_f[k])
    assert float(out["loss_adv"]) == 0.0 and float(out["frames"]) == float(sum(lens))
    assert abs(float(out["real_correct"]) - ref["real_correct"]) <= 3
    assert abs(float(out["fake_correct"]) - got_f["fake_correct"]) <= 3
    assert rel_err(npy(ys), ys_ref.numpy()) < 1e-4
    assert_equal_lists(g0, snapshot(*mg.parameters()), "G parameters")
    for q, qf, r in zip(md.parameters(), md_f.parameters(), [t for pair in d_layers for t in pair]):
        for other in (r.detach().numpy(), npy(qf)):
            dd = np.abs(npy(q) - other)
            assert np.median(dd) < 5e-6 and dd.max() <= 0.0201


def ref_discriminator(n_in, seed, dev):
    """A reference discriminator with dropout 0.5 (it must run with dropout off) left in train mode."""
    import gantts_b200
    torch.manual_seed(seed)
    return gantts_b200.models.MLP(n_in, 1, 2, 16, dropout=0.5, last_sigmoid=True).to(dev).train()


def centre(ref_d, ys, hp):
    """Scale and shift ref_d's last layer so that its outputs on ys fall on both sides of 0.5."""
    with torch.no_grad():
        ref_d.last_linear.weight.mul_(10.0)
        ref_d.last_linear.bias.zero_()
        z = torch.logit(gp.reference_output(gp.DiscriminatorOracle(sd_numpy(ref_d)), ys, None, hp))
        ref_d.last_linear.bias.fill_(-float(z.median()))


def check_count(got, ref_d, ys, lens, hp):
    """got == the oracle's count on ys, up to the frames where the CPU's |D_ref - 0.5| < 1e-5."""
    d = gp.DiscriminatorOracle(sd_numpy(ref_d))
    mask = gp.sequence_mask(lens, ys.size(1)).unsqueeze(-1)
    want = gp.spoof_count(d, ys, lens, mask, hp)
    close = float(((gp.reference_output(d, ys, lens, hp) - 0.5).abs() < 1e-5).float().mul(mask).sum())
    assert abs(float(got) - want) <= close, (float(got), want, close)
    return want


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["mlp", "highway"])
def test_spoof_count_fused_and_gan_trainer_match_oracle(dev, kind):
    """The spoof count of FusedGanStep and of GanTrainer, in training (full and D-only steps) and in the test phase,
    equals the oracle's count (train.py:549-558) on the product's own pre-update y_hat_static; the reference D runs with
    dropout off and is never updated; loss_dict() reports it only when a reference D is configured."""
    from gantts_b200 import step as gstep
    B, T = 4, 60
    mg, md, hp, d_in, d_out, _, _, _ = build(kind, 60)
    mg.to(dev).train(), md.to(dev).train()
    n_adv = md.layers[0].weight.shape[1]
    ref_d = ref_discriminator(n_adv, 61, dev)
    lens = ragged_lengths(B, T, 62)
    x, y = make_batch(B, T, d_in, d_out, lens, 63)
    xd, yd, ld = x.to(dev), y.to(dev), torch.LongTensor(lens).to(dev)
    mg.eval(), md.eval()
    plain = fused(mg, md, hp, B, T, seed=64)
    plain.step(xd, yd, ld)
    assert "spoof_count" not in plain.loss_dict()
    centre(ref_d, plain.y_hat_static.cpu(), hp)
    r0 = snapshot(*ref_d.parameters())
    fs = fused(mg, md, hp, B, T, seed=64, reference_discriminator=ref_d)
    for i, (train, update_g) in enumerate(((False, True), (True, False), (True, True), (False, True))):
        mg.train(train), md.train(train)
        fs.step(xd, yd, ld, update_g=update_g)
        got = fs.loss_dict()
        want = check_count(got["spoof_count"], ref_d, fs.y_hat_static.cpu(), lens, hp)
        if i == 0:
            assert 0 < want < sum(lens)                        # the reference D's outputs straddle 0.5
        assert float(fs.spoof_count) == got["spoof_count"]
    assert ref_d.training
    assert_equal_lists(r0, snapshot(*ref_d.parameters()), "reference D")
    R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, T)).to(dev)
    tr = gstep.GanTrainer(mg, md, step_hp(hp), w_d=1.0, reference_discriminator=ref_d)
    assert not ref_d.training                                   # train.py:445
    for train, update_g in ((True, True), (True, False), (False, True)):
        mg.train(train), md.train(train)
        out, _, ys = tr.step(xd, yd, lens, R, train=train, update_g=update_g)
        check_count(out["spoof_count"], ref_d, ys.detach().cpu(), lens, hp)
    assert_equal_lists(r0, snapshot(*ref_d.parameters()), "reference D")


@pytest.mark.gpu
def test_conditioned_reference_discriminator_and_d_only_without_d_are_refused(dev):
    """A reference D whose input is not the n_adv adversarial columns alone (a linguistically conditioned one) is refused
    citing train.py:549-555; update_g=False without a discriminator (w_d = 0) is refused by both paths."""
    from gantts_b200 import step as gstep
    mg, md, hp, d_in, d_out, _, _, _ = build("mlp", 70)
    mg.to(dev).train(), md.to(dev).train()
    cond = ref_discriminator(d_in + 58, 71, dev)
    with pytest.raises(RuntimeError, match="train.py:549-555"):
        fused(mg, md, hp, 2, 16, reference_discriminator=cond)
    with pytest.raises(RuntimeError, match="train.py:549-555"):
        gstep.GanTrainer(mg, md, step_hp(hp), reference_discriminator=cond)
    lens = [16, 12]
    x, y = make_batch(2, 16, d_in, d_out, lens, 72)
    fs = fused(mg, md, hp, 2, 16, w_d=0.0, seed=73)
    with pytest.raises(RuntimeError, match="needs w_d > 0"):
        fs.step(x.to(dev), y.to(dev), torch.LongTensor(lens).to(dev), adv_w=0.0, update_g=False)
    tr = gstep.GanTrainer(mg, md, step_hp(hp), w_d=0.0)
    R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, 16)).to(dev)
    with pytest.raises(RuntimeError, match="needs w_d > 0"):
        tr.step(x.to(dev), y.to(dev), lens, R, update_g=False)
