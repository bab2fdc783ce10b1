"""The fused GAN step (gantts_gan_step / FusedGanStep) with the SRURNN generator of hparams `tts_acoustic` and
`tts_duration` (reference gantts/models.py:144-167): the SRU stack's GEMMs and scans, its backward and its optimiser
step inside the one-call step.

The checker is the CPU restatement of the SRU recurrence in oracle/gantts_port.py (sru_layer_forward) composed into an
SRURNN by GeneratorOracle("sru"); SRU parity with the upstream `cuda_functional` package stays unpinned (it is not
vendored).  Train-mode parity injects the step's own masks: every SRU mask is gantts_dropout(ones, p,
gantts_sru_mask_seed(seed, layer, which)), the discriminator's masks come from gantts_gan_step_seed as in
test_gpu_fused_highway.py.  Tolerances: losses, outputs and gradient norms 2e-4 relative; post-step weights median
|delta| < 5e-6 and max <= 0.0201 (a first Adagrad / Adam step moves a weight by lr * sign(g)).  The configuration-rule
test is host-only (no mark).
"""
import numpy as np
import pytest
import torch

from conftest import WINDOWS, TTS_HP, rel_err
from fused_step_helpers import (_sru_step_config, adv_loss_with, check_weights, config_checker, d_masks,  # noqa: F401
                                dev, generator_oracle, loss_errors, make_batch, npy, ragged_lengths, resync_oracle,
                                sd_numpy, sru_masks, sru_models, step_hp, use_adam)
from oracle import gantts_port as gp
from oracle import nnmnkwii_port as nnp

ACOUSTIC_HP = dict(TTS_HP, discriminator_linguistic_condition=True)
DURATION_HP = dict(stream_sizes=[5], has_dynamic_features=[False], adversarial_streams=[True],
                   mask_nth_mgc_for_adv_loss=0, num_windows=1, discriminator_linguistic_condition=True)
LOSS_KEYS = ("loss_d", "loss_fake_d", "loss_real_d", "loss_mge", "loss_mse", "loss_adv", "loss_g")
TOL = 2e-4


def run_vs_oracle(dev, mg, md, ohp, B, T, steps, mse_w, p_d, d_hidden, seed, tag, with_outputs=True):
    from gantts_b200 import fused
    in_dim = mg.gru.rnn_lst[0].n_in
    out_dim = mg.hidden2out.weight.shape[0]
    gen = generator_oracle(mg)
    d_layers = gp.discriminator_layers(sd_numpy(md))
    d_sum = [torch.zeros_like(t) for pair in d_layers for t in pair]
    mg.to(dev).train(), md.to(dev).train()
    fs = fused.FusedGanStep(mg, md, step_hp(ohp), B, T, w_d=1.0, mse_w=mse_w, mge_w=1.0, weight_decay=0.0, seed=seed)
    R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, T))
    for it in range(steps):
        lens = ragged_lengths(B, T, seed + 10 * it)
        x, y = make_batch(B, T, in_dim, out_dim, lens, seed + 10 * it + 1)
        fs.step(x.to(dev), y.to(dev), torch.LongTensor(lens).to(dev), frames=sum(lens))
        got = fs.loss_dict()
        gm, dm = sru_masks(fs, mg, B, dev), d_masks(fs, B * T, [d_hidden] * (len(d_layers) - 1), p_d, dev)
        ref, yh_ref, ys_ref = gp.gan_step(lambda: gen.forward(x, R, lens, ohp, masks=gm), gen.params(), gen.sums,
                                          d_layers, d_sum, x, y, lens, R, ohp, w_d=1.0, mse_w=mse_w, mge_w=1.0,
                                          adv_w=1.0, dropout_d=p_d, training=True, weight_decay=0.0, d_masks=dm)
        ref = dict(ref, loss_adv=adv_loss_with(gp.DiscriminatorOracle(sd_numpy(md)), x, ys_ref, lens, ohp, dm["adv"]))
        errs = loss_errors(got, ref, LOSS_KEYS + ("d_grad_norm", "g_grad_norm"))
        if with_outputs:
            errs["y_hat"] = rel_err(npy(fs.y_hat), yh_ref.numpy())
            errs["y_hat_static"] = rel_err(npy(fs.y_hat_static), ys_ref.numpy())
        assert max(errs.values()) < TOL, (tag, it, errs)
        assert abs(got["real_correct"] - ref["real_correct"]) <= 3 and abs(got["fake_correct"] - ref["fake_correct"]) <= 3
        check_weights(mg, gen.named, "%s step %d" % (tag, it))
        resync_oracle(fs, mg, md, gen, [t for pair in d_layers for t in pair], d_sum)
    return fs


@pytest.mark.gpu
@pytest.mark.parametrize("mse_w", [0.0, 1.0])
@pytest.mark.parametrize("k0", [4, 3])
@pytest.mark.parametrize("relu", [True, False])
@pytest.mark.parametrize("bidir", [True, False])
def test_fused_sru_toy_vs_oracle(dev, bidir, relu, k0, mse_w):
    """A small SRURNN (3 layers, 16 hidden units per direction; layer 0 with k = 4 or, when in_dim = ncols, k = 3) on the
    tts_acoustic stream layout with a conditioned D, dropout 0.2 / rnn_dropout 0.2 in G and 0.5 in D, two training steps
    against the oracle.  mse_w = 0 takes the MLPG adjoint that writes the operand planes directly, 1 the fp32 one."""
    nc = 16 * (2 if bidir else 1)
    in_dim = nc if k0 == 3 else 20
    mg, md = sru_models(100 + 8 * bidir + 4 * relu + k0, in_dim, 187, 3, 16, bidir, relu, 0.2, 0.2, 32, 3, 0.5, 58)
    assert mg.gru.rnn_lst[0].k == k0
    run_vs_oracle(dev, mg, md, ACOUSTIC_HP, 3, 40, 2, mse_w, 0.5, 32, 200 + k0, "toy")


@pytest.mark.gpu
def test_fused_sru_tts_acoustic_full_width(dev):
    """hparams tts_acoustic: SRURNN 425 -> 6 x 512 bidirectional ReLU -> 187, dropout 0.2, rnn_dropout 0.2; D 483 ->
    256 x 3 -> 1 conditioned on x, dropout 0.5; Adagrad.  B = 4 x T = 200 ragged, train mode, one step against the
    oracle: the losses, y_hat, y_hat_static, both gradient norms and every updated generator weight."""
    mg, md = sru_models(7, 425, 187, 6, 512, True, True, 0.2, 0.2, 256, 3, 0.5, 58)
    run_vs_oracle(dev, mg, md, ACOUSTIC_HP, 4, 200, 1, 0.0, 0.5, 256, 300, "tts_acoustic")


@pytest.mark.gpu
def test_fused_sru_tts_duration_adam_and_resume(dev):
    """hparams tts_duration: SRURNN 416 -> 6 x 512 bidirectional ReLU -> 5 (one static stream), D 421 -> 256 x 3 -> 1
    conditioned, Adam lr 1e-3 betas (0.5, 0.9).  Three steps against the oracle's Adam, each starting from the product's
    weights and moments; then a step resumed from state_dict() is bit-identical to the uninterrupted one."""
    from gantts_b200 import fused
    B, T, p, pd = 4, 128, 0.2, 0.5
    okw = dict(lr=1e-3, betas=(0.5, 0.9), weight_decay=0.0, eps=1e-8)

    def build():
        return sru_models(11, 416, 5, 6, 512, True, True, p, p, 256, 3, pd, 5)
    mg, md = build()
    gen = generator_oracle(mg)
    d_layers = gp.discriminator_layers(sd_numpy(md))
    d_params = [t for pair in d_layers for t in pair]
    g_opt, d_opt = gp.AdamStepper(gen.params(), **okw), gp.AdamStepper(d_params, **okw)
    mg.to(dev).train(), md.to(dev).train()
    hp = step_hp(DURATION_HP)
    fs = fused.FusedGanStep(mg, md, hp, B, T, w_d=1.0, mse_w=1.0, mge_w=0.0, seed=12, optimizer="Adam",
                            optimizer_params=okw)
    for it in range(3):
        lens = ragged_lengths(B, T, 40 + it)
        x, y = make_batch(B, T, 416, 5, lens, 50 + it)
        fs.step(x.to(dev), y.to(dev), torch.LongTensor(lens).to(dev), frames=sum(lens))
        got = fs.loss_dict()
        gm, dm = sru_masks(fs, mg, B, dev), d_masks(fs, B * T, [256] * 3, pd, dev)
        ref, yh_ref, ys_ref = gp.gan_step(lambda: gen.forward(x, None, lens, DURATION_HP, masks=gm), gen.params(), None,
                                          d_layers, None, x, y, lens, None, DURATION_HP, w_d=1.0, mse_w=1.0, mge_w=0.0,
                                          adv_w=1.0, dropout_d=pd, training=True, d_masks=dm, d_opt=d_opt, g_opt=g_opt)
        ref = dict(ref, loss_adv=adv_loss_with(gp.DiscriminatorOracle(sd_numpy(md)), x, ys_ref, lens, DURATION_HP,
                                               dm["adv"]))
        errs = loss_errors(got, ref, ("loss_d", "loss_mse", "loss_adv", "loss_g", "d_grad_norm", "g_grad_norm"))
        errs["y_hat"] = rel_err(npy(fs.y_hat), yh_ref.numpy())
        errs["y_hat_static"] = rel_err(npy(fs.y_hat_static), ys_ref.numpy())
        assert max(errs.values()) < TOL, (it, errs)
        check_weights(mg, gen.named, "tts_duration optimizer_g step %d" % it)
        check_weights(md, dict(zip([n for n, _ in md.named_parameters()], d_params)), "tts_duration optimizer_d step %d" % it)
        resync_oracle(fs, mg, md, gen, d_params, None, g_opt, d_opt)
    snap = [q.detach().clone() for q in list(mg.parameters()) + list(md.parameters())]
    sd = fs.state_dict()
    lens = ragged_lengths(B, T, 60)
    x, y = make_batch(B, T, 416, 5, lens, 61)
    xd, yd, ld = x.to(dev), y.to(dev), torch.LongTensor(lens).to(dev)
    fs.step(xd, yd, ld)
    want = fs.loss_dict()
    after = [q.detach().clone() for q in list(mg.parameters()) + list(md.parameters())]
    g2, d2 = build()
    g2.to(dev).train(), d2.to(dev).train()
    with torch.no_grad():
        for q, v in zip(list(g2.parameters()) + list(d2.parameters()), snap):
            q.copy_(v)
    fs2 = fused.FusedGanStep(g2, d2, hp, B, T, w_d=1.0, mse_w=1.0, mge_w=0.0, seed=999, optimizer="Adam",
                             optimizer_params=okw)
    fs2.load_state_dict(sd)
    fs2.step(xd, yd, ld)
    assert fs2.loss_dict() == want
    for q, v in zip(list(g2.parameters()) + list(d2.parameters()), after):
        assert torch.equal(q.detach(), v)


@pytest.mark.gpu
def test_fused_sru_matches_gan_trainer(dev):
    """tts_acoustic widths with every dropout 0: two training steps of FusedGanStep and of the modular GanTrainer from
    the same weights agree on the losses, y_hat, y_hat_static and the updated weights; so do their eval phases on the
    same weights (the fused step's, copied over: a first Adagrad step moves a weight whose gradient is near zero by
    +-lr on either side, which alone moves the outputs by more than the tolerance)."""
    from gantts_b200 import fused, step as gstep
    B, T = 4, 200
    hp = step_hp(ACOUSTIC_HP)
    mk = lambda: sru_models(21, 425, 187, 6, 512, True, True, 0.0, 0.0, 256, 3, 0.0, 58)
    (mg, md), (tg, td) = mk(), mk()
    for m in (mg, md, tg, td):
        m.to(dev).train()
    fs = fused.FusedGanStep(mg, md, hp, B, T, w_d=1.0, mse_w=0.5, mge_w=1.0, weight_decay=0.0, seed=22)
    tr = gstep.GanTrainer(tg, td, hp, w_d=1.0, mse_w=0.5, mge_w=1.0, weight_decay=0.0)
    R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, T)).to(dev)
    for it in range(3):
        train = it < 2
        if not train:
            with torch.no_grad():
                for a, b in zip(list(mg.parameters()) + list(md.parameters()),
                                list(tg.parameters()) + list(td.parameters())):
                    b.copy_(a)
            for m in (mg, md, tg, td):
                m.eval()
        lens = ragged_lengths(B, T, 23 + it)
        x, y = make_batch(B, T, 425, 187, lens, 24 + it)
        xd, yd = x.to(dev), y.to(dev)
        fs.step(xd, yd, torch.LongTensor(lens).to(dev))
        got = fs.loss_dict()
        out, yh, ys = tr.step(xd, yd, lens, R, train=train)
        errs = loss_errors(got, {k: float(out[k]) for k in LOSS_KEYS}, LOSS_KEYS)
        errs["y_hat"] = rel_err(npy(fs.y_hat), npy(yh))
        errs["y_hat_static"] = rel_err(npy(fs.y_hat_static), npy(ys))
        assert max(errs.values()) < TOL, (it, errs)
        for i, (a, b) in enumerate(zip(list(mg.parameters()) + list(md.parameters()),
                                       list(tg.parameters()) + list(td.parameters()))):
            d = np.abs(npy(a) - npy(b))
            assert np.median(d) < 5e-6 and d.max() <= 0.0201, (it, i, np.median(d), d.max())


@pytest.mark.gpu
def test_fused_sru_invariants(dev):
    """An eval-phase call leaves every parameter and all optimiser state bit-unchanged; phases 1, 2 and 4 called one by
    one give exactly what one call gives, and grad_buffer(0) holds every generator parameter in model_g.parameters()
    order; state_dict()'s generator part loads into torch.optim.Adagrad(model_g.parameters())."""
    from gantts_b200 import fused
    B, T = 3, 60
    hp = step_hp(ACOUSTIC_HP)
    lens = ragged_lengths(B, T, 31)
    x, y = make_batch(B, T, 30, 187, lens, 32)
    xd, yd, ld = x.to(dev), y.to(dev), torch.LongTensor(lens).to(dev)
    runs = []
    for split in (False, True):
        mg, md = sru_models(33, 30, 187, 3, 24, True, True, 0.2, 0.2, 32, 3, 0.5, 58)
        mg.to(dev).train(), md.to(dev).train()
        fs = fused.FusedGanStep(mg, md, hp, B, T, mse_w=0.5, weight_decay=0.0, seed=34)
        if split:
            fs.cfg.adv_w, fs._step, fs.cfg.opt_step = 1.0, 1, 1
            for ph in (1, 2, 4):
                fs._call(ph, xd, yd, ld, 0.0, fs._seed)
        else:
            fs.step(xd, yd, ld)
            assert fs.last_seed == fs._seed
        gb = fs.grad_buffer(0)
        params = list(mg.parameters())
        assert gb.numel() == sum(q.numel() for q in params)
        off = 0
        for q, s in zip(params, fs._sums):                 # weight decay 0: Adagrad's first state_sum = g^2
            n = q.numel()
            assert torch.equal((gb[off:off + n] * gb[off:off + n]).view_as(q), s)
            off += n
        runs.append([fs.losses.clone(), fs.y_hat.clone(), fs.y_hat_static.clone(), gb.clone(), fs.grad_buffer(1).clone()]
                    + [q.detach().clone() for q in list(mg.parameters()) + list(md.parameters())]
                    + [s.clone() for s in fs._sums])
    for a, b in zip(*runs):
        assert torch.equal(a, b)
    # eval phase: nothing changes
    wsnap = [q.detach().clone() for q in list(mg.parameters()) + list(md.parameters())]
    ssnap = [s.clone() for s in fs._sums]
    mg.eval(), md.eval()
    fs.step(xd, yd, ld)
    assert fs.loss_dict()["g_grad_norm"] == 0.0
    for a, b in zip(wsnap, list(mg.parameters()) + list(md.parameters())):
        assert torch.equal(a, b.detach())
    for a, b in zip(ssnap, fs._sums):
        assert torch.equal(a, b)
    sd = fs.state_dict()
    opt = torch.optim.Adagrad(mg.parameters(), lr=0.01, weight_decay=0.0)
    opt.load_state_dict(sd["optimizer_g"])
    first = mg.gru.rnn_lst[0].weight
    assert torch.equal(opt.state[first]["sum"], fs._sums[0])
    assert len(sd["optimizer_g"]["state"]) == len(list(mg.parameters()))


@pytest.mark.gpu
def test_fused_sru_rejects_sigmoid_output(dev):
    """An SRURNN with last_sigmoid=True is refused like any sigmoid-output generator."""
    import gantts_b200
    from gantts_b200 import fused
    mg = gantts_b200.models.SRURNN(in_dim=20, out_dim=187, num_hidden=2, hidden_dim=8, last_sigmoid=True).to(dev)
    md = gantts_b200.models.MLP(58, 1, 2, 16, dropout=0.0, last_sigmoid=True).to(dev)
    with pytest.raises(RuntimeError, match="linear-output"):
        fused.FusedGanStep(mg, md, step_hp(TTS_HP), 2, 10)


def test_sru_step_config_rules_on_tensor_tables():
    """gantts_gan_step_workspace_bytes (host-only) accepts the SRURNN layout, lays out no SRU workspace without a stack,
    and rejects, with a message naming the rule, every SRU configuration the step does not implement.  The generator's
    table holds [weight, bias] of layers 0, 1, 2, then hidden2out's."""
    from gantts_b200 import _lib
    ws, err, rejected = config_checker()
    lib = _lib.load()
    assert lib.gantts_version() == 104
    c = _sru_step_config()
    assert ws(c) > 0, err()
    with_sru = ws(c)
    c.sru.num_layers = 0                                # the same config without a stack: D then sees g.dims[0] columns
    c.d.dims[0] = 32 + 58
    c.g_tensors.n = 2
    assert 0 < ws(c) < with_sru, err()

    def rej(mutate, needle):
        rejected(_sru_step_config, mutate, needle)
    rej(lambda c: setattr(c.highway, "static_dim", 59), "mutually exclusive")
    rej(lambda c: setattr(c.sru, "num_layers", _lib.MAX_SRU_LAYERS + 1), "SRU layer count")
    rej(lambda c: setattr(c.sru, "num_layers", -1), "SRU layer count")
    rej(lambda c: setattr(c.sru, "act", 3), "activation")
    rej(lambda c: setattr(c.sru, "dropout", 1.0), "dropout")
    rej(lambda c: setattr(c.sru, "rnn_dropout", -0.1), "dropout")
    rej(lambda c: c.g.dims.__setitem__(0, 31), "hidden2out")
    rej(lambda c: setattr(c.g, "num_layers", 2), "hidden2out")
    rej(lambda c: c.g_tensors.param.__setitem__(4, None), "null generator tensor 4")        # layer 2's weight
    rej(lambda c: c.g_tensors.param.__setitem__(1, None), "null generator tensor 1")        # layer 0's bias
    rej(lambda c: c.g_tensors.state.__setitem__(3, None), "null generator optimiser state of tensor 3")
    rej(lambda c: setattr(c.sru, "num_layers", 2), "generator table has 8 tensors, its shapes give 6")
    rej(lambda c: use_adam(c, missing=(4, 5)), "exp_avg_sq for generator tensor 4")           # layer 2's
    rej(lambda c: c.d.dims.__setitem__(0, 32 + 58), "discriminator input width")
    # the seeds of the SRU masks are a stream of their own
    seeds = {lib.gantts_sru_mask_seed(5, l, w) for l in range(8) for w in range(2)}
    assert len(seeds) == 16 and not seeds & {lib.gantts_gan_step_seed(5, w) for w in range(3)}
