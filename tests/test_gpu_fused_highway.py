"""The fused GAN step (gantts_gan_step / FusedGanStep) with the In2OutHighwayNet generator of hparams `vc`
(reference gantts/models.py:21-69): the sigmoid gate T on x_static, the highway combine around the MLPG and their
backward inside the one-call step.

Parity with injected dropout masks as in test_gpu_train_mode.py: the step's keep masks are regenerated from the seed it
used and handed to the oracle port.  Tolerance: 1e-4 relative unless stated.  The last-but-one test is host-only (no
mark): the highway block's configuration rules through the C ABI.
"""
import numpy as np
import pytest
import torch

from conftest import WINDOWS, rel_err
from fused_step_helpers import (FAKE, _vc_step_config, check_weights, config_checker, dev, loss_errors,  # noqa: F401
                                make_batch, npy, ragged_lengths, resync_oracle, sd_numpy)
from oracle import gantts_port as gp
from oracle import nnmnkwii_port as nnp

VC_HP = dict(stream_sizes=[177], has_dynamic_features=[True], adversarial_streams=[True],
             mask_nth_mgc_for_adv_loss=0, num_windows=3, discriminator_linguistic_condition=False)
# The reference's windows take the substitution MLPG kernels, a delta window two frames wide the FIR kernels.
FAMILY_WINDOWS = {"substitution": WINDOWS,
                  "fir": [WINDOWS[0], (2, 2, np.array([-0.2, -0.1, 0.0, 0.1, 0.2])), WINDOWS[2]]}
LOSS_KEYS = ("loss_d", "loss_fake_d", "loss_real_d", "loss_mge", "loss_mse", "loss_adv", "loss_g")
GOLD_KEYS = ("loss_d", "loss_fake_d", "loss_real_d", "loss_mse", "loss_mge", "loss_adv", "loss_g",
             "real_correct", "fake_correct")


def vc_hp(width=177, windows=WINDOWS):
    from gantts_b200 import step as gstep
    return gstep.HParams(windows=windows, stream_sizes=[width], has_dynamic_features=[True], adversarial_streams=[True],
                         mask_nth_mgc_for_adv_loss=0, discriminator_linguistic_condition=False)


def vc_models(seed, p, dev, hidden=512, d_hidden=256, d_layers=2):
    import gantts_b200
    torch.manual_seed(seed)
    mg = gantts_b200.models.In2OutHighwayNet(in_dim=177, out_dim=177, static_dim=59, num_hidden=3, hidden_dim=hidden,
                                             dropout=p)
    md = gantts_b200.models.MLP(59, 1, d_layers, d_hidden, dropout=p, last_sigmoid=True)
    return mg, md


def step_masks(fs, M, g_hidden, d_hidden, p, dev, with_d=True):
    """The keep masks the last training step drew (gantts_gan_step_seed: 0 = G, 1 = stacked real|fake D, 2 = adv D)."""
    from gantts_b200 import ops, _lib
    lib = _lib.load()
    s = fs.last_seed
    g = [m.cpu() for m in ops.mlp_dropout_masks(M, g_hidden, p, lib.gantts_gan_step_seed(s, 0), dev)]
    if not with_d:
        return g, None
    stacked = ops.mlp_dropout_masks(2 * M, d_hidden, p, lib.gantts_gan_step_seed(s, 1), dev)
    dm = {"real": [m[:M].cpu() for m in stacked], "fake": [m[M:].cpu() for m in stacked],
          "adv": [m.cpu() for m in ops.mlp_dropout_masks(M, d_hidden, p, lib.gantts_gan_step_seed(s, 2), dev)]}
    return g, dm


@pytest.mark.gpu
def test_fused_highway_golden(dev, golden_step_models):
    """The `hw_` vectors of the UNMODIFIED reference's train.py step functions (In2OutHighwayNet 27 -> 27, S = 9,
    B = 3, T = 24, w_d = 0, MSE + MGE, two mini-batches, ragged lengths) through FusedGanStep: every loss of both
    batches, y_hat and y_hat_static (the second batch runs on the weights the first step produced)."""
    import gantts_b200
    from gantts_b200 import fused
    g = golden_step_models
    sub = lambda pre: {k[len(pre):]: torch.from_numpy(g[k]) for k in g.files if k.startswith(pre)}
    mg = gantts_b200.models.In2OutHighwayNet(in_dim=27, out_dim=27, static_dim=9, num_hidden=2, hidden_dim=24,
                                             dropout=0.0)
    mg.load_state_dict(sub("hw_g0_"))
    md = gantts_b200.models.MLP(9, 1, 2, 16, dropout=0.0, last_sigmoid=True)
    mg.to(dev).train(), md.to(dev).train()
    w_d, mse_w, mge_w = [float(v) for v in g["hw_cfg"]]
    assert w_d == 0.0
    fs = fused.FusedGanStep(mg, md, vc_hp(27), 3, 24, w_d=w_d, mse_w=mse_w, mge_w=mge_w, seed=5)
    for it in range(2):
        p = "hw_it%d_" % it
        lens = [int(v) for v in g[p + "lengths"]]
        fs.step(torch.from_numpy(g[p + "x"]).to(dev), torch.from_numpy(g[p + "y"]).to(dev),
                torch.LongTensor(lens).to(dev), adv_w=0.0)
        got = fs.loss_dict()
        for k, v in zip(GOLD_KEYS, g[p + "losses"]):
            if np.isnan(v):
                continue
            if k.endswith("correct"):
                assert got[k] == v, (it, k, got[k], v)
            else:
                assert abs(got[k] - v) <= 1e-4 * max(abs(v), 1e-3), (it, k, got[k], v)
        assert rel_err(npy(fs.y_hat), g[p + "y_hat"]) < 1e-4
        assert rel_err(npy(fs.y_hat_static), g[p + "y_hat_static"]) < 1e-4


@pytest.mark.gpu
def test_fused_highway_vc_adversarial_train_mode_injected_masks(dev):
    """hparams `vc` with adversarial training at full width: G 177 -> 512 x 3 -> 177 (S = 59), D 59 -> 256 -> 256 -> 1,
    dropout 0.5 in both, B = 20 x T = 400 ragged, Adagrad lr 0.01 wd 0.  Against the oracle's In2OutHighwayNet step
    with the fused step's own keep masks: seven losses, both gradient norms, y_hat, y_hat_static, the counts and the
    post-step weights of every generator tensor (the gate included)."""
    from gantts_b200 import fused
    B, T, p = 20, 400, 0.5
    M = B * T
    mg, md = vc_models(61, p, dev)
    gen = gp.GeneratorOracle("highway", sd_numpy(mg), static_dim=59)
    d_layers = gp.discriminator_layers(sd_numpy(md))
    d_sum = [torch.zeros_like(t) for pair in d_layers for t in pair]
    mg.to(dev).train(), md.to(dev).train()
    lens = ragged_lengths(B, T, 62)
    x, y = make_batch(B, T, 177, 177, lens, 63)
    fs = fused.FusedGanStep(mg, md, vc_hp(), B, T, w_d=1.0, mse_w=0.0, mge_w=1.0, weight_decay=0.0, seed=64)
    fs.step(x.to(dev), y.to(dev), torch.LongTensor(lens).to(dev), frames=sum(lens))
    got = fs.loss_dict()
    gm, dm = step_masks(fs, M, [512] * 3, [256] * 2, p, dev)
    R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, T))
    ref, yh_ref, ys_ref = gp.gan_step(lambda: gen.forward(x, R, lens, VC_HP, p, True, gm), gen.params(), gen.sums,
                                      d_layers, d_sum, x, y, lens, R, VC_HP, w_d=1.0, mse_w=0.0, mge_w=1.0, adv_w=1.0,
                                      dropout_d=p, training=True, weight_decay=0.0, d_masks=dm)
    errs = loss_errors(got, ref, LOSS_KEYS + ("d_grad_norm",))
    errs["y_hat"] = rel_err(npy(fs.y_hat), yh_ref.numpy())
    errs["y_hat_static"] = rel_err(npy(fs.y_hat_static), ys_ref.numpy())
    assert max(errs.values()) < 1e-4, errs
    # The generator's gradient norm: 2.0e-4 measured.  The adversarial part of dL/dy_hat_static is D's input gradient,
    # in which every LeakyReLU kink flip of D's hidden layers (bf16x3 vs CPU fp32, see test_leaky_kink_flip_count_is_bounded)
    # moves one derivative between 1 and 0.01; here that term is a large share of G's gradient.  Without the
    # discriminator the gate's and last_linear's gradients agree with the oracle to 1e-5 (test_fused_highway_cfg1_two_steps
    # pins the norm at 1e-4); the modular path's test with a highway generator and a D (cfg3) allows 2e-4 likewise.
    g_err = abs(got["g_grad_norm"] - ref["g_grad_norm"]) / ref["g_grad_norm"]
    assert g_err < 5e-4, g_err
    assert abs(got["real_correct"] - ref["real_correct"]) <= 3 and abs(got["fake_correct"] - ref["fake_correct"]) <= 3
    assert got["frames"] == float(sum(lens))
    check_weights(mg, gen.named, "vc", median=2e-6)


@pytest.mark.gpu
@pytest.mark.parametrize("family", ["substitution", "fir"])
def test_fused_highway_cfg1_two_steps(dev, family):
    """BASELINE cfg1 through the fused step: In2OutHighwayNet(177, static 59, 3 x 512, dropout 0.5), B = 8 x T = 200,
    w_d = 0, mse_w = mge_w = 1 (the fp32 MLPG adjoint path), two consecutive steps against the oracle, on the windows of
    each MLPG kernel family (the reference's windows: substitution kernels with the fused combine; a delta window two
    frames wide: FIR kernels with the elementwise highway passes).  The second step starts the oracle from the product's
    post-step weights and accumulators (see test_cfg1_highway_step_full_size)."""
    from gantts_b200 import fused
    windows = FAMILY_WINDOWS[family]
    B, T, p = 8, 200, 0.5
    mg, md = vc_models(3, p, dev, d_hidden=16)
    gen = gp.GeneratorOracle("highway", sd_numpy(mg), static_dim=59)
    mg.to(dev).train(), md.to(dev).train()
    d_before = [q.detach().clone() for q in md.parameters()]
    fs = fused.FusedGanStep(mg, md, vc_hp(windows=windows), B, T, w_d=0.0, mse_w=1.0, mge_w=1.0, seed=70)
    R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(windows, T))
    for it in range(2):
        lens = ragged_lengths(B, T, 20 + it)
        x, y = make_batch(B, T, 177, 177, lens, 30 + it)
        fs.step(x.to(dev), y.to(dev), torch.LongTensor(lens).to(dev), adv_w=0.0)
        got = fs.loss_dict()
        gm, _ = step_masks(fs, B * T, [512] * 3, None, p, dev, with_d=False)
        ref, yh_ref, ys_ref = gp.gan_step(lambda: gen.forward(x, R, lens, VC_HP, p, True, gm), gen.params(), gen.sums,
                                          None, None, x, y, lens, R, VC_HP, w_d=0.0, mse_w=1.0, mge_w=1.0, adv_w=0.0)
        errs = loss_errors(got, ref, ("loss_mse", "loss_mge", "loss_g", "g_grad_norm"))
        errs["y_hat"] = rel_err(npy(fs.y_hat), yh_ref.numpy())
        errs["y_hat_static"] = rel_err(npy(fs.y_hat_static), ys_ref.numpy())
        assert max(errs.values()) < 1e-4, (it, errs)
        assert got["loss_d"] == 0.0 and got["loss_adv"] == 0.0
        check_weights(mg, gen.named, "cfg1 step %d" % it, median=2e-6)
        resync_oracle(fs, mg, md, gen, [], [])
    for a, b in zip(d_before, md.parameters()):
        assert torch.equal(a, b.detach())


@pytest.mark.gpu
def test_fused_highway_matches_gan_trainer_in_eval(dev):
    """Same weights and batch, both models in .eval(): FusedGanStep (eval phase) and the modular GanTrainer agree on
    every loss and on y_hat_static."""
    from gantts_b200 import fused, step as gstep
    B, T = 6, 150
    mg, md = vc_models(80, 0.5, dev)
    mg.to(dev).eval(), md.to(dev).eval()
    lens = ragged_lengths(B, T, 81)
    x, y = make_batch(B, T, 177, 177, lens, 82)
    xd, yd = x.to(dev), y.to(dev)
    fs = fused.FusedGanStep(mg, md, vc_hp(), B, T, w_d=1.0, mse_w=0.5, mge_w=1.0, seed=83)
    fs.step(xd, yd, torch.LongTensor(lens).to(dev))
    got = fs.loss_dict()
    tr = gstep.GanTrainer(mg, md, vc_hp(), w_d=1.0, mse_w=0.5, mge_w=1.0)
    R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, T)).to(dev)
    out, yh, ys = tr.step(xd, yd, lens, R, train=False)
    errs = loss_errors(got, {k: float(out[k]) for k in LOSS_KEYS}, LOSS_KEYS)
    errs["y_hat"] = rel_err(npy(fs.y_hat), npy(yh))
    errs["y_hat_static"] = rel_err(npy(fs.y_hat_static), npy(ys))
    assert max(errs.values()) < 1e-4, errs
    assert got["real_correct"] == float(out["real_correct"]) and got["fake_correct"] == float(out["fake_correct"])


@pytest.mark.gpu
@pytest.mark.parametrize("optimizer", ["Adagrad", "Adam"])
def test_fused_highway_eval_phase_and_resume(dev, optimizer):
    """An eval-phase call between two training steps leaves every parameter and all optimiser state, the gate's
    included, bit-unchanged; a step resumed from state_dict() after step 1 is bit-identical to the uninterrupted
    step 2; the generator's optimiser state loads into torch.optim over model_g.parameters() with T.weight first."""
    from gantts_b200 import fused
    B, T = 4, 80
    lens = [80, 71, 52, 40]
    okw = dict(lr=1e-3, betas=(0.5, 0.9), weight_decay=0.0, eps=1e-8) if optimizer == "Adam" else None

    def build():
        return vc_models(90, 0.5, dev, hidden=64, d_hidden=32)
    mg, md = build()
    mg.to(dev).train(), md.to(dev).train()
    x, y = make_batch(B, T, 177, 177, lens, 91)
    xd, yd, ld = x.to(dev), y.to(dev), torch.LongTensor(lens).to(dev)
    fs = fused.FusedGanStep(mg, md, vc_hp(), B, T, mse_w=0.25, seed=11, optimizer=optimizer, optimizer_params=okw)
    fs.step(xd, yd, ld)
    sd = fs.state_dict()
    wsnap = [q.detach().clone() for q in list(mg.parameters()) + list(md.parameters())]
    ssnap = [s.clone() for s in fs._sums + fs._sqs]
    assert float(fs._sums[0].abs().max()) > 0.0                    # the gate has optimiser state
    mg.eval(), md.eval()
    fs.step(xd, yd, ld)
    assert fs.loss_dict()["g_grad_norm"] == 0.0
    for a, b in zip(wsnap, list(mg.parameters()) + list(md.parameters())):
        assert torch.equal(a, b.detach())
    for a, b in zip(ssnap, fs._sums + fs._sqs):
        assert torch.equal(a, b)
    mg.train(), md.train()
    fs.step(xd, yd, ld)
    want = fs.loss_dict()
    wfinal = [q.detach().clone() for q in mg.parameters()]
    g2, d2 = build()
    g2.to(dev).train(), d2.to(dev).train()
    for q, w in zip(list(g2.parameters()) + list(d2.parameters()), wsnap):
        q.data.copy_(w)
    fs2 = fused.FusedGanStep(g2, d2, vc_hp(), B, T, mse_w=0.25, seed=999, optimizer=optimizer, optimizer_params=okw)
    fs2.load_state_dict(sd)
    fs2.step(xd, yd, ld)
    assert fs2.loss_dict() == want
    for a, b in zip(wfinal, g2.parameters()):
        assert torch.equal(a, b)
    opt = getattr(torch.optim, optimizer)(g2.parameters(), **(okw or dict(lr=0.01, weight_decay=1e-7)))
    opt.load_state_dict(sd["optimizer_g"])
    key = "exp_avg" if optimizer == "Adam" else "sum"
    st0 = opt.state[g2.T.weight][key]
    assert st0.shape == g2.T.weight.shape and torch.equal(st0.to(dev), sd["optimizer_g"]["state"][0][key])
    assert len(sd["optimizer_g"]["state"]) == len(list(g2.parameters()))


@pytest.mark.gpu
def test_fused_highway_phase_split_is_bitwise_equal(dev):
    """Phases 1, 2 and 4 called one by one (the data-parallel schedule, without the all-reduces) give exactly what one
    call of all phases gives.  grad_buffer(0) holds every generator parameter in model_g.parameters() order, the
    gate's S * S + S gradients first (with weight decay 0, Adagrad's first state_sum is the clipped gradient squared)."""
    from gantts_b200 import fused
    B, T, S = 5, 120, 59
    lens = ragged_lengths(B, T, 95)
    x, y = make_batch(B, T, 177, 177, lens, 96)
    xd, yd, ld = x.to(dev), y.to(dev), torch.LongTensor(lens).to(dev)
    runs = []
    for split in (False, True):
        mg, md = vc_models(97, 0.5, dev, hidden=128, d_hidden=64)
        mg.to(dev).train(), md.to(dev).train()
        fs = fused.FusedGanStep(mg, md, vc_hp(), B, T, mse_w=0.5, weight_decay=0.0, seed=98)
        if split:
            fs.cfg.adv_w, fs._step, fs.cfg.opt_step = 1.0, 1, 1
            for ph in (1, 2, 4):
                fs._call(ph, xd, yd, ld, 0.0, fs._seed)
        else:
            fs.step(xd, yd, ld)
            assert fs.last_seed == fs._seed
        gb = fs.grad_buffer(0)
        assert gb.numel() == sum(q.numel() for q in mg.parameters())
        assert torch.equal(gb[:S * S].view(S, S) * gb[:S * S].view(S, S), fs._sums[0])
        assert torch.equal(gb[S * S:S * S + S] * gb[S * S:S * S + S], fs._sums[1])
        runs.append([fs.losses.clone(), fs.y_hat.clone(), fs.y_hat_static.clone(), gb.clone(), fs.grad_buffer(1).clone()]
                    + [q.detach().clone() for q in list(mg.parameters()) + list(md.parameters())]
                    + [s.clone() for s in fs._sums])
    for a, b in zip(*runs):
        assert torch.equal(a, b)


def test_highway_step_config_rules_on_tensor_tables():
    """gantts_gan_step_workspace_bytes (host-only) accepts the VC layout and rejects, with a message naming the rule,
    every highway configuration the gate + combine arithmetic does not describe."""
    from gantts_b200 import _lib, multistream, step as gstep
    ws, err, rejected = config_checker()
    c = _vc_step_config()
    assert ws(c) > 0, err()
    with_gate = ws(c)
    c.highway.static_dim = 0                                   # the same config as a plain MLP generator
    c.g_tensors.n = 4
    assert 0 < ws(c) < with_gate, err()

    def tts_streams(c):                                        # the TTS layout: four streams, one of them static
        hp = gstep.TTS_ACOUSTIC
        entries, _ = multistream.mlpg_stream_entries(hp.stream_sizes, hp.has_dynamic_features, [True] * 4, 3)
        c.streams = _lib.make_streams(entries)

    def n_static(c):
        c.n_static = c.n_static_cols = 58
    rejected(_vc_step_config, tts_streams, "one dynamic stream")
    rejected(_vc_step_config, n_static, "n_static")
    rejected(_vc_step_config, lambda c: c.g.dims.__setitem__(2, 176), "output width")
    rejected(_vc_step_config, lambda c: c.g_tensors.param.__setitem__(0, None), "null generator tensor 0")
    rejected(_vc_step_config, lambda c: c.g_tensors.param.__setitem__(1, FAKE + 4), "gate bias must be 16-byte aligned")
    rejected(_vc_step_config, lambda c: c.g_tensors.state.__setitem__(1, None),
             "null generator optimiser state of tensor 1")


def test_step_tensor_table_rules():
    """Each model's tensor table must hold exactly the tensors its shapes give, each with its optimiser state; the
    discriminator's table is read only when there is a discriminator (w_d > 0)."""
    ws, err, rejected = config_checker()
    rejected(_vc_step_config, lambda c: setattr(c.g_tensors, "n", 4), "generator table has 4 tensors, its shapes give 6")
    rejected(_vc_step_config, lambda c: setattr(c.g_tensors, "n", 7), "generator table has 7 tensors, its shapes give 6")
    rejected(_vc_step_config, lambda c: setattr(c.d_tensors, "n", 0), "discriminator table has 0 tensors, its shapes give 4")
    rejected(_vc_step_config, lambda c: c.d_tensors.param.__setitem__(2, None), "null discriminator tensor 2")
    rejected(_vc_step_config, lambda c: c.d_tensors.state.__setitem__(3, None),
             "null discriminator optimiser state of tensor 3")
    c = _vc_step_config()
    c.w_d, c.d_tensors.n = 0.0, 0
    assert ws(c) > 0, err()


@pytest.mark.gpu
def test_fused_step_rejects_recurrent_generator(dev):
    """A generator the fused step has no kernels for gets a RuntimeError that points to GanTrainer."""
    import gantts_b200
    from gantts_b200 import fused
    mg = gantts_b200.models.LSTMRNN(in_dim=20, out_dim=177, num_hidden=1, hidden_dim=16).to(dev)
    md = gantts_b200.models.MLP(59, 1, 2, 16, dropout=0.0, last_sigmoid=True).to(dev)
    with pytest.raises(RuntimeError, match="GanTrainer"):
        fused.FusedGanStep(mg, md, vc_hp(), 2, 10)
