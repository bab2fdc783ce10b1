"""Parity of the BENCHMARKED mode: train mode with dropout 0.5 at BASELINE sizes.

torch's Philox dropout stream cannot be reproduced on the device (the product derives every keep decision from
a counter hash, csrc/common.cuh), so parity is established with INJECTED masks (SURVEY.md 7, hard part 4): the
product's dropout multipliers {0, 1/(1-p)} are regenerated with gantts_dropout() from the seeds the step used
and handed to the oracle port, whose mlp_forward applies them where the reference applies F.dropout
(Linear -> LeakyReLU -> Dropout, gantts/models.py:137-139).  Everything else in the oracle is the reference's
arithmetic (pinned by tests/test_oracle_golden.py), so a bug in the product's dropout scaling, its 2-bit
derivative code plane under dropout, the per-forward seeds or the real|fake stacking shows up as a loss /
gradient mismatch here.

Tolerance: 1e-4 relative (the north-star bar for fp32 outputs and losses).
"""
import numpy as np
import pytest
import torch

from conftest import WINDOWS, TTS_HP, rel_err
from oracle import gantts_port as gp
from oracle import nnmnkwii_port as nnp

pytestmark = pytest.mark.gpu

NAMES4 = ["layers.0", "layers.1", "layers.2", "last_linear"]
VC_HP = dict(stream_sizes=[177], has_dynamic_features=[True], adversarial_streams=[True],
             mask_nth_mgc_for_adv_loss=0, num_windows=3, discriminator_linguistic_condition=False)


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__
    __graft_entry__.build()
    return torch.device("cuda:0")


def npy(t):
    return t.detach().cpu().numpy()


def ragged_lengths(B, T, seed):
    rng = np.random.RandomState(seed)
    return sorted([T] + [int(v) for v in rng.randint(T // 2, T, B - 1)], reverse=True)


def make_batch(B, T, d_in, d_out, lens, seed, uniform_x=True):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(B, T, d_in, generator=g) * 0.98 + 0.01 if uniform_x else torch.randn(B, T, d_in, generator=g)
    y = torch.randn(B, T, d_out, generator=g)
    for b, n in enumerate(lens):
        x[b, n:] = 0
        y[b, n:] = 0
    return x, y


def layers_of(m, names=NAMES4):
    sd = m.state_dict()
    return [(sd[n + ".weight"].detach().cpu().clone(), sd[n + ".bias"].detach().cpu().clone()) for n in names]


def cfg2_models(p, dev):
    import gantts_b200
    torch.manual_seed(1234)
    mg = gantts_b200.models.MLP(425, 187, 3, 512, dropout=p, last_sigmoid=False)
    md = gantts_b200.models.MLP(58, 1, 3, 256, dropout=p, last_sigmoid=True)
    state = gp.GanStepState(layers_of(mg), layers_of(md))
    return mg.to(dev).train(), md.to(dev).train(), state


def loss_errors(got, ref, keys):
    return {k: abs(float(got[k]) - ref[k]) / max(abs(ref[k]), 1e-12) for k in keys}


LOSS_KEYS = ("loss_d", "loss_fake_d", "loss_real_d", "loss_mge", "loss_mse", "loss_adv", "loss_g")


def test_fused_step_cfg2_full_size_train_mode_injected_masks(dev):
    """gantts_gan_step at the benchmarked configuration -- B=32 x T=1000, G 425-512-512-512-187, D 58-256-256-256-1,
    dropout 0.5 in train mode, ragged lengths -- against the oracle driven with the step's own keep masks: all seven
    losses, both gradient norms (i.e. every weight gradient of G and D), y_hat, y_hat_static, the counts."""
    from gantts_b200 import step as gstep, fused, ops, _lib
    lib = _lib.load()
    B, T, p = 32, 1000, 0.5
    M = B * T
    mg, md, state = cfg2_models(p, dev)
    lens = ragged_lengths(B, T, 7)
    x, y = make_batch(B, T, 425, 187, lens, 99)
    fs = fused.FusedGanStep(mg, md, gstep.TTS_ACOUSTIC, B, T, w_d=1.0, mse_w=0.5, mge_w=1.0, seed=4242)
    fs.step(x.to(dev), y.to(dev), torch.LongTensor(lens).to(dev), frames=sum(lens))
    got = fs.loss_dict()
    s = fs.last_seed
    cpu = lambda ms: [m.cpu() for m in ms]
    masks = {"g": cpu(ops.mlp_dropout_masks(M, [512] * 3, p, lib.gantts_gan_step_seed(s, 0), dev))}
    stacked = ops.mlp_dropout_masks(2 * M, [256] * 3, p, lib.gantts_gan_step_seed(s, 1), dev)
    masks["real"] = [m[:M].cpu() for m in stacked]
    masks["fake"] = [m[M:].cpu() for m in stacked]
    del stacked
    masks["adv"] = cpu(ops.mlp_dropout_masks(M, [256] * 3, p, lib.gantts_gan_step_seed(s, 2), dev))
    keep = float(np.mean([float((m != 0).float().mean()) for m in masks["g"] + masks["adv"]]))
    assert abs(keep - 0.5) < 2e-3 and float(masks["g"][0].max()) == 2.0
    R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, T))
    ref, yh_ref, ys_ref = gp.gan_step_mlp(state, x, y, lens, R, TTS_HP, mse_w=0.5, dropout_g=p, dropout_d=p,
                                          training=True, masks=masks)
    errs = loss_errors(got, ref, LOSS_KEYS + ("d_grad_norm", "g_grad_norm"))
    errs["y_hat"] = rel_err(npy(fs.y_hat), yh_ref.numpy())
    errs["y_hat_static"] = rel_err(npy(fs.y_hat_static), ys_ref.numpy())
    assert max(errs.values()) < 1e-4, errs
    # counts: (D > 0.5) on 26k frames -- a value within fp32 rounding of 0.5 may fall on either side
    assert abs(got["real_correct"] - ref["real_correct"]) <= 3 and abs(got["fake_correct"] - ref["fake_correct"]) <= 3
    assert got["frames"] == float(sum(lens))
    # post-step weights (Adagrad's first step is lr * sign(g): ill-conditioned only where g ~ 0)
    for mod, st in ((mg, state.g), (md, state.d)):
        dW = np.abs(npy(mod.layers[1].weight) - st[1][0].detach().numpy())
        assert np.median(dW) < 1e-6 and dW.max() <= 0.0201, (np.median(dW), dW.max())


def test_gan_trainer_cfg2_full_size_train_mode_injected_masks(dev):
    """The modular path (GanTrainer: python-orchestrated native ops through autograd) at the same configuration."""
    from gantts_b200 import step as gstep, ops
    B, T, p = 32, 1000, 0.5
    M = B * T
    mg, md, state = cfg2_models(p, dev)
    lens = ragged_lengths(B, T, 8)
    x, y = make_batch(B, T, 425, 187, lens, 100)
    tr = gstep.GanTrainer(mg, md, gstep.TTS_ACOUSTIC, w_d=1.0, mse_w=0.0, mge_w=1.0)
    torch.manual_seed(77)
    sg, sr, sf, sa = ops.peek_seeds(4)          # G forward, D(real), D(fake), D(adv): one draw per mlp_stack call
    R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, T))
    out, yh, ys = tr.step(x.to(dev), y.to(dev), torch.LongTensor(lens).to(dev), R.to(dev))
    cpu = lambda ms: [m.cpu() for m in ms]
    masks = {"g": cpu(ops.mlp_dropout_masks(M, [512] * 3, p, sg, dev)),
             "real": cpu(ops.mlp_dropout_masks(M, [256] * 3, p, sr, dev)),
             "fake": cpu(ops.mlp_dropout_masks(M, [256] * 3, p, sf, dev)),
             "adv": cpu(ops.mlp_dropout_masks(M, [256] * 3, p, sa, dev))}
    ref, yh_ref, ys_ref = gp.gan_step_mlp(state, x, y, lens, R, TTS_HP, dropout_g=p, dropout_d=p, training=True,
                                          masks=masks)
    errs = loss_errors(out, ref, ("loss_d", "loss_fake_d", "loss_real_d", "loss_mge", "loss_adv", "loss_g"))
    errs["y_hat"] = rel_err(npy(yh), yh_ref.numpy())
    errs["y_hat_static"] = rel_err(npy(ys), ys_ref.numpy())
    errs["g_grad_norm"] = abs(float(tr.opt_g.grad_norm()) - ref["g_grad_norm"]) / ref["g_grad_norm"]
    errs["d_grad_norm"] = abs(float(tr.opt_d.grad_norm()) - ref["d_grad_norm"]) / ref["d_grad_norm"]
    assert max(errs.values()) < 1e-4, errs


DUR_HP = dict(stream_sizes=[5], has_dynamic_features=[False], adversarial_streams=[True], mask_nth_mgc_for_adv_loss=0,
              num_windows=1, discriminator_linguistic_condition=False)


def _duration_models(dev, p=0.0):
    import gantts_b200
    torch.manual_seed(5)
    mg = gantts_b200.models.MLP(20, 5, 2, 64, dropout=p, last_sigmoid=False)
    md = gantts_b200.models.MLP(5, 1, 2, 32, dropout=p, last_sigmoid=True)
    names = ["layers.0", "layers.1", "last_linear"]
    state = gp.GanStepState(layers_of(mg, names), layers_of(md, names))
    return mg.to(dev).train(), md.to(dev).train(), state


def _duration_hp():
    from gantts_b200 import step as gstep
    return gstep.HParams(windows=[(0, 0, np.array([1.0]))], stream_sizes=[5], has_dynamic_features=[False],
                         adversarial_streams=[True], mask_nth_mgc_for_adv_loss=0, discriminator_linguistic_condition=False)


def test_gan_trainer_duration_config_adam_and_no_R(dev):
    """The duration model's configuration (reference hparams.py:98-130): static-only stream (has_dynamic_features = [False]
    => train.py:510-515 passes R = None and multi_stream_mlpg is the identity), adversarial loss on the whole stream, Adam
    (lr 1e-3, betas (0.5, 0.9)) for both models.  GanTrainer with optimizer="Adam" against the oracle stepping with
    AdamStepper: losses, both gradient norms and the post-step weights of two consecutive steps (the oracle is re-synchronised
    to the product's weights and moments before step 2: a first Adam step is lr * sign(g), ill-conditioned where g ~ 0)."""
    from gantts_b200 import step as gstep
    B, T = 6, 50
    mg, md, state = _duration_models(dev)
    okw = dict(lr=1e-3, betas=(0.5, 0.9), weight_decay=0.0, eps=1e-8)
    tr = gstep.GanTrainer(mg, md, _duration_hp(), w_d=1.0, mse_w=1.0, mge_w=0.0, optimizer="Adam", optimizer_params=okw)
    g_opt = gp.AdamStepper(state.g_params(), **okw)
    d_opt = gp.AdamStepper(state.d_params(), **okw)
    for it in range(2):
        lens = ragged_lengths(B, T, 30 + it)
        x, y = make_batch(B, T, 20, 5, lens, 200 + it)
        out, yh, ys = tr.step(x.to(dev), y.to(dev), lens, None)
        ref, yh_ref, ys_ref = gp.gan_step_mlp(state, x, y, lens, None, DUR_HP, w_d=1.0, mse_w=1.0, mge_w=0.0, d_opt=d_opt,
                                              g_opt=g_opt)
        errs = loss_errors(out, ref, ("loss_d", "loss_fake_d", "loss_real_d", "loss_mse", "loss_mge", "loss_adv", "loss_g"))
        errs["y_hat"] = rel_err(npy(yh), yh_ref.numpy())
        errs["g_grad_norm"] = abs(float(tr.opt_g.grad_norm()) - ref["g_grad_norm"]) / ref["g_grad_norm"]
        errs["d_grad_norm"] = abs(float(tr.opt_d.grad_norm()) - ref["d_grad_norm"]) / ref["d_grad_norm"]
        assert max(errs.values()) < 1e-4, (it, errs)
        assert torch.equal(ys, yh)                                       # static-only: MLPG is the identity
        for mod, params in ((mg, state.g_params()), (md, state.d_params())):
            for q, r in zip(mod.parameters(), params):
                dW = np.abs(npy(q) - r.detach().numpy())
                assert np.median(dW) < 2e-6 and dW.max() <= 2.01e-3, (it, np.median(dW), dW.max())
        # re-synchronise the oracle: weights and Adam moments
        with torch.no_grad():
            for mod, params, opt, st in ((mg, state.g_params(), tr.opt_g, g_opt), (md, state.d_params(), tr.opt_d, d_opt)):
                sd = opt.state_dict()["state"]
                for i, (q, r) in enumerate(zip(mod.parameters(), params)):
                    r.copy_(q.detach().cpu())
                    st.m[i].copy_(sd[i]["exp_avg"].cpu())
                    st.v[i].copy_(sd[i]["exp_avg_sq"].cpu())


def test_fused_step_adam(dev):
    """gantts_gan_step with optimizer = Adam (reference hparams.py:125-130: lr 1e-3, betas (0.5, 0.9)) against the oracle
    stepping with AdamStepper (pinned to torch.optim.Adam on the CPU): three consecutive steps -- losses, gradient norms,
    post-step weights -- with the oracle re-synchronised to the product's weights and moments between steps (a first Adam
    step is lr * sign(g)); and the state_dict is torch.optim.Adam's layout and round-trips."""
    from gantts_b200 import fused, step as gstep
    B, T = 4, 120
    import gantts_b200
    torch.manual_seed(9)
    mg = gantts_b200.models.MLP(425, 187, 2, 128, dropout=0.0, last_sigmoid=False)
    md = gantts_b200.models.MLP(58, 1, 2, 64, dropout=0.0, last_sigmoid=True)
    names = ["layers.0", "layers.1", "last_linear"]
    state = gp.GanStepState(layers_of(mg, names), layers_of(md, names))
    mg, md = mg.to(dev).train(), md.to(dev).train()
    okw = dict(lr=1e-3, betas=(0.5, 0.9), weight_decay=0.0, eps=1e-8)
    fs = fused.FusedGanStep(mg, md, gstep.TTS_ACOUSTIC, B, T, w_d=1.0, mse_w=0.0, mge_w=1.0, seed=1, optimizer="Adam",
                            optimizer_params=okw)
    g_opt, d_opt = gp.AdamStepper(state.g_params(), **okw), gp.AdamStepper(state.d_params(), **okw)
    R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, T))
    for it in range(3):
        lens = ragged_lengths(B, T, 50 + it)
        x, y = make_batch(B, T, 425, 187, lens, 400 + it)
        fs.step(x.to(dev), y.to(dev), torch.LongTensor(lens).to(dev), frames=sum(lens))
        got = fs.loss_dict()
        ref, yh_ref, ys_ref = gp.gan_step_mlp(state, x, y, lens, R, TTS_HP, d_opt=d_opt, g_opt=g_opt)
        errs = loss_errors(got, ref, LOSS_KEYS + ("d_grad_norm", "g_grad_norm"))
        errs["y_hat_static"] = rel_err(npy(fs.y_hat_static), ys_ref.numpy())
        assert max(errs.values()) < 1e-4, (it, errs)
        sd = fs.state_dict()
        for mod, params, key, st in ((mg, state.g_params(), "optimizer_g", g_opt), (md, state.d_params(), "optimizer_d", d_opt)):
            assert set(sd[key]["state"][0]) == {"step", "exp_avg", "exp_avg_sq"} and tuple(sd[key]["param_groups"][0]["betas"]) == (0.5, 0.9)
            for i, (q, r) in enumerate(zip(mod.parameters(), params)):
                dW = np.abs(npy(q) - r.detach().numpy())
                assert np.median(dW) < 2e-6 and dW.max() <= 4e-3, (it, key, i, np.median(dW), dW.max())
                with torch.no_grad():                                    # re-synchronise the oracle
                    r.copy_(q.detach().cpu())
                    st.m[i].copy_(sd[key]["state"][i]["exp_avg"].cpu())
                    st.v[i].copy_(sd[key]["state"][i]["exp_avg_sq"].cpu())
    # resume: a second object loaded from the state_dict takes the same next step
    snap = [q.detach().clone() for q in list(mg.parameters()) + list(md.parameters())]
    sd = fs.state_dict()
    lens = ragged_lengths(B, T, 60)
    x, y = make_batch(B, T, 425, 187, lens, 500)
    fs.step(x.to(dev), y.to(dev), torch.LongTensor(lens).to(dev), frames=sum(lens))
    after = [q.detach().clone() for q in list(mg.parameters()) + list(md.parameters())]
    with torch.no_grad():
        for q, v in zip(list(mg.parameters()) + list(md.parameters()), snap):
            q.copy_(v)
    fs2 = fused.FusedGanStep(mg, md, gstep.TTS_ACOUSTIC, B, T, w_d=1.0, mse_w=0.0, mge_w=1.0, seed=77, optimizer="Adam",
                             optimizer_params=okw)
    fs2.load_state_dict(sd)
    fs2.step(x.to(dev), y.to(dev), torch.LongTensor(lens).to(dev), frames=sum(lens))
    for q, v in zip(list(mg.parameters()) + list(md.parameters()), after):
        assert torch.equal(q.detach(), v)


def test_fused_step_static_only_streams(dev):
    """The same static-only configuration on the fused entry point (Adagrad): no stream has dynamic features, MLPG
    degenerates to a copy (reference train.py:510-515: R = None), the discriminator sees the whole stream."""
    from gantts_b200 import fused
    B, T = 6, 50
    mg, md, state = _duration_models(dev)
    lens = ragged_lengths(B, T, 41)
    x, y = make_batch(B, T, 20, 5, lens, 300)
    fs = fused.FusedGanStep(mg, md, _duration_hp(), B, T, w_d=1.0, mse_w=1.0, mge_w=1.0, seed=3)
    fs.step(x.to(dev), y.to(dev), torch.LongTensor(lens).to(dev), frames=sum(lens))
    got = fs.loss_dict()
    ref, yh_ref, ys_ref = gp.gan_step_mlp(state, x, y, lens, None, DUR_HP, w_d=1.0, mse_w=1.0, mge_w=1.0)
    errs = loss_errors(got, ref, LOSS_KEYS + ("d_grad_norm", "g_grad_norm"))
    errs["y_hat"] = rel_err(npy(fs.y_hat), yh_ref.numpy())
    errs["y_hat_static"] = rel_err(npy(fs.y_hat_static), ys_ref.numpy())
    assert max(errs.values()) < 1e-4, errs
    assert torch.equal(fs.y_hat, fs.y_hat_static)


@pytest.mark.parametrize("rows,cols,p", [(257, 256, 0.5), (64, 187, 0.2), (33, 58, 0.5), (5, 3, 0.9)])
def test_dropout_mask_matches_numpy_mirror(dev, rows, cols, p):
    """gantts_dropout (the kernel the injected-mask parity tests regenerate masks with) against tests/dropout_mirror.py, the
    numpy statement of csrc/common.cuh's counter hash: bit-exact, including widths that are not multiples of 4; and the
    tensor-core epilogue applies the same mask (a Linear layer with zero weights and bias 1 outputs exactly the multiplier)."""
    import dropout_mirror as dm
    from gantts_b200 import ops, _lib
    seed = 0x1234567 * (rows + cols)
    keep = dm.keep_mask(seed, rows, cols, p)
    scale = 1.0 / (1.0 - p)

    def check(got, what):
        assert np.array_equal(got != 0, keep), what                         # the mask: bit-exact
        assert np.allclose(got[keep], scale, rtol=1e-6, atol=0), what       # the multiplier 1 / (1 - p)
    check(npy(ops.dropout_mask(rows, cols, p, seed, dev)), "gantts_dropout")
    if cols >= 16:
        W = torch.zeros(cols, 16, device=dev)
        b = torch.ones(cols, device=dev)
        x = torch.zeros(rows, 16, device=dev)
        for engine in ("simt", "tc"):
            y = ops.linear_act(x, W, b, act=_lib.ACT_LEAKY_DROPOUT, p=p, training=True, engine=engine, seed=seed)
            check(npy(y), engine)


@pytest.mark.parametrize("mse_w,mge_w", [(0.0, 1.0), (1.0, 0.0)])
def test_fused_step_without_discriminator(dev, mse_w, mge_w):
    """BASELINE configs[3] (TTS acoustic MLP + MGE loss, no adversarial term) and the MSE-only objective of configs[0] on the
    fused entry point: w_d = 0 -- no discriminator forward/backward/update, loss_g = mse_w MSE + mge_w MGE -- train mode with
    the injected generator mask, against the oracle; the discriminator's weights must come out untouched."""
    from gantts_b200 import step as gstep, fused, ops, _lib
    lib = _lib.load()
    B, T, p = 4, 250, 0.5
    M = B * T
    mg, md, state = cfg2_models(p, dev)
    d_before = [q.detach().clone() for q in md.parameters()]
    lens = ragged_lengths(B, T, 21)
    x, y = make_batch(B, T, 425, 187, lens, 123)
    fs = fused.FusedGanStep(mg, md, gstep.TTS_ACOUSTIC, B, T, w_d=0.0, mse_w=mse_w, mge_w=mge_w, seed=99)
    fs.step(x.to(dev), y.to(dev), torch.LongTensor(lens).to(dev), frames=sum(lens))
    got = fs.loss_dict()
    masks = {"g": [m.cpu() for m in ops.mlp_dropout_masks(M, [512] * 3, p, lib.gantts_gan_step_seed(fs.last_seed, 0), dev)]}
    R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, T))
    ref, yh_ref, ys_ref = gp.gan_step_mlp(state, x, y, lens, R, TTS_HP, w_d=0.0, mse_w=mse_w, mge_w=mge_w, dropout_g=p,
                                          dropout_d=p, training=True, masks=masks)
    errs = loss_errors(got, ref, ("loss_mge", "loss_mse", "loss_g", "g_grad_norm"))
    errs["y_hat"] = rel_err(npy(fs.y_hat), yh_ref.numpy())
    errs["y_hat_static"] = rel_err(npy(fs.y_hat_static), ys_ref.numpy())
    assert max(errs.values()) < 1e-4, errs
    assert got["loss_d"] == 0.0 and got["loss_adv"] == 0.0 and got["frames"] == float(sum(lens))
    for a, b in zip(d_before, md.parameters()):
        assert torch.equal(a, b.detach())
    dW = np.abs(npy(mg.layers[1].weight) - state.g[1][0].detach().numpy())
    assert np.median(dW) < 1e-6 and dW.max() <= 0.0201


def test_cfg1_highway_step_full_size(dev):
    """BASELINE cfg1: In2OutHighwayNet(177 -> 177, static 59, 3 x 512, dropout 0.5), B=8 x T=200, no discriminator
    (w_d = 0), MSE + MGE, train mode with injected masks; two consecutive steps incl. post-step weights."""
    import gantts_b200
    from gantts_b200 import step as gstep, ops
    B, T, p = 8, 200, 0.5
    torch.manual_seed(3)
    m = gantts_b200.models.In2OutHighwayNet(in_dim=177, out_dim=177, static_dim=59, num_hidden=3, hidden_dim=512,
                                            dropout=p)
    gen = gp.GeneratorOracle("highway", {k: v.detach().numpy() for k, v in m.state_dict().items()}, static_dim=59)
    m.to(dev).train()
    hp = gstep.HParams(windows=WINDOWS, stream_sizes=[177], has_dynamic_features=[True], adversarial_streams=[True],
                       mask_nth_mgc_for_adv_loss=0, discriminator_linguistic_condition=False)
    tr = gstep.GanTrainer(m, None, hp, w_d=0.0, mse_w=1.0, mge_w=1.0)
    R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, T))
    for it in range(2):
        lens = ragged_lengths(B, T, 20 + it)
        x, y = make_batch(B, T, 177, 177, lens, 30 + it, uniform_x=False)
        torch.manual_seed(500 + it)
        (sg,) = ops.peek_seeds(1)
        out, yh, ys = tr.step(x.to(dev), y.to(dev), lens, R.to(dev), adv_w=0.0)
        masks = [mm.cpu() for mm in ops.mlp_dropout_masks(B * T, [512] * 3, p, sg, dev)]
        ref, yh_ref, ys_ref = gp.gan_step(lambda: gen.forward(x, R, lens, VC_HP, p, True, masks), gen.params(),
                                          gen.sums, None, None, x, y, lens, R, VC_HP, w_d=0.0, mse_w=1.0, mge_w=1.0,
                                          adv_w=0.0)
        errs = loss_errors(out, ref, ("loss_mse", "loss_mge", "loss_g"))
        errs["y_hat"] = rel_err(npy(yh), yh_ref.numpy())
        errs["y_hat_static"] = rel_err(npy(ys), ys_ref.numpy())
        errs["g_grad_norm"] = abs(float(tr.opt_g.grad_norm()) - ref["g_grad_norm"]) / ref["g_grad_norm"]
        assert max(errs.values()) < 1e-4, (it, errs)
        for k, v in m.state_dict().items():
            d = np.abs(npy(v) - gen.named[k].detach().numpy())
            assert np.median(d) < 2e-6 and d.max() <= 0.0201, (it, k, np.median(d), d.max())
        # Adagrad's first steps are lr * sign(g) per element: an element whose gradient is ~0 moves by +-lr with a
        # sign decided by rounding, and the NEXT forward amplifies that (the oracle run twice with a 1e-7 input
        # perturbation already differs by 9e-5 in the second step's y_hat).  The second step is therefore taken
        # from the product's own post-step state (weights and Adagrad accumulators), which pins its arithmetic
        # -- non-zero accumulators, weight decay -- without compounding the sign chaos.
        sums = dict(zip([n for n, _ in m.named_parameters()], tr.opt_g._sums))
        with torch.no_grad():
            for i, (k, t) in enumerate(gen.named.items()):
                t.copy_(m.state_dict()[k].cpu())
                gen.sums[i].copy_(sums[k].cpu())


def test_leaky_kink_flip_count_is_bounded(dev):
    """How many hidden activations land on the other side of the LeakyReLU kink than in the fp32 reference
    (bf16x3 tensor-core accumulation vs torch CPU fp32): each such element swaps a derivative 1 <-> 0.01 in the
    backward, which is why weight gradients are compared in norm.  Bound: < 1e-4 of the elements, and only where
    the pre-activation is within 1e-5 of the layer's scale."""
    from gantts_b200 import ops, _lib
    torch.manual_seed(21)
    M, dims = 32000, [425, 512, 512, 512]
    h_ref = torch.rand(M, dims[0]) * 0.98 + 0.01
    h_dev = h_ref.to(dev)
    for i, o in zip(dims[:-1], dims[1:]):
        lin = torch.nn.Linear(i, o)
        z_ref = torch.nn.functional.linear(h_ref, lin.weight, lin.bias)
        h_new = ops.linear_act(h_dev, lin.weight.detach().to(dev), lin.bias.detach().to(dev), _lib.ACT_LEAKY_DROPOUT,
                               p=0.0, engine="tc")
        # feed BOTH chains the reference activations so that every layer is judged on identical inputs
        flips = (h_new.cpu() > 0) != (z_ref > 0)
        frac = float(flips.float().mean())
        worst = float(z_ref[flips].abs().max() / z_ref.abs().max()) if flips.any() else 0.0
        assert frac < 1e-4 and worst < 1e-5, (i, o, frac, worst)
        h_ref = torch.nn.functional.leaky_relu(z_ref, 0.01).detach()
        h_dev = h_ref.to(dev)


def test_mlp_stack_weight_gradients_fp32_grade_away_from_the_kink(dev):
    """gW / gb / gx of the fused stack against fp64 at the reference's slope 0.01, with the upstream gradient
    zeroed on the rows that own a pre-activation within 1e-5 of the layer scale (the only elements that can sit on
    different sides of the LeakyReLU kink in two fp32 summation orders, see the count test above): what remains
    must agree to 1e-4 of each gradient's norm -- i.e. the 2e-2 Frobenius allowance of the round-1 tests is
    entirely explained by kink-flipped elements, not by the GEMM arithmetic."""
    from gantts_b200 import ops
    torch.manual_seed(22)
    M, dims = 4096, [425, 512, 512, 187]
    Ws = [torch.randn(o, i) / np.sqrt(i) for i, o in zip(dims[:-1], dims[1:])]
    bs = [torch.randn(o) * 0.1 for o in dims[1:]]
    x, g = torch.rand(M, dims[0]), torch.randn(M, dims[-1])
    Wr = [w.double().requires_grad_(True) for w in Ws]
    br = [b.double().requires_grad_(True) for b in bs]
    xr = x.double().requires_grad_(True)
    h = xr
    near = torch.zeros(M, dtype=torch.bool)
    for W, b in zip(Wr[:-1], br[:-1]):
        z = torch.nn.functional.linear(h, W, b)
        near |= (z.abs() < 1e-5 * z.abs().max()).any(dim=1)
        h = torch.nn.functional.leaky_relu(z, 0.01)
    assert float(near.float().mean()) < 0.2, float(near.float().mean())
    g[near] = 0
    torch.nn.functional.linear(h, Wr[-1], br[-1]).backward(g.double())
    Wd = [w.to(dev).requires_grad_(True) for w in Ws]
    bd = [b.to(dev).requires_grad_(True) for b in bs]
    xd = x.to(dev).requires_grad_(True)
    ops.mlp_stack(xd, Wd, bd, slope=0.01).backward(g.to(dev))
    errs = {}
    for i, (a, b) in enumerate(zip([xd] + Wd + bd, [xr] + Wr + br)):
        a64, b64 = npy(a.grad).astype(np.float64), npy(b.grad)
        errs[i] = float(np.linalg.norm(a64 - b64) / np.linalg.norm(b64))
    assert max(errs.values()) < 1e-4, errs


# ------------------------------------------------------------------------------ recurrent generators
def _sd_numpy(m):
    return {k: v.detach().cpu().numpy() for k, v in m.state_dict().items()}


def _check_weights(model, named, lr_steps, tag):
    for k, v in model.state_dict().items():
        d = np.abs(npy(v) - named[k].detach().numpy())
        assert np.median(d) < 5e-6 and d.max() <= 0.0201 * lr_steps, (tag, k, np.median(d), d.max())


def test_cfg3_rnn_highway_gan_step_vs_oracle(dev):
    """BASELINE cfg3 model: In2OutRNNHighwayNet(177, 177, static 59, 3 x 512 bidirectional LSTM) + MLP D
    (59-256-256-1) on hparams.vc, full widths, reduced batch (B=4, T=300), ragged lengths passed as a host list
    like train.py:503,542.  Inter-layer LSTM dropout off (torch's nn.LSTM cannot take an injected mask); the
    discriminator runs train-mode dropout 0.5 with injected masks.  Losses, outputs, grad norms, post-step weights
    (incl. weight_hh of every layer and direction)."""
    import gantts_b200
    from gantts_b200 import step as gstep, ops
    B, T, p = 4, 300, 0.5
    torch.manual_seed(5)
    mg = gantts_b200.models.In2OutRNNHighwayNet(in_dim=177, out_dim=177, static_dim=59, num_hidden=3, hidden_dim=512,
                                                bidirectional=True, dropout=0.0)
    md = gantts_b200.models.MLP(59, 1, 2, 256, dropout=p, last_sigmoid=True)
    gen = gp.GeneratorOracle("rnn_highway", _sd_numpy(mg), static_dim=59, num_hidden=3, hidden_dim=512,
                             bidirectional=True)
    d_layers = gp.discriminator_layers(_sd_numpy(md))
    d_sum = [torch.zeros_like(t) for pair in d_layers for t in pair]
    mg.to(dev).train(), md.to(dev).train()
    hp = gstep.HParams(windows=WINDOWS, stream_sizes=[177], has_dynamic_features=[True], adversarial_streams=[True],
                       mask_nth_mgc_for_adv_loss=0, discriminator_linguistic_condition=False)
    tr = gstep.GanTrainer(mg, md, hp, w_d=1.0, mse_w=0.0, mge_w=1.0, weight_decay=0.0)
    R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, T))
    lens = ragged_lengths(B, T, 41)
    x, y = make_batch(B, T, 177, 177, lens, 42, uniform_x=False)
    torch.manual_seed(9)
    sr, sf, sa = ops.peek_seeds(3)
    out, yh, ys = tr.step(x.to(dev), y.to(dev), lens, R.to(dev))
    dm = {k: [m.cpu() for m in ops.mlp_dropout_masks(B * T, [256] * 2, p, s, dev)]
          for k, s in (("real", sr), ("fake", sf), ("adv", sa))}
    ref, yh_ref, ys_ref = gp.gan_step(lambda: gen.forward(x, R, lens, VC_HP), gen.params(), gen.sums, d_layers, d_sum,
                                      x, y, lens, R, VC_HP, w_d=1.0, mse_w=0.0, mge_w=1.0, adv_w=1.0, dropout_d=p,
                                      training=True, weight_decay=0.0, d_masks=dm)
    assert torch.equal(yh.cpu(), x)                                                # models.py:118: returns its input
    errs = loss_errors(out, ref, ("loss_d", "loss_fake_d", "loss_real_d", "loss_mge", "loss_adv", "loss_g"))
    errs["y_hat_static"] = rel_err(npy(ys), ys_ref.numpy())
    errs["g_grad_norm"] = abs(float(tr.opt_g.grad_norm()) - ref["g_grad_norm"]) / ref["g_grad_norm"]
    errs["d_grad_norm"] = abs(float(tr.opt_d.grad_norm()) - ref["d_grad_norm"]) / ref["d_grad_norm"]
    assert max(errs.values()) < 2e-4, errs
    _check_weights(mg, gen.named, 1, "cfg3")


def test_cfg5_lstm_gan_step_vs_oracle(dev):
    """BASELINE cfg5 model: LSTMRNN(425 -> 187, 3 x 512 bidirectional) + MLP D (58-256-256-256-1) on
    hparams.tts_acoustic (MLPG over mgc/lf0/bap, adversarial mgc with mask_nth = 2), full widths, B=4 x T=200."""
    import gantts_b200
    from gantts_b200 import step as gstep, ops
    B, T, p = 4, 200, 0.5
    torch.manual_seed(6)
    mg = gantts_b200.models.LSTMRNN(in_dim=425, out_dim=187, num_hidden=3, hidden_dim=512, bidirectional=True,
                                    dropout=0.0, last_sigmoid=False)
    md = gantts_b200.models.MLP(58, 1, 3, 256, dropout=p, last_sigmoid=True)
    gen = gp.GeneratorOracle("lstm", _sd_numpy(mg), num_hidden=3, hidden_dim=512, bidirectional=True)
    d_layers = gp.discriminator_layers(_sd_numpy(md))
    d_sum = [torch.zeros_like(t) for pair in d_layers for t in pair]
    mg.to(dev).train(), md.to(dev).train()
    tr = gstep.GanTrainer(mg, md, gstep.TTS_ACOUSTIC, w_d=1.0, mse_w=0.5, mge_w=1.0)
    R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, T))
    lens = ragged_lengths(B, T, 51)
    x, y = make_batch(B, T, 425, 187, lens, 52)
    torch.manual_seed(10)
    sr, sf, sa = ops.peek_seeds(3)
    out, yh, ys = tr.step(x.to(dev), y.to(dev), lens, R.to(dev))
    dm = {k: [m.cpu() for m in ops.mlp_dropout_masks(B * T, [256] * 3, p, s, dev)]
          for k, s in (("real", sr), ("fake", sf), ("adv", sa))}
    ref, yh_ref, ys_ref = gp.gan_step(lambda: gen.forward(x, R, lens, TTS_HP), gen.params(), gen.sums, d_layers, d_sum,
                                      x, y, lens, R, TTS_HP, w_d=1.0, mse_w=0.5, mge_w=1.0, adv_w=1.0, dropout_d=p,
                                      training=True, d_masks=dm)
    errs = loss_errors(out, ref, ("loss_d", "loss_fake_d", "loss_real_d", "loss_mge", "loss_mse", "loss_adv", "loss_g"))
    errs["y_hat"] = rel_err(npy(yh), yh_ref.numpy())
    errs["y_hat_static"] = rel_err(npy(ys), ys_ref.numpy())
    errs["g_grad_norm"] = abs(float(tr.opt_g.grad_norm()) - ref["g_grad_norm"]) / ref["g_grad_norm"]
    errs["d_grad_norm"] = abs(float(tr.opt_d.grad_norm()) - ref["d_grad_norm"]) / ref["d_grad_norm"]
    assert max(errs.values()) < 2e-4, errs
    _check_weights(mg, gen.named, 1, "cfg5")


STEP_MODEL_CASES = {
    "hw_": ("In2OutHighwayNet", dict(in_dim=27, out_dim=27, static_dim=9, num_hidden=2, hidden_dim=24, dropout=0.0),
            None, True),
    "rhw_": ("In2OutRNNHighwayNet", dict(in_dim=27, out_dim=27, static_dim=9, num_hidden=2, hidden_dim=12,
                                          bidirectional=True, dropout=0.0),
             dict(in_dim=9, out_dim=1, num_hidden=2, hidden_dim=16, dropout=0.0, last_sigmoid=True), True),
    "lstm_": ("LSTMRNN", dict(in_dim=20, out_dim=187, num_hidden=2, hidden_dim=16, bidirectional=True, dropout=0.0,
                              last_sigmoid=False),
              dict(in_dim=58, out_dim=1, num_hidden=3, hidden_dim=16, dropout=0.0, last_sigmoid=True), False),
}
GOLD_KEYS = ("loss_d", "loss_fake_d", "loss_real_d", "loss_mse", "loss_mge", "loss_adv", "loss_g",
             "real_correct", "fake_correct")


@pytest.mark.parametrize("engine", ["simt", "tc"])
@pytest.mark.parametrize("tag", sorted(STEP_MODEL_CASES))
def test_gan_step_non_mlp_generators_golden(dev, golden_step_models, tag, engine):
    """GanTrainer with the reference's non-MLP generators against vectors produced by the UNMODIFIED reference's
    train.py step functions (tests/golden/make_golden.py gen_step_models): two mini-batches, ragged host lengths."""
    import gantts_b200
    from gantts_b200 import step as gstep
    g = golden_step_models
    cls, gkw, dkw, vc = STEP_MODEL_CASES[tag]
    sub = lambda pre: {k[len(pre):]: torch.from_numpy(g[k]) for k in g.files if k.startswith(pre)}
    mg = getattr(gantts_b200.models, cls)(**gkw)
    mg.load_state_dict(sub(tag + "g0_"))
    mg.to(dev).train()
    mg.engine = engine
    md = None
    if dkw is not None:
        md = gantts_b200.models.MLP(**dkw)
        md.load_state_dict(sub(tag + "d0_"))
        md.to(dev).train()
        md.engine = engine
    w_d, mse_w, mge_w = [float(v) for v in g[tag + "cfg"]]
    hp = gstep.HParams(windows=WINDOWS, stream_sizes=[27], has_dynamic_features=[True], adversarial_streams=[True],
                       mask_nth_mgc_for_adv_loss=0, discriminator_linguistic_condition=False) if vc else gstep.TTS_ACOUSTIC
    tr = gstep.GanTrainer(mg, md, hp, w_d=w_d, mse_w=mse_w, mge_w=mge_w)
    R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, 24)).to(dev)
    tol = 2e-5 if engine == "simt" else 1e-4
    for it in range(2):
        p = "%sit%d_" % (tag, it)
        lens = [int(v) for v in g[p + "lengths"]]
        out, y_hat, y_hat_static = tr.step(torch.from_numpy(g[p + "x"]).to(dev), torch.from_numpy(g[p + "y"]).to(dev),
                                           lens, R, adv_w=1.0 if w_d > 0 else 0.0)
        ref = dict(zip(GOLD_KEYS, g[p + "losses"]))
        for k, v in ref.items():
            if np.isnan(v):
                continue
            if k.endswith("correct"):
                assert float(out[k]) == v, (k, float(out[k]), v)
            elif k == "loss_mse" and tag == "rhw_":
                assert abs(float(out[k]) - v) <= 1e-6 * abs(v)          # MSE between the returned input x and y
            else:
                assert abs(float(out[k]) - v) <= tol * max(abs(v), 1e-3), (k, float(out[k]), v)
        assert rel_err(npy(y_hat), g[p + "y_hat"]) < tol
        assert rel_err(npy(y_hat_static), g[p + "y_hat_static"]) < tol
        if engine == "simt":
            for k, v in mg.state_dict().items():
                assert rel_err(npy(v), g[p + "g_" + k]) < 5e-4, (k, rel_err(npy(v), g[p + "g_" + k]))


# ------------------------------------------------------------------------------ fused step: eval / resume
def test_fused_step_eval_phase_and_resume(dev):
    """(a) "test" phase of train.py:481-486: model.eval() -> forwards and losses only, parameters and Adagrad state
    untouched, losses equal the oracle's forward-only step; (b) state_dict()/load_state_dict() in torch.optim.Adagrad
    layout: a resumed FusedGanStep continues bit-identically, and the state loads into torch.optim.Adagrad."""
    import gantts_b200
    from gantts_b200 import step as gstep, fused
    B, T = 4, 60
    lens = [60, 51, 44, 30]

    def build():
        torch.manual_seed(15)
        g = gantts_b200.models.MLP(40, 187, 3, 64, dropout=0.5, last_sigmoid=False)
        d = gantts_b200.models.MLP(58, 1, 3, 32, dropout=0.5, last_sigmoid=True)
        return g, d
    mg, md = build()
    state = gp.GanStepState(layers_of(mg), layers_of(md))
    mg.to(dev), md.to(dev)
    R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, T))
    x, y = make_batch(B, T, 40, 187, lens, 5)
    xd, yd, ld = x.to(dev), y.to(dev), torch.LongTensor(lens).to(dev)
    fs = fused.FusedGanStep(mg, md, gstep.TTS_ACOUSTIC, B, T, mse_w=0.25, seed=11)
    mg.eval(), md.eval()
    before = [p.detach().clone() for p in list(mg.parameters()) + list(md.parameters())]
    fs.step(xd, yd, ld, frames=sum(lens))
    got = fs.loss_dict()
    ref, yh_ref, ys_ref = gp.gan_step_mlp(state, x, y, lens, R, TTS_HP, mse_w=0.25, dropout_g=0.5, dropout_d=0.5,
                                          training=False, update=False)
    errs = loss_errors(got, ref, LOSS_KEYS)
    errs["y_hat_static"] = rel_err(npy(fs.y_hat_static), ys_ref.numpy())
    assert max(errs.values()) < 1e-4, errs
    assert got["real_correct"] == ref["real_correct"] and got["fake_correct"] == ref["fake_correct"]
    assert got["d_grad_norm"] == 0.0 and got["g_grad_norm"] == 0.0
    for a, b in zip(before, list(mg.parameters()) + list(md.parameters())):
        assert torch.equal(a, b)
    assert all(float(s.abs().max()) == 0.0 for s in fs._sums)
    # (b) two training steps, checkpoint after the first
    mg.train(), md.train()
    fs.step(xd, yd, ld, frames=sum(lens))
    sd = fs.state_dict()
    wsnap = [p.detach().clone() for p in list(mg.parameters()) + list(md.parameters())]
    fs.step(xd, yd, ld, frames=sum(lens))
    want = fs.loss_dict()
    wfinal = [p.detach().clone() for p in mg.parameters()]
    g2, d2 = build()
    g2.to(dev).train(), d2.to(dev).train()
    for p, w in zip(list(g2.parameters()) + list(d2.parameters()), wsnap):
        p.data.copy_(w)
    fs2 = fused.FusedGanStep(g2, d2, gstep.TTS_ACOUSTIC, B, T, mse_w=0.25, seed=999)
    fs2.load_state_dict(sd)
    fs2.step(xd, yd, ld, frames=sum(lens))
    assert fs2.loss_dict() == want
    for a, b in zip(wfinal, g2.parameters()):
        assert torch.equal(a, b)
    opt = torch.optim.Adagrad(g2.parameters(), lr=0.01, weight_decay=1e-7)
    opt.load_state_dict(sd["optimizer_g"])
    assert torch.equal(opt.state[next(iter(g2.parameters()))]["sum"].to(dev), sd["optimizer_g"]["state"][0]["sum"])
    with pytest.raises(RuntimeError):
        fs2.step(xd, yd, ld, frames=sum(lens) + 1)
        fs2.loss_dict()


def test_clip_optimizers_vs_torch(dev):
    """ClipAdagrad on a 34-tensor parameter list (4-layer bidirectional LSTM + hidden2out: more than one 32-tensor
    kernel chunk) and ClipAdam (hparams.py:125-130: lr 1e-3, betas (0.5, 0.9)) against clip_grad_norm_ + torch.optim."""
    from gantts_b200 import optim
    for name, kw in (("Adagrad", dict(lr=0.01, weight_decay=1e-7)), ("Adam", dict(lr=1e-3, betas=(0.5, 0.9)))):
        torch.manual_seed(31)
        net = torch.nn.ModuleList([torch.nn.LSTM(12, 16, 4, bidirectional=True), torch.nn.Linear(32, 5)]).to(dev)
        ref = [p.detach().clone().requires_grad_(True) for p in net.parameters()]
        assert len(ref) == 34
        ours = optim.make_optimizer(name, net.parameters(), **kw)
        topt = getattr(torch.optim, name)(ref, **kw)
        for it in range(3):
            ours.zero_grad()
            topt.zero_grad()
            for p, r in zip(net.parameters(), ref):
                g = torch.randn_like(p) * (0.3 if it else 3.0)
                p.grad.copy_(g)
                r.grad = g.clone()
            ours.step()
            norm = torch.nn.utils.clip_grad_norm_(ref, 1.0)
            topt.step()
            assert abs(float(ours.grad_norm()) - float(norm)) <= 2e-6 * float(norm)
            for p, r in zip(net.parameters(), ref):
                assert rel_err(npy(p), npy(r)) < 2e-6
        sd = ours.state_dict()
        topt2 = getattr(torch.optim, name)(ref, **kw)
        topt2.load_state_dict(sd)                     # torch accepts our layout


def test_sru_train_mode_masks_vs_port(dev):
    """SRUCell in train mode with rnn_dropout (variational input mask) and dropout (mask on g(c_t)), k = 3 so the
    highway term is the layer input: upstream masks ONLY the GEMM input, the highway keeps the unmasked x
    (cuda_functional.SRUCell.forward).  Masks regenerated from the seeds the cell drew.  Parity unpinned (the
    upstream package is not vendored): checked against the restatement in oracle/gantts_port.py."""
    from gantts_b200 import rnn, ops
    torch.manual_seed(18)
    B, Tn, d, bidir = 3, 13, 8, True
    n_in = 2 * d
    cell = rnn.SRUCell(n_in, d, dropout=0.3, rnn_dropout=0.25, bidirectional=bidir, use_tanh=0, use_relu=1)
    assert cell.k == 3
    cell.bias.data.uniform_(-0.5, 0.5)
    x = torch.randn(B, Tn, n_in)
    xr = x.clone().requires_grad_(True)
    Wr = cell.weight.detach().clone().requires_grad_(True)
    br = cell.bias.detach().clone().requires_grad_(True)
    cell.to(dev).train()
    torch.manual_seed(44)
    s_x, s_h = ops.peek_seeds(2)
    xg = x.to(dev).requires_grad_(True)
    yg = cell(xg, engine="simt")
    g = torch.randn(B, Tn, 2 * d)
    yg.backward(g.to(dev))
    mask_x = ops.dropout_mask(B, n_in, 0.25, s_x, dev).cpu()
    mask_h = ops.dropout_mask(B, 2 * d, 0.3, s_h, dev).cpu()
    assert 0 < float((mask_x == 0).float().mean()) < 1
    bport = torch.stack([br[:2 * d].view(2, d), br[2 * d:].view(2, d)], 1).reshape(-1)
    yr = gp.sru_layer_forward(xr.transpose(0, 1), Wr, bport, bidirectional=True, use_tanh=False, use_relu=True,
                              mask_x=mask_x, mask_h=mask_h).transpose(0, 1)
    yr.backward(g)
    errs = {"y": rel_err(npy(yg), npy(yr)), "gx": rel_err(npy(xg.grad), npy(xr.grad)),
            "gW": rel_err(npy(cell.weight.grad), npy(Wr.grad)), "gb": rel_err(npy(cell.bias.grad), npy(br.grad))}
    assert max(errs.values()) < 2e-5, errs


# ------------------------------------------------------------------------------ single-output sigmoid stack (discriminator)
@pytest.mark.parametrize("dims,M", [([58, 256, 256, 256, 1], 5000), ([59, 256, 256, 1], 1300), ([58, 32, 32, 32, 1], 700),
                                    ([40, 128, 192, 64, 1], 513), ([40, 64, 1], 70), ([58, 384, 384, 1], 777),
                                    ([58, 256, 520, 1], 300), ([58, 100, 100, 1], 450)])
@pytest.mark.parametrize("slope", [1.0, 0.01])
def test_sigmoid_stack_train_mode_vs_per_layer_fp32(dev, dims, M, slope):
    """The per-layer tensor-core stack with the GEMV + sigmoid tail in TRAIN mode (dropout 0.5) against the exact-fp32
    per-layer engine driven with the same per-layer seeds: output, input gradient and every weight / bias gradient.
    Row counts that are not multiples of the 64-row tile, hidden widths below and between the 64-column chunks, one
    hidden layer, and last hidden widths that select each GEMV kernel (<= 256, <= 512 and wider multiples of 8, and an
    even width that is not a multiple of 8).  slope 1.0 removes the LeakyReLU kink (everything to 1e-4); with the
    reference's slope 0.01 gradients are compared in norm (kink flips)."""
    from gantts_b200 import ops, _lib
    lib = _lib.load()
    torch.manual_seed(41)
    L = len(dims) - 1
    Ws = [(torch.randn(o, i) / np.sqrt(i)).to(dev).requires_grad_(True) for i, o in zip(dims[:-1], dims[1:])]
    bs = [(torch.randn(o) * 0.1).to(dev).requires_grad_(True) for o in dims[1:]]
    x = torch.randn(M, dims[0], device=dev, requires_grad=True)
    g = torch.randn(M, 1, device=dev)
    seed = 24681357
    y = ops.mlp_stack(x, Ws, bs, p=0.5, training=True, seed=seed, slope=slope, last_act=_lib.ACT_SIGMOID)
    y.backward(g)
    got = [npy(y), npy(x.grad)] + [npy(w.grad) for w in Ws] + [npy(b.grad) for b in bs]
    for t in [x] + Ws + bs:
        t.grad = None
    h = x
    for l in range(L - 1):
        h = ops.linear_act(h, Ws[l], bs[l], _lib.ACT_LEAKY_DROPOUT, p=0.5, training=True, engine="simt",
                           seed=lib.gantts_mlp_layer_seed(seed, l), slope=slope)
    y2 = ops.linear_act(h, Ws[-1], bs[-1], _lib.ACT_SIGMOID, engine="simt")
    y2.backward(g)
    ref = [npy(y2), npy(x.grad)] + [npy(w.grad) for w in Ws] + [npy(b.grad) for b in bs]
    names = ["y", "gx"] + ["gW%d" % i for i in range(L)] + ["gb%d" % i for i in range(L)]
    frob = lambda a, b: float(np.linalg.norm(a.astype(np.float64) - b) / max(np.linalg.norm(b), 1e-30))
    if slope == 1.0:
        errs = {n: rel_err(a, b) for n, a, b in zip(names, got, ref)}
        assert max(errs.values()) < 1e-4, errs
    else:
        errs = {n: frob(a, b) for n, a, b in zip(names, got, ref)}
        assert errs["y"] < 1e-4 and max(errs.values()) < 2e-2, errs


def test_mlp_bwd_input_grad_only_and_weight_grads_only(dev):
    """The backward call shapes of the fused step through the C ABI against the full backward: input gradient only
    (adversarial pass), weight gradients only."""
    import ctypes
    from gantts_b200 import ops, _lib
    lib = _lib.load()
    torch.manual_seed(43)
    dims, M = [58, 256, 256, 256, 1], 1024
    Ws = [(torch.randn(o, i) / np.sqrt(i)).to(dev) for i, o in zip(dims[:-1], dims[1:])]
    bs = [(torch.randn(o) * 0.1).to(dev) for o in dims[1:]]
    x = torch.randn(M, 58, device=dev)
    g = torch.randn(M, 1, device=dev)
    Wr = [w.clone().requires_grad_(True) for w in Ws]
    br = [b.clone().requires_grad_(True) for b in bs]
    xr = x.clone().requires_grad_(True)
    ops.mlp_stack(xr, Wr, br, slope=1.0, last_act=_lib.ACT_SIGMOID).backward(g)
    d = _lib.MlpT()
    d.num_layers = 4
    for i, v in enumerate(dims):
        d.dims[i] = v
    for i in range(4):
        d.W[i], d.b[i] = Ws[i].data_ptr(), bs[i].data_ptr()
    d.slope, d.dropout_p, d.last_act, d.seed = 1.0, 0.0, _lib.ACT_SIGMOID, 0
    y = torch.empty(M, 1, device=dev)
    tape = torch.empty(lib.gantts_mlp_tape_bytes(ctypes.byref(d), M), dtype=torch.uint8, device=dev)
    ws = torch.empty(lib.gantts_mlp_workspace_bytes(ctypes.byref(d), M), dtype=torch.uint8, device=dev)
    st = ops._stream()
    _lib.check(lib.gantts_mlp_fwd(ctypes.byref(d), x.data_ptr(), 58, M, y.data_ptr(), 1, tape.data_ptr(), tape.numel(), st))
    gx = torch.zeros(M, 58, device=dev)
    none4 = (ctypes.c_void_p * 4)(None, None, None, None)
    _lib.check(lib.gantts_mlp_bwd(ctypes.byref(d), g.data_ptr(), 1, y.data_ptr(), 1, M, tape.data_ptr(), tape.numel(),
                                  gx.data_ptr(), 58, none4, none4, 0, ws.data_ptr(), ws.numel(), st))
    assert rel_err(npy(gx), npy(xr.grad)) < 2e-5          # input gradient only
    gWs = [torch.empty_like(w) for w in Ws]
    gbs = [torch.empty_like(b) for b in bs]
    arr = lambda ts: (ctypes.c_void_p * 4)(*[t.data_ptr() for t in ts])
    _lib.check(lib.gantts_mlp_bwd(ctypes.byref(d), g.data_ptr(), 1, y.data_ptr(), 1, M, tape.data_ptr(), tape.numel(),
                                  None, 58, arr(gWs), arr(gbs), 0, ws.data_ptr(), ws.numel(), st))
    for a, b in zip(gWs + gbs, Wr + br):
        assert rel_err(npy(a), npy(b.grad)) < 2e-5


# The shape picks the MLPG kernel family: the reference's windows (half bandwidth l + u = 2) take the banded-Cholesky
# substitution kernels, a delta window two frames wide (l + u = 4) the 49-tap FIR kernels.
WIDE_DELTA = (2, 2, np.array([-0.2, -0.1, 0.0, 0.1, 0.2]))
FAMILY_WINDOWS = {"substitution": WINDOWS, "fir": [WINDOWS[0], WIDE_DELTA, WINDOWS[2]]}


@pytest.mark.parametrize("family", ["substitution", "fir"])
@pytest.mark.parametrize("B,Tn", [(3, 257), (2, 31), (1, 1000), (2, 5)])
def test_mlpg_both_kernel_families_vs_dense_R(dev, family, B, Tn):
    """The MLPG forward and backward on the windows of each kernel family against the dense R matmul of the reference
    path (oracle/nnmnkwii_port), TTS stream layout (three dynamic streams + the static vuv column), lengths that do not
    divide the time chunks."""
    from gantts_b200 import multistream, ops
    wins = FAMILY_WINDOWS[family]
    torch.manual_seed(Tn)
    x = torch.randn(B, Tn, 187)
    g = torch.randn(B, Tn, 63)
    R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(wins, Tn))
    xr = x.clone().requires_grad_(True)
    yr = gp.multi_stream_mlpg(xr, R)
    yr.backward(g)
    entries, ncols = multistream.mlpg_stream_entries([180, 3, 1, 3], [True, True, False, True], [True] * 4, len(wins))
    xd = x.to(dev).requires_grad_(True)
    yd = ops.mlpg(xd, [(l, u, tuple(float(v) for v in c)) for l, u, c in wins], entries, ncols)
    yd.backward(g.to(dev))
    assert rel_err(npy(yd), npy(yr)) < 5e-6
    assert rel_err(npy(xd.grad), npy(xr.grad)) < 5e-6
    assert torch.equal(yd[:, :, 61].cpu(), x[:, :, 183])          # static stream copied bit-exactly


DENSE_DELTA = {"substitution": (1, 1, np.array([-0.4, 0.1, 0.5])),
               "fir": (2, 2, np.array([-0.2, -0.1, 0.1, 0.1, 0.2]))}


@pytest.mark.parametrize("family", ["substitution", "fir"])
@pytest.mark.parametrize("case", ["two_windows", "dense_delta"])
def test_mlpg_generic_window_patterns(dev, family, case):
    """Window sets that do NOT have the sparsity pattern the substitution kernels are specialised for (`STD3`): static +
    delta only, and three windows whose delta window has a non-zero centre tap -- the generic path of both kernel families,
    forward and backward, against the dense R matmul."""
    from gantts_b200 import ops
    base = FAMILY_WINDOWS[family]
    if case == "two_windows":
        wins = base[:2]
    else:
        wins = [base[0], DENSE_DELTA[family], base[2]]
    nw, sd, B, Tn = len(wins), 7, 3, 203
    torch.manual_seed(11)
    x = torch.randn(B, Tn, nw * sd + 2)                 # one dynamic stream of 7 static dims + a static stream of 2
    g = torch.randn(B, Tn, sd + 2)
    R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(wins, Tn))
    xr = x.clone().requires_grad_(True)
    yr = gp.multi_stream_mlpg(xr, R, (nw * sd, 2), (True, False), (True, True))
    yr.backward(g)
    entries = [(0, sd, True, 0), (nw * sd, 2, False, sd)]
    xd = x.to(dev).requires_grad_(True)
    yd = ops.mlpg(xd, [(l, u, tuple(float(v) for v in c)) for l, u, c in wins], entries, sd + 2)
    yd.backward(g.to(dev))
    assert rel_err(npy(yd), npy(yr)) < 5e-6
    assert rel_err(npy(xd.grad), npy(xr.grad)) < 5e-6

