"""CPU-only tests of the recurrent discriminator (LSTMRNN / GRURNN) of the fused GAN step:

* the oracle's gan_step with a DiscriminatorOracle pinned to tests/golden/rnn_d.npz (written by
  tests/golden/make_golden_rnn_d.py from the unmodified reference) -- losses, counts, y_hat_static, post-step weights
  of both models, optimiser state;
* the host-only rules of gantts_gan_step_t.d_lstm that gantts_gan_step_workspace_bytes applies, the workspace of a
  zero-filled block, the mask-seed stream and the ctypes binding (placeholder device pointers: only the configuration
  check and the workspace layout run)."""
import ctypes
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, TTS_HP, WINDOWS, rel_err
from fused_step_helpers import _rnn_d_config, config_checker, use_adam

F32_TOL = 1e-6
VC_TOY_HP = dict(stream_sizes=[27], has_dynamic_features=[True], adversarial_streams=[True],
                 mask_nth_mgc_for_adv_loss=0, num_windows=3, discriminator_linguistic_condition=False)


def test_rnn_d_config_rules():
    from gantts_b200 import _lib
    ws, err, rejected = config_checker()
    for kw in (dict(), dict(bidir=0), dict(layers=1), dict(layers=3, cond=True)):
        assert ws(_rnn_d_config(**kw)) > 0, (kw, err())
    c = _rnn_d_config()
    use_adam(c)
    assert ws(c) > 0, err()

    def rej(mutate, needle, **kw):
        rejected(lambda: _rnn_d_config(**kw), mutate, needle)
    rej(lambda c: setattr(c, "B", 65), "2B sequences")
    rej(lambda c: setattr(c, "B", 65), "GanTrainer")
    rej(lambda c: setattr(c.d_lstm, "num_layers", _lib.MAX_LSTM_LAYERS + 1), "discriminator LSTM layer count")
    rej(lambda c: setattr(c.d_lstm, "num_layers", -1), "discriminator LSTM layer count")
    rej(lambda c: setattr(c.d_lstm, "hidden", 18), "not a positive multiple of 4")
    rej(lambda c: setattr(c.d_lstm, "bidirectional", 2), "bidirectional")
    rej(lambda c: setattr(c.d_lstm, "dropout", 1.0), "discriminator LSTM dropout")
    rej(lambda c: setattr(c.d_lstm, "dropout", -0.1), "discriminator LSTM dropout")
    rej(lambda c: setattr(c.d_tensors, "n", c.d_tensors.n - 1), "discriminator table has 17 tensors, its shapes give 18")
    rej(lambda c: setattr(c.d_lstm, "num_layers", 1), "discriminator table has 18 tensors, its shapes give 10")
    rej(lambda c: c.d_tensors.state.__setitem__(5, None), "null discriminator optimiser state of tensor 5")
    rej(lambda c: use_adam(c) or c.d_tensors.state2.__setitem__(17, None), "exp_avg_sq for discriminator tensor 17")
    # d is hidden2out alone: one layer of width ndir * hidden, a single sigmoid output
    rej(lambda c: c.d.dims.__setitem__(0, 16), "hidden2out alone")
    rej(lambda c: setattr(c.d, "num_layers", 2), "hidden2out alone")
    rej(lambda c: c.d.dims.__setitem__(1, 2), "single sigmoid output")
    rej(lambda c: setattr(c.d, "last_act", _lib.ACT_NONE), "single sigmoid output")
    rej(lambda c: setattr(c.d_lstm, "in_dim", 10), "discriminator input width 10 != 0 conditioning + 9")
    rej(lambda c: setattr(c.d_lstm, "in_dim", 9), "discriminator input width 9 != 20 conditioning + 9", cond=True)


def test_zero_filled_d_lstm_keeps_the_workspace():
    """A zero-filled d_lstm block is the MLP discriminator: the workspace is what it was before the field existed (the
    value below is the size the layout gave this configuration then), and a recurrent D only adds to it."""
    ws, err, _ = config_checker()
    c = _rnn_d_config()
    rnn = ws(c)
    ctypes.memset(ctypes.addressof(c.d_lstm), 0, ctypes.sizeof(c.d_lstm))
    c.d.num_layers, c.d.dims[0], c.d.dims[1], c.d.dims[2] = 2, 9, 16, 1
    c.d_tensors.n = 4
    assert ws(c) == 1210112, err()
    assert rnn > ws(c)


def test_d_lstm_mask_seeds_are_a_stream_of_their_own():
    from gantts_b200 import _lib
    lib = _lib.load()
    for seed in (0, 5, 12345, (1 << 61) - 1):
        d_seeds = {lib.gantts_d_lstm_mask_seed(seed, w, l) for w in (1, 2) for l in range(_lib.MAX_LSTM_LAYERS)}
        others = {lib.gantts_gan_step_seed(seed, w) for w in range(4)}
        others |= {lib.gantts_sru_mask_seed(seed, l, w) for l in range(_lib.MAX_SRU_LAYERS) for w in range(2)}
        others |= {lib.gantts_lstm_mask_seed(seed, l) for l in range(_lib.MAX_LSTM_LAYERS)}
        others |= {lib.gantts_mlp_layer_seed(lib.gantts_gan_step_seed(seed, w), l) for w in range(3)
                   for l in range(_lib.MAX_LAYERS)}
        assert len(d_seeds) == 2 * _lib.MAX_LSTM_LAYERS and not d_seeds & others


def test_d_lstm_ctypes_binding():
    from gantts_b200 import _lib
    lib = _lib.load()
    assert _lib.SIGNATURES["gantts_d_lstm_mask_seed"] == (ctypes.c_uint64, [ctypes.c_uint64, ctypes.c_int, ctypes.c_int])
    assert lib.gantts_d_lstm_mask_seed.argtypes == _lib.SIGNATURES["gantts_d_lstm_mask_seed"][1]
    # appended after opt_step: every earlier field keeps its offset
    names = [f for f, _ in _lib.GanStepT._fields_]
    assert names[-2:] == ["opt_step", "d_lstm"] and _lib.GanStepT.d_lstm.offset >= _lib.GanStepT.opt_step.offset + 8


# ---- the oracle's gan_step with a DiscriminatorOracle pinned to tests/golden/rnn_d.npz (tests/golden/make_golden_rnn_d.py:
# the unmodified reference's apply_generator / update_discriminator / update_generator with a recurrent discriminator)
GOLD_KEYS = ("loss_d", "loss_fake_d", "loss_real_d", "loss_mse", "loss_mge", "loss_adv", "loss_g",
             "real_correct", "fake_correct")
GOLD_CASES = {  # tag: (hparams set, D state_dict prefix, bidirectional, conditioned, update_g)
    "lstm_uni": ("tts_acoustic", "lstm", False, False, True),
    "lstm_bi_cond": ("tts_acoustic", "lstm", True, True, True),
    "gru_bi": ("tts_acoustic", "gru", True, False, True),
    "hw_lstm_bi": ("vc", "lstm", True, False, True),
    "lstm_bi_d_only": ("tts_acoustic", "lstm", True, False, False),
}


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN, "rnn_d.npz"))


@pytest.mark.parametrize("case,opt", [(c, o) for c in sorted(GOLD_CASES) for o in ("adagrad", "adam")
                                      if GOLD_CASES[c][4] or o == "adagrad"])
def test_restatement_matches_reference(golden, case, opt):
    """Two mini-batches of the restatement against the reference: the losses and counts of each, then y_hat_static, the
    weights of both models and the discriminator optimiser's state."""
    from oracle import gantts_port as gp
    from oracle import nnmnkwii_port as nnp
    g = golden
    hp_name, prefix, bidir, cond, update_g = GOLD_CASES[case]
    tag = "%s_%s_" % (case, opt)
    sub = lambda pre: {k[len(pre):]: g[k] for k in g.files if k.startswith(pre)}
    hp = dict(VC_TOY_HP if hp_name == "vc" else TTS_HP, discriminator_linguistic_condition=cond)
    kind = "highway" if hp_name == "vc" else "mlp"
    gen = gp.GeneratorOracle(kind, sub(hp_name + "_g0_"), static_dim=9 if kind == "highway" else None)
    d = gp.DiscriminatorOracle(sub(tag + "d0_"))
    assert (d.layers[0].hidden_size, len(d.layers), d.layers[0].bidirectional) == (4, 2, bidir)
    assert list(d.named)[0].startswith(prefix + ".")
    d_sum = [torch.zeros_like(t) for t in d.params()]
    akw = dict(lr=1e-3, betas=(0.5, 0.9), eps=1e-8, weight_decay=0.0)
    g_opt = gp.AdamStepper(gen.params(), **akw) if opt == "adam" else None
    d_opt = gp.AdamStepper(d.params(), **akw) if opt == "adam" else None
    g0 = [q.detach().clone() for q in gen.params()]
    for it in range(2):
        p = "%s_it%d_" % (hp_name, it)
        x, y = torch.from_numpy(g[p + "x"]), torch.from_numpy(g[p + "y"])
        lens = [int(v) for v in g[p + "lengths"]]
        R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, x.size(1)))
        out, _, y_hat_static = gp.gan_step(lambda: gen.forward(x, R, lens, hp, training=True), gen.params(), gen.sums,
                                           d, d_sum, x, y, lens, R, hp, update_g=update_g, d_opt=d_opt, g_opt=g_opt)
        for k, v in zip(GOLD_KEYS, g["%sit%d_losses" % (tag, it)]):
            if np.isnan(v):
                continue
            if k.endswith("correct"):
                assert out[k] == v, (it, k, out[k], v)
            else:
                assert abs(out[k] - v) <= F32_TOL * max(abs(v), 1e-6), (it, k, out[k], v)
    assert rel_err(y_hat_static.numpy(), g[tag + "y_hat_static"]) < F32_TOL
    for pre, named in (("g_", gen.named), ("d_", d.named)):
        gold = sub(tag + pre)
        assert sorted(gold) == sorted(named)
        for k, v in named.items():
            assert rel_err(v.detach().numpy(), gold[k]) < 1e-5, pre + k
    if not update_g:                                     # the D-only steps leave the generator alone
        for a, b in zip(g0, gen.params()):
            assert torch.equal(a, b.detach())
    # the reference's optimiser state is indexed in model.parameters() (= state_dict) order
    for i, name in enumerate(sub(tag + "d0_")):
        key, j = "%sdopt%d_" % (tag, i), list(d.named).index(name)
        if opt == "adam":
            assert float(g[key + "step"]) == d_opt.t == 2
            assert rel_err(d_opt.m[j].numpy(), g[key + "exp_avg"]) < 1e-5, key
            assert rel_err(d_opt.v[j].numpy(), g[key + "exp_avg_sq"]) < 1e-5, key
        else:
            assert rel_err(d_sum[j].numpy(), g[key + "sum"]) < 1e-5, key
