"""CPU-only tests of the discriminator warm-up step (update_g = False) and of the spoofing-rate count:

* the oracle's gan_step(update_g=False) and spoof_count pinned to tests/golden/dwarmup.npz (written by
  tests/golden/make_golden_dwarmup.py), the vectors of the UNMODIFIED
  reference's apply_generator + update_discriminator (train.py:336-355, 245-279; update_generator not called, :696) and
  of its spoofing-rate block (train.py:549-558) -- losses, counts, post-step discriminator weights and optimiser state,
  unchanged generator weights, spoof counts;
* the host-only configuration rules of GANTTS_STEP_D_ONLY and of gantts_spoof_count through the C ABI (placeholder
  device pointers: the checks run before anything touches the device).
"""
import ctypes
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, TTS_HP, WINDOWS, rel_err
from fused_step_helpers import FAKE, config_checker, fill_tables, step_config
from oracle import gantts_port as gp
from oracle import nnmnkwii_port as nnp

F32_TOL = 1e-6
VC_TOY_HP = dict(stream_sizes=[27], has_dynamic_features=[True], adversarial_streams=[True],
                 mask_nth_mgc_for_adv_loss=0, num_windows=3, discriminator_linguistic_condition=False)
CASES = {"vc": VC_TOY_HP, "tts": TTS_HP}
LOSS_KEYS = ("loss_d", "loss_fake_d", "loss_real_d", "real_correct", "fake_correct")


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN, "dwarmup.npz"))


def sub(g, pre):
    return {k[len(pre):]: g[k] for k in g.files if k.startswith(pre)}


@pytest.mark.parametrize("opt", ["adagrad", "adam"])
@pytest.mark.parametrize("case", ["vc", "tts"])
def test_d_only_step_and_spoof_count_match_reference(golden, case, opt):
    g, hp, tag = golden, CASES[case], "%s_%s_" % (case, opt)
    gen = gp.GeneratorOracle("mlp", sub(g, tag + "g0_"))
    d_layers = gp.discriminator_layers(sub(g, tag + "d0_"))
    d_params = [t for pair in d_layers for t in pair]
    d_sum = [torch.zeros_like(t) for t in d_params]
    d_opt = gp.AdamStepper(d_params, lr=1e-3, betas=(0.5, 0.9), eps=1e-8, weight_decay=0.0) if opt == "adam" else None
    ref_d = gp.DiscriminatorOracle(sub(g, tag + "ref_"))
    g0 = [p.detach().clone() for p in gen.params()]
    for it in range(2):
        p = "%sit%d_" % (tag, it)
        x, y = torch.from_numpy(g[p + "x"]), torch.from_numpy(g[p + "y"])
        lens = [int(v) for v in g[p + "lengths"]]
        R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, x.size(1)))
        out, y_hat, y_hat_static = gp.gan_step(lambda: gen.forward(x, R, lens, hp, training=True), gen.params(), None,
                                               d_layers, d_sum, x, y, lens, R, hp, update_g=False, d_opt=d_opt)
        assert rel_err(y_hat.numpy(), g[p + "y_hat"]) < F32_TOL
        assert rel_err(y_hat_static.numpy(), g[p + "y_hat_static"]) < F32_TOL
        for k, v in zip(LOSS_KEYS, g[p + "losses"]):
            if k.endswith("correct"):
                assert out[k] == v, (it, k, out[k], v)
            else:
                assert abs(out[k] - v) <= F32_TOL * abs(v), (it, k, out[k], v)
        assert out["loss_adv"] == 0.0 and out["g_grad_norm"] == 0.0
        assert out["loss_g"] == pytest.approx(out["loss_mge"], rel=1e-7)          # mse_w = 0, mge_w = 1
        mask = gp.sequence_mask(lens, x.size(1)).unsqueeze(-1)
        assert gp.spoof_count(ref_d, y_hat_static, lens, mask, hp) == float(g[p + "spoof"])
        gold_d = sub(g, p + "d_")
        names = ["layers.%d" % i for i in range(len(d_layers) - 1)] + ["last_linear"]
        for n, (W, b) in zip(names, d_layers):
            assert rel_err(W.detach().numpy(), gold_d[n + ".weight"]) < 1e-5, (it, n)
            assert rel_err(b.detach().numpy(), gold_d[n + ".bias"]) < 1e-5, (it, n)
        for i in range(len(d_params)):
            if opt == "adam":
                assert float(g["%sdopt%d_step" % (p, i)]) == d_opt.t == it + 1
                assert rel_err(d_opt.m[i].numpy(), g["%sdopt%d_exp_avg" % (p, i)]) < 1e-5
                assert rel_err(d_opt.v[i].numpy(), g["%sdopt%d_exp_avg_sq" % (p, i)]) < 1e-5
            else:
                assert rel_err(d_sum[i].numpy(), g["%sdopt%d_sum" % (p, i)]) < 1e-5
        # the generator is never stepped, in the reference and in the restatement
        gold_g = sub(g, p + "g_")
        for k, v in sub(g, tag + "g0_").items():
            assert np.array_equal(gold_g[k], v), (it, k)
        for a, b in zip(g0, gen.params()):
            assert torch.equal(a, b.detach())


def _mlp_step_config():
    """A valid plain-MLP configuration of gantts_gan_step_t (VC toy layout: one dynamic stream of 9 x 3 columns)."""
    c = step_config((27, 16, 27), (9, 8, 1), [(0, 9, True, 0)], range(9), range(9))
    return fill_tables(c, 4)


def _gan_step(lib, c, phases):
    return lib.gantts_gan_step(ctypes.byref(c), phases, FAKE, FAKE, FAKE, 0.0, 1, FAKE, FAKE, FAKE, FAKE, 1 << 40, FAKE)


def test_d_only_phase_rules():
    """GANTTS_STEP_D_ONLY is refused, with a message naming the rule, without a discriminator (w_d = 0) and together
    with GANTTS_STEP_EVAL."""
    from gantts_b200 import _lib
    ws, err, _ = config_checker()
    lib = _lib.load()
    c = _mlp_step_config()
    assert ws(c) > 0, err()
    c.w_d, c.d_tensors.n = 0.0, 0
    assert ws(c) > 0, err()                                  # a valid configuration without a discriminator ...
    for phases in (7 | _lib.STEP_D_ONLY, 1 | _lib.STEP_D_ONLY):
        assert _gan_step(lib, c, phases) == 1
        assert "GANTTS_STEP_D_ONLY trains the discriminator and needs w_d > 0" in err(), err()
    c = _mlp_step_config()
    assert _gan_step(lib, c, _lib.STEP_EVAL | _lib.STEP_D_ONLY) == 1
    assert "GANTTS_STEP_D_ONLY cannot be combined with GANTTS_STEP_EVAL" in err(), err()


def _ref_desc(dims=(9, 8, 8, 1), sigmoid=True):
    from gantts_b200 import _lib
    d = _lib.MlpT()
    d.num_layers = len(dims) - 1
    for i, v in enumerate(dims):
        d.dims[i] = v
    for l in range(d.num_layers):
        d.W[l] = d.b[l] = FAKE
    d.last_act = _lib.ACT_SIGMOID if sigmoid else _lib.ACT_NONE
    return d


def test_spoof_count_configuration_rules():
    """gantts_spoof_count_workspace_bytes / gantts_spoof_count (host-only): a sigmoid single-output reference
    discriminator over exactly the n_adv adversarial columns (no linguistic conditioning, train.py:554-555), B * T below
    2^24, no null pointer."""
    from gantts_b200 import _lib
    _, err, _ = config_checker()
    lib = _lib.load()
    wsb = lambda d, rows: lib.gantts_spoof_count_workspace_bytes(ctypes.byref(d) if d is not None else None, rows)
    assert wsb(_ref_desc(), 2 * 16) > 0, err()
    assert wsb(_ref_desc(sigmoid=False), 32) == 0 and "single sigmoid output" in err()
    assert wsb(_ref_desc(dims=(9, 8, 2)), 32) == 0 and "single sigmoid output" in err()
    assert wsb(None, 32) == 0 and "null reference discriminator" in err()
    assert wsb(_ref_desc(), 1 << 24) == 0 and "2^24" in err()
    cols = (ctypes.c_int * 9)(*range(9))

    def count(d, n_adv, ys=FAKE, ad=cols, ln=FAKE, out=FAKE):
        return lib.gantts_spoof_count(ctypes.byref(d), ys, 12, ad, n_adv, ln, 2, 16, out, FAKE, 1 << 40, FAKE)
    assert count(_ref_desc(), 8) == 1 and "8 adversarial columns != reference discriminator input width 9" in err(), err()
    assert count(_ref_desc(dims=(9 + 27, 8, 1)), 9) == 1 and "linguistic conditioning" in err(), err()
    assert count(_ref_desc(sigmoid=False), 9) == 1 and "single sigmoid output" in err()
    for kw in (dict(ys=None), dict(ad=None), dict(ln=None), dict(out=None)):
        assert count(_ref_desc(), 9, **kw) == 1 and "null pointer" in err(), (kw, err())
    bad = (ctypes.c_int * 9)(*range(4, 13))
    assert count(_ref_desc(), 9, ad=bad) == 1 and "out of range" in err(), err()
