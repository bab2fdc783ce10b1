"""CPU-only tests of the spoofing-rate count with a recurrent reference discriminator (LSTMRNN / GRURNN):

* the oracle's spoof_count on a DiscriminatorOracle pinned to tests/golden/spoof_rnn.npz (written by
  tests/golden/make_golden_spoof_rnn.py from the UNMODIFIED reference's spoof block, train.py:549-558) -- the generator
  output it counts on, the reference discriminator's output and the count, exactly;
* the host-only configuration rules of gantts_spoof_count_lstm_workspace_bytes / gantts_spoof_count_lstm through the C ABI
  (placeholder device pointers: the checks run before anything touches the device);
* the Python-side rules of check_reference_discriminator (CPU modules: nothing runs).
"""
import ctypes
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, TTS_HP, WINDOWS, rel_err
from fused_step_helpers import FAKE, config_checker
from oracle import gantts_port as gp
from oracle import nnmnkwii_port as nnp

VC_TOY_HP = dict(stream_sizes=[27], has_dynamic_features=[True], adversarial_streams=[True],
                 mask_nth_mgc_for_adv_loss=0, num_windows=3, discriminator_linguistic_condition=False)
CASES = {"vc": VC_TOY_HP, "tts": TTS_HP}


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN, "spoof_rnn.npz"))


def sub(g, pre):
    return {k[len(pre):]: g[k] for k in g.files if k.startswith(pre)}


@pytest.mark.parametrize("ref_cls", ["lstmrnn", "grurnn"])
@pytest.mark.parametrize("case", ["vc", "tts"])
def test_spoof_count_rnn_matches_reference(golden, case, ref_cls):
    """Over a D-only step and then a full step, the restatement's generator output, reference discriminator output and
    count equal the reference's; the count is exact (it is an integer)."""
    g, hp, tag = golden, CASES[case], "%s_%s_" % (case, ref_cls)
    gen = gp.GeneratorOracle("mlp", sub(g, tag + "g0_"))
    ref_d = gp.DiscriminatorOracle(sub(g, tag + "ref_"))
    assert list(ref_d.named)[0].startswith("lstm." if ref_cls == "lstmrnn" else "gru.")
    for it in range(2):
        p = "%sit%d_" % (tag, it)
        x = torch.from_numpy(g[p + "x"])
        lens = [int(v) for v in g[p + "lengths"]]
        R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, x.size(1)))
        with torch.no_grad():       # neither step changes the generator before it is applied
            _, y_hat_static = gen.forward(x, R, lens, hp, training=True)
        assert rel_err(y_hat_static.numpy(), g[p + "y_hat_static"]) < 1e-6, (it, "y_hat_static")
        ys = torch.from_numpy(g[p + "y_hat_static"])
        target = gp.reference_output(ref_d, ys, lens, hp)
        assert rel_err(target.numpy(), g[p + "target"]) < 1e-6, (it, "target")
        mask = gp.sequence_mask(lens, x.size(1)).unsqueeze(-1)
        want = float(g[p + "spoof"])
        assert gp.spoof_count(ref_d, ys, lens, mask, hp) == want, it
        assert gp.spoof_count(ref_d, y_hat_static, lens, mask, hp) == want, it
        if it == 0:
            assert 0 < want < sum(lens)                    # the reference D's outputs straddle 0.5


def _stack(layers=2, in_dim=9, hidden=8, bidir=1):
    from gantts_b200 import _lib
    s = _lib.LstmStackT()
    s.num_layers, s.in_dim, s.hidden, s.bidirectional, s.dropout = layers, in_dim, hidden, bidir, 0.5
    return s


def _head(n_in=16, n_out=1, layers=1, sigmoid=True):
    from gantts_b200 import _lib
    d = _lib.MlpT()
    d.num_layers = layers
    d.dims[0] = n_in
    for l in range(layers):
        d.dims[l + 1] = n_out if l == layers - 1 else n_in
        d.W[l] = d.b[l] = FAKE
    d.last_act = _lib.ACT_SIGMOID if sigmoid else _lib.ACT_NONE
    return d


def test_spoof_count_lstm_configuration_rules():
    """gantts_spoof_count_lstm_workspace_bytes / gantts_spoof_count_lstm (host-only) refuse, with a message naming the
    rule: null pointers, a layer count outside [1, 3], a hidden size that is not a multiple of 4, bidirectional not 0 / 1,
    B above LSTM_MAX_B, B * T >= 2^24, a tensor count other than 4 ndir layers, an input width other than n_adv (no
    linguistic conditioning, train.py:554-555), a head that is not one sigmoid layer ndir H -> 1, a small workspace."""
    from gantts_b200 import _lib
    _, err, _ = config_checker()
    lib = _lib.load()

    def wsb(s=None, h=None, B=2, T=16, null_s=False, null_h=False):
        s = None if null_s else ctypes.byref(s or _stack())
        h = None if null_h else ctypes.byref(h or _head())
        return lib.gantts_spoof_count_lstm_workspace_bytes(s, h, B, T)
    assert wsb() > 0, err()
    assert wsb(_stack(layers=3, bidir=0, hidden=4), _head(n_in=4), B=128, T=1000) > 0, err()
    assert wsb(null_s=True) == 0 and "null reference discriminator" in err()
    assert wsb(null_h=True) == 0 and "null reference discriminator" in err()
    for n in (0, 4):
        assert wsb(_stack(layers=n)) == 0 and "layer count %d not in [1, 3]" % n in err(), err()
    assert wsb(_stack(hidden=6), _head(n_in=12)) == 0 and "not a positive multiple of 4" in err(), err()
    assert wsb(_stack(bidir=2)) == 0 and "bidirectional 2" in err(), err()
    assert wsb(B=129) == 0 and "LSTM_MAX_B = 128" in err(), err()
    assert wsb(B=128, T=1 << 17) == 0 and "2^24" in err(), err()
    for h in (_head(n_in=8), _head(n_out=2), _head(layers=2), _head(sigmoid=False)):
        assert wsb(h=h) == 0 and "hidden2out alone, 1 layer of 16 -> 1 with a sigmoid" in err(), err()
    # a larger workspace than the call's shape needs is accepted: a step's (B, T) holds every (b, t) it is called with
    assert wsb(B=2, T=16) < wsb(B=4, T=16) and wsb(B=2, T=15) < wsb(B=2, T=16)

    cols = (ctypes.c_int * 9)(*range(9))
    tensors = (ctypes.c_void_p * 16)(*([FAKE] * 16))

    def count(s=None, n_tensors=16, h=None, n_adv=9, ts=tensors, ys=FAKE, ad=cols, ln=FAKE, out=FAKE, wsp=FAKE,
              ws_bytes=1 << 40):
        return lib.gantts_spoof_count_lstm(ctypes.byref(s or _stack()), ts, n_tensors, ctypes.byref(h or _head()), ys, 12,
                                           ad, n_adv, ln, 2, 16, out, wsp, ws_bytes, FAKE)
    assert count(n_tensors=8) == 1 and "8 LSTM tensors, the stack has 16" in err(), err()
    assert count(_stack(bidir=0), h=_head(n_in=8)) == 1 and "16 LSTM tensors, the stack has 8" in err(), err()
    assert count(n_adv=8) == 1 and "8 adversarial columns != reference discriminator input width 9" in err(), err()
    assert count(_stack(in_dim=9 + 27)) == 1 and "linguistic conditioning, train.py:554-555" in err(), err()
    for kw in (dict(ts=None), dict(ys=None), dict(ad=None), dict(ln=None), dict(out=None)):
        assert count(**kw) == 1 and "null pointer" in err(), (kw, err())
    holed = (ctypes.c_void_p * 16)(*([FAKE] * 15 + [None]))
    assert count(ts=holed) == 1 and "null pointer (LSTM tensor 15)" in err(), err()
    h = _head()
    h.W[0] = None
    assert count(h=h) == 1 and "null pointer" in err(), err()
    bad = (ctypes.c_int * 9)(*range(4, 13))
    assert count(ad=bad) == 1 and "out of range" in err(), err()
    need = wsb()
    assert count(ws_bytes=need - 1) == 4 and "workspace too small" in err(), err()
    assert count(wsp=None) == 4 and "workspace too small" in err(), err()


def test_check_reference_discriminator_accepts_recurrent_ones():
    """LSTMRNN and GRURNN reference discriminators with a sigmoid output over the n_adv adversarial columns pass the check
    of both paths; a conditioned one is refused citing train.py:549-555, one without a sigmoid output and one the fused
    step has no kernel for (more than 3 layers) are refused."""
    import gantts_b200
    from gantts_b200.fused import check_reference_discriminator as check
    M = gantts_b200.models
    for cls in (M.LSTMRNN, M.GRURNN):
        for who in ("FusedGanStep", "GanTrainer"):
            check(cls(9, 1, 2, 8, bidirectional=True, dropout=0.5, last_sigmoid=True), 9, who)
            with pytest.raises(RuntimeError, match="train.py:549-555"):
                check(cls(9 + 27, 1, 2, 8, bidirectional=True, last_sigmoid=True), 9, who)
            with pytest.raises(RuntimeError, match="sigmoid output"):
                check(cls(9, 1, 2, 8, last_sigmoid=False), 9, who)
            with pytest.raises(RuntimeError, match="4 layers"):
                check(cls(9, 1, 4, 8, last_sigmoid=True), 9, who)
    check(M.MLP(9, 1, 2, 16, last_sigmoid=True), 9, "GanTrainer")          # the MLP branch is unchanged
    with pytest.raises(RuntimeError, match="train.py:549-555"):
        check(M.MLP(36, 1, 2, 16, last_sigmoid=True), 9, "GanTrainer")
