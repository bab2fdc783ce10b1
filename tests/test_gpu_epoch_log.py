"""EpochLog (gantts_epoch_log_add) against a restatement of train.py:562-637 fed per batch by FusedGanStep.loss_dict()
and gantts_b200.metrics.compute_distortions: ragged batches of vc, tts_acoustic and tts_duration, train and test phases,
update_g on and off, with and without a reference discriminator."""
import math

import numpy as np
import pytest
import torch

import train_cli_helpers as H

pytestmark = pytest.mark.gpu

HPS = {"vc": H.vc_hp, "tts_acoustic": H.tts_acoustic_hp, "tts_duration": H.tts_duration_hp}
DIMS = {"vc": (12, 12), "tts_acoustic": (20, 187), "tts_duration": (16, 5)}


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__
    __graft_entry__.build()
    return torch.device("cuda:0")


def _setup(name, dev, spoof, seed=0):
    from gantts_b200 import fused, models, train
    hp = HPS[name]()
    d_in, d_out = DIMS[name]
    if name == "vc":
        hp.generator_params.update(in_dim=d_in, out_dim=d_out)
    else:
        train.derive_tts_dims(hp, d_in, d_out)
    torch.manual_seed(seed)
    mg = getattr(models, hp.generator)(**hp.generator_params).to(dev)
    md = getattr(models, hp.discriminator)(**hp.discriminator_params).to(dev)
    ref = None
    if spoof:
        n_adv = len(fused.adversarial_columns(hp))
        ref = models.MLP(n_adv, 1, 2, 8, dropout=0.0, last_sigmoid=True).to(dev).eval()
    fs = fused.FusedGanStep(mg, md, hp, 6, 40, w_d=1.0, optimizer=hp.optimizer_g, optimizer_params=hp.optimizer_g_params,
                            optimizer_d=hp.optimizer_d, optimizer_d_params=hp.optimizer_d_params,
                            reference_discriminator=ref, seed=1)
    rng = np.random.RandomState(seed)
    Ym, Ys = rng.randn(d_out) * 0.3, rng.rand(d_out) + 0.5
    if name == "tts_acoustic":
        Ym[183], Ys[183] = 0.5, 1.0          # V/UV column: normalised 0 is the threshold
    return hp, fs, mg, md, Ym, Ys


def _batches(name, n, seed, unvoiced=False):
    d_in, d_out = DIMS[name]
    rng = np.random.RandomState(seed)
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(n):
        b = 6 if i < n - 1 else 3                                   # a short last batch, like train.py's loader
        lens = sorted((int(v) for v in rng.randint(5, 41, b)), reverse=True)
        t = lens[0]
        x, y = torch.randn(b, t, d_in, generator=g), torch.randn(b, t, d_out, generator=g)
        if name == "tts_acoustic":
            y[:, :, 183] = torch.where(torch.rand(b, t, generator=g) > 0.3, 1.0, -1.0)
            if unvoiced and i == 1:
                y[:, :, 183] = -1.0                                  # no frame voiced in the target
        for k, n_ in enumerate(lens):
            x[k, n_:] = 0
            y[k, n_:] = 0
        out.append((x, y, lens))
    return out


@pytest.mark.parametrize("name", ["vc", "tts_acoustic", "tts_duration"])
@pytest.mark.parametrize("update_g", [True, False])
@pytest.mark.parametrize("spoof", [False, True])
def test_epoch_log_equals_train_py_restatement(dev, name, update_g, spoof):
    from gantts_b200 import metrics, multistream
    from gantts_b200.epochlog import EpochLog
    hp, fs, mg, md, Ym, Ys = _setup(name, dev, spoof)
    log = EpochLog(hp, Ym, Ys, dev)
    for phase in ("train", "test"):
        for m in (mg, md):
            m.train() if phase == "train" else m.eval()
        log.reset()
        host = []
        for x, y, lens in _batches(name, 4, 7 if phase == "train" else 8, unvoiced=True):
            x, y, ld = x.to(dev), y.to(dev), torch.tensor(lens, dtype=torch.int64, device=dev)
            losses = fs.step(x, y, ld, adv_w=0.7, update_g=update_g)
            log.add(losses, y, fs.y_hat_static, ld, True, update_g, fs.spoof_count if spoof else None)
            v = fs.loss_dict()
            ys = multistream.get_static_features(y, len(hp.windows), hp.stream_sizes, hp.has_dynamic_features)
            v["distortions"] = metrics.compute_distortions(ys, fs.y_hat_static, Ym, Ys, ld, hp=hp)
            v["lengths"] = lens
            host.append(v)
        got = log.read(phase, mse_w=0.0, mge_w=1.0)
        want = H.trainpy_phase_log(host, phase, True, update_g, spoof)
        assert list(got) == list(want)
        s = log.sums
        assert s["N"] == len(host) and s["total_num_frames"] == sum(sum(v["lengths"]) for v in host)
        for k in ("real_correct", "fake_correct", "loss_d", "loss_fake_d", "loss_real_d"):
            assert s[k] == sum(v[k] for v in host), k
        if spoof:
            assert s["spoof_count"] == sum(v["spoof_count"] for v in host)
        for k, w in want.items():
            g = got[k]
            if " metric" in k:
                if math.isnan(w):
                    assert math.isnan(g), k
                else:
                    assert abs(g - w) <= 2e-6 * abs(w), (k, g, w)
            else:
                assert g == w, (k, g, w)           # the same fp32 scalars summed in fp64 in batch order
        if name == "tts_acoustic" and update_g:
            assert math.isnan(got["%s f0_rmse metric" % phase])     # batch 1 has no voiced target frame


def test_epoch_log_reads_y_hat_static_with_strides(dev):
    """y_hat_static as a strided view (a slice of a wider buffer) gives the values of its contiguous copy."""
    from gantts_b200.epochlog import EpochLog
    hp = H.tts_acoustic_hp()
    rng = np.random.RandomState(2)
    Ym, Ys = rng.randn(187) * 0.3, rng.rand(187) + 0.5
    Ym[183], Ys[183] = 0.5, 1.0
    x, y, lens = _batches("tts_acoustic", 1, 3)[0]
    y, ld = y.to(dev), torch.tensor(lens, dtype=torch.int64, device=dev)
    wide = torch.randn(y.shape[1], y.shape[0], 70, device=dev)
    yhs = wide.transpose(0, 1)[:, :, 3:66]
    losses = torch.rand(12, device=dev)
    a, b = EpochLog(hp, Ym, Ys, dev), EpochLog(hp, Ym, Ys, dev)
    a.add(losses, y, yhs, ld, True, True)
    b.add(losses, y, yhs.contiguous(), ld, True, True)
    assert a.read("train") == b.read("train")
