"""Voice conversion on the GPU (gantts_vc_inputs, gantts_mc2b, gantts_mlsa_filter, convert.VoiceConverter and the
convert command) against numpy: the generator inputs bit for bit, the MLSA filter against
oracle.mlsa_port.mlsa_synthesis on seeded ragged harmonic wavs at 16, 22.05 and 48 kHz and orders 24 and 59, every row
bit-identical to its B = 1 run under other padding, the converter end to end against the per-utterance reference chain,
and the command."""
import os

import numpy as np
import pytest
import torch

from conftest import WINDOWS, rel_err
from oracle import gantts_port as gp
from oracle import nnmnkwii_port as nnp
from oracle import mlsa_port
from oracle import sptk_port
from oracle import world_analysis_port as A
from test_gpu_world_analysis import wave

pytestmark = pytest.mark.gpu

FP = 5.0
# |y - y_oracle| / max |y_oracle| per row, on the same x and b.  FILTER_TOL is about 10x the worst seen on an H100
# (8.6e-16): the kernel runs each stage's tap recursion as a warp scan and sums in another order.
FILTER_TOL = 1e-14
GEN_TOL = 2e-4              # test_gpu_generate.py's generation tolerance


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__
    __graft_entry__.build()
    return torch.device("cuda:0")


def _hop(fs):
    return int(fs * (FP * 0.001))


def _min_dio_samples(fs):
    """The fewest samples DIO analyses: FixF0Contour needs more frames than its 7-frame window."""
    from gantts_b200 import ops
    S = 1
    while ops.world_dio_frames(S, fs, FP) <= 7:
        S += 1
    return S


def _coefficients(rng, frames, order, alpha):
    """mc2b of smooth random mel-cepstra with c0 = 0, (frames, order + 1)."""
    base = rng.randn(order + 1) * 0.4 * np.exp(-0.25 * np.arange(order + 1))
    drift = np.cumsum(rng.randn(frames, order + 1) * 0.03, axis=0) * np.exp(-0.25 * np.arange(order + 1))
    mc = base + drift
    mc[:, 0] = 0.0
    return sptk_port.mc2b(mc, alpha)


def _pad(rows, width, value):
    out = np.full((len(rows), width) + rows[0].shape[1:], value)
    for i, r in enumerate(rows):
        out[i, :len(r)] = r
    return out


def _filter(dev, xs, bs, alpha, hop, pad=0.0, S=None, T=None):
    from gantts_b200 import ops
    S = S or max(len(x) for x in xs)
    T = T or max(len(b) for b in bs)
    x = torch.from_numpy(_pad(xs, S, pad)).to(dev)
    b = torch.from_numpy(_pad(bs, T, pad)).to(dev)
    L = torch.tensor([len(v) for v in xs], dtype=torch.int64, device=dev)
    F = torch.tensor([len(v) for v in bs], dtype=torch.int64, device=dev)
    return ops.mlsa_filter(x, L, b, F, alpha, hop).cpu().numpy()


@pytest.mark.parametrize("fs", [16000, 22050, 48000])
@pytest.mark.parametrize("order", [24, 59])
def test_mlsa_filter_against_the_restatement(dev, fs, order):
    from gantts_b200 import generate, ops
    rng = np.random.RandomState(fs + order)
    hop, alpha = _hop(fs), generate.mcep_alpha(fs)
    lengths = [int(0.3 * fs) + 37, _min_dio_samples(fs), int(0.17 * fs), int(0.3 * fs) - hop + 1]
    xs = [wave(rng, fs, 0.35)[0][:n] for n in lengths]
    bs = [_coefficients(rng, ops.world_dio_frames(n, fs, FP), order, alpha) for n in lengths]
    got = _filter(dev, xs, bs, alpha, hop)
    want = mlsa_port.mlsa_synthesis(xs, bs, alpha, hop)
    worst = 0.0
    for r, (x, w) in enumerate(zip(xs, want)):
        assert np.all(got[r, len(x):] == 0)
        worst = max(worst, float(np.max(np.abs(got[r, :len(x)] - w)) / np.max(np.abs(w))))
    print("mlsa_filter fs=%d order=%d: worst |y - oracle| / peak %.3g" % (fs, order, worst))
    assert worst <= FILTER_TOL


def test_mlsa_filter_tail_beyond_the_frames_is_zero(dev):
    """22.05 kHz: hop 110 samples for 110.25 per frame, so from about 20 s on the frames end before the samples."""
    from gantts_b200 import generate, ops
    fs, S = 22050, 50000
    rng = np.random.RandomState(1)
    T = ops.world_dio_frames(S, fs, FP)
    assert T * 110 < S
    alpha = generate.mcep_alpha(fs)
    y = _filter(dev, [rng.randn(S) * 1000], [_coefficients(rng, T, 24, alpha)], alpha, 110)
    assert np.all(y[0, T * 110:] == 0) and np.all(y[0, :T * 110] != 0)


def _vc_inputs(dev, mcs, mean, std, pad=0.0, T=None):
    from gantts_b200 import ops
    T = T or max(len(m) for m in mcs)
    mc = torch.from_numpy(_pad(mcs, T, pad)).to(dev)
    L = torch.tensor([len(m) for m in mcs], dtype=torch.int64, device=dev)
    xin, st = ops.vc_inputs(mc, L, WINDOWS, mean, std)
    return xin.cpu().numpy(), st.cpu().numpy()


def test_vc_inputs_bit_identical_to_numpy(dev):
    rng = np.random.RandomState(2)
    D = 24
    lens = [1, 2, 3, 57, 200]
    mcs = [rng.randn(n, D) * np.exp(-0.1 * np.arange(D)) for n in lens]
    mean, std = rng.randn(3 * D), rng.uniform(0.2, 2.0, 3 * D)
    xin, st = _vc_inputs(dev, mcs, mean, std, pad=np.nan)
    for b, m in enumerate(mcs):
        d = nnp.delta_features(m, WINDOWS).astype(np.float32)      # P.delta_features(mc, hp.windows).astype(float32)
        assert np.array_equal(st[b, :len(m)], d[:, :D])
        assert np.array_equal(xin[b, :len(m)], ((d - mean) / std).astype(np.float32))     # P.scale, normalize_input
        assert np.all(xin[b, len(m):] == 0) and np.all(st[b, len(m):] == 0)            # NaN padding never read


def test_rows_are_bit_identical_at_any_position_and_padding(dev):
    from gantts_b200 import generate, ops
    fs, order = 16000, 24
    rng = np.random.RandomState(3)
    alpha = generate.mcep_alpha(fs)
    lengths = [5000, _min_dio_samples(fs), 3333]
    xs = [wave(rng, fs, 0.4)[0][:n] for n in lengths]
    bs = [_coefficients(rng, ops.world_dio_frames(n, fs, FP), order, alpha) for n in lengths]
    mcs = [rng.randn(len(b), order) for b in bs]
    mean, std = rng.randn(3 * order), rng.uniform(0.5, 2.0, 3 * order)
    full_y = _filter(dev, xs, bs, alpha, 80)
    full_in = _vc_inputs(dev, mcs, mean, std)
    preds = [rng.randn(len(b), order).astype(np.float32) for b in bs]

    def mc2b(ps, ss, pad=0.0, T=None):
        T = T or max(len(p) for p in ps)
        p = torch.from_numpy(_pad(ps, T, pad).astype(np.float32)).to(dev)
        s = torch.from_numpy(_pad(ss, T, pad).astype(np.float32)).to(dev)
        return ops.mc2b(p, s, torch.tensor([len(v) for v in ps], device=dev), alpha).cpu().numpy()

    full_b = mc2b(preds, [m.astype(np.float32) for m in mcs])
    for r in range(3):
        n, F = lengths[r], len(bs[r])
        other = (r + 1) % 3
        for pad, pos in ((np.nan, 0), (1e30, 1)):
            sel = [r] if pos == 0 else [other, r]
            y = _filter(dev, [xs[i] for i in sel], [bs[i] for i in sel], alpha, 80, pad=pad, S=max(lengths) + 501,
                        T=max(len(b) for b in bs) + 9)
            assert np.array_equal(y[pos, :n], full_y[r, :n]), (r, pad)
            Tp = max(len(bs[i]) for i in sel) + 20
            xin, st = _vc_inputs(dev, [mcs[i] for i in sel], mean, std, pad=pad, T=Tp)
            assert np.array_equal(xin[pos, :F], full_in[0][r, :F]) and np.array_equal(st[pos, :F], full_in[1][r, :F])
            b = mc2b([preds[i] for i in sel], [mcs[i].astype(np.float32) for i in sel], pad=pad, T=Tp)
            assert np.array_equal(b[pos, :F], full_b[r, :F])
        # mc2b is the oracle's, operation for operation
        want = sptk_port.mc2b(np.hstack([np.zeros((F, 1)), preds[r].astype(np.float64)
                                         - mcs[r].astype(np.float32).astype(np.float64)]), alpha)
        assert np.array_equal(full_b[r, :F], want)


def _generator(name, order):
    from gantts_b200 import models
    D = 3 * order
    if name == "In2OutHighwayNet":
        return models.In2OutHighwayNet(D, D, order, num_hidden=2, hidden_dim=32, dropout=0.0)
    return models.In2OutRNNHighwayNet(D, D, order, num_hidden=1, hidden_dim=16, bidirectional=True, dropout=0.0)


def _oracle(model, name):
    sd = {k: v.detach().cpu() for k, v in model.state_dict().items()}
    if name == "In2OutHighwayNet":
        return gp.GeneratorOracle("highway", sd, static_dim=model.static_dim)
    return gp.GeneratorOracle("rnn_highway", sd, static_dim=model.static_dim, num_hidden=model.lstm.num_layers,
                              hidden_dim=model.lstm.hidden_size, bidirectional=bool(model.lstm.bidirectional))


@pytest.mark.parametrize("name", ["In2OutHighwayNet", "In2OutRNNHighwayNet"])
def test_voice_converter_against_the_reference_chain(dev, name):
    """test_vc_from_path per utterance on the restatements: WORLD analysis, modspec smoothing of mc[:, 1:], delta,
    scale, the generator, the difference, mc2b and the filter."""
    import train_cli_helpers as H
    from gantts_b200 import analysis, convert, generate, ops
    fs, order = 16000, 24
    torch.manual_seed(5)
    rng = np.random.RandomState(5)
    hp = H.vc_hp(order=order, generator=name)
    model = _generator(name, order)
    stats = {"data_mean": rng.randn(3 * order) * 0.1, "data_std": rng.uniform(0.5, 1.5, 3 * order)}
    conv = convert.VoiceConverter(model.to(dev), hp, stats, fs)
    waves = [wave(rng, fs, s)[0].astype(np.int16) for s in (0.9, 0.6, 0.75)]
    got = conv.convert_utterances(waves, batch_size=3)
    orc, alpha, hop = _oracle(model, name), generate.mcep_alpha(fs), _hop(fs)
    n = sptk_port.cheaptrick_fft_size(fs)
    stream = A.randn_stream(400 * (2 * n + 2))
    worst = 0.0
    for i, w in enumerate(waves):
        x = w.astype(np.float64)
        f0, t = A.dio(x, fs, FP)
        sp = A.cheaptrick(x, A.stonemask(x, f0, t, fs), t, fs, n, stream)
        mc = A.sp2mc(sp, order, alpha)
        src = A.modspec_smoothing(mc, analysis.modulation_rate(fs, FP))[:, 1:]
        d = nnp.delta_features(src, WINDOWS).astype(np.float32)
        xin = ((d - stats["data_mean"]) / stats["data_std"]).astype(np.float32)
        R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, len(d)))
        with torch.no_grad():
            _, y_static = orc.forward(torch.from_numpy(xin)[None], R, [len(d)], {})
        mc_want = y_static[0].numpy().astype(np.float64) * stats["data_std"][:order] + stats["data_mean"][:order]
        assert got[i]["mc"].shape == mc_want.shape and len(got[i]["waveform"]) == len(w)
        assert rel_err(got[i]["mc"], mc_want) <= GEN_TOL, (i, rel_err(got[i]["mc"], mc_want))
        # the waveform: the restated diff, mc2b and filter on the device's converted mc and source statics
        xt, L = analysis.pad_waves([x], dev)
        s_dev, _, frames = conv.analyse(xt, L)
        static = ops.vc_inputs(s_dev, frames, WINDOWS, conv.mean, conv.std)[1][0].cpu().numpy()
        assert np.max(np.abs(static - d[:, :order])) <= 1e-6 * np.max(np.abs(d[:, :order]))
        b = sptk_port.mc2b(np.hstack([np.zeros((len(d), 1)), got[i]["mc"].astype(np.float64) - static]), alpha)
        y = mlsa_port.mlsa_synthesis([x], [b], alpha, hop)[0]
        worst = max(worst, float(np.max(np.abs(got[i]["waveform"] - y)) / np.max(np.abs(y))))
        alone = conv.convert_utterances([w], batch_size=1)[0]
        assert np.array_equal(alone["waveform"], got[i]["waveform"]) and np.array_equal(alone["mc"], got[i]["mc"])
    print("VoiceConverter %s: worst waveform |y - chain| / peak %.3g" % (name, worst))
    assert worst <= FILTER_TOL


def test_converter_names_the_utterance_analysis_refuses(dev):
    import train_cli_helpers as H
    from gantts_b200 import convert
    rng = np.random.RandomState(6)
    conv = convert.VoiceConverter(_generator("In2OutHighwayNet", 4).to(dev), H.vc_hp(), {
        "data_mean": np.zeros(12), "data_std": np.ones(12)}, 16000)
    good = wave(rng, 16000, 0.5)[0]
    with pytest.raises(RuntimeError, match="utterance b.wav: .*too short for DIO"):
        conv.convert_utterances([good, good[:300]], 2, names=["a.wav", "b.wav"])
    bad = good.copy()
    bad[77] = np.inf
    with pytest.raises(RuntimeError, match="utterance 1: .*not finite"):
        conv.convert_utterances([good, bad], 2)


def test_command_end_to_end(dev, tmp_path):
    from scipy.io import wavfile
    from gantts_b200 import convert, models, train
    import train_cli_helpers as H
    root = str(tmp_path / "data")
    xd, yd = H.write_vc_data(root, n_files=12)
    hp = H.vc_hp()
    train.load_data(hp, xd, yd, -1)                   # writes data_mean.npy / data_var.npy
    torch.manual_seed(7)
    model = getattr(models, hp.generator)(**hp.generator_params)
    ck = str(tmp_path / "ck")
    os.makedirs(ck)
    train.save_checkpoint(model, torch.optim.Adagrad(model.parameters()), 3, ck, "Generator")
    ckpt = os.path.join(ck, "checkpoint_epoch3_Generator.pth")
    wd = str(tmp_path / "wavs")
    os.makedirs(wd)
    rng = np.random.RandomState(8)
    waves = {}
    for f in sorted(os.listdir(xd)):
        name = os.path.splitext(f)[0]
        waves[name] = wave(rng, 16000, rng.uniform(0.4, 0.9))[0].astype(np.int16)
        wavfile.write(os.path.join(wd, name + ".wav"), 16000, waves[name])
    out = str(tmp_path / "out")
    with pytest.raises(SystemExit, match="--diffvc is required"):
        convert.main([ckpt, root, wd, out], hp=H.vc_hp())
    assert convert.main(["--diffvc", "--batch-size=4", ckpt, root, wd, out], hp=H.vc_hp()) == 0
    stats = {"data_mean": np.load(os.path.join(root, "data_mean.npy")),
             "data_std": np.sqrt(np.load(os.path.join(root, "data_var.npy")))}
    hp2 = H.vc_hp()
    hp2.generator_params["in_dim"] = hp2.generator_params["out_dim"] = 12
    model_g = getattr(models, hp2.generator)(**hp2.generator_params)
    train.load_checkpoint(model_g, ckpt)
    conv = convert.VoiceConverter(model_g.to(dev), hp2, stats, 16000)
    for sub, files in convert.wav_files(root, wd):
        names = [os.path.splitext(os.path.basename(p))[0] for p in files]
        assert sorted(os.listdir(os.path.join(out, sub))) == sorted(nm + ".wav" for nm in names)
        want = conv.convert_utterances([waves[nm] for nm in names], 2)
        for nm, r in zip(names, want):
            rate, data = wavfile.read(os.path.join(out, sub, nm + ".wav"))
            assert rate == 16000 and data.dtype == np.int16 and len(data) == len(waves[nm])
            assert np.array_equal(data, r["waveform"].astype(np.int16))
