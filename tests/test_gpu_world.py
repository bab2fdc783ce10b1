"""WORLD waveform synthesis on the GPU (gantts_world_*, ops.world_*, Synthesizer(waveform=True), synthesize --waveform)
against the per-utterance numpy restatement oracle.world_port on seeded ragged batches: pulses, counts, y_lengths and
V/UV exact, the noise stream bit for bit, ap and the shifts within 1e-12, y within 1e-10 of max|y|, every row bit-identical
to its B = 1 run, the status word and the rules, and the command end to end."""
import os

import numpy as np
import pytest
import torch

from oracle import world_port as W
import tts_data_helpers as TH

pytestmark = pytest.mark.gpu

NAN = float("nan")
FP = 5.0
Y_TOL = 1e-10       # y against the oracle, relative to max|y|: the FFTs differ from numpy's only in rounding


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__
    __graft_entry__.build()
    return torch.device("cuda:0")


def _f0_track(rng, F, mode):
    t = np.arange(F)
    if mode == "voiced":
        return (120 + 40 * np.sin(t / 13.0) + rng.rand(F)).astype(np.float32)
    if mode == "unvoiced":
        return np.zeros(F, np.float32)
    if mode == "alternating":
        return np.where(t % 2 == 0, 150 + 30 * rng.rand(F), 0.0).astype(np.float32)
    if mode == "jumps":                          # voiced runs of 100-250 Hz with unvoiced gaps and octave jumps
        f = np.where((t // 17) % 3 == 2, 0.0, 100 + 150 * rng.rand(F).round(1))
        f[t % 29 == 5] = 10.0                    # below lowest_f0: unvoiced
        return f.astype(np.float32)
    raise ValueError(mode)


def _envelopes(dev, rng, lens, fs, T):
    """sp from smooth random order-59 mgc through ops.mc2sp, padding NaN; f0 and bap too."""
    from gantts_b200 import generate, ops
    B = len(lens)
    n = generate.cheaptrick_fft_size(fs)
    mc = np.zeros((B, T, 60), np.float32)
    for b, F in enumerate(lens):
        base = rng.randn(60) * np.exp(-0.15 * np.arange(60))
        drift = np.cumsum(rng.randn(F, 60) * 0.02, axis=0) * np.exp(-0.2 * np.arange(60))
        mc[b, :F] = base + drift
    mc[:, :, 0] -= 2.0
    L = torch.tensor(lens, dtype=torch.int64, device=dev)
    sp = ops.mc2sp(torch.from_numpy(mc).to(dev), L, generate.mcep_alpha(fs), n)
    sp_np = sp.cpu().numpy()
    for b, F in enumerate(lens):
        sp_np[b, F:] = NAN
    return torch.from_numpy(sp_np).to(dev), L, n


def _batch(dev, seed, lens, fs, modes):
    from gantts_b200 import ops
    rng = np.random.RandomState(seed)
    T = max(lens) + 3
    sp, L, n = _envelopes(dev, rng, lens, fs, T)
    nb = ops.world_band_count(fs)
    f0 = np.full((len(lens), T), NAN, np.float32)
    bap = np.full((len(lens), T, nb), NAN, np.float32)
    for b, F in enumerate(lens):
        f0[b, :F] = _f0_track(rng, F, modes[b % len(modes)])
        bap[b, :F] = np.where(f0[b, :F, None] > 0, -25 + 8 * rng.randn(F, nb), -0.1 * rng.rand(F, nb))
    return torch.from_numpy(f0).to(dev), sp, torch.from_numpy(bap).to(dev), L, n


CASES = [  # fs, lengths, f0 modes, pulses per response chunk (None: one chunk)
    (16000, [400, 2, 37, 150, 3, 251], ["voiced", "unvoiced", "alternating", "jumps"], None),
    (48000, [120, 2, 61, 5], ["jumps", "voiced", "unvoiced", "alternating"], None),
    (16000, [2 + (b * 173) % 399 for b in range(20)], ["jumps", "voiced", "alternating", "unvoiced", "voiced"], 97),
]


@pytest.mark.parametrize("fs,lens,modes,chunk", CASES)
def test_against_the_oracle(dev, fs, lens, modes, chunk):
    from gantts_b200 import ops
    f0, sp, bap, L, n = _batch(dev, fs + len(lens), lens, fs, modes)
    ap = ops.world_decode_aperiodicity(bap, L, fs, n)
    tb = ops.world_time_base(f0, L, fs, FP, n)
    old = ops.WORLD_CHUNK_BYTES
    if chunk:
        ops.WORLD_CHUNK_BYTES = chunk * 8 * n
    try:
        y, ylen = ops.world_synthesize(f0, sp, ap, L, fs, FP, pulses=tb)
    finally:
        ops.WORLD_CHUNK_BYTES = old
    ap_h, y_h, sp_h = ap.cpu().numpy(), y.cpu().numpy(), sp.cpu().numpy()
    f0_h, bap_h = f0.cpu().numpy(), bap.cpu().numpy()
    idx, sh, vv = tb["index"].cpu().numpy(), tb["shift"].cpu().numpy(), tb["vuv"].cpu().numpy()
    for b, F in enumerate(lens):
        want_ap = W.decode_aperiodicity(bap_h[b, :F], fs, n)
        assert np.max(np.abs(ap_h[b, :F] - want_ap) / want_ap) <= 1e-12, b
        assert not ap_h[b, F:].any()
        want_y, det = W.synthesize(f0_h[b, :F], sp_h[b, :F], want_ap, fs, FP, details=True)
        P = int(tb["counts"][b])
        assert ylen[b] == len(want_y) == W.y_length(F, fs, FP), b
        assert P == len(det["index"]) and np.array_equal(idx[b, :P], det["index"]), b
        assert np.array_equal(vv[b, :P], det["vuv"]), b
        assert np.all(np.abs(sh[b, :P] - det["shift"]) <= 1e-12 * np.abs(det["shift"]) + 1e-300), b
        scale = max(np.max(np.abs(want_y)), 1e-300)
        dev_y = np.max(np.abs(y_h[b, :ylen[b]] - want_y)) / scale
        print("fs %d row %d: max|y - oracle| / max|y| = %.3g" % (fs, b, dev_y))
        assert dev_y <= Y_TOL, (b, dev_y)
        assert not y_h[b, ylen[b]:].any()


def test_noise_stream_is_bit_exact(dev):
    from gantts_b200 import ops
    for count in (1, 255, 256, 257, 3 * 256 * 256 + 17):
        got = ops.world_randn(count, dev).cpu().numpy()
        if count < 5000:
            want = W.Randn().draws(count)
        else:                                   # the tail by jump-ahead in the oracle, the head sequentially
            want = W.Randn().draws(600)
            assert np.array_equal(got[:600].view(np.int64), want.view(np.int64))
            k = count - 300
            r = W.Randn(W.jump(W.SEED, 12 * k))
            want = r.draws(300)
            got = got[k:]
        assert np.array_equal(got.view(np.int64), want.view(np.int64)), count


def test_rows_are_batch_invariant(dev):
    from gantts_b200 import ops
    fs, lens = 16000, [300, 41, 2, 120]
    f0, sp, bap, L, n = _batch(dev, 7, lens, fs, ["jumps", "voiced", "alternating"])
    ap = ops.world_decode_aperiodicity(bap, L, fs, n)
    y, ylen = ops.world_synthesize(f0, sp, ap, L, fs, FP)
    y = y.cpu().numpy()
    ap_h = ap.cpu().numpy()
    for b, F in enumerate(lens):
        one = lambda t: t[b:b + 1, :F].contiguous()
        L1 = torch.tensor([F], dtype=torch.int64, device=dev)
        ap1 = ops.world_decode_aperiodicity(one(bap), L1, fs, n)
        assert np.array_equal(ap1.cpu().numpy()[0].view(np.int64), ap_h[b, :F].view(np.int64)), b
        y1, yl1 = ops.world_synthesize(one(f0), one(sp), ap1, L1, fs, FP)
        assert yl1[0] == ylen[b] and np.array_equal(y1.cpu().numpy()[0].view(np.int64), y[b, :ylen[b]].view(np.int64)), b
    # reversed rows with 50 more padded frames of junk, in chunks of 7 pulses
    Tp = f0.shape[1] + 50
    rev = list(range(len(lens)))[::-1]
    pad = lambda t, v: torch.cat([t[rev], torch.full((len(lens), 50) + tuple(t.shape[2:]), v, dtype=t.dtype,
                                                      device=dev)], 1)
    f0r, spr, apr = pad(f0, 333.0), pad(sp, 7.0), pad(ap, 0.5)
    Lr = L[rev].contiguous()
    old = ops.WORLD_CHUNK_BYTES
    ops.WORLD_CHUNK_BYTES = 7 * 8 * n
    try:
        yr, ylr = ops.world_synthesize(f0r, spr, apr, Lr, fs, FP)
    finally:
        ops.WORLD_CHUNK_BYTES = old
    assert f0r.shape[1] == Tp
    ys, _ = ops.world_synthesize(f0r, spr, apr, Lr, fs, FP, noise=ops.world_randn(int(ylr.max()) + 1000, dev))
    assert np.array_equal(ys.cpu().numpy().view(np.int64), yr.cpu().numpy().view(np.int64))   # a stream made once
    with pytest.raises(RuntimeError, match="noise must be world_randn's contiguous float64 CUDA draws, at least"):
        ops.world_synthesize(f0r, spr, apr, Lr, fs, FP, noise=ops.world_randn(int(ylr.max()) - 1, dev))
    yr = yr.cpu().numpy()
    for j, b in enumerate(rev):
        assert ylr[j] == ylen[b] and np.array_equal(yr[j, :ylen[b]].view(np.int64), y[b, :ylen[b]].view(np.int64)), b


def test_status_word_and_rules(dev):
    from gantts_b200 import ops
    fs = 16000
    f0, sp, bap, L, n = _batch(dev, 3, [30, 20], fs, ["voiced"])
    ap = ops.world_decode_aperiodicity(bap, L, fs, n)
    for bad in (NAN, float("inf")):
        g = f0.clone()
        g[1, 7] = bad
        with pytest.raises(RuntimeError, match="world_time_base: an f0 value within a row's length is not finite"):
            ops.world_synthesize(g, sp, ap, L, fs, FP)
    g = f0.clone()
    g[1, 25] = NAN                              # padding: never read
    ops.world_synthesize(g, sp, ap, L, fs, FP)
    with pytest.raises(RuntimeError, match="a row has fewer than 2 frames"):
        ops.world_synthesize(f0, sp, ap, torch.tensor([30, 1], dtype=torch.int64, device=dev), fs, FP)
    with pytest.raises(RuntimeError, match="nb = 1 coded bands, but WORLD codes 5 at fs = 48000"):
        ops.world_decode_aperiodicity(bap, L, 48000, 2048)
    with pytest.raises(RuntimeError, match="fftlen = 8192 must be a power of two in"):
        ops.world_decode_aperiodicity(bap, L, fs, 8192)
    with pytest.raises(RuntimeError, match="frame_period = -5 ms must be finite and > 0"):
        ops.world_synthesize(f0, sp, ap, L, fs, -5.0)
    with pytest.raises(RuntimeError, match="CUDA tensor required"):
        ops.world_synthesize(f0, sp.cpu(), ap, L, fs, FP)
    torch.cuda.synchronize()


# ---- the synthesizer and the command ----

@pytest.fixture(scope="module")
def data(tmp_path_factory):
    return TH.write_tts_data(str(tmp_path_factory.mktemp("tts") / "data"), n_files=10)


def _checkpoints(tmp_path, dev, data, seed=5):
    from gantts_b200 import generate, models, train
    hp_a, hp_d = TH.srurnn_hps()
    sd, sa = generate.load_stats(TH.duration_hp(), data), generate.load_stats(TH.acoustic_hp(), data)
    generate.derive_dims(hp_a, sa), generate.derive_dims(hp_d, sd)
    torch.manual_seed(seed)
    md = models.SRURNN(**hp_d.generator_params).to(dev)
    ma = models.SRURNN(**hp_a.generator_params).to(dev)
    ck = str(tmp_path / "ck")
    os.makedirs(ck)
    paths = []
    for m, tag in ((ma, "Acoustic"), (md, "Duration")):
        train.save_checkpoint(m, torch.optim.Adagrad(m.parameters()), 1, ck, tag)
        paths.append(os.path.join(ck, "checkpoint_epoch1_%s.pth" % tag))
    return paths


def test_command_writes_the_oracles_waveforms(dev, data, tmp_path):
    from scipy.io import wavfile
    from gantts_b200 import synthesize
    ck_a, ck_d = _checkpoints(tmp_path, dev, data)
    plain, wav = str(tmp_path / "plain"), str(tmp_path / "wav")
    hp = TH.srurnn_hps
    assert synthesize.main(["--batch-size=3", ck_a, ck_d, data, plain], hp_acoustic=hp()[0], hp_duration=hp()[1]) == 0
    assert synthesize.main(["--waveform", "--batch-size=3", ck_a, ck_d, data, wav], hp_acoustic=hp()[0],
                           hp_duration=hp()[1]) == 0
    for sub, names in synthesize.utterance_names(data):
        assert sorted(os.listdir(os.path.join(plain, sub))) == sorted(n + ".npz" for n in names)
        assert sorted(os.listdir(os.path.join(wav, sub))) == sorted([n + ".npz" for n in names] +
                                                                    [n + ".wav" for n in names])
        for n in names:
            a, z = np.load(os.path.join(plain, sub, n + ".npz")), np.load(os.path.join(wav, sub, n + ".npz"))
            assert a.files == z.files
            for k in a.files:
                assert a[k].dtype == z[k].dtype and a[k].tobytes() == z[k].tobytes(), (n, k)
            rate, s = wavfile.read(os.path.join(wav, sub, n + ".wav"))
            assert rate == 16000 and s.dtype == np.int16
            f0 = z["f0"][:, 0].astype(np.float64)
            from gantts_b200 import generate
            fs, fftlen = 16000, generate.cheaptrick_fft_size(16000)
            # the oracle's waveform of the features the command wrote; sp through mc2sp on the device
            from gantts_b200 import ops
            T = len(f0)
            L = torch.tensor([T], dtype=torch.int64, device=dev)
            sp = ops.mc2sp(torch.from_numpy(z["mgc"][None]).to(dev), L, generate.mcep_alpha(fs), fftlen)[0].cpu().numpy()
            ap = W.decode_aperiodicity(z["bap"], fs, fftlen)
            y = W.synthesize(z["f0"][:, 0], sp, ap, fs, FP)
            want = (y / np.max(np.abs(y)) * 32767).astype(np.int16)
            assert len(s) == len(want) == W.y_length(T, fs, FP), n
            assert np.max(np.abs(s.astype(np.int32) - want.astype(np.int32))) <= 1, n


def test_synthesizer_waveform_outputs(dev, data):
    from gantts_b200 import generate, models, synthesize
    hp_a, hp_d = TH.srurnn_hps()
    sd, sa = generate.load_stats(TH.duration_hp(), data), generate.load_stats(TH.acoustic_hp(), data)
    generate.derive_dims(hp_a, sa), generate.derive_dims(hp_d, sd)
    torch.manual_seed(2)
    md = models.SRURNN(**hp_d.generator_params).to(dev)
    ma = models.SRURNN(**hp_a.generator_params).to(dev)
    names = sorted(os.path.splitext(f)[0] for f in os.listdir(os.path.join(data, "X_duration")))
    X = [np.load(os.path.join(data, "X_duration", n + ".npy")) for n in names]
    plain = synthesize.Synthesizer(md, ma, hp_d, hp_a, sd, sa).synthesize_utterances(X, 4)
    both = synthesize.Synthesizer(md, ma, hp_d, hp_a, sd, sa, spectrogram=True, waveform=True)
    got = both.synthesize_utterances(X, 4)
    wave_only = synthesize.Synthesizer(md, ma, hp_d, hp_a, sd, sa, waveform=True).synthesize_utterances(X, 4)
    for p, g, w in zip(plain, got, wave_only):
        assert sorted(g) == sorted(list(p) + ["sp", "waveform"]) and sorted(w) == sorted(list(p) + ["waveform"])
        for k in p:
            assert p[k].tobytes() == g[k].tobytes() == w[k].tobytes(), k
        T = len(p["f0"])
        assert g["waveform"].dtype == np.float64 and len(g["waveform"]) == W.y_length(T, 16000, FP)
        assert g["waveform"].tobytes() == w["waveform"].tobytes()
    out, _ = both.synthesize(torch.from_numpy(X[0][None]).to(dev), torch.tensor([len(X[0])], device=dev))
    assert out["waveform"].dtype == torch.float64 and out["waveform"].is_cuda
