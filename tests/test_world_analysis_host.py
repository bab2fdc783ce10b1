"""The numpy restatement of WORLD analysis, sp2mc and modulation-spectrum smoothing (oracle.world_analysis_port), pinned
by properties that need neither pyworld, pysptk nor nnmnkwii; the sp2mc operator of gantts_mcep_operator against it; and
the rules of the objective's --wav-dir option that are checked before any device work."""
import os

import numpy as np
import pytest

from oracle import sptk_port
from oracle import world_analysis_port as A
from oracle import world_port as W

FP = 5.0


def harmonic(fs, f0_frames, rng, fp=FP):
    """A seven-harmonic signal whose f0 is f0_frames[j] over frame j's hop (silent where 0), plus a little noise."""
    hop = int(fs * fp / 1000)
    f = np.repeat(np.asarray(f0_frames, np.float64), hop)
    ph = np.cumsum(2 * np.pi * f / fs)
    x = sum(np.where(f > 0, np.cos(k * ph) / k, 0.0) for k in range(1, 8))
    return 3000.0 * x + rng.randn(len(f))


@pytest.mark.parametrize("fs", [16000, 48000])
def test_dio_and_stonemask_recover_a_known_f0(fs):
    rng = np.random.RandomState(fs)
    F = 320
    f0 = np.zeros(F)
    f0[20:120] = np.linspace(80, 120, 100)
    f0[150:230] = np.linspace(250, 400, 80)
    f0[250:300] = 180.0
    x = harmonic(fs, f0, rng)
    got, t = A.dio(x, fs, FP)
    assert len(got) == A.dio_frames(len(x), fs, FP) and np.array_equal(t, np.arange(len(got)) * FP / 1000.0)
    refined = A.stonemask(x, got, t, fs)
    # away from the voicing edges (a window of 10 frames) every frame is voiced, within 1 % of the true f0 (the signal's f0
    # changes in steps of one hop, the frame sits at the step)
    for a, b in ((20, 120), (150, 230), (250, 300)):
        inner = slice(a + 10, b - 10)
        assert np.all(np.abs(got[inner] / f0[inner] - 1) < 0.01)
        assert np.all(np.abs(refined[inner] / f0[inner] - 1) < 0.01)
    for a, b in ((0, 10), (130, 140), (310, len(got))):
        assert np.all(got[a:b] == 0) and np.all(refined[a:b] == 0)


def test_dio_refuses_rows_too_short():
    assert A.voice_range_minimum(FP) == 7
    with pytest.raises(ValueError, match="more than 7 frames"):
        A.dio(np.ones(400), 16000, FP)             # int(1000 * 400 / 16000 / 5) + 1 = 6 frames
    f0, _ = A.dio(np.random.RandomState(0).randn(700), 16000, FP)
    assert len(f0) == 9


def test_dio_frame_count_is_getsamplesfordio():
    for L, fs in ((16000, 16000), (16079, 16000), (16080, 16000), (48000 * 3 + 7, 48000)):
        assert A.dio_frames(L, fs, FP) == int(1000.0 * L / fs / FP) + 1


def test_block_sum_is_the_fixed_order_sum():
    rng = np.random.RandomState(1)
    for n in (1, 255, 256, 257, 10000):
        v = rng.randn(n) * 1e4
        assert abs(A.block_sum(v) - np.sum(v)) <= 1e-9 * np.sum(np.abs(v))
    v = rng.randn(1000)
    assert A.block_sum(v) == A.block_sum(np.concatenate([v, np.zeros(300)]))


def test_sp2mc_inverts_mc2sp():
    rng = np.random.RandomState(2)
    for fs, order in ((16000, 24), (16000, 59), (48000, 59)):
        n = sptk_port.cheaptrick_fft_size(fs)
        alpha = sptk_port.mcepalpha(fs)
        mc = rng.randn(5, order + 1) * np.exp(-0.3 * np.arange(order + 1))
        back = A.sp2mc(sptk_port.mc2sp(mc, alpha, n), order, alpha)
        assert np.max(np.abs(back - mc)) < 1e-8, (fs, order)


def test_sp2mc_operator_matches_the_chain():
    """gantts_sp2mc_operator applied to log sp against the literal chain (irfft, c0 halved, freqt)."""
    from gantts_b200 import ops
    rng = np.random.RandomState(3)
    for fs, order in ((16000, 59), (48000, 24)):
        n = sptk_port.cheaptrick_fft_size(fs)
        alpha = sptk_port.mcepalpha(fs)
        op = ops.sp2mc_operator_host(alpha, order, n)
        assert op.shape == (n // 2 + 1, order + 1)
        sp = np.exp(rng.randn(4, n // 2 + 1) * 0.3 + np.linspace(8, -4, n // 2 + 1))
        want = A.sp2mc(sp, order, alpha)
        assert np.max(np.abs(np.log(sp) @ op - want)) < 1e-10 * max(1.0, np.max(np.abs(want)))


def min_phase_pulse(n_taps, rng):
    """A short minimum-phase impulse response: a product of first-order sections with zeros inside the unit circle."""
    h = np.array([1.0])
    for r in rng.uniform(-0.6, 0.6, n_taps):
        h = np.convolve(h, [1.0, r])
    return h


@pytest.mark.parametrize("fs", [16000, 48000])
def test_cheaptrick_recovers_a_pulse_train_envelope(fs):
    """A 200 Hz pulse train through a known minimum-phase filter: CheapTrick's envelope is within 1 dB (0.115 in natural
    log of the power) of |H|^2 times the pulse train's power per harmonic, fs / f0, over the bins from f0 to 0.9 fs / 2.
    (CheapTrick's spectral recovery is exact only for a smooth envelope; the filter's few taps keep it smooth.)"""
    rng = np.random.RandomState(5)
    f0 = 200.0
    period = int(fs / f0)
    x = np.zeros(fs)
    x[::period] = 1.0
    h = min_phase_pulse(4, rng)
    x = np.convolve(x, h)[:len(x)] * 1000.0
    n = sptk_port.cheaptrick_fft_size(fs)
    t = np.arange(40, 60) * FP / 1000.0
    sp = A.cheaptrick(x, np.full(len(t), fs / period), t, fs, n)
    H = np.fft.rfft(h, n)
    want = np.abs(H) ** 2 * 1e6 * fs / f0 / fs           # |H|^2 times the harmonics' power density
    k = np.arange(n // 2 + 1) * fs / n
    band = (k > f0) & (k < 0.9 * fs / 2)
    ratio = np.log(sp[:, band]) - np.log(want[band])
    ratio -= np.median(ratio)                            # the level depends on the window's normalisation
    assert np.max(np.abs(ratio)) < 0.115


def test_cheaptrick_draw_offsets_follow_the_sequential_stream():
    fs, n = 16000, 1024
    f0 = np.array([0.0, 120.0, 47.5, 300.0, 47.0, 88.5])
    counts = A.draw_counts(f0, fs, n)
    cur = A.current_f0(f0, fs, n)
    assert np.array_equal(counts, [2 * A.matlab_round(1.5 * fs / f) + 1 + n // 2 + 1 for f in cur])
    assert cur[0] == cur[4] == 500.0 and cur[2] == 47.5 and 47.0 < A.cheaptrick_f0_floor(fs, n) < 47.5
    off = A.draw_offsets(f0, fs, n)
    seq = W.Randn().draws(int(off[-1] + counts[-1]))
    stream = A.randn_stream(len(seq))
    assert np.array_equal(stream, seq)
    M = W.step_matrix()
    for j in (1, 3, 5):                                  # frame j starts at draw off[j]: jump 12 off[j] xorshift steps
        state = W.jump(W.SEED, 12 * int(off[j]), M)
        assert np.array_equal(W.Randn(state).draws(5), seq[off[j]:off[j] + 5])


def test_smoothing_leaves_a_band_limited_column_unchanged():
    n, modfs = 4096, 200.0
    kc = A.smoothing_bin(n, modfs)
    assert kc == 1024
    T = n                                               # a periodic column of n frames below the cut-off
    t = np.arange(T)
    col = 1.5 + np.cos(2 * np.pi * 37 * t / n) - 0.3 * np.sin(2 * np.pi * 1000 * t / n)
    x = np.stack([col, -2 * col], axis=1)
    assert np.max(np.abs(A.modspec_smoothing(x, modfs, n) - x)) < 1e-12
    # above the cut-off it is removed
    hi = np.cos(2 * np.pi * 1500 * t / n)
    assert np.max(np.abs(A.modspec_smoothing((col + hi)[:, None], modfs, n)[:, 0] - col)) < 1e-12
    with pytest.raises(ValueError, match="more than n"):
        A.modspec_smoothing(np.zeros((n + 1, 2)), modfs, n)


def _write_wav(path, fs, data):
    from scipy.io import wavfile
    wavfile.write(path, fs, data)


def test_objective_refuses_bad_wavs_before_any_device_work(tmp_path):
    from gantts_b200 import objective
    import train_cli_helpers as H
    root = str(tmp_path / "data")
    xd, yd = H.write_vc_data(root, n_files=12)
    wd = tmp_path / "wavs"
    wd.mkdir()
    names = [os.path.splitext(os.path.basename(f))[0] for _, xf, _ in objective.paired_files(xd, yd) for f in xf]
    rng = np.random.RandomState(0)
    for name in names:
        _write_wav(str(wd / (name + ".wav")), 16000, (rng.randn(3200) * 1000).astype(np.int16))
    args = ["--hparams_name=vc", "--wav-dir=" + str(wd), xd, yd, str(tmp_path / "out"), "missing.pth"]
    os.remove(str(wd / (names[3] + ".wav")))
    with pytest.raises(SystemExit, match="%s.wav" % names[3]):
        objective.main(args, hp=H.vc_hp())
    _write_wav(str(wd / (names[3] + ".wav")), 22050, np.zeros(3200, np.int16))
    with pytest.raises(SystemExit, match="22050 Hz.*--fs=16000"):
        objective.main(args, hp=H.vc_hp())
    _write_wav(str(wd / (names[3] + ".wav")), 16000, np.zeros((3200, 2), np.int16))
    with pytest.raises(SystemExit, match="2 channels"):
        objective.main(args, hp=H.vc_hp())
    _write_wav(str(wd / (names[3] + ".wav")), 16000, np.zeros(3200, np.int16))
    with pytest.raises(SystemExit, match="natural_wav"):
        objective.main(args[:-1] + ["--labels=natural_wav", "x.pth"], hp=H.vc_hp())
