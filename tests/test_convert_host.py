"""Voice conversion on the host: the MLSA filter restatement (oracle.mlsa_port.mlsadf / mlsa_synthesis) pinned by its
properties, the delta restatement against the compat shim, and the convert command's host logic (arguments, the files of
get_wav_files, each refusal before any model is loaded)."""
import os

import numpy as np
import pytest

from oracle import nnmnkwii_port
from oracle import mlsa_port as P
from oracle import sptk_port

ALPHA = 0.41                  # mcepalpha(16000)


def _impulse_response(b, alpha, n):
    x = np.zeros(n)
    x[0] = 1.0
    return P.mlsa_synthesis([x], [np.tile(b, (n // 80 + 1, 1))], alpha, 80)[0]


def test_zero_coefficients_pass_the_input_through_bit_for_bit():
    rng = np.random.RandomState(0)
    x = np.round(rng.randn(700) * 3000)
    y = P.mlsa_synthesis([x], [np.zeros((10, 25))], ALPHA, 80)[0]
    assert np.array_equal(y, x)


def test_the_filter_is_linear_in_its_input():
    rng = np.random.RandomState(1)
    b = rng.randn(8, 13) * 0.1
    x1, x2 = rng.randn(600), rng.randn(600)
    y1, y2, y12 = P.mlsa_synthesis([x1, x2, x1 - 2.5 * x2], [b, b, b], ALPHA, 80)
    assert np.max(np.abs(y12 - (y1 - 2.5 * y2))) <= 1e-12 * np.max(np.abs(y12))


def test_constant_coefficients_equal_one_long_run_and_the_tail_is_zero():
    rng = np.random.RandomState(2)
    bc = rng.randn(25) * 0.1
    x = rng.randn(800)
    d = np.zeros((1, P.mlsa_delay_size(24)))
    long_run = np.array([P.mlsadf(np.array([v]), bc[None], ALPHA, d)[0] for v in x])
    # 800 samples = 10 hops of 80: the 11th frame's hop has no samples
    y = P.mlsa_synthesis([x], [np.tile(bc, (11, 1))], ALPHA, 80)[0]
    assert np.array_equal(y, long_run)
    # 22.05 kHz: hop int(110.25) = 110, DIO makes int(S / 110.25) + 1 frames, and from about 20 s on T hop < S: the
    # samples from T hop on stay 0 (a small order keeps the Python loop short)
    S = 50000
    T = int(1000.0 * S / 22050 / 5.0) + 1
    assert T * 110 < S
    y = P.mlsa_synthesis([np.resize(x, S)], [np.tile(bc[:3], (T, 1))], ALPHA, 110)[0]
    assert len(y) == S and np.all(y[T * 110:] == 0) and np.any(y[:T * 110] != 0)


def test_rows_in_lockstep_equal_rows_alone():
    rng = np.random.RandomState(3)
    xs = [rng.randn(n) for n in (530, 800, 81)]
    bs = [rng.randn(n // 80 + 1, 11) * 0.2 for n in (530, 800, 81)]
    together = P.mlsa_synthesis(xs, bs, ALPHA, 80)
    for x, b, y in zip(xs, bs, together):
        assert np.array_equal(P.mlsa_synthesis([x], [b], ALPHA, 80)[0], y)


def _pade_log_error(r, pd=5):
    """max |log R(w) - w| over |w| = r, R the Pade approximant of exp with SPTK's coefficients: log R(w) - w is analytic
    on the disk (R has no zeros or poles there for the r used), so its maximum modulus is on the circle."""
    w = r * np.exp(1j * np.linspace(0, 2 * np.pi, 4096, endpoint=False))
    num = sum(P.MLSA_PADE5[k] * w ** k for k in range(pd + 1))
    den = sum(P.MLSA_PADE5[k] * (-w) ** k for k in range(pd + 1))
    return float(np.max(np.abs(np.log(num / den) - w)))


def test_impulse_response_magnitude_is_the_mel_cepstrum_envelope_without_gain():
    """Pins alpha's sign, mc2b and the gain convention together: with c0 = 0, |FFT(h)| = sqrt(mc2sp(mc)) exp(-b[0]).
    The filter approximates exp(F1) exp(F2), F1 = b[1] Phi_1 and F2 = sum_{m>=2} b[m] Phi_m, each by the order-5 Pade
    approximant, so the log-magnitude error is at most e(r1) + e(r2), e(r) = max |log R(w) - w| over |w| = r and rk the
    peak of |Fk| on the unit circle."""
    rng = np.random.RandomState(4)
    M, n = 24, 4096
    mc = rng.randn(M + 1) * 0.3 * np.exp(-0.3 * np.arange(M + 1))
    mc[0] = 0.0
    b = sptk_port.mc2b(mc, ALPHA)
    h = _impulse_response(b, ALPHA, n)
    got = np.log(np.abs(np.fft.rfft(h)))
    want = 0.5 * np.log(sptk_port.mc2sp(mc, ALPHA, n)) - b[0]
    omega = np.pi * np.arange(n // 2 + 1) / (n // 2)
    z1 = np.exp(-1j * omega)
    phi1 = (1 - ALPHA ** 2) * z1 / (1 - ALPHA * z1)
    warp = (z1 - ALPHA) / (1 - ALPHA * z1)
    F1 = b[1] * phi1
    F2 = sum(b[m] * phi1 * warp ** (m - 1) for m in range(2, M + 1))
    bound = _pade_log_error(np.max(np.abs(F1))) + _pade_log_error(np.max(np.abs(F2)))
    err = float(np.max(np.abs(got - want)))
    print("impulse response: |log|H| - log envelope| %.3g, Pade bound %.3g (r1 %.3f, r2 %.3f)"
          % (err, bound, np.max(np.abs(F1)), np.max(np.abs(F2))))
    assert 0 < bound < 1e-3 and err <= bound + 1e-9
    # the other conventions break it: the gain applied, alpha's sign flipped
    assert np.max(np.abs(got - (want + b[0]))) > 10 * bound
    h_neg = _impulse_response(sptk_port.mc2b(mc, -ALPHA), -ALPHA, n)
    assert np.max(np.abs(np.log(np.abs(np.fft.rfft(h_neg))) - want)) > 10 * bound


def test_delta_restatement_equals_the_compat_shim():
    from compat.nnmnkwii import preprocessing
    rng = np.random.RandomState(5)
    windows = [(0, 0, np.array([1.0])), (1, 1, np.array([-0.5, 0.0, 0.5])), (1, 1, np.array([1.0, -2.0, 1.0])),
               (2, 1, np.array([0.1, -0.3, 0.7, 0.2]))]
    for T in (1, 2, 3, 57):
        x = rng.randn(T, 6)
        got = nnmnkwii_port.delta_features(x, windows)
        assert np.array_equal(got, preprocessing.delta_features(x, windows))
        # nnmnkwii's definition for its centred windows: np.correlate(x[:, d], window, mode="same") per column (which
        # swaps its arguments when the window is the longer)
        for wi, (l, u, coef) in enumerate(windows[:3]):
            for dcol in range(6 if T >= 3 else 0):
                ref = np.correlate(x[:, dcol], coef, mode="same")
                assert np.allclose(got[:, wi * 6 + dcol], ref, rtol=0, atol=1e-12)


# ---- the command's host logic ----

def _tree(tmp_path, n_files=12, fs=16000, seconds=0.3):
    from scipy.io import wavfile
    import train_cli_helpers as H
    root = str(tmp_path / "data")
    xd, _ = H.write_vc_data(root, n_files=n_files)
    wd = tmp_path / "wavs"
    wd.mkdir()
    rng = np.random.RandomState(0)
    names = sorted(os.path.splitext(f)[0] for f in os.listdir(xd))
    for name in names:
        wavfile.write(str(wd / (name + ".wav")), fs, (rng.randn(int(fs * seconds)) * 1000).astype(np.int16))
    return root, str(wd), names


def test_arguments_and_files_follow_evaluation_vc(tmp_path):
    from gantts_b200 import convert, train
    args = convert.parse_args(["--diffvc", "--batch-size=3", "--hparams=order=4", "ck.pth", "d", "w", "o"])
    assert args["--diffvc"] and args["--batch-size"] == "3" and args["--hparams"] == "order=4"
    assert (args["<checkpoint>"], args["<data_dir>"], args["<wav_dir>"], args["<outputs_dir>"]) == ("ck.pth", "d", "w",
                                                                                                   "o")
    assert not convert.parse_args(["a", "b", "c", "d"])["--diffvc"]
    root, wd, names = _tree(tmp_path)
    splits = convert.wav_files(root, wd)
    xd = os.path.join(root, "X")
    # get_wav_files (evaluation_vc.py:121-129) through NPYDataSource.collect_files
    for (sub, got), files in zip(splits, (train.npy_files(xd, train=False), train.npy_files(xd, test=True))):
        assert got == [os.path.join(wd, os.path.splitext(os.path.basename(f))[0] + ".wav") for f in files]
    assert [s for s, _ in splits] == ["eval", "test"] and len(splits[1][1]) == 5


def test_refusals_come_before_any_model_is_loaded(tmp_path):
    from scipy.io import wavfile
    from gantts_b200 import convert
    import train_cli_helpers as H
    root, wd, names = _tree(tmp_path)
    test_names = [os.path.splitext(os.path.basename(p))[0] for p in convert.wav_files(root, wd)[1][1]]
    victim = os.path.join(wd, test_names[2] + ".wav")
    base = [root, wd, str(tmp_path / "out")]
    run = lambda extra: convert.main(extra + ["missing.pth"] + base, hp=H.vc_hp())
    with pytest.raises(SystemExit, match="--diffvc is required.*D4C"):
        run([])
    with pytest.raises(SystemExit, match="--batch-size must be >= 1"):
        run(["--diffvc", "--batch-size=0"])
    os.remove(victim)
    with pytest.raises(SystemExit, match="%s is missing" % victim):
        run(["--diffvc"])
    wavfile.write(victim, 22050, np.zeros(3200, np.int16))
    with pytest.raises(SystemExit, match="%s is at 22050 Hz, but .* is at 16000 Hz" % victim):
        run(["--diffvc"])
    wavfile.write(victim, 16000, np.zeros((3200, 2), np.int16))
    with pytest.raises(SystemExit, match="%s has 2 channels" % victim):
        run(["--diffvc"])
    # 4097 frames at 5 ms: 20.48 s of 16 kHz audio
    wavfile.write(victim, 16000, np.zeros(16000 * 20480 // 1000, np.int16))
    with pytest.raises(SystemExit, match="%s has 4097 frames; modspec_smoothing is defined for at most 4096" % victim):
        run(["--diffvc"])
    wavfile.write(victim, 16000, np.zeros(16000 * 20480 // 1000 - 1, np.int16))
    # every wav is now acceptable: the next failure is the model's (no GPU here) or its missing checkpoint
    with pytest.raises((SystemExit, FileNotFoundError, OSError), match="CUDA|missing.pth|data_mean"):
        run(["--diffvc"])
