"""Host-side pieces of the spectral post-processing of generation (Merlin's post filter and mc2sp): the identities that pin
the conventions of the CPU restatement (oracle.sptk_port), the all-pass constant and FFT size per sampling rate, the
operator builder gantts_mcep_operator against the restatement, the argument rules of gantts_mcep_postfilter and
gantts_mcep_to_sp (refused before any device work), and the command's new options.  No GPU needed."""
import ctypes

import numpy as np
import pytest

from oracle import sptk_port as sp
import train_cli_helpers as H

FAKE = 1 << 20          # placeholder device pointer: the argument checks never dereference it
FS = (16000, 22050, 48000)


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__
    __graft_entry__.build()
    from gantts_b200 import _lib
    return _lib.load()


def _frames(n, seed, M1=60):
    """Mel-cepstra shaped like generated mgc: a c0 of a few units and coefficients decaying with the index."""
    rng = np.random.RandomState(seed)
    mc = rng.randn(n, M1) * np.exp(-0.1 * np.arange(M1))
    mc[:, 0] = rng.uniform(-2.0, 2.0, n)
    return mc


def _direct_envelope(mc, alpha, n):
    """exp(2 Re sum_m c_m z~^-m), z~^-1 = (e^-jw - alpha) / (1 - alpha e^-jw): the power of a mel-cepstrum evaluated on the
    warped unit circle."""
    z = np.exp(-1j * 2 * np.pi * np.arange(n // 2 + 1) / n)
    zt = (z - alpha) / (1 - alpha * z)
    return np.exp(2 * np.real(np.polynomial.polynomial.polyval(zt, mc.T)))


@pytest.mark.parametrize("fs", FS)
def test_freqt_inverts_with_the_opposite_alpha(fs):
    alpha = sp.mcepalpha(fs)
    mc = _frames(4, 1)
    back = sp.freqt(sp.freqt(mc, 1023, -alpha), 59, alpha)
    assert np.abs(back - mc).max() <= 1e-12


@pytest.mark.parametrize("fs", FS)
def test_mc2sp_is_the_warped_spectrum(fs):
    alpha, n = sp.mcepalpha(fs), sp.cheaptrick_fft_size(fs)
    mc = _frames(4, 2)
    got, want = sp.mc2sp(mc, alpha, n), _direct_envelope(mc, alpha, n)
    assert got.shape == (4, n // 2 + 1)
    assert np.abs(got / want - 1).max() <= 1e-12


@pytest.mark.parametrize("fs", FS)
def test_post_filter_keeps_the_energy_and_only_moves_c0(fs):
    alpha = sp.mcepalpha(fs)
    mc = _frames(5, 3)
    w = np.full(60, 1.4)
    w[:2] = 1
    out = sp.merlin_post_filter(mc, alpha)
    r0 = lambda c: sp.c2acr0(sp.freqt(c, 511, -alpha), 1024)
    assert np.abs(r0(out) / r0(mc) - 1).max() <= 1e-12
    assert np.abs(out[:, 1:] - w[1:] * mc[:, 1:]).max() <= 1e-12
    assert np.abs(sp.merlin_post_filter(mc, alpha, coef=1.0) - mc).max() <= 1e-12


def test_all_pass_constant_and_fft_size_per_sampling_rate():
    from gantts_b200 import generate
    want = {8000: 0.312, 16000: 0.41, 22050: 0.455, 44100: 0.544, 48000: 0.554}
    for fs, a in want.items():
        assert generate.mcep_alpha(fs) == pytest.approx(a, abs=1e-12)
        assert sp.mcepalpha(fs) == pytest.approx(a, abs=1e-12)
    for fs, n in ((8000, 512), (16000, 1024), (22050, 1024), (44100, 2048), (48000, 2048)):
        assert generate.cheaptrick_fft_size(fs) == sp.cheaptrick_fft_size(fs) == n


@pytest.mark.parametrize("fs", FS)
def test_operator_builder_against_the_chain(lib, fs):
    from gantts_b200 import _lib, ops
    alpha, n = sp.mcepalpha(fs), sp.cheaptrick_fft_size(fs)
    mc = _frames(6, 4)
    op_s = ops.mcep_operator_host(alpha, 59, n, _lib.MCEP_SP)
    assert op_s.shape == (n // 2 + 1, 60)
    want = sp.mc2sp(mc, alpha, n)
    assert np.abs(np.exp(mc @ op_s.T) / want - 1).max() <= 1e-12
    # the post filter's energy operator, at merlin_post_filter's fftlen 1024 whatever the sampling rate
    op_r = ops.mcep_operator_host(alpha, 59, 1024, _lib.MCEP_R0)
    bins = np.full(513, 2.0)
    bins[[0, -1]] = 1.0
    r0 = lambda c: np.exp(c @ op_r.T) @ bins / 1024
    assert np.abs(r0(mc) / sp.c2acr0(sp.freqt(mc, 511, -alpha), 1024) - 1).max() <= 1e-12
    w = np.full(60, 1.4)
    w[:2] = 1
    closed = w * mc
    closed[:, 0] += 0.5 * np.log(r0(mc) / r0(w * mc))
    assert np.abs(closed - sp.merlin_post_filter(mc, alpha)).max() <= 1e-12


def _op_rc(lib, alpha=0.41, order=59, fftlen=1024, kind=0, out=FAKE):
    return lib.gantts_mcep_operator(alpha, order, fftlen, kind, out)


@pytest.mark.parametrize("kw,needle", [
    (dict(alpha=1.0), "alpha = 1 must satisfy |alpha| < 1"),
    (dict(alpha=-1.5), "alpha = -1.5 must satisfy |alpha| < 1"),
    (dict(alpha=float("nan")), "must satisfy |alpha| < 1"),
    (dict(order=-1), "order M = -1: M + 1 must be in [1, 128]"),
    (dict(order=128), "order M = 128: M + 1 must be in [1, 128]"),
    (dict(fftlen=32), "fftlen = 32 must be a power of two in [64, 4096]"),
    (dict(fftlen=8192), "fftlen = 8192 must be a power of two"),
    (dict(fftlen=1000), "fftlen = 1000 must be a power of two"),
    (dict(kind=2), "kind 2 must be GANTTS_MCEP_R0 (0) or GANTTS_MCEP_SP (1)"),
    (dict(out=None), "mcep_operator: null output"),
])
def test_operator_rules(lib, kw, needle):
    from gantts_b200 import _lib
    assert _op_rc(lib, **kw) == _lib.GANTTS_E_BADARG
    assert needle in lib.gantts_last_error_string().decode()


def test_operator_accepts_the_edges(lib):
    for order, fftlen in ((0, 64), (127, 64), (0, 4096)):
        for kind in (0, 1):
            out = np.full((fftlen // 2 + 1, order + 1), np.nan)
            assert _op_rc(lib, alpha=-0.99, order=order, fftlen=fftlen, kind=kind, out=out.ctypes.data) == 0
            assert np.isfinite(out).all()
    out = np.zeros((33, 1))
    _op_rc(lib, alpha=0.3, order=0, fftlen=64, kind=1, out=out.ctypes.data)
    assert np.array_equal(out[:, 0], np.full(33, 2.0))             # freqt sends e0 to e0: log power 2 c0 at every bin


def _kernel_rc(lib, name, lengths=FAKE, B=2, T=16, M=59, K=513, coef=1.4, mc=FAKE, out=FAKE, op=FAKE):
    if name == "postfilter":
        return lib.gantts_mcep_postfilter(mc, 1, 60, out, 1, 60, op, coef, lengths, B, T, M, K, None)
    return lib.gantts_mcep_to_sp(mc, 1, 60, out, 1, 513, op, lengths, B, T, M, K, None)


@pytest.mark.parametrize("name", ["postfilter", "to_sp"])
@pytest.mark.parametrize("kw,needle", [
    (dict(lengths=None), "null lengths"),
    (dict(B=0), "batch size B = 0 must be in [1, 65535]"),
    (dict(B=65536), "batch size B = 65536 must be in [1, 65535]"),
    (dict(T=0), "padded length T = 0 must be in [1, 16777216]"),
    (dict(T=(1 << 24) + 1), "padded length T = 16777217"),
    (dict(M=-1), "order M = -1: M + 1 must be in [1, 128]"),
    (dict(M=128), "order M = 128: M + 1 must be in [1, 128]"),
    (dict(K=17), "K = 17 bins: fftlen = 2 (K - 1) must be a power of two in [64, 4096]"),
    (dict(K=2050), "K = 2050 bins"),
    (dict(K=4097), "K = 4097 bins"),
    (dict(K=1), "K = 1 bins"),
    (dict(op=None), "null input, output or operator"),
    (dict(mc=None), "null input, output or operator"),
])
def test_kernel_rules(lib, name, kw, needle):
    from gantts_b200 import _lib
    assert _kernel_rc(lib, name, **kw) == _lib.GANTTS_E_BADARG
    msg = lib.gantts_last_error_string().decode()
    assert msg.startswith("mcep_" + name) and needle in msg, msg


@pytest.mark.parametrize("coef", [float("inf"), float("-inf"), float("nan")])
def test_postfilter_coef_must_be_finite(lib, coef):
    from gantts_b200 import _lib
    assert _kernel_rc(lib, "postfilter", coef=coef) == _lib.GANTTS_E_BADARG
    assert "coef = %g must be finite" % coef in lib.gantts_last_error_string().decode()


def test_new_symbols_have_their_ctypes_signatures(lib):
    from gantts_b200 import _lib
    res, args = _lib.SIGNATURES["gantts_mcep_operator"]
    assert res is ctypes.c_int and args[0] is ctypes.c_double and len(args) == 5
    res, args = _lib.SIGNATURES["gantts_mcep_postfilter"]
    assert res is ctypes.c_int and len(args) == 14 and args[7] is ctypes.c_double
    res, args = _lib.SIGNATURES["gantts_mcep_to_sp"]
    assert res is ctypes.c_int and len(args) == 13
    for name in ("gantts_mcep_operator", "gantts_mcep_postfilter", "gantts_mcep_to_sp"):
        assert hasattr(lib, name)


def test_new_options():
    from gantts_b200 import generate
    a = generate.parse_args(["c", "i", "o"])
    assert a["--fs"] == "16000" and not a["--post-filter"] and not a["--spectrogram"]
    a = generate.parse_args(["--hparams_name=tts_acoustic", "--post-filter", "--spectrogram", "--fs=48000", "c", "i", "o"])
    assert (a["--post-filter"], a["--spectrogram"], a["--fs"]) == (True, True, "48000")


@pytest.mark.parametrize("hp,argv,needle", [
    (H.vc_hp, ["--post-filter"], "--post-filter applies to tts_acoustic only"),
    (H.tts_duration_hp, ["--post-filter"], "--post-filter applies to tts_acoustic only"),
    (H.vc_hp, ["--spectrogram"], "--spectrogram applies to tts_acoustic only"),
    (H.tts_duration_hp, ["--spectrogram"], "--spectrogram applies to tts_acoustic only"),
    (H.tts_acoustic_hp, ["--fs=0"], "--fs must be > 0 (got 0)"),
    (H.tts_acoustic_hp, ["--fs=-16000", "--post-filter"], "--fs must be > 0 (got -16000)"),
    (H.tts_acoustic_hp, ["--fs=16k"], "--fs must be an integer"),
    (H.tts_acoustic_hp, ["--fs=192000", "--spectrogram"], "needs a 8192-point FFT; at most 4096"),
])
def test_command_refusals(hp, argv, needle):
    from gantts_b200 import generate
    with pytest.raises(SystemExit) as e:
        generate.main(argv + ["ckpt.pth", "data/X", "out"], hp=hp())
    assert needle in str(e.value)


def test_generator_refuses_the_flags_outside_tts_acoustic():
    from gantts_b200 import generate
    with pytest.raises(ValueError, match="applies to tts_acoustic only"):
        generate.check_hparams(H.vc_hp(), post_filter=True)
    generate.check_hparams(H.tts_acoustic_hp(), post_filter=True, spectrogram=True, fs=96000)


def test_utterances_carry_the_keys_generate_returns():
    import torch
    from gantts_b200 import generate
    pg = generate.ParameterGenerator.__new__(generate.ParameterGenerator)
    pg.hp, pg.kind, pg.device = H.tts_acoustic_hp(), "acoustic", torch.device("cpu")
    pg.stats = {"X_min": np.zeros(3), "X_max": np.ones(3)}

    def fake_generate(x, lengths):
        return {"mgc": x[..., :2], "vuv": x[..., 2], generate.SPECTROGRAM_NAME: x.repeat(1, 1, 3)}
    pg.generate = fake_generate
    arrays = [np.random.RandomState(n).rand(n, 3).astype(np.float32) for n in (5, 2, 7)]
    out = pg.generate_utterances(arrays, 2)
    for a, r in zip(arrays, out):
        x = 0.01 + a * 0.98
        assert list(r) == ["mgc", "vuv", "sp"]
        np.testing.assert_allclose(r["sp"], np.tile(x, 3), rtol=1e-6)
        np.testing.assert_allclose(r["vuv"], x[:, 2], rtol=1e-6)
