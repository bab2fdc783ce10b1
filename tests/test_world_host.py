"""Host-side pieces of WORLD waveform synthesis: the numpy restatement oracle.world_port pinned by properties that hold
for WORLD's algorithm whatever the restatement (randn's stream and jump-ahead, decode_aperiodicity's knots, the time
base's pulse spacing, the responses' DC removal and minimum-phase magnitude), the C entry points' argument rules, which
are refused before any device work, and synthesize --waveform's options and refusals.  No GPU needed."""
import os

import numpy as np
import pytest

from oracle import sptk_port
from oracle import world_port as W
import tts_data_helpers as TH

FAKE = 1 << 20          # placeholder device pointer: the argument checks never dereference it


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__
    __graft_entry__.build()
    from gantts_b200 import _lib
    return _lib.load()


# ---- randn ----

def test_randn_reseeds_and_is_standardised():
    a, b = W.Randn().draws(1000), W.Randn().draws(1000)
    assert np.array_equal(a, b)
    x = W.Randn().draws(100000)
    assert abs(x.mean()) < 0.01 and abs(x.var() - 1.0) < 0.02     # a sum of 12 uniforms minus 6
    assert x.min() >= -6.0 and x.max() <= 6.0


@pytest.mark.parametrize("steps", [1, 11, 12, 12 * 255, 12 * 256, 12 * 257, 12 * 512 + 5])
def test_jump_ahead_equals_single_steps(steps):
    r = W.Randn()
    for _ in range(steps):
        r.step()
    assert W.jump(W.SEED, steps) == r.s


# ---- decode_aperiodicity ----

@pytest.mark.parametrize("fs,nb", [(16000, 1), (22050, 2), (48000, 5), (44100, 5), (12000, 1), (11999, 0)])
def test_band_count(lib, fs, nb):
    assert W.band_count(fs) == nb and lib.gantts_world_band_count(fs) == nb


@pytest.mark.parametrize("fs,n", [(16000, 1024), (48000, 2048)])
def test_decode_knots(fs, n):
    nb = W.band_count(fs)
    rng = np.random.RandomState(fs)
    bap = -20 - 10 * rng.rand(6, nb)
    ap = W.decode_aperiodicity(bap, fs, n)
    k_per_hz = n / float(fs)
    for j in range(1, nb + 1):
        k = 3000 * j * k_per_hz
        if k == int(k):                                                     # the knot falls on a bin
            assert np.allclose(ap[:, int(k)], 10 ** (bap[:, j - 1] / 20), rtol=1e-13)
    assert np.allclose(ap[:, 0], 10 ** (-60 / 20.0), rtol=1e-13)
    assert np.allclose(ap[:, -1], 10 ** (-1e-12 / 20.0), rtol=1e-13)
    unv = np.full((3, nb), -0.4)
    assert np.array_equal(W.decode_aperiodicity(unv, fs, n), np.full((3, n // 2 + 1), 1 - 1e-12))


# ---- the time base ----

def test_constant_voiced_f0_spacing():
    fs = 16000
    idx, shift, vuv, Y = W.time_base(np.full(200, 100.0), fs, 5.0, 1024)
    assert Y == W.y_length(200, fs, 5.0) == 16000
    d = np.diff(idx)
    assert np.all(np.abs(d - 160) <= 1)
    exact = idx + shift * fs
    assert np.max(np.abs(np.diff(exact) - fs / 100.0)) < 1e-9
    assert np.all(vuv == 1)


@pytest.mark.parametrize("f0", [0.0, 15.9])
def test_unvoiced_gives_the_500_hz_grid(f0):
    fs = 16000                                  # lowest_f0 = 16000 // 1024 + 1 = 16: below it is unvoiced
    idx, shift, vuv, Y = W.time_base(np.full(100, f0), fs, 5.0, 1024)
    assert np.all(vuv == 0)
    assert np.all(np.abs(np.diff(idx) - 32) <= 1)
    assert np.max(np.abs(np.diff(idx + shift * fs) - 32.0)) < 1e-9


def test_y_length_formula(lib):
    for F, fs, fp in [(2, 16000, 5.0), (1000, 48000, 5.0), (77, 22050, 5.0), (13, 16000, 2.5), (3, 44100, 7.3)]:
        assert W.y_length(F, fs, fp) == int(F * fp * fs / 1000) == lib.gantts_world_y_length(F, fs, fp)


# ---- the responses ----

def _env(seed, fs=16000, n=1024, frames=3):
    rng = np.random.RandomState(seed)
    mc = rng.randn(frames, 60) * np.exp(-0.15 * np.arange(60))
    from gantts_b200 import generate
    return np.stack([sptk_port.mc2sp(m, generate.mcep_alpha(fs), n) for m in mc])


def test_periodic_responses_sum_to_zero_and_last_pulse_is_silent():
    fs = 16000
    F = 60
    f0 = np.where(np.arange(F) < 40, 130.0, 0.0)
    sp = np.repeat(_env(1, frames=1), F, 0)
    ap = np.full((F, 513), 0.05)
    y, det = W.synthesize(f0, sp, ap, fs, 5.0, details=True)
    dcr = W.dc_remover(1024)
    nz = 0
    for i, (n_i, v) in enumerate(zip(det["index"], det["vuv"])):
        env, ratio = W.envelope_ratio(sp, ap, n_i, fs, 0.005)
        p = W.periodic_response(env, ratio, float(v), det["shift"][i], fs, dcr)
        if v == 0:
            assert not p.any()                                              # unvoiced: no periodic part
        else:
            nz += 1
            assert abs(p.sum()) < 1e-12 * np.abs(p).max()
    assert nz > 10
    assert not det["responses"][-1].any()                                   # N = 0
    assert np.all(np.isfinite(y))


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_min_phase_magnitude(seed):
    sp = _env(seed, frames=1)[0]
    ratio = np.full_like(sp, 0.3)
    X = W.periodic_spectrum(sp, ratio)
    want = np.sqrt(sp * (1 - ratio) + 1e-12)
    assert np.max(np.abs(np.abs(X) / want - 1)) < 1e-6                      # cepstral aliasing only


# ---- the C entry points' argument rules ----

def _decode(lib, bap=FAKE, bs=3, ts=1, lengths=FAKE, B=2, T=10, nb=1, fs=16000, n=1024, ap=FAKE):
    return lib.gantts_world_decode_aperiodicity(bap, bs, ts, lengths, B, T, nb, fs, n, ap, None)


def _time_base(lib, f0=FAKE, bs=10, ts=1, lengths=FAKE, B=2, T=10, fs=16000, fp=5.0, n=1024, cap=800, idx=FAKE,
               sh=FAKE, vuv=FAKE, info=FAKE):
    return lib.gantts_world_time_base(f0, bs, ts, lengths, B, T, fs, fp, n, cap, idx, sh, vuv, info, None)


def _synth(lib, cap=800, total=10, B=2, T=10, fs=16000, fp=5.0, n=1024, y_max=800, ws=1 << 30, sps=1):
    return lib.gantts_world_synthesize(FAKE, 5130, 513, FAKE, 5130, sps * 513, FAKE, FAKE, FAKE, FAKE, FAKE, cap, total,
                                       FAKE, B, T, fs, fp, n, y_max, FAKE, FAKE, ws, None)


@pytest.mark.parametrize("call,kw,needle", [
    ("decode", dict(nb=2), "nb = 2 coded bands, but WORLD codes 1 at fs = 16000"),
    ("decode", dict(fs=8000, nb=0), "fs = 8000 has no aperiodicity band"),
    ("decode", dict(n=1000), "fftlen = 1000 must be a power of two in [64, 4096]"),
    ("decode", dict(n=8192), "fftlen = 8192 must be a power of two"),
    ("decode", dict(B=0), "batch size B = 0 must be in [1, 65535]"),
    ("decode", dict(T=0), "padded length T = 0 must be in [1, 16777216]"),
    ("decode", dict(bap=None), "null pointer"),
    ("decode", dict(ts=-1), "bap_tstride = -1"),
    ("time_base", dict(fp=0.0), "frame_period = 0 ms must be finite and > 0"),
    ("time_base", dict(fp=float("nan")), "must be finite and > 0"),
    ("time_base", dict(fs=0), "fs = 0 must be >= 1"),
    ("time_base", dict(cap=799), "cap = 799 pulses per row, but a row of T = 10 frames has 800 samples"),
    ("time_base", dict(info=None), "null pointer"),
    ("time_base", dict(n=32), "fftlen = 32 must be a power of two"),
    ("time_base", dict(T=1, fs=100, fp=1.0), "T = 1 frames make 0 samples"),
    ("synth", dict(y_max=801), "y_max = 801 must be in [1, 800]"),
    ("synth", dict(total=-1), "total_pulses = -1 must be >= 0"),
    ("synth", dict(ws=100), "holds no pulse response"),
    ("synth", dict(sps=-1), "ap_tstride = -513"),
])
def test_entry_point_rules(lib, call, kw, needle):
    from gantts_b200 import _lib
    fn = {"decode": _decode, "time_base": _time_base, "synth": _synth}[call]
    assert fn(lib, **kw) in (_lib.GANTTS_E_BADARG, 4)
    msg = lib.gantts_last_error_string().decode()
    assert msg.startswith("world_") and needle in msg, msg


def test_randn_rules(lib):
    assert lib.gantts_world_randn(0, FAKE, FAKE, 1 << 20, None) == 1
    assert "count = 0 must be in" in lib.gantts_last_error_string().decode()
    assert lib.gantts_world_randn(1000, FAKE, FAKE, 16, None) == 4
    assert "workspace of 16 bytes" in lib.gantts_last_error_string().decode()


def test_ops_refuse_cpu_tensors():
    import torch
    from gantts_b200 import ops
    with pytest.raises(RuntimeError, match="CUDA tensor required"):
        ops.world_decode_aperiodicity(torch.zeros(1, 4, 1), torch.tensor([4]), 16000, 1024)
    with pytest.raises(RuntimeError, match="CUDA tensor required"):
        ops.world_time_base(torch.zeros(1, 4), torch.tensor([4]), 16000, 5.0, 1024)


# ---- the command ----

def test_waveform_option():
    from gantts_b200 import synthesize
    assert synthesize.parse_args(["a", "d", "x", "o"])["--waveform"] is False
    assert synthesize.parse_args(["--waveform", "a", "d", "x", "o"])["--waveform"] is True
    assert "--waveform" in synthesize.__doc__ and ".wav" in synthesize.__doc__


@pytest.fixture(scope="module")
def data_dir(tmp_path_factory):
    return TH.write_tts_data(str(tmp_path_factory.mktemp("tts") / "data"), n_files=8)


@pytest.mark.parametrize("argv,hp_a,needle", [
    (["--waveform", "--fs=48000"], None, "the bap stream has 1 static columns, but WORLD codes 5 aperiodicity bands "
                                         "at --fs=48000"),
    (["--waveform", "--fs=22050"], None, "WORLD codes 2 aperiodicity bands at --fs=22050"),
    (["--waveform", "--fs=192000"], None, "at most 4096 points are supported"),
])
def test_waveform_refusals(lib, data_dir, tmp_path, argv, hp_a, needle):
    from gantts_b200 import synthesize
    out = str(tmp_path / "out")
    hp = hp_a() if hp_a else TH.acoustic_hp()
    with pytest.raises(SystemExit) as e:
        synthesize.main(argv + ["ck/a.pth", "ck/d.pth", data_dir, out], hp_acoustic=hp, hp_duration=TH.duration_hp())
    assert str(e.value).startswith("gantts_b200.synthesize: ") and needle in str(e.value), str(e.value)
    assert not os.path.exists(out)


def test_waveform_rules_follow_the_bap_width(lib):
    from gantts_b200 import synthesize
    synthesize.check_tts_hparams(TH.acoustic_hp(), TH.duration_hp(), fs=16000, waveform=True)
    five = TH.acoustic_hp(stream_sizes=[180, 3, 1, 15])
    synthesize.check_tts_hparams(five, TH.duration_hp(), fs=48000, waveform=True)
    with pytest.raises(ValueError, match="the bap stream has 5 static columns, but WORLD codes 1"):
        synthesize.check_tts_hparams(five, TH.duration_hp(), fs=16000, waveform=True)
    synthesize.check_tts_hparams(five, TH.duration_hp(), fs=16000)          # no rule without the waveform


def test_wav_scaling(tmp_path):
    from scipy.io import wavfile
    from gantts_b200 import synthesize
    y = np.array([0.0, 0.5, -2.0, 1.0, 1e-9])
    p = str(tmp_path / "a.wav")
    synthesize.write_wav(p, y, 16000)
    rate, s = wavfile.read(p)
    assert rate == 16000 and s.dtype == np.int16
    assert np.array_equal(s, (y / 2.0 * 32767).astype(np.int16))
