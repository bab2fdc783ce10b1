"""Host-side pieces of the objective measures (gantts_b200.objective): the restatement of the notebooks' global variance
and log modulation spectrum (objective_oracle) against their literal definitions, the command's usage text and
refusals, the npz layout and the summary formula on fabricated statistics, and the argument rules of gantts_modspec and
gantts_global_variance, which are refused before any device work.  No GPU needed."""
import ctypes
import os

import numpy as np
import pytest

import objective_oracle as ref
import train_cli_helpers as H

FAKE = 1 << 20          # placeholder device pointer: the argument checks never dereference it


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__
    __graft_entry__.build()
    from gantts_b200 import _lib
    return _lib.load()


def _dft_power(x, n):
    """|sum_{t < min(T, n)} x[t] exp(-2 pi i k t / n)|^2 for k = 0 .. n/2, by the explicit sum in float64."""
    x = np.asarray(x, dtype=np.float64)[:n]
    t, k = np.arange(len(x)), np.arange(n // 2 + 1)
    X = np.exp(-2j * np.pi * np.outer(k, t) / n) @ x
    return X.real ** 2 + X.imag ** 2


@pytest.mark.parametrize("T,n", [(1, 64), (37, 64), (64, 64), (65, 64), (300, 64), (200, 512)])
def test_modspec_is_the_literal_dft_power(T, n):
    x = np.random.RandomState(T).randn(T, 3) + 2.0
    got, want = ref.modspec(x, n), _dft_power(x, n)
    assert got.shape == (n // 2 + 1, 3) and got.dtype == np.float64
    assert np.abs(got - want).max() <= 1e-12 * want.max()
    assert np.allclose(ref.log_modspec(x, n), np.log(want), rtol=0, atol=1e-9)


def test_modspec_crops_at_n_and_zero_pads():
    x = np.random.RandomState(1).randn(100, 2)
    assert np.array_equal(ref.modspec(x, 64), ref.modspec(x[:64], 64))
    assert np.array_equal(ref.modspec(x[:40], 64), ref.modspec(np.concatenate([x[:40], np.zeros((24, 2))]), 64))


def test_modspec_of_a_silent_column_is_minus_inf():
    x = np.zeros((7, 2))
    x[:, 1] = 1.0                                       # 7 frames: no bin of its spectrum is 0
    ms = ref.log_modspec(x, 64)
    assert np.all(ms[:, 0] == -np.inf) and np.isfinite(ms[:, 1]).all()
    assert np.all(ref.log_modspec(np.zeros((0, 3)), 64) == -np.inf)


def test_float32_input_is_computed_in_double():
    x = (np.random.RandomState(2).randn(50, 4) * 3 + 1).astype(np.float32)
    got = ref.modspec(x, 128)
    assert got.dtype == np.float64
    assert np.array_equal(got, ref.modspec(x.astype(np.float64), 128))
    gv = ref.global_variance(x)
    assert gv.dtype == np.float64 and np.array_equal(gv, np.var(x.astype(np.float64), axis=0))


def test_global_variance_definition():
    x = np.random.RandomState(3).randn(30, 5) * np.arange(1, 6)
    assert np.allclose(ref.global_variance(x), ((x - x.mean(0)) ** 2).sum(0) / 30, rtol=1e-14)
    assert np.all(np.isnan(ref.global_variance(np.zeros((0, 5)))))
    assert np.array_equal(ref.global_variance(np.full((1, 2), 7.0)), np.zeros(2))


def test_usage_and_options():
    from gantts_b200 import objective
    a = objective.parse_args(["X", "Y", "out", "ck/baseline/g.pth", "ck/gan/g.pth"])
    assert (a["<inputs_dir>"], a["<outputs_dir>"], a["<dst_dir>"]) == ("X", "Y", "out")
    assert a["<checkpoint>"] == ["ck/baseline/g.pth", "ck/gan/g.pth"]
    assert (a["--hparams_name"], a["--hparams"], a["--labels"], a["--batch-size"], a["--no-mge"]) == \
        ("vc", "", None, None, False)
    assert (a["--ms-fftlen"], a["--fs"]) == ("4096", "16000")
    a = objective.parse_args(["--hparams_name=tts_acoustic", "--labels=a,b", "--batch-size=3", "--no-mge",
                              "--ms-fftlen=8192", "--fs=48000", "X", "Y", "o", "c"])
    assert (a["--labels"], a["--batch-size"], a["--no-mge"], a["--ms-fftlen"], a["--fs"]) == \
        ("a,b", "3", True, "8192", "48000")
    assert "WORLD" in objective.__doc__ and "prepared targets" in objective.__doc__
    with pytest.raises(SystemExit, match="usage: objective.py"):
        objective.parse_args(["X", "Y", "out"])                             # at least one checkpoint


def test_default_labels_are_the_checkpoint_directories():
    from gantts_b200 import objective
    assert objective.check_labels(None, ["ck/baseline/a.pth", "ck/gan/a.pth"]) == ["baseline", "gan"]
    assert objective.check_labels("x,y", ["a.pth", "b.pth"]) == ["x", "y"]


def _data(tmp_path):
    return H.write_vc_data(str(tmp_path / "data"), n_files=12)


@pytest.mark.parametrize("hp,argv,ckpts,needle", [
    (H.tts_duration_hp, [], ["c/a.pth"], "the notebooks compute neither"),
    (lambda: H.tts_acoustic_hp(generator="In2OutHighwayNet"), [], ["c/a.pth"], "cannot generate under the TTS"),
    (lambda: H.vc_hp(generator_add_noise=True), [], ["c/a.pth"], "generator_add_noise"),
    (H.vc_hp, ["--no-mge"], ["c/a.pth"], "--no-mge applies to tts_acoustic only"),
    (H.vc_hp, ["--batch-size=0"], ["c/a.pth"], "--batch-size must be >= 1"),
    (H.vc_hp, ["--ms-fftlen=1000"], ["c/a.pth"], "--ms-fftlen must be a power of two in [64, 8192] (got 1000)"),
    (H.vc_hp, ["--ms-fftlen=32"], ["c/a.pth"], "--ms-fftlen must be a power of two in [64, 8192] (got 32)"),
    (H.vc_hp, ["--ms-fftlen=16384"], ["c/a.pth"], "(got 16384)"),
    (H.vc_hp, ["--ms-fftlen=4k"], ["c/a.pth"], "must be integers"),
    (H.vc_hp, ["--fs=0"], ["c/a.pth"], "--fs must be > 0 (got 0)"),
    (H.vc_hp, ["--fs=100"], ["c/a.pth"], "--fs=100 gives a hop of 0 samples"),
    (H.vc_hp, ["--labels=a"], ["c/a.pth", "c/b.pth"], "--labels has 1 labels for 2 checkpoints"),
    (H.vc_hp, ["--labels=a,b,c"], ["c/a.pth", "c/b.pth"], "--labels has 3 labels for 2 checkpoints"),
    (H.vc_hp, ["--labels=a,a"], ["c/a.pth", "c/b.pth"], "label 'a' is used twice"),
    (H.vc_hp, ["--labels=natural"], ["c/a.pth"], "label 'natural' is used twice"),
    (H.vc_hp, ["--labels=a,"], ["c/a.pth", "c/b.pth"], "a label must not be empty"),
    (H.vc_hp, [], ["ck/gan/a.pth", "ck/gan/b.pth"], "label 'gan' is used twice"),
])
def test_command_refusals(tmp_path, hp, argv, ckpts, needle):
    from gantts_b200 import objective
    xd, yd = _data(tmp_path)
    with pytest.raises(SystemExit) as e:
        objective.main(argv + [xd, yd, str(tmp_path / "out")] + ckpts, hp=hp())
    assert str(e.value).startswith("gantts_b200.objective: ") and needle in str(e.value), str(e.value)
    assert not os.path.exists(str(tmp_path / "out"))


def test_command_refuses_x_and_y_that_differ(tmp_path):
    from gantts_b200 import objective
    xd, yd = _data(tmp_path)
    last = sorted(os.listdir(yd))[-1]
    os.rename(os.path.join(yd, last), os.path.join(yd, "zz_" + last))
    with pytest.raises(SystemExit, match="test split: the utterances of .* differ"):
        objective.main([xd, yd, str(tmp_path / "out"), "c/a.pth"], hp=H.vc_hp())
    os.rename(os.path.join(yd, "zz_" + last), os.path.join(yd, last))
    y = np.load(os.path.join(yd, last))
    np.save(os.path.join(yd, last), y[:-1])
    with pytest.raises(SystemExit) as e:
        objective.main([xd, yd, str(tmp_path / "out"), "c/a.pth"], hp=H.vc_hp())
    assert "%s: %d input frames but %d target frames" % (last, len(y), len(y) - 1) in str(e.value)


def test_modulation_frequencies():
    from gantts_b200 import objective
    f = objective.modulation_frequencies(4096, 16000)
    assert f.shape == (2049,) and f[0] == 0 and f[-1] == 100.0            # modfs = 16000 / 80 = 200 Hz
    assert np.allclose(objective.modulation_frequencies(64, 22050), np.arange(33) / 64 * (22050 / 110))
    assert objective.modulation_frequencies(64, 16000, frame_period=10)[-1] == 50.0


def test_natural_columns_are_the_first_streams_statics():
    from gantts_b200 import objective
    assert objective.natural_columns(H.vc_hp(order=59)) == slice(0, 59)
    assert objective.natural_columns(H.tts_acoustic_hp()) == slice(0, 60)


def _fabricated(rng, U=4, D=3, K=5, nl=3):
    return [(rng.rand(U, D) + 0.1, rng.rand(D) + 0.1, rng.randn(K, D)) for _ in range(nl)]


def test_npz_layout(tmp_path):
    from gantts_b200 import objective
    rng = np.random.RandomState(0)
    res = _fabricated(rng)
    files = ["/d/X/utt%d.npy" % i for i in range(4)]
    Y = [np.zeros((n, 6)) for n in (5, 9, 2, 7)]
    arrays = objective.split_arrays(["natural", "baseline", "gan"], files, Y, np.arange(5.0), res)
    np.savez(str(tmp_path / "eval.npz"), **arrays)
    z = np.load(str(tmp_path / "eval.npz"))                               # loads without pickle
    assert sorted(z.files) == ["gv", "gv_mean", "labels", "lengths", "ms_freq", "ms_mean", "names"]
    assert list(z["labels"]) == ["natural", "baseline", "gan"]
    assert list(z["names"]) == ["utt0", "utt1", "utt2", "utt3"]
    assert z["lengths"].dtype == np.int64 and list(z["lengths"]) == [5, 9, 2, 7]
    assert z["gv"].shape == (3, 4, 3) and z["gv_mean"].shape == (3, 3) and z["ms_mean"].shape == (3, 5, 3)
    for i, (gv, gvm, ms) in enumerate(res):
        assert np.array_equal(z["gv"][i], gv) and np.array_equal(z["gv_mean"][i], gvm)
        assert np.array_equal(z["ms_mean"][i], ms)


def test_summary_formula():
    from gantts_b200 import objective
    gv_mean = np.array([[1.0, 2.0, 4.0], [1.0, 2.0, 4.0], [10.0, 0.2, 4.0]])
    ms_mean = np.zeros((3, 2, 3))
    ms_mean[2] = [[1.0, -1.0, 1.0], [-1.0, 1.0, 3.0]]
    rows = objective.summary(["natural", "same", "other"], gv_mean, ms_mean)
    assert [r[0] for r in rows] == ["same", "other"]
    assert rows[0][1:] == (0.0, 0.0)
    assert rows[1][1] == pytest.approx((1.0 - 1.0 + 0.0) / 3)
    assert rows[1][2] == pytest.approx(np.sqrt((1 + 1 + 1 + 1 + 1 + 9) / 6.0))


def test_feature_stats_refuses_cpu_tensors():
    import torch
    from gantts_b200 import ops
    x, lengths = torch.zeros(2, 5, 3), torch.tensor([5, 3])
    with pytest.raises(RuntimeError, match="CUDA tensor required"):
        ops.modspec(x, lengths, 64)
    with pytest.raises(RuntimeError, match="CUDA tensor required"):
        ops.global_variance(x, lengths)


def _rc(lib, name, x=FAKE, bs=600, ts=60, lengths=FAKE, B=2, T=10, D=60, n=4096, out=FAKE, sum_=None):
    if name == "modspec":
        return lib.gantts_modspec(x, bs, ts, lengths, B, T, D, n, out, sum_, None)
    return lib.gantts_global_variance(x, bs, ts, lengths, B, T, D, out, None)


@pytest.mark.parametrize("name", ["modspec", "global_variance"])
@pytest.mark.parametrize("kw,needle", [
    (dict(lengths=None), "null lengths"),
    (dict(B=0), "batch size B = 0 must be in [1, 65535]"),
    (dict(B=65536), "batch size B = 65536 must be in [1, 65535]"),
    (dict(T=0), "padded length T = 0 must be in [1, 16777216]"),
    (dict(T=(1 << 24) + 1), "padded length T = 16777217"),
    (dict(D=0), "feature width D = 0 must be in [1, 65535]"),
    (dict(D=65536), "feature width D = 65536"),
    (dict(bs=-1), "strides x_bstride = -1 and x_tstride = 60 must be >= 0"),
    (dict(ts=-60), "x_tstride = -60 must be >= 0"),
    (dict(x=None), "null input or output"),
    (dict(out=None), "null input or output"),
])
def test_kernel_rules(lib, name, kw, needle):
    from gantts_b200 import _lib
    assert _rc(lib, name, **kw) == _lib.GANTTS_E_BADARG
    msg = lib.gantts_last_error_string().decode()
    assert msg.startswith(name + ":") and needle in msg, msg


@pytest.mark.parametrize("n", [0, 32, 63, 96, 1000, 16384, -4096])
def test_modspec_n_rule(lib, n):
    from gantts_b200 import _lib
    assert _rc(lib, "modspec", n=n, sum_=FAKE) == _lib.GANTTS_E_BADARG
    assert "modspec: n = %d must be a power of two in [64, 8192]" % n in lib.gantts_last_error_string().decode()


def test_new_symbols_have_their_ctypes_signatures(lib):
    from gantts_b200 import _lib
    res, args = _lib.SIGNATURES["gantts_modspec"]
    assert res is ctypes.c_int and len(args) == 11 and args[1] is ctypes.c_int64 and args[2] is ctypes.c_int64
    res, args = _lib.SIGNATURES["gantts_global_variance"]
    assert res is ctypes.c_int and len(args) == 9 and args[1] is ctypes.c_int64 and args[2] is ctypes.c_int64
    assert hasattr(lib, "gantts_modspec") and hasattr(lib, "gantts_global_variance")
