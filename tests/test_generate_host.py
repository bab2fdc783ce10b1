"""Host-side pieces of feature generation (gantts_b200.generate): usage and refusals of the command, the eval/test file
split, input normalisation, batching order, and the argument rules of the two length-exact entry points
(gantts_mlpg_ragged, gantts_sru_fwd_lengths), which are refused before any device work.  No GPU needed."""
import ctypes

import numpy as np
import pytest
import torch

from conftest import WINDOWS
import train_cli_helpers as H

FAKE = 1 << 20          # placeholder device pointer: the argument checks never dereference it


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__
    __graft_entry__.build()
    from gantts_b200 import _lib
    return _lib.load()


def test_usage_and_options():
    from gantts_b200 import generate
    a = generate.parse_args(["ckpt.pth", "data/X", "out"])
    assert (a["<checkpoint>"], a["<inputs_dir>"], a["<dst_dir>"]) == ("ckpt.pth", "data/X", "out")
    assert a["--hparams_name"] == "vc" and a["--hparams"] == "" and a["--batch-size"] is None and not a["--no-mge"]
    a = generate.parse_args(["--hparams_name=tts_acoustic", "--hparams=batch_size=3", "--batch-size=7", "--no-mge",
                             "c", "i", "o"])
    assert (a["--hparams_name"], a["--hparams"], a["--batch-size"], a["--no-mge"]) == \
        ("tts_acoustic", "batch_size=3", "7", True)


@pytest.mark.parametrize("hp,argv,needle", [
    (lambda: H.tts_acoustic_hp(generator="In2OutHighwayNet"), [], "cannot generate under the TTS hparams"),
    (lambda: H.tts_duration_hp(generator="In2OutRNNHighwayNet"), [], "cannot generate under the TTS hparams"),
    (lambda: H.vc_hp(generator_add_noise=True), [], "generator_add_noise"),
    (lambda: H.vc_hp(), ["--no-mge"], "--no-mge applies to tts_acoustic only"),
    (lambda: H.tts_duration_hp(), ["--no-mge"], "--no-mge applies to tts_acoustic only"),
    (lambda: H.vc_hp(), ["--batch-size=0"], "--batch-size must be >= 1"),
])
def test_command_refusals(hp, argv, needle):
    from gantts_b200 import generate
    with pytest.raises(SystemExit) as e:
        generate.main(argv + ["ckpt.pth", "data/X", "out"], hp=hp())
    assert needle in str(e.value)


def test_eval_and_test_split_is_the_training_commands(tmp_path):
    from gantts_b200 import generate, train
    for i in range(23):
        np.save(str(tmp_path / ("u%02d.npy" % i)), np.zeros((2, 1), np.float32))
    split = generate.utterance_files(str(tmp_path))
    assert [s for s, _ in split] == ["eval", "test"]
    assert split[0][1] == train.npy_files(str(tmp_path), train=False)
    assert split[1][1] == train.npy_files(str(tmp_path), test=True) == sorted(split[1][1])
    assert len(split[1][1]) == 5 and not set(split[0][1]) & set(split[1][1])


def test_input_normalisation():
    from gantts_b200 import generate
    rng = np.random.RandomState(0)
    x = rng.randn(9, 6).astype(np.float32) * 3
    mean, var = rng.randn(6), 0.5 + rng.rand(6)
    got = generate.normalize_input(x, H.vc_hp(), {"data_mean": mean, "data_std": np.sqrt(var)})
    assert got.dtype == np.float32
    np.testing.assert_allclose(got, (x.astype(np.float64) - mean) / np.sqrt(var), rtol=1e-6, atol=1e-6)
    xmin, xmax = x.min(0) - 1, x.max(0) + 1
    xmax[2] = xmin[2]                                      # a constant column: range 1, as nnmnkwii handles zeros
    for hp in (H.tts_acoustic_hp(), H.tts_duration_hp()):
        got = generate.normalize_input(x, hp, {"X_min": xmin, "X_max": xmax})
        rng_ = np.where(xmax - xmin == 0, 1.0, xmax - xmin)
        np.testing.assert_allclose(got, 0.01 + (x - xmin) * 0.98 / rng_, rtol=1e-6, atol=1e-6)


def test_statistics_are_read_from_the_inputs_parent(tmp_path):
    from gantts_b200 import generate
    np.save(str(tmp_path / "data_mean.npy"), np.arange(3.0))
    np.save(str(tmp_path / "data_var.npy"), np.full(3, 4.0))
    s = generate.load_stats(H.vc_hp(), str(tmp_path))
    assert np.array_equal(s["data_mean"], np.arange(3.0)) and np.array_equal(s["data_std"], np.full(3, 2.0))
    for ty, hp in (("acoustic", H.tts_acoustic_hp()), ("duration", H.tts_duration_hp())):
        for k, v in (("X_%s_data_min", 0.0), ("X_%s_data_max", 1.0), ("Y_%s_data_mean", 2.0), ("Y_%s_data_var", 9.0)):
            np.save(str(tmp_path / ((k % ty) + ".npy")), np.full(2, v))
        s = generate.load_stats(hp, str(tmp_path))
        assert [float(s[k][0]) for k in ("X_min", "X_max", "Y_mean", "Y_std")] == [0.0, 1.0, 2.0, 3.0]


def test_batches_are_sorted_split_and_results_come_back_in_input_order():
    from gantts_b200 import generate
    assert generate.plan_batches([3, 7, 7, 1, 5], 2) == [[1, 2], [4, 0], [3]]
    assert [len(b) for b in generate.plan_batches([1] * 300, 1000)] == [128, 128, 44]      # LSTM_MAX_B
    with pytest.raises(ValueError):
        generate.plan_batches([1], 0)
    # generate_utterances around a stand-in generator that doubles its input: each result is its own utterance
    pg = generate.ParameterGenerator.__new__(generate.ParameterGenerator)
    pg.hp, pg.kind, pg.device = H.vc_hp(), "vc", torch.device("cpu")
    pg.stats = {"data_mean": np.zeros(3), "data_std": np.ones(3)}
    seen = []

    def fake_generate(x, lengths):
        seen.append(lengths.tolist())
        return {"mc": 2 * x}
    pg.generate = fake_generate
    rng = np.random.RandomState(1)
    arrays = [rng.randn(n, 3).astype(np.float32) for n in (4, 9, 1, 9, 6)]
    out = pg.generate_utterances(arrays, 2)
    assert seen == [[9, 9], [6, 4], [1]]
    assert [sorted(r) for r in out] == [["mc"]] * 5
    for a, r in zip(arrays, out):
        assert r["mc"].dtype == np.float32 and np.array_equal(r["mc"], 2 * a)


def _streams(entries):
    from gantts_b200 import _lib
    return _lib.make_streams(entries)


def test_mlpg_ragged_workspace_query_accepts_valid_shapes(lib):
    from gantts_b200 import _lib
    w = _lib.make_windows(WINDOWS)
    for entries, B, T in (([(0, 60, 1, 0), (180, 1, 1, 60), (183, 1, 0, 61), (184, 1, 1, 62)], 20, 1000),
                          ([(0, 59, 1, 0)], 1, 1), ([(0, 5, 0, 0)], 128, 1 << 24)):
        s = _streams(entries)
        n_static = sum(e[1] for e in entries)
        got = lib.gantts_mlpg_ragged_workspace_bytes(ctypes.byref(s), ctypes.byref(w), FAKE, B, T)
        assert got == T * (2 + 2) * B * n_static * 8 + 256


def _reject(lib, needle, s=None, w=None, lengths=FAKE, B=2, T=16):
    from gantts_b200 import _lib
    s = s if s is not None else _streams([(0, 4, 1, 0)])
    w = w if w is not None else _lib.make_windows(WINDOWS)
    assert lib.gantts_mlpg_ragged_workspace_bytes(ctypes.byref(s), ctypes.byref(w), lengths, B, T) == 0
    msg = lib.gantts_last_error_string().decode()
    assert needle in msg, msg
    rc = lib.gantts_mlpg_ragged(FAKE, 1, 1, None, None, None, FAKE, 1, 1, None, None, ctypes.byref(s), ctypes.byref(w),
                                lengths, B, T, FAKE, 1 << 40, None)
    assert rc == _lib.GANTTS_E_BADARG and needle in lib.gantts_last_error_string().decode()


def test_mlpg_ragged_rules(lib):
    from gantts_b200 import _lib
    _reject(lib, "null lengths", lengths=None)
    _reject(lib, "batch size B = 0 must be >= 1", B=0)
    _reject(lib, "padded length T = 0 must be in [1, 16777216]", T=0)
    _reject(lib, "padded length T = 16777217 must be in [1, 16777216]", T=(1 << 24) + 1)
    s = _streams([(0, 1, 0, 0)])
    s.n = _lib.MAX_STREAMS + 1
    _reject(lib, "stream count 9 must be in [1, 8]", s=s)
    s.n = 0
    _reject(lib, "stream count 0 must be in [1, 8]", s=s)
    _reject(lib, "stream 1 static width sd = 0 must be in [1, 256]", s=_streams([(0, 3, 1, 0), (9, 0, 0, 3)]))
    _reject(lib, "stream 0 static width sd = 257 must be in [1, 256]", s=_streams([(0, 257, 0, 0)]))
    w = _lib.make_windows(WINDOWS)
    w.l[2] = 4                                             # 6 taps
    _reject(lib, "window 2 taps out of range", w=w)


def test_mlpg_ragged_needs_both_halves_of_an_affine_map(lib):
    from gantts_b200 import _lib
    s, w = _streams([(0, 4, 1, 0)]), _lib.make_windows(WINDOWS)
    rc = lib.gantts_mlpg_ragged(FAKE, 1, 1, None, FAKE, None, FAKE, 1, 1, None, None, ctypes.byref(s), ctypes.byref(w),
                                FAKE, 2, 16, FAKE, 1 << 40, None)
    assert rc == _lib.GANTTS_E_BADARG
    assert "needs both its scale and its shift" in lib.gantts_last_error_string().decode()


@pytest.mark.parametrize("kw,needle", [
    (dict(lengths=None), "null lengths"),
    (dict(T=0), "padded length T = 0 must be in [1, 16777216]"),
    (dict(T=(1 << 24) + 1), "padded length T = 16777217"),
    (dict(B=0), "B = 0 and d = 8 must be >= 1"),
    (dict(d=0), "B = 2 and d = 0 must be >= 1"),
    (dict(k=5), "sru: bad shape"),
    (dict(act=3), "sru: bad activation 3"),
    (dict(h=None), "sru_fwd_lengths: null output"),
])
def test_sru_fwd_lengths_rules(lib, kw, needle):
    from gantts_b200 import _lib
    a = dict(u=FAKE, x=None, bias=FAKE, lengths=FAKE, h=FAKE, B=2, T=16, d=8, k=4, bidir=1, act=2)
    a.update(kw)
    rc = lib.gantts_sru_fwd_lengths(a["u"], a["x"], a["bias"], a["lengths"], a["h"], a["B"], a["T"], a["d"], a["k"],
                                    a["bidir"], a["act"], None)
    assert rc == _lib.GANTTS_E_BADARG
    assert needle in lib.gantts_last_error_string().decode()


def test_new_symbols_have_their_ctypes_signatures(lib):
    from gantts_b200 import _lib
    assert _lib.SIGNATURES["gantts_sru_fwd_lengths"][1][:5] == [ctypes.c_void_p] * 5
    res, args = _lib.SIGNATURES["gantts_mlpg_ragged"]
    assert res is ctypes.c_int and len(args) == 19
    assert _lib.SIGNATURES["gantts_mlpg_ragged_workspace_bytes"][0] is ctypes.c_size_t
    for name in ("gantts_sru_fwd_lengths", "gantts_mlpg_ragged", "gantts_mlpg_ragged_workspace_bytes"):
        assert hasattr(lib, name)
