"""Host-side pieces of TTS synthesis with predicted durations (gantts_b200.synthesize): the restatement of Merlin's
"full" subphone features (oracle.merlin_port) against a hand-worked phone and its identities, the argument rules of
gantts_state_frame_offsets and gantts_expand_state_frames, which are refused before any device work, and the command's
usage, options and refusals.  No GPU needed."""
import ctypes
import os

import numpy as np
import pytest

from oracle import merlin_port
import tts_data_helpers as TH

FAKE = 1 << 20          # placeholder device pointer: the argument checks never dereference it


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__
    __graft_entry__.build()
    from gantts_b200 import _lib
    return _lib.load()


def test_hand_worked_phone():
    # durations [1, 2, 3, 1, 1]: N = 8, bases 0, 1, 3, 6, 7
    want = np.array([
        # (i+1)/d  (d-i)/d  d   s  S+1-s  N  d/N    (N-i-base)/N  (base+i+1)/N
        [1,       1,       1,  1, 5,     8, 1 / 8, 8 / 8,        1 / 8],
        [1 / 2,   1,       2,  2, 4,     8, 2 / 8, 7 / 8,        2 / 8],
        [2 / 2,   1 / 2,   2,  2, 4,     8, 2 / 8, 6 / 8,        3 / 8],
        [1 / 3,   1,       3,  3, 3,     8, 3 / 8, 5 / 8,        4 / 8],
        [2 / 3,   2 / 3,   3,  3, 3,     8, 3 / 8, 4 / 8,        5 / 8],
        [3 / 3,   1 / 3,   3,  3, 3,     8, 3 / 8, 3 / 8,        6 / 8],
        [1,       1,       1,  4, 2,     8, 1 / 8, 2 / 8,        7 / 8],
        [1,       1,       1,  5, 1,     8, 1 / 8, 1 / 8,        8 / 8],
    ], dtype=np.float64)
    got = merlin_port.frame_features([1, 2, 3, 1, 1])
    assert got.shape == (8, 9) and got.dtype == np.float64
    assert np.array_equal(got, want)
    x = np.array([[0.5, -2.0, 3.0]], dtype=np.float32)
    e = merlin_port.expand(x, np.array([[1, 2, 3, 1, 1]], dtype=np.float32))
    assert e.dtype == np.float32 and e.shape == (8, 12)
    assert np.array_equal(e[:, :3], np.repeat(x, 8, axis=0))
    assert np.array_equal(e[:, 3:], want.astype(np.float32))


@pytest.mark.parametrize("S", [1, 3, 5, 16])
def test_identities(S):
    rng = np.random.RandomState(S)
    P, L = 17, 6
    x = rng.randn(P, L).astype(np.float32)
    dur = TH.random_durations(rng, P, S, hi=12)
    e = merlin_port.expand(x, dur)
    assert len(e) == int(dur.sum())                                      # the frame count is the sum of durations
    t = 0
    for p in range(P):
        d = dur[p].astype(int)
        N = int(d.sum())
        f = merlin_port.frame_features(d)
        assert np.array_equal(e[t:t + N, :L], np.repeat(x[p:p + 1], N, axis=0))   # repeated linguistic rows
        assert np.array_equal(e[t:t + N, L:], f.astype(np.float32))
        assert f[0, 7] == 1.0 and f[-1, 8] == 1.0                        # first / last frame of the phone
        last = np.cumsum(d) - 1
        assert np.all(f[last, 0] == 1.0)                                 # last frame of each state
        assert abs(f[last, 6].sum() - 1.0) < 1e-12                       # state shares sum to 1
        assert np.array_equal(f[:, 3] + f[:, 4], np.full(N, S + 1.0))
        assert np.all(f[:, 5] == N)
        t += N


def test_oracle_refuses_zero_durations():
    with pytest.raises(ValueError, match="must be >= 1"):
        merlin_port.frame_features([1, 0, 2])


# ---- the C entry points' argument rules ----

def _offsets(lib, dur=FAKE, bs=100, ps=5, lengths=FAKE, B=2, P=20, S=5, offsets=FAKE, fl=FAKE, status=FAKE):
    return lib.gantts_state_frame_offsets(dur, bs, ps, lengths, B, P, S, offsets, fl, status, None)


def _expand(lib, x=FAKE, xbs=8320, xps=416, dur=FAKE, bs=100, ps=5, offsets=FAKE, fl=FAKE, scale=FAKE, mn=FAKE, B=2,
            P=20, L=416, S=5, T=1000, out=FAKE):
    return lib.gantts_expand_state_frames(x, xbs, xps, dur, bs, ps, offsets, fl, scale, mn, B, P, L, S, T, out, None)


COMMON = [
    (dict(B=0), "batch size B = 0 must be in [1, 65535]"),
    (dict(B=65536), "batch size B = 65536 must be in [1, 65535]"),
    (dict(P=0), "phones P = 0 must be >= 1"),
    (dict(S=0), "states S = 0 must be in [1, 16]"),
    (dict(S=17), "states S = 17 must be in [1, 16]"),
    (dict(dur=None), "null pointer"),
    (dict(offsets=None), "null pointer"),
    (dict(fl=None), "null pointer"),
    (dict(bs=-1), "dur_bstride = -1"),
    (dict(ps=-5), "dur_pstride = -5"),
]


@pytest.mark.parametrize("kw,needle", COMMON + [
    (dict(lengths=None), "null pointer"),
    (dict(status=None), "null pointer"),
])
def test_offsets_rules(lib, kw, needle):
    from gantts_b200 import _lib
    assert _offsets(lib, **kw) == _lib.GANTTS_E_BADARG
    msg = lib.gantts_last_error_string().decode()
    assert msg.startswith("state_frame_offsets:") and needle in msg, msg


@pytest.mark.parametrize("kw,needle", COMMON + [
    (dict(L=0), "linguistic width L = 0 must be in [1, 65535]"),
    (dict(L=65536), "linguistic width L = 65536 must be in [1, 65535]"),
    (dict(T=0), "padded length T = 0 must be in [1, 16777216]"),
    (dict(T=(1 << 24) + 1), "padded length T = 16777217 must be in [1, 16777216]"),
    (dict(xbs=-1), "x_bstride = -1"),
    (dict(xps=-416), "x_pstride = -416"),
    (dict(x=None), "null pointer"),
    (dict(scale=None), "null pointer"),
    (dict(mn=None), "null pointer"),
    (dict(out=None), "null pointer"),
])
def test_expand_rules(lib, kw, needle):
    from gantts_b200 import _lib
    assert _expand(lib, **kw) == _lib.GANTTS_E_BADARG
    msg = lib.gantts_last_error_string().decode()
    assert msg.startswith("expand_state_frames:") and needle in msg, msg


def test_new_symbols_have_their_ctypes_signatures(lib):
    from gantts_b200 import _lib
    res, args = _lib.SIGNATURES["gantts_state_frame_offsets"]
    assert res is ctypes.c_int and len(args) == 11 and args[1] is ctypes.c_int64 and args[2] is ctypes.c_int64
    res, args = _lib.SIGNATURES["gantts_expand_state_frames"]
    assert res is ctypes.c_int and len(args) == 17 and args[4] is ctypes.c_int64 and args[5] is ctypes.c_int64
    assert hasattr(lib, "gantts_state_frame_offsets") and hasattr(lib, "gantts_expand_state_frames")


def test_ops_refuse_cpu_tensors():
    import torch
    from gantts_b200 import ops
    with pytest.raises(RuntimeError, match="CUDA tensor required"):
        ops.state_frame_offsets(torch.ones(2, 3, 5), torch.tensor([3, 2]))
    with pytest.raises(RuntimeError, match="CUDA tensor required"):
        ops.expand_state_frames(torch.ones(2, 3, 4), torch.ones(2, 3, 5), None, None, None, None, 10)


# ---- the command ----

def test_usage_and_options():
    from gantts_b200 import synthesize
    a = synthesize.parse_args(["ac.pth", "dur.pth", "data", "out"])
    assert (a["<acoustic_checkpoint>"], a["<duration_checkpoint>"], a["<data_dir>"], a["<dst_dir>"]) == \
        ("ac.pth", "dur.pth", "data", "out")
    assert (a["--fs"], a["--disable-duraton-gen"], a["--post-filter"], a["--spectrogram"], a["--batch-size"],
            a["--no-mge"]) == ("16000", False, False, False, None, False)
    a = synthesize.parse_args(["--fs=48000", "--disable-duraton-gen", "--post-filter", "--spectrogram",
                               "--batch-size=3", "--no-mge", "a", "d", "x", "o"])
    assert (a["--fs"], a["--disable-duraton-gen"], a["--post-filter"], a["--spectrogram"], a["--batch-size"],
            a["--no-mge"]) == ("48000", True, True, True, "3", True)
    assert "silence" in synthesize.__doc__ and "WORLD" in synthesize.__doc__
    with pytest.raises(SystemExit, match="usage: synthesize.py"):
        synthesize.parse_args(["a", "d", "x"])
    with pytest.raises(SystemExit, match="unknown option --hparams_name"):
        synthesize.parse_args(["--hparams_name=vc", "a", "d", "x", "o"])


@pytest.fixture(scope="module")
def data_dir(tmp_path_factory):
    return TH.write_tts_data(str(tmp_path_factory.mktemp("tts") / "data"))


def _main(data, out, argv=(), hp_a=None, hp_d=None):
    from gantts_b200 import synthesize
    return synthesize.main(list(argv) + ["ck/a.pth", "ck/d.pth", data, out],
                           hp_acoustic=hp_a if hp_a is not None else TH.acoustic_hp(),
                           hp_duration=hp_d if hp_d is not None else TH.duration_hp())


@pytest.mark.parametrize("argv,hp_a,hp_d,needle", [
    ([], lambda: TH.duration_hp(), None, "the acoustic hyper parameters must have name 'acoustic'"),
    ([], None, lambda: TH.acoustic_hp(), "the duration hyper parameters must have name 'duration'"),
    ([], lambda: TH.acoustic_hp(generator_add_noise=True), None, "generator_add_noise"),
    ([], None, lambda: TH.duration_hp(generator_add_noise=True), "generator_add_noise"),
    ([], lambda: TH.acoustic_hp(generator="In2OutHighwayNet"), None, "cannot generate under the TTS"),
    ([], None, lambda: TH.duration_hp(generator="In2OutRNNHighwayNet"), "cannot generate under the TTS"),
    (["--fs=0"], None, None, "--fs must be > 0 (got 0)"),
    (["--fs=16k"], None, None, "--fs and --batch-size must be integers"),
    (["--spectrogram", "--fs=192000"], None, None, "at most 4096 points are supported"),
    (["--batch-size=0"], None, None, "--batch-size must be >= 1 (got 0)"),
    ([], lambda: TH.acoustic_hp(subphone_features="coarse_coding"), None,
     "hp.subphone_features must be \"full\" (got 'coarse_coding')"),
    ([], lambda: TH.acoustic_hp(subphone_features=None), None, "hp.subphone_features must be \"full\" (got None)"),
    ([], lambda: TH.acoustic_hp(add_frame_features=False), None, "hp.add_frame_features must be True"),
    ([], lambda: TH.acoustic_hp(use_phone_alignment=True), None, "the acoustic hp.use_phone_alignment=True"),
    ([], None, lambda: TH.duration_hp(use_phone_alignment=True), "the duration hp.use_phone_alignment=True"),
    ([], None, lambda: TH.duration_hp(stream_sizes=[3]), "5 state columns but hp_duration.stream_sizes totals 3"),
])
def test_command_refusals(data_dir, tmp_path, argv, hp_a, hp_d, needle):
    out = str(tmp_path / "out")
    with pytest.raises(SystemExit) as e:
        _main(data_dir, out, argv, hp_a() if hp_a else None, hp_d() if hp_d else None)
    assert str(e.value).startswith("gantts_b200.synthesize: ") and needle in str(e.value), str(e.value)
    assert not os.path.exists(out)


def test_command_refuses_mismatched_statistics(tmp_path):
    data = TH.write_tts_data(str(tmp_path / "data"), n_files=8)
    p = os.path.join(data, "X_acoustic_data_min.npy")
    np.save(p, np.load(p)[:-1])
    with pytest.raises(SystemExit) as e:
        _main(data, str(tmp_path / "out"))
    assert "the acoustic input statistics have %d columns but the duration ones %d" % (TH.L_PHONE + 8, TH.L_PHONE) \
        in str(e.value), str(e.value)
    p = os.path.join(data, "Y_duration_data_mean.npy")
    np.save(p, np.zeros(17))
    with pytest.raises(SystemExit, match="S = 17 states per phone must be in"):
        _main(data, str(tmp_path / "out"), hp_d=TH.duration_hp(stream_sizes=[17], has_dynamic_features=[False]))


def test_command_refuses_missing_phone_files(tmp_path):
    from gantts_b200 import synthesize
    data = TH.write_tts_data(str(tmp_path / "data"), n_files=8)
    (_, names), (_, test_names) = synthesize.utterance_names(data)
    assert len(test_names) == 5 and names
    os.remove(os.path.join(data, "Y_duration", test_names[2] + ".npy"))
    out = str(tmp_path / "out")
    with pytest.raises(SystemExit) as e:
        _main(data, out, ["--disable-duraton-gen"])
    assert "test split: %s has no Y_duration/%s.npy" % (test_names[2], test_names[2]) in str(e.value)
    os.remove(os.path.join(data, "X_duration", names[0] + ".npy"))
    with pytest.raises(SystemExit) as e:
        _main(data, out)
    assert "eval split: %s has no X_duration/%s.npy" % (names[0], names[0]) in str(e.value)
    assert not os.path.exists(out)


def test_utterances_are_get_lab_files_picks(tmp_path):
    from gantts_b200 import generate, synthesize
    data = TH.write_tts_data(str(tmp_path / "data"), n_files=12)
    got = synthesize.utterance_names(data)
    want = generate.utterance_files(os.path.join(data, "X_acoustic"))
    assert [s for s, _ in got] == ["eval", "test"]
    for (_, names), (_, files) in zip(got, want):
        assert names == [os.path.splitext(os.path.basename(f))[0] for f in files]


def test_prepared_directory_holds_the_expansion(tmp_path):
    data = TH.write_tts_data(str(tmp_path / "data"), n_files=4)
    for n in sorted(os.listdir(os.path.join(data, "X_acoustic"))):
        x, d = (np.load(os.path.join(data, k, n)) for k in ("X_duration", "Y_duration"))
        xa = np.load(os.path.join(data, "X_acoustic", n))
        assert xa.shape == (int(d.sum()), TH.L_PHONE + 9) and np.array_equal(xa, merlin_port.expand(x, d))
    assert np.load(os.path.join(data, "X_acoustic_data_min.npy")).dtype == np.float32
