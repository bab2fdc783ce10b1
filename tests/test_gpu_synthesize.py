"""TTS synthesis with predicted durations on the GPU (gantts_b200.synthesize): gantts_state_frame_offsets and
gantts_expand_state_frames against the per-phone restatement (oracle.merlin_port) bit for bit on ragged batches, the
status word on bad durations, natural durations against generate.normalize_input of the prepared X_acoustic,
Synthesizer against the per-utterance chain of evaluation_tts.py's tts_from_label, and the command end to end."""
import os

import numpy as np
import pytest
import torch

from conftest import rel_err
from oracle import merlin_port
import tts_data_helpers as TH

pytestmark = pytest.mark.gpu

TOL = 2e-4          # test_gpu_generate's tolerance
NAN = float("nan")


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__
    __graft_entry__.build()
    return torch.device("cuda:0")


def _batch(rng, lens, L, S, mode):
    """Ragged phone rows and durations, padding poisoned with NaN.  mode: random 1..8, ones, long (500-frame states)."""
    B, P = len(lens), max(lens)
    x = np.full((B, P, L), NAN, np.float32)
    d = np.full((B, P, S), NAN, np.float32)
    for b, n in enumerate(lens):
        x[b, :n] = rng.randn(n, L) * 3
        if mode == "ones":
            d[b, :n] = 1
        elif mode == "long":
            d[b, :n] = 500
            d[b, :n, rng.randint(S)] = 1
        else:
            d[b, :n] = TH.random_durations(rng, n, S)
    return x, d


def _run(dev, x, d, lens, T_pad=0, scale=None, min_=None, views=False):
    from gantts_b200 import _lib, ops
    B, P, L = x.shape
    W = L + _lib.SUBPHONE_FEATURES
    if views:                                   # batch and phone strides of a wider tensor, as a generator's output
        xw = np.full((B, P + 1, L + 3), NAN, np.float32)
        xw[:, :P, 1:L + 1] = x
        dw = np.full((B, P, d.shape[2] + 2), NAN, np.float32)
        dw[:, :, :d.shape[2]] = d
        xt = torch.from_numpy(xw).to(dev)[:, :P, 1:L + 1]
        dt = torch.from_numpy(dw).to(dev)[:, :, :d.shape[2]]
        assert not xt.is_contiguous() and not dt.is_contiguous()
    else:
        xt, dt = torch.from_numpy(x).to(dev), torch.from_numpy(d).to(dev)
    pl = torch.tensor(lens, dtype=torch.int64, device=dev)
    offsets, fl, fl_host = ops.state_frame_offsets(dt, pl)
    T = int(fl_host.max()) + T_pad
    scale = np.ones(W, np.float32) if scale is None else scale
    min_ = np.zeros(W, np.float32) if min_ is None else min_
    out = ops.expand_state_frames(xt, dt, offsets, fl, torch.from_numpy(scale).to(dev), torch.from_numpy(min_).to(dev),
                                  T)
    return offsets.cpu().numpy(), fl.cpu().numpy(), fl_host, out.cpu().numpy()


CASES = [  # P, S, L, durations, lengths of the other rows as fractions of P
    (1, 5, 416, "random"), (1, 5, 7, "long"), (2, 3, 1, "long"), (2, 5, 416, "ones"), (37, 5, 416, "random"),
    (37, 3, 7, "random"), (37, 5, 1, "ones"), (300, 5, 416, "random"), (300, 3, 7, "ones"), (300, 5, 1, "random"),
]


def _lens(P):
    return sorted({P, max(1, P // 2), 1, max(1, P - 1)}, reverse=True) + [max(1, P // 3)]


@pytest.mark.parametrize("P,S,L,mode", CASES)
def test_kernels_against_the_oracle(dev, P, S, L, mode):
    rng = np.random.RandomState(P * 100 + S * 10 + L)
    lens = _lens(P)
    x, d = _batch(rng, lens, L, S, mode)
    offsets, fl, fl_host, out = _run(dev, x, d, lens, T_pad=5, views=(P == 37))
    B, T, W = out.shape
    assert W == L + 9 and np.array_equal(fl, fl_host)
    for b, n in enumerate(lens):
        N = d[b, :n].sum(axis=1).astype(np.int64)
        want_off = np.concatenate([[0], np.cumsum(N), np.full(P - n, N.sum())])
        assert np.array_equal(offsets[b], want_off), b                    # offsets and lengths exact
        assert fl[b] == N.sum()
        want = merlin_port.expand(x[b, :n], d[b, :n])
        assert np.array_equal(out[b, :fl[b]].view(np.int32), want.view(np.int32)), (b, n)
        assert not out[b, fl[b]:].view(np.int32).any(), "0 at and beyond the frame length"


@pytest.mark.parametrize("P,S,L,mode", [(37, 5, 416, "random"), (300, 3, 7, "random"), (2, 5, 1, "long")])
def test_rows_are_independent_of_the_batch(dev, P, S, L, mode):
    rng = np.random.RandomState(P + S + L)
    lens = _lens(P)
    x, d = _batch(rng, lens, L, S, mode)
    W = L + 9
    scale = (rng.rand(W) * 2 + 0.01).astype(np.float32)
    min_ = rng.randn(W).astype(np.float32)
    _, fl, _, out = _run(dev, x, d, lens, scale=scale, min_=min_)
    for b, n in enumerate(lens):
        # normalised in float32 as generate.normalize_input does on float32 statistics
        want = merlin_port.expand(x[b, :n], d[b, :n]) * scale + min_
        assert want.dtype == np.float32
        assert np.array_equal(out[b, :fl[b]].view(np.int32), want.view(np.int32)), b
        _, _, _, alone = _run(dev, x[b:b + 1, :n].copy(), d[b:b + 1, :n].copy(), [n], scale=scale, min_=min_)
        assert np.array_equal(alone[0].view(np.int32), out[b, :fl[b]].view(np.int32)), b
    # reversed batch, 7 more padding phones of junk and 300 more padded frames
    rev = lens[::-1]
    xr, dr = _batch(rng, [P + 7] * len(lens), L, S, mode)
    for j, b in enumerate(range(len(lens) - 1, -1, -1)):
        xr[j, :lens[b]], dr[j, :lens[b]] = x[b, :lens[b]], d[b, :lens[b]]
    _, flr, _, outr = _run(dev, xr, dr, rev, T_pad=300, scale=scale, min_=min_)
    for j, b in enumerate(range(len(lens) - 1, -1, -1)):
        assert flr[j] == fl[b]
        assert np.array_equal(outr[j, :fl[b]].view(np.int32), out[b, :fl[b]].view(np.int32)), b
        assert not outr[j, fl[b]:].any()


@pytest.mark.parametrize("bad", [NAN, 0.0, -3.0, 2.5, float("inf"), float(1 << 25)])
def test_bad_duration_raises(dev, bad):
    from gantts_b200 import ops
    d = np.full((3, 4, 5), 2.0, np.float32)
    d[:, 3] = NAN                                                        # padding: never read
    d[1, 2, 3] = bad
    pl = torch.tensor([3, 3, 2], dtype=torch.int64, device=dev)
    with pytest.raises(RuntimeError, match=r"state_frame_offsets: a state duration is not a finite integer in "
                                           r"\[1, 16777216\]"):
        ops.state_frame_offsets(torch.from_numpy(d).to(dev), pl)
    d[1, 2, 3] = 2.0
    offsets, fl, host = ops.state_frame_offsets(torch.from_numpy(d).to(dev), pl)
    assert list(host) == [30, 30, 20]
    torch.cuda.synchronize()


def test_too_many_frames_raises(dev):
    from gantts_b200 import ops
    d = torch.full((2, 3, 1), float(1 << 23), device=dev)
    pl = torch.tensor([2, 3], dtype=torch.int64, device=dev)
    with pytest.raises(RuntimeError, match=r"a row has more than 16777216 frames \(max 25165824\)"):
        ops.state_frame_offsets(d, pl)
    offsets, fl, host = ops.state_frame_offsets(d, torch.tensor([2, 1], dtype=torch.int64, device=dev))
    assert list(host) == [1 << 24, 1 << 23]


# ---- against the prepared data ----

@pytest.fixture(scope="module")
def data(tmp_path_factory):
    return TH.write_tts_data(str(tmp_path_factory.mktemp("tts") / "data"), n_files=14)


def _load(data, sub, names):
    return [np.load(os.path.join(data, sub, n + ".npy")) for n in names]


def _names(data):
    return sorted(os.path.splitext(f)[0] for f in os.listdir(os.path.join(data, "X_acoustic")))


def _stats(data):
    from gantts_b200 import generate
    return generate.load_stats(TH.duration_hp(), data), generate.load_stats(TH.acoustic_hp(), data)


def _synth(dev, data, seed=0, **kw):
    from gantts_b200 import generate, models, synthesize
    hp_a, hp_d = TH.srurnn_hps()
    sd, sa = _stats(data)
    generate.derive_dims(hp_a, sa), generate.derive_dims(hp_d, sd)
    torch.manual_seed(seed)
    md = models.SRURNN(**hp_d.generator_params).to(dev)
    ma = models.SRURNN(**hp_a.generator_params).to(dev)
    return synthesize.Synthesizer(md, ma, hp_d, hp_a, sd, sa, **kw), (md, ma, hp_d, hp_a, sd, sa)


def test_natural_durations_give_normalize_input_bits(dev, data):
    from gantts_b200 import generate, ops
    syn, _ = _synth(dev, data)
    names = _names(data)
    X, D, XA = _load(data, "X_duration", names), _load(data, "Y_duration", names), _load(data, "X_acoustic", names)
    hp_a, (sd, sa) = TH.acoustic_hp(), _stats(data)
    assert sa["X_min"].dtype == np.float32
    lens = [len(a) for a in X]
    B, P = len(X), max(lens)
    xb = np.zeros((B, P, TH.L_PHONE), np.float32)
    db = np.full((B, P, TH.S_STATES), NAN, np.float32)
    for b in range(B):
        xb[b, :lens[b]], db[b, :lens[b]] = X[b], D[b]
    pl = torch.tensor(lens, dtype=torch.int64, device=dev)
    xt, dt = torch.from_numpy(xb).to(dev), torch.from_numpy(db).to(dev)
    offsets, fl, host = ops.state_frame_offsets(dt, pl)
    out = ops.expand_state_frames(xt, dt, offsets, fl, syn.scale_a, syn.min_a, int(host.max())).cpu().numpy()
    for b in range(B):
        want = generate.normalize_input(XA[b], hp_a, sa)
        assert host[b] == len(XA[b])
        assert np.array_equal(out[b, :host[b]].view(np.int32), want.view(np.int32)), names[b]
    # the duration model's inputs, scaled on the device
    xd = syn.duration_inputs(xt, pl).cpu().numpy()
    for b in range(B):
        want = generate.normalize_input(X[b], TH.duration_hp(), sd)
        assert np.array_equal(xd[b, :lens[b]].view(np.int32), want.view(np.int32)), names[b]
        assert not xd[b, lens[b]:].any()


def _unrounded_durations(pg, x, dev):
    """The duration model's de-normalised output for one normalised utterance at B = 1, before rounding."""
    from gantts_b200 import ops
    xt = torch.from_numpy(x[None]).to(dev)
    l = torch.tensor([len(x)], dtype=torch.int64, device=dev)
    with torch.no_grad():
        y = ops.mlpg_ragged(pg._generator_output(xt, l), l, pg.windows, pg.entries, pg.ncols, var=pg.var,
                            in_affine=pg.in_affine, out_affine=pg.out_affine)
    return y[0].cpu().numpy().astype(np.float64)


@pytest.mark.parametrize("mge,post", [(True, False), (False, True)])
def test_synthesizer_against_the_per_utterance_chain(dev, data, mge, post):
    from gantts_b200 import generate
    syn, (md, ma, hp_d, hp_a, sd, sa) = _synth(dev, data, seed=3, mge_training=mge, post_filter=post,
                                              spectrogram=post)
    names = _names(data)
    X = _load(data, "X_duration", names)
    got = syn.synthesize_utterances(X, 5)
    pa = syn.gen_acoustic
    compared = 0
    for n, x, g in zip(names, X, got):
        assert g["duration"].shape == (len(x), TH.S_STATES)
        # the chain: duration generate at B = 1, durations to the host, the restated expansion and normalize_input in
        # numpy, acoustic generate at B = 1
        raw = _unrounded_durations(syn.gen_duration, generate.normalize_input(x, hp_d, sd), dev)
        want_d = np.round(raw)
        want_d[want_d <= 0] = 1
        near = np.abs(np.abs(raw - np.floor(raw)) - 0.5) < 1e-4
        assert np.array_equal(g["duration"][~near], want_d[~near]), n
        if not np.array_equal(g["duration"], want_d):
            continue                                                     # a duration on a rounding boundary
        xa = generate.normalize_input(merlin_port.expand(x, want_d), hp_a, sa)
        want = pa.generate_utterances([merlin_port.expand(x, want_d)], 1)[0]
        assert sorted(g) == sorted(["duration"] + list(want))
        for k, w in want.items():
            assert g[k].shape == w.shape, (n, k)
            if k == "vuv":
                near_v = np.abs(w - 0.5) < 1e-4
                assert np.array_equal((g[k] >= 0.5)[~near_v], (w >= 0.5)[~near_v])
            if k != "f0":
                assert rel_err(g[k], w) <= TOL, (n, k, rel_err(g[k], w))
        assert len(xa) == int(want_d.sum())
        compared += 1
    assert compared >= len(names) - 2


def _checkpoints(tmp_path, dev, data, seed=5):
    from gantts_b200 import train
    _, (md, ma, _, _, _, _) = _synth(dev, data, seed=seed)
    ck = str(tmp_path / "ck")
    os.makedirs(ck)
    paths = []
    for m, tag in ((ma, "Acoustic"), (md, "Duration")):
        train.save_checkpoint(m, torch.optim.Adagrad(m.parameters()), 1, ck, tag)
        paths.append(os.path.join(ck, "checkpoint_epoch1_%s.pth" % tag))
    return paths


def test_command_with_natural_durations_matches_generate(dev, data, tmp_path):
    from gantts_b200 import generate, synthesize
    ck_a, ck_d = _checkpoints(tmp_path, dev, data)
    dst = str(tmp_path / "syn")
    hp_a, hp_d = TH.srurnn_hps()
    assert synthesize.main(["--disable-duraton-gen", "--batch-size=4", ck_a, ck_d, data, dst],
                           hp_acoustic=hp_a, hp_duration=hp_d) == 0
    gen = str(tmp_path / "gen")
    assert generate.main(["--hparams_name=tts_acoustic", "--batch-size=4", ck_a, os.path.join(data, "X_acoustic"), gen],
                         hp=TH.srurnn_hps()[0]) == 0
    for sub, names in synthesize.utterance_names(data):
        assert sorted(os.listdir(os.path.join(dst, sub))) == sorted(n + ".npz" for n in names)
        for n in names:
            s, g = np.load(os.path.join(dst, sub, n + ".npz")), np.load(os.path.join(gen, sub, n + ".npz"))
            assert sorted(s.files) == sorted(["duration"] + list(g.files))
            assert np.array_equal(s["duration"], np.load(os.path.join(data, "Y_duration", n + ".npy")))
            for k in g.files:
                assert s[k].shape == g[k].shape and rel_err(s[k], g[k]) <= TOL, (sub, n, k)


@pytest.mark.parametrize("extra", [[], ["--post-filter", "--spectrogram"]])
def test_command_with_predicted_durations(dev, data, tmp_path, extra):
    from gantts_b200 import synthesize
    ck_a, ck_d = _checkpoints(tmp_path, dev, data)
    dst = str(tmp_path / "syn")
    hp_a, hp_d = TH.srurnn_hps()
    assert synthesize.main(extra + [ck_a, ck_d, data, dst], hp_acoustic=hp_a, hp_duration=hp_d) == 0
    keys = sorted(["bap", "duration", "f0", "lf0", "mgc", "vuv"] + (["sp"] if extra else []))
    for sub, names in synthesize.utterance_names(data):
        assert sorted(os.listdir(os.path.join(dst, sub))) == sorted(n + ".npz" for n in names)
        for n in names:
            z = np.load(os.path.join(dst, sub, n + ".npz"))
            P = len(np.load(os.path.join(data, "X_duration", n + ".npy")))
            assert sorted(z.files) == keys
            d = z["duration"]
            assert d.shape == (P, TH.S_STATES) and d.dtype == np.float32
            assert np.all(d >= 1) and np.array_equal(d, np.round(d))
            T = int(d.sum())
            assert z["mgc"].shape == (T, 60) and z["lf0"].shape == (T, 1) and z["vuv"].shape == (T,)
            assert z["bap"].shape == (T, 1) and z["f0"].shape == (T, 1)
            if extra:
                assert z["sp"].shape == (T, 513) and np.all(z["sp"] > 0)
            assert all(np.isfinite(z[k]).all() for k in keys)
