"""Spectral post-processing of generation on the GPU: gantts_mcep_postfilter (Merlin's post filter) and gantts_mcep_to_sp
(mc2sp) against the literal per-frame chain of oracle.sptk_port on ragged batches, zeros beyond each length, each row bit
for bit equal to its utterance alone, ParameterGenerator's post_filter / spectrogram against the unflagged output followed
by the chain, and the command's files."""
import os

import numpy as np
import pytest
import torch

from oracle import sptk_port as sp
import train_cli_helpers as H

pytestmark = pytest.mark.gpu

FS = (16000, 22050, 48000)
LENS = [300, 1, 33, 32, 64, 257, 150]      # B = 7: a full row, one frame, the 32-frame tile edges, T - 43


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__
    __graft_entry__.build()
    return torch.device("cuda:0")


def _batch(lens, M1, seed, pad_cols=3):
    """A padded batch of mel-cepstra shaped like generated mgc, junk beyond each length, as a column slice of a wider
    array (the mgc columns of the acoustic features)."""
    rng = np.random.RandomState(seed)
    B, T = len(lens), max(lens)
    x = rng.randn(B, T, M1 + pad_cols) * 3.0
    x[..., :M1] = rng.randn(B, T, M1) * np.exp(-0.1 * np.arange(M1))
    x[..., 0] = rng.uniform(-2.0, 2.0, (B, T))
    for b, L in enumerate(lens):
        x[b, L:, :M1] = rng.randn(T - L, M1) * 5.0
    return x.astype(np.float32)


def _check_mgc(got, want):
    np.testing.assert_allclose(got, want, rtol=1e-6, atol=1e-6)


def _check_sp(got, want):
    assert np.all(np.abs(got - want) <= 2e-6 * np.abs(want)), float(np.max(np.abs(got / want - 1)))


def _run(kind, x, lens, alpha, fftlen, M1, dev):
    from gantts_b200 import ops
    xt = torch.from_numpy(x).to(dev)[..., :M1]
    lengths = torch.tensor(lens, dtype=torch.int64, device=dev)
    if kind == "postfilter":
        return ops.mcep_postfilter(xt, lengths, alpha).cpu().numpy()
    return ops.mc2sp(xt, lengths, alpha, fftlen).cpu().numpy()


@pytest.mark.parametrize("fs,M1", [(fs, 60) for fs in FS] + [(48000, 1), (48000, 128)])     # mgc width, its edges
@pytest.mark.parametrize("kind", ["postfilter", "mc2sp"])
def test_kernels_vs_the_chain_frame_by_frame(dev, fs, kind, M1):
    from gantts_b200 import generate
    alpha, fftlen = generate.mcep_alpha(fs), generate.cheaptrick_fft_size(fs)
    x = _batch(LENS, M1, seed=fs + M1)
    got = _run(kind, x, LENS, alpha, fftlen, M1, dev)
    B, T = len(LENS), max(LENS)
    assert got.shape == ((B, T, M1) if kind == "postfilter" else (B, T, fftlen // 2 + 1))
    assert got.dtype == np.float32
    valid = np.concatenate([x[b, :L, :M1] for b, L in enumerate(LENS)]).astype(np.float64)
    want = sp.merlin_post_filter(valid, alpha) if kind == "postfilter" else sp.mc2sp(valid, alpha, fftlen)
    (_check_mgc if kind == "postfilter" else _check_sp)(np.concatenate([got[b, :L] for b, L in enumerate(LENS)]), want)
    for b, L in enumerate(LENS):
        assert not got[b, L:].any(), "frames at or beyond the length must be exactly 0"
        alone = _run(kind, np.ascontiguousarray(x[b:b + 1, :L]), [L], alpha, fftlen, M1, dev)
        assert np.array_equal(alone[0], got[b, :L]), (b, L)


def test_postfilter_coef(dev):
    from gantts_b200 import generate, ops
    alpha = generate.mcep_alpha(16000)
    x = _batch(LENS, 60, seed=3)
    xt, lengths = torch.from_numpy(x).to(dev)[..., :60], torch.tensor(LENS, dtype=torch.int64, device=dev)
    valid = np.concatenate([x[b, :L, :60] for b, L in enumerate(LENS)]).astype(np.float64)
    for coef in (1.0, 0.7, 2.0):
        got = ops.mcep_postfilter(xt, lengths, alpha, coef).cpu().numpy()
        _check_mgc(np.concatenate([got[b, :L] for b, L in enumerate(LENS)]), sp.merlin_post_filter(valid, alpha,
                                                                                                    coef=coef))


def _acoustic_setup(dev, seed=7):
    from gantts_b200 import models
    torch.manual_seed(seed)
    rng = np.random.RandomState(seed)
    hp = H.tts_acoustic_hp()
    model = models.MLP(20, 187, 2, 32, dropout=0.0, last_sigmoid=False).to(dev)
    mean, std = 0.2 * rng.randn(187), 0.05 + 0.2 * rng.rand(187)
    mean[0], std[0] = 1.0, 0.5
    mean[183], std[183] = 0.5, 0.5
    stats = {"X_min": np.zeros(20), "X_max": np.ones(20), "Y_mean": mean, "Y_std": std}
    arrays = [rng.rand(n, 20).astype(np.float32) for n in (40, 3, 77, 1, 65, 32)]
    return hp, model, stats, arrays


@pytest.mark.parametrize("fs", [16000, 48000])
def test_generate_utterances_with_post_filter_and_spectrogram(dev, fs):
    from gantts_b200 import generate
    hp, model, stats, arrays = _acoustic_setup(dev)
    plain = generate.ParameterGenerator(model, hp, stats).generate_utterances(arrays, 4)
    flagged = generate.ParameterGenerator(model, hp, stats, post_filter=True, spectrogram=True,
                                          fs=fs).generate_utterances(arrays, 4)
    alpha, fftlen = generate.mcep_alpha(fs), generate.cheaptrick_fft_size(fs)
    for a, p, f in zip(arrays, plain, flagged):
        assert list(p) == list(generate.OUTPUT_NAMES["acoustic"])                 # unflagged: unchanged keys
        assert list(f) == list(generate.OUTPUT_NAMES["acoustic"]) + [generate.SPECTROGRAM_NAME]
        for k in ("lf0", "vuv", "bap", "f0"):
            assert np.array_equal(f[k], p[k]), k
        mgc = sp.merlin_post_filter(p["mgc"].astype(np.float64), alpha)
        _check_mgc(f["mgc"], mgc)
        assert f["sp"].shape == (len(a), fftlen // 2 + 1) and f["sp"].dtype == np.float32
        _check_sp(f["sp"], sp.mc2sp(mgc, alpha, fftlen))
    # spectrogram alone: the envelope of the unfiltered mgc, which stays as it was
    only_sp = generate.ParameterGenerator(model, hp, stats, spectrogram=True, fs=fs).generate_utterances(arrays, 4)
    for p, s in zip(plain, only_sp):
        assert np.array_equal(s["mgc"], p["mgc"])
        _check_sp(s["sp"], sp.mc2sp(p["mgc"].astype(np.float64), alpha, fftlen))


def test_command_writes_filtered_mgc_and_sp(dev, tmp_path):
    from gantts_b200 import generate, train
    hp, model, stats, _ = _acoustic_setup(dev, seed=9)
    root = str(tmp_path / "data")
    xd = os.path.join(root, "X_acoustic")
    os.makedirs(xd)
    rng = np.random.RandomState(9)
    for i in range(12):
        np.save(os.path.join(xd, "utt%03d.npy" % i), rng.rand(int(rng.randint(5, 90)), 20).astype(np.float32))
    for k, v in (("X_acoustic_data_min", stats["X_min"]), ("X_acoustic_data_max", stats["X_max"]),
                 ("Y_acoustic_data_mean", stats["Y_mean"]), ("Y_acoustic_data_var", stats["Y_std"] ** 2)):
        np.save(os.path.join(root, k + ".npy"), v)
    ck = str(tmp_path / "ck")
    os.makedirs(ck)
    train.save_checkpoint(model, torch.optim.Adagrad(model.parameters()), 2, ck, "Generator")
    ckpt = os.path.join(ck, "checkpoint_epoch2_Generator.pth")
    hpc = lambda: H.tts_acoustic_hp(generator_params={"in_dim": 20, "out_dim": 187, "num_hidden": 2, "hidden_dim": 32,
                                                      "dropout": 0.0, "last_sigmoid": False})
    dst, dst_plain = str(tmp_path / "gen"), str(tmp_path / "gen_plain")
    assert generate.main(["--batch-size=5", "--post-filter", "--spectrogram", "--fs=22050", ckpt, xd, dst], hp=hpc()) == 0
    assert generate.main(["--batch-size=5", ckpt, xd, dst_plain], hp=hpc()) == 0
    st = generate.load_stats(hpc(), root)
    pg = generate.ParameterGenerator(model, hpc(), st)
    alpha, fftlen = generate.mcep_alpha(22050), generate.cheaptrick_fft_size(22050)
    for sub, files in generate.utterance_files(xd):
        want = pg.generate_utterances([np.load(f) for f in files], 5)
        for f, w in zip(files, want):
            name = os.path.splitext(os.path.basename(f))[0] + ".npz"
            got, plain = np.load(os.path.join(dst, sub, name)), np.load(os.path.join(dst_plain, sub, name))
            assert sorted(plain.files) == sorted(generate.OUTPUT_NAMES["acoustic"])
            assert sorted(got.files) == sorted(generate.OUTPUT_NAMES["acoustic"] + ("sp",))
            for k in plain.files:
                assert np.array_equal(plain[k], w[k]), k
            mgc = sp.merlin_post_filter(w["mgc"].astype(np.float64), alpha)
            _check_mgc(got["mgc"], mgc)
            _check_sp(got["sp"], sp.mc2sp(mgc, alpha, fftlen))
