"""The objective measures on the GPU (gantts_modspec, gantts_global_variance, gantts_b200.objective): both kernels against
the fp64 restatement of the notebooks' definitions (objective_oracle) on ragged batches, padding that is never read,
a column's bits independent of its batch position, padded length and neighbours, the running sum in row order, means
with the same bits for any batch size, and the command end to end against generate_utterances and the restatement."""
import os

import numpy as np
import pytest
import torch

import objective_oracle as ref
import train_cli_helpers as H

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__
    __graft_entry__.build()
    return torch.device("cuda:0")


def _batch(rng, lens, D, T=None, pad=0.0):
    """(B, T, D) float32 with mgc-like columns (an offset and a scale per column, a slow drift) and `pad` beyond each
    length."""
    T = T or max(max(lens), 1)
    x = np.full((len(lens), T, D), pad, dtype=np.float32)
    for b, L in enumerate(lens):
        t = np.arange(L)[:, None]
        x[b, :L] = (rng.randn(L, D) * rng.uniform(0.1, 2.0, D) + rng.randn(D) * 3
                    + np.sin(t * rng.uniform(0.001, 0.2, D)))
    return x


def _run(dev, x, lens, n, out_sum=None):
    from gantts_b200 import ops
    xt = torch.from_numpy(x).to(dev) if isinstance(x, np.ndarray) else x
    lengths = torch.tensor(lens, dtype=torch.int64, device=dev)
    ms = ops.modspec(xt, lengths, n, out_sum=out_sum)
    gv = ops.global_variance(xt, lengths)
    return ms.cpu().numpy(), gv.cpu().numpy()


def check_ms(got_log, x, n):
    """got_log (K, D) against log_modspec(x, n): the power within 1e-9 of the column's largest power; the log power
    within 1e-6 wherever the power is above 1e-3 of the column's largest."""
    want = ref.modspec(x, n)
    peak = want.max(axis=0, keepdims=True)
    assert got_log.shape == want.shape
    assert np.all(np.abs(np.exp(got_log) - want) <= 1e-9 * peak)
    big = want > 1e-3 * peak
    assert np.all(np.abs(got_log - np.log(want))[big] <= 1e-6)


def check_gv(got, x):
    want = ref.global_variance(x)
    assert np.all(np.abs(got - want) <= 1e-12 * np.abs(want))


@pytest.mark.parametrize("n", [64, 4096, 8192])
@pytest.mark.parametrize("D", [1, 7, 59, 60])
def test_kernels_against_the_definitions(dev, n, D):
    rng = np.random.RandomState(n + D)
    lens = [1, 2, n - 1, n, n + 1, 3 * n + 5, 0]
    x = _batch(rng, lens, D)
    ms, gv = _run(dev, x, lens, n)
    assert ms.shape == (len(lens), n // 2 + 1, D) and ms.dtype == np.float64 and gv.shape == (len(lens), D)
    for b, L in enumerate(lens[:-1]):
        check_ms(ms[b], x[b, :L], n)
        check_gv(gv[b], x[b, :L])
    assert np.all(ms[-1] == -np.inf) and np.all(np.isnan(gv[-1]))      # no frames: np.log(0), np.var of nothing


def test_silent_and_constant_columns(dev):
    x = np.zeros((1, 9, 3), np.float32)
    x[0, :, 1] = 2.5
    x[0, :, 2] = np.arange(9)
    ms, gv = _run(dev, x, [9], 64)
    assert np.all(ms[0, :, 0] == -np.inf) and np.isfinite(ms[0, :, 1:]).all()
    assert np.array_equal(gv[0, :2], [0.0, 0.0])
    check_ms(ms[0, :, 1:], x[0, :, 1:], 64)
    check_gv(gv[0], x[0])


def test_lengths_are_clamped(dev):
    rng = np.random.RandomState(4)
    x = _batch(rng, [50, 50], 5)
    ms, gv = _run(dev, x, [-3, 10 ** 6], 64)
    assert np.all(ms[0] == -np.inf) and np.all(np.isnan(gv[0]))
    check_ms(ms[1], x[1], 64)
    check_gv(gv[1], x[1])


@pytest.mark.parametrize("n", [64, 4096])
def test_padding_is_never_read(dev, n):
    rng = np.random.RandomState(7)
    lens = [30, 1, n + 3, 200]
    x = _batch(rng, lens, 7, T=max(lens) + 40)
    y = x.copy()
    for b, L in enumerate(lens):
        y[b, L:] = np.nan
    a, b_ = _run(dev, x, lens, n), _run(dev, y, lens, n)
    assert np.array_equal(a[0], b_[0]) and np.array_equal(a[1], b_[1])
    assert np.isfinite(b_[0]).all() and np.isfinite(b_[1]).all()


def test_rows_and_columns_are_independent_bitwise(dev):
    rng = np.random.RandomState(9)
    n, D = 4096, 60
    lens = [900, 17, 4500, 333, 1]
    x = _batch(rng, lens, D)
    ms, gv = _run(dev, x, lens, n)
    # each row alone, at its own length, and at another position of a batch with another padded length
    for b, L in enumerate(lens):
        alone = _run(dev, np.ascontiguousarray(x[b:b + 1, :L]), [L], n)
        assert np.array_equal(alone[0][0], ms[b]) and np.array_equal(alone[1][0], gv[b])
        other = _batch(rng, [L + 77, 5, 12], D, T=max(L, 12) + 500, pad=3.0)
        other[1, :L] = x[b, :L]
        got = _run(dev, other, [L + 77, L, 12], n)
        assert np.array_equal(got[0][1], ms[b]) and np.array_equal(got[1][1], gv[b])
    # columns permuted, and a column slice read in place through its strides
    perm = rng.permutation(D)
    pm = _run(dev, np.ascontiguousarray(x[:, :, perm]), lens, n)
    assert np.array_equal(pm[0], ms[:, :, perm]) and np.array_equal(pm[1], gv[:, perm])
    wide = np.concatenate([rng.randn(len(lens), x.shape[1], 3).astype(np.float32), x,
                           rng.randn(len(lens), x.shape[1], 120).astype(np.float32)], axis=2)
    view = torch.from_numpy(wide).to(dev)[:, :, 3:3 + D]
    assert not view.is_contiguous()
    sl = _run(dev, view, lens, n)
    assert np.array_equal(sl[0], ms) and np.array_equal(sl[1], gv)


def test_running_sum_adds_rows_in_order(dev):
    rng = np.random.RandomState(11)
    n, D = 512, 7
    lens = [300, 20, 511, 64, 2]
    x = _batch(rng, lens, D)
    base = rng.randn(n // 2 + 1, D)
    out_sum = torch.from_numpy(base.copy()).to(dev)
    ms, _ = _run(dev, x, lens, n, out_sum=out_sum)
    want = base.copy()
    for b in range(len(lens)):
        want = want + ms[b]
    assert np.array_equal(out_sum.cpu().numpy(), want)
    from gantts_b200 import ops
    with pytest.raises(RuntimeError, match="out_sum must be a contiguous float64"):
        ops.modspec(torch.from_numpy(x).to(dev), torch.tensor(lens, device=dev), n,
                    out_sum=torch.zeros(n // 2, D, dtype=torch.float64, device=dev))


def _fixed_arrays(rng, lens, D):
    return [_batch(rng, [L], D)[0] for L in lens]


def test_means_have_the_same_bits_for_any_batch_size(dev):
    from gantts_b200 import objective
    rng = np.random.RandomState(13)
    lens = list(rng.randint(1, 700, 37)) + [300, 300, 5]
    Y = _fixed_arrays(rng, lens, 60 * 3)
    hp = H.tts_acoustic_hp()
    runs = {bs: objective.split_stats(hp, [], None, Y, bs, 4096, dev)[0] for bs in (1, 3, 20)}
    gv, gv_mean, ms_mean = runs[1]
    for bs in (3, 20):
        for a, b in zip(runs[bs], runs[1]):
            assert np.array_equal(a, b), bs
    assert gv.shape == (len(lens), 60)
    for i, y in enumerate(Y):
        check_gv(gv[i], y[:, :60])
    want_gv = np.mean([ref.global_variance(y[:, :60]) for y in Y], axis=0)
    assert np.all(np.abs(gv_mean - want_gv) <= 1e-12 * want_gv)
    logs = [ref.modspec(y[:, :60], 4096) for y in Y]
    want_ms = np.mean([np.log(p) for p in logs], axis=0)
    big = np.all([p > 1e-3 * p.max(axis=0, keepdims=True) for p in logs], axis=0)
    assert np.all(np.abs(ms_mean - want_ms)[big] <= 1e-6)


def test_feature_stats_refuses_another_width(dev):
    from gantts_b200 import objective
    fs = objective.FeatureStats(4, 64, dev)
    with pytest.raises(RuntimeError, match="FeatureStats of D = 4 columns"):
        fs.add(torch.zeros(2, 5, 3, device=dev), torch.tensor([5, 5], device=dev))
    with pytest.raises(RuntimeError, match="no utterances"):
        fs.result()


def _expected(pg, files, yfiles, n, cols, key, batch_size):
    """gv, gv_mean, ms_mean per label from generate_utterances' host features and the restatement."""
    feats = [r[key] for r in pg.generate_utterances([np.load(f) for f in files], batch_size)] if pg else \
        [np.load(f)[:, cols] for f in yfiles]
    gv = np.array([ref.global_variance(f) for f in feats])
    powers = [ref.modspec(f, n) for f in feats]
    return gv, gv.mean(axis=0), np.mean([np.log(p) for p in powers], axis=0), powers


def _check_split(z, label_idx, want):
    gv, gv_mean, ms_mean, powers = want
    assert np.all(np.abs(z["gv"][label_idx] - gv) <= 1e-12 * np.abs(gv))
    assert np.all(np.abs(z["gv_mean"][label_idx] - gv_mean) <= 1e-12 * gv_mean)
    big = np.all([p > 1e-3 * p.max(axis=0, keepdims=True) for p in powers], axis=0)
    assert np.all(np.abs(z["ms_mean"][label_idx] - ms_mean)[big] <= 1e-6)


@pytest.mark.parametrize("kind", ["vc", "tts_acoustic"])
def test_command_end_to_end(dev, tmp_path, capsys, kind):
    from gantts_b200 import generate, models, objective, train
    root = str(tmp_path / "data")
    if kind == "vc":
        xd, yd = H.write_vc_data(root)
        make_hp = H.vc_hp
    else:
        xd, yd = os.path.join(root, "X_acoustic"), os.path.join(root, "Y_acoustic")
        os.makedirs(xd), os.makedirs(yd)
        rng = np.random.RandomState(2)
        for i in range(14):
            L = int(rng.randint(20, 90))
            np.save(os.path.join(xd, "utt%03d.npy" % i), rng.rand(L, 20).astype(np.float32))
            np.save(os.path.join(yd, "utt%03d.npy" % i), (rng.randn(L, 187) + 1).astype(np.float32))
        make_hp = H.tts_acoustic_hp
    hp = make_hp()
    train.load_data(hp, xd, yd, -1)                      # writes the statistics next to X and Y
    ckpts = []
    for seed, label in ((3, "baseline"), (4, "gan")):
        torch.manual_seed(seed)
        model = getattr(models, hp.generator)(**hp.generator_params)
        ck = str(tmp_path / "ck" / label)
        os.makedirs(ck)
        train.save_checkpoint(model, torch.optim.Adagrad(model.parameters()), 4, ck, "Generator")
        ckpts.append(os.path.join(ck, "checkpoint_epoch4_Generator.pth"))
    name = ["--hparams_name=" + kind]
    for dst, extra in (("gen", []), ("gen1", ["--batch-size=1"])):
        assert objective.main(name + extra + [xd, yd, str(tmp_path / dst)] + ckpts, hp=make_hp()) == 0
    printed = capsys.readouterr().out
    stats = generate.load_stats(hp, root)
    pgs = []
    for c in ckpts:
        model = getattr(models, hp.generator)(**hp.generator_params)
        train.load_checkpoint(model, c)
        pgs.append(generate.ParameterGenerator(model.to(dev), hp, stats))
    cols, key = objective.natural_columns(hp), objective.FEATURES[hp.name]
    for sub, files in generate.utterance_files(xd):
        z, z1 = (np.load(str(tmp_path / d / (sub + ".npz"))) for d in ("gen", "gen1"))
        assert list(z["labels"]) == ["natural", "baseline", "gan"]
        assert list(z["names"]) == [os.path.splitext(os.path.basename(f))[0] for f in files]
        assert list(z["lengths"]) == [len(np.load(f)) for f in files]
        assert np.array_equal(z["ms_freq"], np.arange(2049) / 4096 * 200.0)
        for k in ("gv", "gv_mean", "ms_mean"):
            assert np.array_equal(z[k], z1[k]), (sub, k)            # --batch-size=1 and the default: the same bits
        yfiles = [os.path.join(yd, os.path.basename(f)) for f in files]
        for i, pg in enumerate([None] + pgs):
            _check_split(z, i, _expected(pg, files, yfiles, 4096, cols, key, hp.batch_size))
        for label, gv_ratio, ms_rms in objective.summary(list(z["labels"]), z["gv_mean"], z["ms_mean"]):
            assert ("%s %s: mean log10 GV ratio to natural %+.4f, RMS log MS difference to natural %.4f"
                    % (sub, label, gv_ratio, ms_rms)) in printed
