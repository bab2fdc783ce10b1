"""Feature generation on the GPU (gantts_b200.generate): the length-exact MLPG (gantts_mlpg_ragged) against the dense
fp64 nnmnkwii.paramgen.mlpg restatement run on each row alone at its own length, the golden gen_parameters outputs through
the new path, the length-exact SRU forward (gantts_sru_fwd_lengths) against the SRU restatement per utterance, every
generator class end to end against GeneratorOracle at B = 1 followed by the evaluation scripts' post-processing, and the
command against generate_utterances."""
import os
import types

import numpy as np
import pytest
import torch
from torch import nn

from conftest import ROOT, WINDOWS, rel_err
from oracle import gantts_port as gp
from oracle import nnmnkwii_port as nnp
import evaltts_mirror
import train_cli_helpers as H

pytestmark = pytest.mark.gpu

ACOUSTIC = [(0, 60, True, 0), (180, 1, True, 60), (183, 1, False, 61), (184, 1, True, 62)]     # 187 -> 63 columns
VC = [(0, 4, True, 0)]                                                                        # 12 -> 4 columns
TOL = 2e-4
P = types.SimpleNamespace(inv_scale=lambda x, m, s: x * s + m)     # nnmnkwii.preprocessing.inv_scale


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__
    __graft_entry__.build()
    return torch.device("cuda:0")


def _mlpg_row(x, entries, var=None, in_aff=None, out_aff=None):
    """One utterance (L, D) as the evaluation scripts generate it: float64 dense per-stream MLPG."""
    x = np.asarray(x, dtype=np.float64)
    if in_aff is not None:
        x = x * in_aff[0] + in_aff[1]
    ncols = sum(e[1] for e in entries)
    out = np.zeros((len(x), ncols))
    for a, sd, dyn, o in entries:
        if dyn:
            v = np.ones(3 * sd) if var is None else np.asarray(var[a:a + 3 * sd], dtype=np.float64)
            out[:, o:o + sd] = nnp.mlpg(x[:, a:a + 3 * sd], v, WINDOWS)
        else:
            out[:, o:o + sd] = x[:, a:a + sd]
    if out_aff is not None:
        out = out * out_aff[0] + out_aff[1]
    return out


@pytest.mark.parametrize("layout", ["acoustic", "vc"])
@pytest.mark.parametrize("mode", ["unit", "unit_out_affine", "var_in_affine"])
@pytest.mark.parametrize("lens", [[1, 2, 40, 17, 9], [1, 2, 31, 17, 9]])
def test_mlpg_ragged_vs_each_row_alone(dev, layout, mode, lens):
    from gantts_b200 import ops
    entries = ACOUSTIC if layout == "acoustic" else VC
    D, ncols = (187, 63) if layout == "acoustic" else (12, 4)
    rng = np.random.RandomState(len(mode) + lens[2])
    B, T = len(lens), 40
    x = rng.randn(B, T, D).astype(np.float32)
    var = in_aff = out_aff = None
    if mode == "unit_out_affine":
        out_aff = ((0.5 + rng.rand(ncols)).astype(np.float32), rng.randn(ncols).astype(np.float32))
    if mode == "var_in_affine":
        std = (0.3 + rng.rand(D)).astype(np.float32)
        in_aff, var = (std, rng.randn(D).astype(np.float32)), (std.astype(np.float64) ** 2).astype(np.float32)
    td = lambda a: None if a is None else torch.from_numpy(np.asarray(a)).to(dev)
    lengths = torch.tensor(lens, dtype=torch.int64, device=dev)
    run = lambda xx: ops.mlpg_ragged(td(xx), lengths, ops.windows_key(WINDOWS), entries, ncols, var=td(var),
                                     in_affine=None if in_aff is None else tuple(map(td, in_aff)),
                                     out_affine=None if out_aff is None else tuple(map(td, out_aff)))
    got = run(x)
    assert tuple(got.shape) == (B, T, ncols)
    g = got.cpu().numpy()
    for b, L in enumerate(lens):
        want = _mlpg_row(x[b, :L], entries, var, in_aff, out_aff)
        np.testing.assert_allclose(g[b, :L], want, rtol=2e-5, atol=2e-6 * np.abs(want).max())
        assert not g[b, L:].any(), "frames beyond the length must be exactly 0"
    # the same rows padded by 13 more frames of junk: the valid frames are bit-identical
    xp = np.concatenate([x, rng.randn(B, 13, D).astype(np.float32)], 1)
    for b, L in enumerate(lens):
        xp[b, L:] = rng.randn(T + 13 - L, D)
    gp_ = run(xp).cpu().numpy()
    for b, L in enumerate(lens):
        assert np.array_equal(gp_[b, :L], g[b, :L]) and not gp_[b, L:].any()


class _Passthrough(nn.Module):
    """A generator whose output is its input (the golden vectors are generator outputs)."""

    def __init__(self):
        super().__init__()
        self.w = nn.Parameter(torch.zeros(1))

    def include_parameter_generation(self):
        return False

    def forward(self, x, lengths):
        return x


def test_golden_gen_parameters_through_the_batched_path(dev):
    from gantts_b200 import generate
    g = np.load(os.path.join(ROOT, "tests", "golden", "eval.npz"))
    y = g["eval_y"].astype(np.float32)
    L, D = y.shape
    rng = np.random.RandomState(5)
    B, T = 3, L + 11
    x = rng.randn(B, T, D).astype(np.float32)
    x[1, :L] = y
    lengths = torch.tensor([T, L, 7], dtype=torch.int64, device=dev)
    stats = {"Y_mean": g["eval_mean"], "Y_std": g["eval_std"]}
    for tag, mge in (("mge", True), ("var", False)):
        pg = generate.ParameterGenerator(_Passthrough().to(dev), H.tts_acoustic_hp(), stats, mge_training=mge)
        out = pg.generate(torch.from_numpy(x).to(dev), lengths)
        for k in ("mgc", "lf0", "vuv", "bap"):
            want = g["eval_%s_%s" % (tag, k)]
            got = out[k][1, :L].cpu().numpy().astype(np.float64).reshape(want.shape)
            assert np.abs(got - want).max() <= 2e-5 * np.abs(want).max(), (tag, k)


@pytest.mark.parametrize("bidir", [False, True])
@pytest.mark.parametrize("layers", [1, 2, 3])
def test_sru_forward_with_lengths(dev, bidir, layers):
    from gantts_b200 import rnn
    torch.manual_seed(layers + 10 * bidir)
    sru = rnn.SRU(10, 8, layers, bidirectional=bidir, use_relu=1).to(dev).eval()
    lens = [33, 1, 2, 20, 7]
    B, T = len(lens), 33
    x = torch.randn(B, T, 10)
    lengths = torch.tensor(lens, dtype=torch.int64, device=dev)
    with torch.no_grad():
        got = sru(x.to(dev), lengths=lengths).cpu()
        full = torch.full((B,), T, dtype=torch.int64, device=dev)
        assert torch.equal(sru(x.to(dev), lengths=full), sru(x.to(dev)))      # all lengths T: gantts_sru_fwd's bits
    ncols = 8 * (2 if bidir else 1)
    cells = [(c.weight.detach().cpu(), c.bias.detach().cpu()) for c in sru.rnn_lst]
    ident = (torch.eye(ncols), torch.zeros(ncols))
    for b, L in enumerate(lens):
        want = gp.sru_forward(x[b:b + 1, :L], cells, ident, bidir, 2)[0]
        assert rel_err(got[b, :L].numpy(), want.detach().numpy()) <= TOL, (b, L)
        assert not got[b, L:].any()
    with pytest.raises(RuntimeError, match="eval-only"):
        sru.train()(x.to(dev), lengths=lengths)


def _models(kind, name):
    from gantts_b200 import models
    if kind == "vc":
        return {"In2OutHighwayNet": lambda: models.In2OutHighwayNet(12, 12, 4, num_hidden=2, hidden_dim=32, dropout=0.5),
                "In2OutRNNHighwayNet": lambda: models.In2OutRNNHighwayNet(12, 12, 4, num_hidden=2, hidden_dim=16,
                                                                          bidirectional=True, dropout=0.0),
                "MLP": lambda: models.MLP(12, 12, 2, 32, dropout=0.5, last_sigmoid=False)}[name]()
    out = 187 if kind == "acoustic" else 5
    return {"MLP": lambda: models.MLP(20, out, 2, 32, dropout=0.5, last_sigmoid=False),
            "SRURNN": lambda: models.SRURNN(20, out, 2, 16, bidirectional=True, use_relu=1),
            "LSTMRNN": lambda: models.LSTMRNN(20, out, 2, 16, bidirectional=True),
            "GRURNN": lambda: models.GRURNN(20, out, 1, 16, bidirectional=False)}[name]()


def _oracle(model, name):
    sd = {k: v.detach().cpu() for k, v in model.state_dict().items()}
    kind = {"MLP": "mlp", "In2OutHighwayNet": "highway", "In2OutRNNHighwayNet": "rnn_highway", "LSTMRNN": "lstm",
            "GRURNN": "lstm", "SRURNN": "sru"}[name]
    rnn_ = getattr(model, "lstm", None) or getattr(model, "gru", None)
    num_hidden = getattr(rnn_, "num_layers", None)
    hidden = getattr(rnn_, "hidden_size", None)
    bidir = bool(getattr(rnn_, "bidirectional", False)) if not name == "SRURNN" else model.gru.rnn_lst[0].bidirectional
    act = model.gru.rnn_lst[0].activation_type if name == "SRURNN" else 2
    return gp.GeneratorOracle(kind, sd, static_dim=getattr(model, "static_dim", None), num_hidden=num_hidden,
                              hidden_dim=hidden, bidirectional=bidir, rnn_attr="gru" if name == "GRURNN" else "lstm",
                              activation_type=act)


def _want(orc, hp, x, mean, std, mge):
    """What the evaluation scripts compute for one normalised utterance x (L, D)."""
    L = len(x)
    R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, L)) if any(hp.has_dynamic_features) else None
    ohp = {"stream_sizes": hp.stream_sizes, "has_dynamic_features": hp.has_dynamic_features}
    with torch.no_grad():
        y_hat, y_hat_static = orc.forward(torch.from_numpy(x)[None], R, [L], ohp)
    if hp.name == "vc":                                                        # evaluation_vc.py:85-89
        S = y_hat_static.shape[-1]
        return {"mc": y_hat_static[0].numpy().astype(np.float64) * std[:S] + mean[:S]}
    y = y_hat[0].numpy()
    if hp.name == "duration":                                                  # evaluation_tts.py:171-176
        return {"duration": y.astype(np.float64) * std + mean}                 # rounded by the comparison
    mgc, lf0, vuv, bap = evaltts_mirror.gen_parameters(y, mean, std, mge, hp.stream_sizes, WINDOWS, nnp, P)
    f0 = lf0.copy()                                                            # gen_waveform :117-119
    f0[vuv < 0.5] = 0
    f0[np.nonzero(f0)] = np.exp(f0[np.nonzero(f0)])
    return {"mgc": mgc, "lf0": lf0, "vuv": vuv, "bap": bap, "f0": f0}


def _compare(got, want, name):
    if name == "duration":
        near = np.abs(np.abs(want - np.floor(want)) - 0.5) < 1e-4                # within 1e-4 of a rounding boundary
        w = np.round(want)
        w[w <= 0] = 1
        assert np.array_equal(got[~near], w[~near]), name
        return
    if name == "vuv":
        near = np.abs(want - 0.5) < 1e-4
        assert np.array_equal((got >= 0.5)[~near], (want >= 0.5)[~near])
    if name == "f0":
        return
    assert rel_err(got, want) <= TOL, (name, rel_err(got, want))


def _check_f0(got, want):
    near = (np.abs(want["vuv"] - 0.5) < 1e-4)[:, None]
    gz, wz = got["f0"] == 0, want["f0"] == 0
    assert np.array_equal(gz | near, wz | near)
    both = ~gz & ~wz
    assert np.all(np.abs(got["f0"][both] - want["f0"][both]) <= TOL * np.abs(want["f0"][both]))


CASES = [("vc", "In2OutHighwayNet", True), ("vc", "In2OutRNNHighwayNet", True), ("vc", "MLP", True),
         ("acoustic", "MLP", True), ("acoustic", "SRURNN", True), ("acoustic", "SRURNN", False),
         ("acoustic", "LSTMRNN", True), ("acoustic", "GRURNN", False), ("duration", "SRURNN", True),
         ("duration", "LSTMRNN", True)]


@pytest.mark.parametrize("kind,name,mge", CASES)
def test_generator_end_to_end(dev, kind, name, mge):
    from gantts_b200 import generate
    hp = {"vc": lambda: H.vc_hp(order=4), "acoustic": H.tts_acoustic_hp, "duration": H.tts_duration_hp}[kind]()
    hp.generator = name
    torch.manual_seed(7)
    model = _models(kind, name)
    orc = _oracle(model, name)
    D, Dout = (12, 12) if kind == "vc" else (20, 187 if kind == "acoustic" else 5)
    rng = np.random.RandomState(11)
    mean, std = rng.randn(Dout), 0.5 + rng.rand(Dout)
    if kind == "acoustic":
        mean[183], std[183] = 0.5, 0.5                     # V/UV around its 0.5 threshold
        mean[180], std[180] = 5.0, 0.3                     # log-F0
    if kind == "duration":
        mean, std = 3.0 + rng.rand(Dout), 2.0 + rng.rand(Dout)
    stats = {"data_mean": mean, "data_std": std} if kind == "vc" else {"Y_mean": mean, "Y_std": std}
    pg = generate.ParameterGenerator(model.to(dev), hp, stats, mge_training=mge)
    lens = [37, 5, 23, 1, 40, 2, 18]
    B, T = len(lens), max(lens)
    x = np.zeros((B, T, D), np.float32)
    for b, L in enumerate(lens):
        x[b, :L] = rng.randn(L, D) if kind == "vc" else rng.uniform(0.01, 0.99, (L, D))
    out = pg.generate(torch.from_numpy(x).to(dev), torch.tensor(lens, dtype=torch.int64, device=dev))
    assert sorted(out) == sorted(generate.OUTPUT_NAMES[hp.name])
    host = {k: v.cpu().numpy() for k, v in out.items()}
    for b, L in enumerate(lens):
        want = _want(orc, hp, x[b, :L], mean, std, mge)
        got = {k: v[b, :L] for k, v in host.items()}
        for k in want:
            _compare(got[k].astype(np.float64).reshape(np.shape(want[k])), np.asarray(want[k], np.float64), k)
        if "f0" in want:
            _check_f0(got, want)
        # the same utterance in a batch of its own
        alone = pg.generate(torch.from_numpy(x[b:b + 1, :L].copy()).to(dev),
                            torch.tensor([L], dtype=torch.int64, device=dev))
        for k, v in alone.items():
            a = v[0].cpu().numpy()
            assert np.allclose(a, got[k], rtol=1e-5, atol=1e-5 * max(np.abs(got[k]).max(), 1e-30)), (k, b)


def test_command_writes_eval_and_test_features(dev, tmp_path):
    from gantts_b200 import generate, models, train
    root = str(tmp_path / "data")
    xd, yd = H.write_vc_data(root)
    hp = H.vc_hp()
    train.load_data(hp, xd, yd, -1)                      # writes data_mean / data_var next to X and Y
    torch.manual_seed(3)
    model = models.In2OutHighwayNet(**hp.generator_params)
    ck = str(tmp_path / "ck")
    os.makedirs(ck)
    train.save_checkpoint(model, torch.optim.Adagrad(model.parameters()), 4, ck, "Generator")
    dst = str(tmp_path / "gen")
    assert generate.main(["--batch-size=4", os.path.join(ck, "checkpoint_epoch4_Generator.pth"), xd, dst],
                         hp=H.vc_hp()) == 0
    stats = generate.load_stats(hp, root)
    pg = generate.ParameterGenerator(model.to(dev), hp, stats)
    for sub, files in generate.utterance_files(xd):
        names = sorted(os.path.splitext(os.path.basename(f))[0] + ".npz" for f in files)
        assert sorted(os.listdir(os.path.join(dst, sub))) == names
        want = pg.generate_utterances([np.load(f) for f in files], 4)
        for f, w in zip(files, want):
            got = np.load(os.path.join(dst, sub, os.path.splitext(os.path.basename(f))[0] + ".npz"))
            assert sorted(got.files) == ["mc"] and got["mc"].shape == (len(np.load(f)), 4)
            assert np.array_equal(got["mc"], w["mc"])
