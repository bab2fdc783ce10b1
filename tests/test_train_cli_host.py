"""Host-side pieces of the training command (gantts_b200.train) and the epoch log (gantts_b200.epochlog): the data split,
statistics, derived dims, batching, LR schedule, checkpoint layout, usage, the per-batch metric formulas and the
configuration rules of gantts_epoch_log_add.  No GPU needed."""
import ctypes
import json
import math
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
import train_cli_helpers as H


@pytest.mark.parametrize("n", [6, 10, 37, 100, 1127])
def test_split_equals_sklearn(n):
    sk = pytest.importorskip("sklearn.model_selection")
    from gantts_b200 import train
    files = ["f%05d.npy" % i for i in range(n)]
    tr, te = sk.train_test_split(files, test_size=0.112, random_state=1234)
    assert train.train_test_split_files(files) == (list(tr), list(te))


def test_npy_files_hold_out_last_five_and_honour_max_files(tmp_path):
    from gantts_b200 import train
    for i in range(20):
        np.save(str(tmp_path / ("u%02d.npy" % i)), np.zeros((2, 1), np.float32))
    (tmp_path / "notes.txt").write_text("x")
    every = sorted(str(tmp_path / ("u%02d.npy" % i)) for i in range(20))
    assert train.npy_files(str(tmp_path), test=True) == every[15:]
    tr, te = train.npy_files(str(tmp_path), train=True), train.npy_files(str(tmp_path), train=False)
    assert sorted(tr + te) == every[:15] and len(te) == math.ceil(0.112 * 15)
    assert sorted(train.npy_files(str(tmp_path), True, 8) + train.npy_files(str(tmp_path), False, 8)) == every[:8]


def test_vc_joint_statistics_over_valid_frames():
    from gantts_b200 import train
    rng = np.random.RandomState(3)
    X = [rng.randn(n, 7).astype(np.float32) * 3 + 1 for n in (9, 14, 30)]
    Y = [rng.randn(n, 7).astype(np.float32) - 2 for n in (9, 14, 30)]
    lengths = np.array([9, 10, 25])         # shorter than the arrays: only the valid frames count
    mean, var = train.meanvar([X, Y], lengths)
    cat = np.concatenate([a[:n] for a, n in zip(X, lengths)] + [a[:n] for a, n in zip(Y, lengths)]).astype(np.float64)
    np.testing.assert_allclose(mean, cat.mean(axis=0), rtol=1e-13, atol=1e-13)
    np.testing.assert_allclose(var, cat.var(axis=0), rtol=1e-12, atol=1e-13)


def test_tts_dims_are_derived_as_train_py():
    from gantts_b200 import train
    hp = H.tts_acoustic_hp()
    train.derive_tts_dims(hp, 425, 187)
    # 60 static mgc columns minus the 2 masked ones, plus the 425 linguistic features of the conditioning
    assert (hp.generator_params["in_dim"], hp.generator_params["out_dim"]) == (425, 187)
    assert hp.discriminator_params["in_dim"] == 60 - 2 + 425
    hp = H.tts_duration_hp()
    train.derive_tts_dims(hp, 416, 5)
    assert (hp.generator_params["in_dim"], hp.generator_params["out_dim"], hp.discriminator_params["in_dim"]) == \
        (416, 5, 421)
    hp = H.tts_acoustic_hp(discriminator_linguistic_condition=False)
    hp.generator_params["in_dim"] = 7
    train.derive_tts_dims(hp, 425, 187)
    assert hp.generator_params["in_dim"] == 7 and hp.discriminator_params["in_dim"] == 58


def test_collate_pads_and_sort_orders_by_length():
    from gantts_b200 import train
    rng = np.random.RandomState(0)
    batch = [(rng.randn(n, 3), rng.randn(n, 2)) for n in (4, 9, 6)]
    x, y, lengths = train.collate_fn(batch)
    assert x.dtype == y.dtype == torch.float32 and lengths.dtype == torch.int64
    assert tuple(x.shape) == (3, 9, 3) and tuple(y.shape) == (3, 9, 2) and lengths.tolist() == [4, 9, 6]
    assert float(x[0, 4:].abs().sum()) == 0 and np.allclose(x[0, :4].numpy(), batch[0][0].astype(np.float32))
    xs, ys, ls = train.sort_batch(x, y, lengths)
    assert ls.tolist() == [9, 6, 4]
    assert torch.equal(xs[0], x[1]) and torch.equal(ys[2], y[0])


def test_lr_schedule_per_epoch():
    from gantts_b200 import train
    opt = torch.optim.Adagrad([torch.nn.Parameter(torch.zeros(2))], lr=0.5)
    got = []
    for epoch in range(1, 31):                          # train_loop calls it with global_epoch - 1
        train.exp_lr_scheduler(opt, epoch - 1, 30, init_lr=0.01, lr_decay_epoch=10)
        got.append(opt.param_groups[0]["lr"])
    assert got == [0.01 * 0.1 ** ((e - 1) // 10) for e in range(1, 31)]


def test_checkpoint_layout(tmp_path):
    from gantts_b200 import models, train
    m = models.MLP(3, 1, 2, 4, dropout=0.0)
    opt = torch.optim.Adam(m.parameters(), lr=1e-3)
    train.save_checkpoint(m, opt, 7, str(tmp_path), "Discriminator")
    ck = torch.load(str(tmp_path / "checkpoint_epoch7_Discriminator.pth"))
    assert set(ck) == {"state_dict", "optimizer", "global_epoch"} and ck["global_epoch"] == 7
    assert set(ck["state_dict"]) == set(m.state_dict()) and set(ck["optimizer"]) == {"state", "param_groups"}
    m2 = models.MLP(3, 1, 2, 4, dropout=0.0)
    ck2 = train.load_checkpoint(m2, str(tmp_path / "checkpoint_epoch7_Discriminator.pth"))
    assert all(torch.equal(a, b) for a, b in zip(m.state_dict().values(), m2.state_dict().values()))
    torch.optim.Adam(m2.parameters()).load_state_dict(ck2["optimizer"])


def test_usage_options_and_defaults_equal_the_reference():
    from gantts_b200 import train
    from oracle import reference_loader
    from compat.docopt import docopt
    got = train.parse_args(["IN", "OUT"])
    if reference_loader.available():
        import ast
        with open(os.path.join(reference_loader.REFERENCE_ROOT, "train.py")) as f:
            want = docopt(ast.get_docstring(ast.parse(f.read())), argv=["IN", "OUT"])
    else:
        with open(os.path.join(GOLDEN, "train_usage.json")) as f:
            want = json.load(f)["args"]
    assert got == want
    flags = ["--hparams_name=tts_acoustic", "--w_d=0", "--discriminator-warmup", "--reset_optimizers",
             "--restart_epoch=3", "--checkpoint-g=g.pth", "--disable-slack", "A", "B"]
    a = train.parse_args(flags)
    assert (a["--hparams_name"], a["--w_d"], a["--discriminator-warmup"], a["--reset_optimizers"], a["--restart_epoch"],
            a["--checkpoint-g"], a["<inputs_dir>"]) == ("tts_acoustic", "0", True, True, "3", "g.pth", "A")


def fold_mirror(kind, s):
    """The fold kernel's per-batch formulas (epochlog.cu) on the eight sums s, in fp64."""
    logdb = 10.0 / math.log(10.0) * math.sqrt(2.0)
    n = s[5]
    if kind == "acoustic":
        return {"mcd": logdb * s[0] / n, "bap_mcd": logdb * s[1] / n / 10.0,
                "f0_rmse": math.sqrt(s[2] / s[3]) if s[3] > 0 else float("nan"), "vuv_err": s[4] / n}
    if kind == "duration":
        return {"dur_rmse": math.sqrt(s[6] / n)}
    return {"mcd": logdb * s[0] / n}


@pytest.mark.parametrize("kind", ["acoustic", "duration", "vc"])
def test_fold_formulas_match_metrics_py(kind, monkeypatch):
    from gantts_b200 import metrics, ops
    hp = {"acoustic": H.tts_acoustic_hp, "duration": H.tts_duration_hp, "vc": H.vc_hp}[kind]()
    D = {"acoustic": 63, "duration": 5, "vc": 4}[kind]
    width = {"acoustic": 187, "duration": 5, "vc": 12}[kind]
    for s in ([12.5, 3.25, 40.0, 17.0, 3.0, 33.0, 9.5, 0.0], [1.0, 2.0, 0.0, 0.0, 7.0, 11.0, 0.25, 0.0]):
        sums = torch.tensor(s, dtype=torch.float32)
        monkeypatch.setattr(ops, "distortion_sums", lambda *a, **k: sums)
        y = torch.zeros(2, 3, D)
        got = metrics.compute_distortions(y, y, np.zeros(width), np.ones(width), [3, 3], hp=hp)
        want = fold_mirror(kind, [float(v) for v in sums])
        assert list(got) == list(want)
        for k in got:
            assert (math.isnan(got[k]) and math.isnan(want[k])) or got[k] == want[k], (k, got[k], want[k])
    if kind == "acoustic":
        assert math.isnan(got["f0_rmse"])           # no frame voiced in both: NaN, as the reference logs it


def test_epoch_log_config_matches_metrics_columns():
    from gantts_b200 import epochlog
    c, scols = epochlog.log_config(H.tts_acoustic_hp())
    assert scols == list(range(60)) + [180, 183, 184] and c.n_static == 63
    assert (c.cols.mcd_start, c.cols.mcd_count, c.cols.bap_start, c.cols.bap_count, c.cols.lf0_col, c.cols.vuv_col) == \
        (1, 59, 62, 1, 60, 61)
    c, scols = epochlog.log_config(H.vc_hp(order=5))
    assert scols == list(range(5)) and (c.cols.mcd_start, c.cols.mcd_count) == (0, 5)
    c, scols = epochlog.log_config(H.tts_duration_hp())
    assert scols == list(range(5)) and (c.cols.mse_start, c.cols.mse_count) == (0, 5)


def test_epoch_log_config_rules_are_rejected_with_named_messages():
    import __graft_entry__
    __graft_entry__.build()
    from gantts_b200 import _lib, epochlog
    lib = _lib.load()
    ws = lambda c: lib.gantts_epoch_log_workspace_bytes(ctypes.byref(c))
    err = lambda: lib.gantts_last_error_string().decode()
    for make in (H.tts_acoustic_hp, H.tts_duration_hp, H.vc_hp):
        assert ws(epochlog.log_config(make())[0]) > 0

    def rejected(make, mutate, needle):
        c = epochlog.log_config(make())[0]
        mutate(c)
        assert ws(c) == 0 and needle in err(), (needle, err())

    rejected(H.vc_hp, lambda c: setattr(c, "kind", 3), "unknown metric kind 3")
    rejected(H.vc_hp, lambda c: setattr(c, "n_static", 0), "n_static 0 outside")
    rejected(H.vc_hp, lambda c: setattr(c, "n_static", _lib.MAX_COLS + 1), "outside [1, 256]")
    rejected(H.vc_hp, lambda c: c.static_cols.__setitem__(2, -1), "static column 2 maps to y column -1")
    rejected(H.vc_hp, lambda c: setattr(c.cols, "mcd_count", 5), "column groups outside [0, n_static)")
    rejected(H.tts_acoustic_hp, lambda c: setattr(c.cols, "vuv_col", 63), "column groups outside")
    rejected(H.tts_acoustic_hp, lambda c: setattr(c.cols, "lf0_col", -1), "acoustic metrics need")
    rejected(H.tts_duration_hp, lambda c: setattr(c.cols, "mcd_count", 1), "duration metric needs the mse group alone")
    rejected(H.vc_hp, lambda c: setattr(c.cols, "mse_count", 1), "vc metric needs the mcd group alone")
    c = epochlog.log_config(H.vc_hp())[0]
    rc = lib.gantts_epoch_log_add(ctypes.byref(c), 8, 1 << 20, None, None, 0, 0, 0, None, 0, 0, 1 << 20, 1, 1, None,
                                  None, 1 << 20, 1 << 20, ws(c), None)
    assert rc == 1 and "unknown flags 0x8" in err()
    rc = lib.gantts_epoch_log_add(ctypes.byref(c), _lib.LOG_SPOOF, 1 << 20, None, None, 0, 0, 0, None, 0, 0, 1 << 20,
                                  1, 1, None, None, 1 << 20, 1 << 20, ws(c), None)
    assert rc == 1 and "LOG_SPOOF needs the spoof count" in err()
    rc = lib.gantts_epoch_log_add(ctypes.byref(c), _lib.LOG_UPDATE_G, 1 << 20, None, 1 << 20, 12 * 9, 12, 3, 1 << 20,
                                  36, 4, 1 << 20, 1, 9, 1 << 20, 1 << 20, 1 << 20, 1 << 20, ws(c), None)
    assert rc == 1 and "static column 3 maps to y column 3 outside [0, 3)" in err()
    rc = lib.gantts_epoch_log_add(ctypes.byref(c), _lib.LOG_UPDATE_G, 1 << 20, None, 1 << 20, 12 * 9, 12, 12, 1 << 20,
                                  36, 4, 1 << 20, 2, 9, 1 << 20, 1 << 20, 1 << 20, 1 << 20, ws(c) - 1, None)
    assert rc == 4 and "workspace too small" in err()


def test_generator_noise_is_refused(tmp_path):
    from gantts_b200 import train
    with pytest.raises(SystemExit, match="generator_add_noise"):
        train.main(["--hparams=generator_add_noise=True", str(tmp_path / "X"), str(tmp_path / "Y")], hp=H.vc_hp())
