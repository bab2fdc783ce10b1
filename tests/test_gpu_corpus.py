"""The training command's device corpus on the GPU: gantts_corpus_gather against a numpy restatement at the widths the
command meets, every batch of two epochs of DeviceBatches against train.py's DataLoader with collate_fn and sort_batch
bit for bit, the five-stage recipe with dropout giving identical scalars and checkpoints on either loader, the fallback
to the host loader over the budget, and a tts_acoustic phase without a host synchronisation before its read with either
loader."""
import json
import os

import numpy as np
import pytest
import torch

import corpus_helpers as C
import train_cli_helpers as H
import test_gpu_train_cli as cli

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__
    __graft_entry__.build()
    return torch.device("cuda:0")


@pytest.mark.parametrize("dx,dy", [(12, 12), (416, 5), (425, 187), (5, 425), (1, 3)])
def test_gather_matches_numpy_and_overwrites_every_element(dev, dx, dy):
    from gantts_b200 import _lib, ops
    rng = np.random.RandomState(dx * 1000 + dy)
    N = 500
    X = rng.randn(N, dx).astype(np.float32)
    Y = rng.randn(N, dy).astype(np.float32)
    X[3, 0] = -0.0
    # every offset parity, a frame at each end of the corpus, a row repeated, length-1 rows, rows shorter than t
    offsets = np.array([0, 1, 2, 3, 499, 7, 7, 250, 37, 498], dtype=np.int64)
    lengths = np.array([40, 33, 1, 17, 1, 40, 2, 1, 39, 2], dtype=np.int64)
    Xd, Yd = torch.from_numpy(X).to(dev), torch.from_numpy(Y).to(dev)
    od, ld = torch.from_numpy(offsets).to(dev), torch.from_numpy(lengths).to(dev)
    for t in (40, 41, 77):
        for b in (1, 3, len(offsets)):
            xo = torch.full((b, t, dx), float("nan"), device=dev)
            yo = torch.full((b, t, dy), float("nan"), device=dev)
            status = torch.zeros((), dtype=torch.int64, device=dev)
            x, y = ops.corpus_gather(Xd, Yd, od[:b], ld[:b], t, x_out=xo, y_out=yo, status=status)
            assert x.data_ptr() == xo.data_ptr() and y.data_ptr() == yo.data_ptr()
            gx, gy = C.gather(X, Y, offsets[:b], lengths[:b], t)
            assert torch.equal(x.cpu(), torch.from_numpy(gx)) and torch.equal(y.cpu(), torch.from_numpy(gy))
            assert int(status) == 0
    assert torch.signbit(ops.corpus_gather(Xd, Yd, od[3:4], ld[3:4], 17)[0][0, 0, 0].cpu())


def test_rows_outside_the_corpus_are_padding_and_flagged(dev):
    from gantts_b200 import _lib, ops
    X = torch.randn(50, 7, device=dev)
    Y = torch.randn(50, 3, device=dev)
    for off, n in ((45, 6), (-1, 2), (0, 11), (3, -1)):             # past N, negative offset, longer than t, negative
        od = torch.tensor([0, off], dtype=torch.int64, device=dev)
        ld = torch.tensor([10, n], dtype=torch.int64, device=dev)
        status = torch.zeros((), dtype=torch.int64, device=dev)
        x, y = ops.corpus_gather(X, Y, od, ld, 10, status=status)
        assert int(status) == _lib.CORPUS_BAD_ROW
        assert torch.equal(x[0], X[:10]) and torch.equal(y[0], Y[:10])
        assert not x[1].any() and not y[1].any()


def _epochs(loader, device, seed):
    from gantts_b200 import train
    torch.manual_seed(seed)
    out = []
    for _ in range(2):
        batches = loader if isinstance(loader, train.DeviceBatches) else train.host_batches(loader, device)
        out.append([(x.cpu(), y.cpu(), lengths.cpu(), cpu) for x, y, lengths, cpu in batches])
    return out, torch.get_rng_state()


@pytest.mark.parametrize("kind", sorted(C.KINDS))
@pytest.mark.parametrize("batch_size", [6, 7])         # 22 train utterances: a last batch of 4, and one of 1
def test_device_batches_equal_the_host_loader(dev, tmp_path, monkeypatch, kind, batch_size):
    from gantts_b200 import train
    make_hp = C.KINDS[kind][0]
    xd, yd = C.write_kind(str(tmp_path), kind)
    on_dev, Ym, Ys, longest = train.load_data(make_hp(batch_size=batch_size), xd, yd, -1)
    monkeypatch.setattr(train, "device_corpus_budget", lambda: 0)
    on_host, Ym2, Ys2, longest2 = train.load_data(make_hp(batch_size=batch_size), xd, yd, -1)
    assert isinstance(on_dev["train"], train.DeviceBatches) and not isinstance(on_host["train"], train.DeviceBatches)
    assert np.array_equal(Ym, Ym2) and np.array_equal(Ys, Ys2) and longest == longest2
    for phase in ("train", "test"):
        assert len(on_dev[phase]) == len(on_host[phase])
        got, rng_dev = _epochs(on_dev[phase], dev, 3)
        want, rng_host = _epochs(on_host[phase], dev, 3)
        assert torch.equal(rng_dev, rng_host)
        sizes = [len(b[3]) for b in got[0]]
        if phase == "train":
            assert sizes[-1] == 22 % batch_size
            assert 1 in [c for e in got for b in e for c in b[3]]        # a length-1 utterance
        for e_got, e_want in zip(got, want):
            assert len(e_got) == len(e_want)
            for (x, y, lengths, cpu), (wx, wy, wl, wcpu) in zip(e_got, e_want):
                assert torch.equal(x, wx) and torch.equal(y, wy) and torch.equal(lengths, wl) and cpu == wcpu
                assert x.dtype == wx.dtype and lengths.dtype == wl.dtype and x.shape == wx.shape


def _dropout_hp():
    return H.vc_hp(generator_params={"in_dim": None, "out_dim": None, "num_hidden": 2, "hidden_dim": 32,
                                     "static_dim": 4, "dropout": 0.3},
                   discriminator_params={"in_dim": 4, "out_dim": 1, "num_hidden": 2, "hidden_dim": 16,
                                         "dropout": 0.4, "last_sigmoid": True})


def test_recipe_is_identical_on_either_loader(dev, tmp_path, monkeypatch, capsys):
    from gantts_b200 import ops, train
    root = str(tmp_path)
    xd, yd = H.write_vc_data(os.path.join(root, "data"))
    # draw_seed counts its draws since the last new torch seed: restart the count so both runs get the same seeds
    monkeypatch.setattr(ops, "_seed_state", [None, 0])
    on_dev = cli._run_recipe(os.path.join(root, "device"), xd, yd, _dropout_hp)
    out = capsys.readouterr().out
    assert "Data loader: device corpus" in out and "Training step: FusedGanStep" in out
    monkeypatch.setattr(train, "device_corpus_budget", lambda: 0)
    monkeypatch.setattr(ops, "_seed_state", [None, 0])
    on_host = cli._run_recipe(os.path.join(root, "host"), xd, yd, _dropout_hp)
    assert "Data loader: host DataLoader" in capsys.readouterr().out
    assert on_dev == on_host
    for stage in on_dev:
        files = sorted(os.listdir(os.path.join(root, "device", stage)))
        assert files and files == sorted(os.listdir(os.path.join(root, "host", stage)))
        for f in files:
            a = torch.load(os.path.join(root, "device", stage, f))
            b = torch.load(os.path.join(root, "host", stage, f))
            assert a["global_epoch"] == b["global_epoch"]
            assert a["state_dict"].keys() == b["state_dict"].keys()
            for k in a["state_dict"]:
                assert torch.equal(a["state_dict"][k], b["state_dict"][k]), (stage, f, k)
            for sa, sb in zip(a["optimizer"]["state"].values(), b["optimizer"]["state"].values()):
                for k in sa:
                    assert torch.equal(torch.as_tensor(sa[k]), torch.as_tensor(sb[k])), (stage, f, k)


def test_corpus_over_the_budget_takes_the_host_loader(dev, tmp_path, monkeypatch, capsys):
    from gantts_b200 import train
    xd, yd = H.write_vc_data(str(tmp_path))
    monkeypatch.setattr(train, "device_corpus_budget", lambda: 1000)
    loaders, _, _, _ = train.load_data(H.vc_hp(), xd, yd, -1)
    assert not any(isinstance(v, train.DeviceBatches) for v in loaders.values())
    assert "Data loader: host DataLoader, corpus" in capsys.readouterr().out
    logdir = os.path.join(str(tmp_path), "log")
    assert train.main(["--hparams=nepoch=1", "--w_d=0", "--checkpoint-dir=%s/ck" % tmp_path,
                       "--log-event-path=%s" % logdir, xd, yd], hp=H.vc_hp()) == 0
    assert "Data loader: host DataLoader" in capsys.readouterr().out
    with open(os.path.join(logdir, "scalars.jsonl")) as f:
        assert any(json.loads(line)["name"] == "train mge loss" for line in f)


@pytest.mark.parametrize("on_device", [True, False])
def test_tts_acoustic_phase_makes_no_host_sync_before_its_read(dev, tmp_path, monkeypatch, on_device):
    """With either loader: the device corpus, or the host DataLoader (budget 0) that a corpus over budget takes."""
    from gantts_b200 import models, train
    from gantts_b200.epochlog import EpochLog
    xd, yd = C.write_kind(str(tmp_path), "tts_acoustic")
    hp = H.tts_acoustic_hp()
    if not on_device:
        monkeypatch.setattr(train, "device_corpus_budget", lambda: 0)
    loaders, Ym, Ys, longest = train.load_data(hp, xd, yd, -1)
    assert isinstance(loaders["train"], train.DeviceBatches) == on_device
    torch.manual_seed(0)
    mg = models.MLP(**hp.generator_params).to(dev)
    md = models.MLP(**hp.discriminator_params).to(dev)
    path = train.make_path(mg, md, hp, hp.batch_size, longest, 1.0, 0.0, 1.0, None, dev)
    assert path.name == "FusedGanStep"
    log = EpochLog(hp, Ym, Ys, dev)
    for phase in ("train", "test"):
        for m in (mg, md):
            m.train() if phase == "train" else m.eval()
        train.run_phase(path, loaders[phase], log, phase, 1.0, True, True, dev)     # warm: tables, allocations
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            train.run_phase(path, loaders[phase], log, phase, 1.0, True, True, dev)
        finally:
            torch.cuda.set_sync_debug_mode("default")
        vals = log.read(phase)
        assert np.isfinite(vals["%s mcd metric" % phase]) and np.isfinite(vals["%s discriminator loss" % phase])
