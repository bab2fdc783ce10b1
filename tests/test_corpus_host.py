"""Host side of the device corpus of the training command: the argument rules of gantts_corpus_gather (refused before
any device work) and its ctypes signature, and BatchPlan, which must give the batches, row order and global torch RNG
draws of train.py's DataLoader with collate_fn and sort_batch.  No GPU needed."""
import ctypes
import os

import numpy as np
import pytest
import torch
from torch.utils import data as data_utils

import corpus_helpers as C

FAKE = 1 << 20          # placeholder device pointer: the argument checks never dereference it


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__
    __graft_entry__.build()
    from gantts_b200 import _lib
    return _lib.load()


def _rc(lib, X=FAKE, Y=FAKE, N=100, Dx=12, Dy=5, offsets=FAKE, lengths=FAKE, b=2, t=16, x_out=FAKE, y_out=FAKE):
    return lib.gantts_corpus_gather(X, Y, N, Dx, Dy, offsets, lengths, b, t, x_out, y_out, None, None)


@pytest.mark.parametrize("kw,needle", [
    (dict(X=None), "null pointer"),
    (dict(Y=None), "null pointer"),
    (dict(offsets=None), "null pointer"),
    (dict(lengths=None), "null pointer"),
    (dict(x_out=None), "null pointer"),
    (dict(y_out=None), "null pointer"),
    (dict(N=0), "corpus frames N = 0 must be >= 1"),
    (dict(Dx=0), "widths Dx = 0 and Dy = 5 must be in [1, 65535]"),
    (dict(Dy=0), "widths Dx = 12 and Dy = 0"),
    (dict(Dx=65536), "widths Dx = 65536"),
    (dict(b=0), "batch size b = 0 must be in [1, 65535]"),
    (dict(b=65536), "batch size b = 65536 must be in [1, 65535]"),
    (dict(t=0), "padded length t = 0 must be in [1, 16777216]"),
    (dict(t=(1 << 24) + 1), "padded length t = 16777217"),
])
def test_gather_rules(lib, kw, needle):
    from gantts_b200 import _lib
    assert _rc(lib, **kw) == _lib.GANTTS_E_BADARG
    msg = lib.gantts_last_error_string().decode()
    assert msg.startswith("corpus_gather") and needle in msg, msg


def test_gather_has_its_ctypes_signature(lib):
    from gantts_b200 import _lib
    res, args = _lib.SIGNATURES["gantts_corpus_gather"]
    assert res is ctypes.c_int and len(args) == 13
    assert args[2] is ctypes.c_int64 and all(args[i] is ctypes.c_int for i in (3, 4, 7, 8))
    assert hasattr(lib, "gantts_corpus_gather")


def _dataset(tmp_path, monkeypatch, kind):
    from gantts_b200 import train
    hp = C.KINDS[kind][0]()
    xd, yd = C.write_kind(str(tmp_path), kind)
    monkeypatch.setattr(train, "device_corpus_budget", lambda: 0)     # the host DataLoaders, with or without a GPU
    loaders, _, _, _ = train.load_data(hp, xd, yd, -1)
    assert isinstance(loaders["train"], data_utils.DataLoader)
    return loaders["train"].dataset


@pytest.mark.parametrize("kind", ["vc", "tts_acoustic_delta"])
@pytest.mark.parametrize("shuffle", [True, False])
@pytest.mark.parametrize("batch_size", [6, 7])       # 22 train utterances: a last batch of 4, and one of 1
def test_plan_matches_the_dataloader(tmp_path, monkeypatch, kind, shuffle, batch_size):
    from gantts_b200 import train
    ds = _dataset(tmp_path, monkeypatch, kind)
    X, Y, L = train.pack_corpus(ds)
    assert len(L) == 22 and L.min() == 1 and X.dtype == Y.dtype == np.float32
    host = data_utils.DataLoader(ds, batch_size=batch_size, shuffle=shuffle, collate_fn=train.collate_fn)
    plan = train.BatchPlan(L, batch_size, shuffle)
    assert len(plan) == len(host)
    torch.manual_seed(11)
    want = [[train.sort_batch(*b) for b in host] for _ in range(2)]
    rng_host = torch.get_rng_state()
    torch.manual_seed(11)
    got = [plan.epoch() for _ in range(2)]
    assert torch.equal(torch.get_rng_state(), rng_host)
    assert len(want[0][-1][2]) == 22 % batch_size
    for epoch_want, (rows, bounds) in zip(want, got):
        assert len(bounds) == len(epoch_want) + 1
        for j, (x, y, lengths) in enumerate(epoch_want):
            s, e = bounds[j], bounds[j + 1]
            assert rows[1, s:e].tolist() == lengths.tolist()
            gx, gy = C.gather(X, Y, rows[0, s:e], rows[1, s:e], int(rows[1, s]))
            assert torch.equal(x, torch.from_numpy(gx)) and torch.equal(y, torch.from_numpy(gy))
    if shuffle:
        assert [r.tolist() for r, _ in got][0] != [r.tolist() for r, _ in got][1]


def test_utterances_without_frames_keep_the_host_loader(tmp_path, monkeypatch, capsys):
    """A batch of 0-frame utterances has t = 0, which collate_fn pads to and the gather kernel refuses: such a corpus
    stays on the host loader whatever the budget, and the choice is made before any device is touched."""
    from gantts_b200 import train
    xd, yd = C.write_kind(str(tmp_path), "vc")
    for d in (xd, yd):
        np.save(str(tmp_path / os.path.basename(d) / "utt003.npy"), np.zeros((0, 12), dtype=np.float32))
    monkeypatch.setattr(train, "device_corpus_budget", lambda: 1 << 50)
    loaders, _, _, _ = train.load_data(C.KINDS["vc"][0](), xd, yd, -1)
    assert all(isinstance(v, data_utils.DataLoader) for v in loaders.values())
    assert "Data loader: host DataLoader (an utterance has no frames)" in capsys.readouterr().out
