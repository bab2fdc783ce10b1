"""The training command (python -m gantts_b200.train) on the GPU: a phase of its loop makes no host synchronisation
before its one read, and the five-stage recipe of train_gan.sh runs end to end on seeded synthetic vc data, with
checkpoints under the reference's names that load into the model classes and torch.optim, and scalars that match the
same loop driven by GanTrainer."""
import json
import os

import numpy as np
import pytest
import torch

import train_cli_helpers as H

pytestmark = pytest.mark.gpu

TOL = 2e-4


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__
    __graft_entry__.build()
    return torch.device("cuda:0")


def test_phase_makes_no_host_sync_before_its_read(dev, tmp_path):
    from gantts_b200 import train
    from gantts_b200.epochlog import EpochLog
    xd, yd = H.write_vc_data(str(tmp_path))
    hp = H.vc_hp()
    loaders, Ym, Ys, longest = train.load_data(hp, xd, yd, -1)
    from gantts_b200 import models
    torch.manual_seed(0)
    mg = models.In2OutHighwayNet(**hp.generator_params).to(dev)
    md = models.MLP(**hp.discriminator_params).to(dev)
    ref = models.MLP(hp.order, 1, 2, 8, dropout=0.0, last_sigmoid=True).to(dev).eval()
    path = train.make_path(mg, md, hp, hp.batch_size, longest, 1.0, 0.0, 1.0, ref, dev)
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
        assert "%s spoofing rate" % phase in vals and np.isfinite(vals["%s mcd metric" % phase])


STAGES = [
    # (name, extra argv, nepoch) -- train_gan.sh: baseline, generator warm-up, discriminator warm-up, adversarial
    ("baseline", ["--w_d=0"], 2),
    ("gan_g_warmup", ["--w_d=0"], 2),
    ("gan_d_warmup", ["--w_d=1", "--checkpoint-g={root}/gan_g_warmup/checkpoint_epoch2_Generator.pth",
                      "--discriminator-warmup", "--restart_epoch=0"], 2),
    ("gan", ["--checkpoint-d={root}/gan_d_warmup/checkpoint_epoch2_Discriminator.pth",
             "--checkpoint-g={root}/gan_g_warmup/checkpoint_epoch2_Generator.pth",
             "--checkpoint-r={root}/gan_d_warmup/checkpoint_epoch2_Discriminator.pth",
             "--w_d=1", "--reset_optimizers", "--restart_epoch=2"], 4),
]


def _run_recipe(root, xd, yd, make_hp, monkeypatch=None, force_modular=False):
    from gantts_b200 import train
    if force_modular:
        def refuse(*a, **k):
            raise RuntimeError("forced GanTrainer path")
        monkeypatch.setattr(train, "FusedGanStep", refuse)
    scalars = {}
    for name, extra, nepoch in STAGES:
        torch.manual_seed(5)
        np.random.seed(5)
        logdir = os.path.join(root, "log", name)
        argv = ["--hparams=nepoch=%d" % nepoch, "--checkpoint-dir=%s/%s" % (root, name),
                "--log-event-path=%s" % logdir, "--disable-slack"] + [a.format(root=root) for a in extra] + [xd, yd]
        assert train.main(argv, hp=make_hp()) == 0
        with open(os.path.join(logdir, "scalars.jsonl")) as f:
            scalars[name] = [json.loads(line) for line in f]
    if force_modular:
        monkeypatch.undo()
    return scalars


def test_recipe_end_to_end(dev, tmp_path, monkeypatch, capsys):
    root = str(tmp_path)
    xd, yd = H.write_vc_data(os.path.join(root, "data"))
    fused = _run_recipe(os.path.join(root, "fused"), xd, yd, H.vc_hp)
    assert "Training step: FusedGanStep" in capsys.readouterr().out
    modular = _run_recipe(os.path.join(root, "modular"), xd, yd, H.vc_hp, monkeypatch, force_modular=True)
    assert "Training step: GanTrainer" in capsys.readouterr().out
    # statistics under the reference's names
    assert os.path.exists(os.path.join(root, "data", "data_mean.npy"))
    assert os.path.exists(os.path.join(root, "data", "data_var.npy"))
    # checkpoints: names, layout, and they load into the model classes and torch.optim
    from gantts_b200 import models
    hp = H.vc_hp()
    expect = {"baseline": ["checkpoint_epoch2_Generator.pth"], "gan_g_warmup": ["checkpoint_epoch2_Generator.pth"],
              "gan_d_warmup": ["checkpoint_epoch2_Discriminator.pth"],
              "gan": ["checkpoint_epoch4_Discriminator.pth", "checkpoint_epoch4_Generator.pth"]}
    for stage, files in expect.items():
        assert sorted(os.listdir(os.path.join(root, "fused", stage))) == files, stage
        for f in files:
            ck = torch.load(os.path.join(root, "fused", stage, f))
            assert set(ck) == {"state_dict", "optimizer", "global_epoch"}
            assert ck["global_epoch"] == int(f.split("epoch")[1].split("_")[0])
            if "Generator" in f:
                m = models.In2OutHighwayNet(**dict(hp.generator_params, in_dim=12, out_dim=12))
            else:
                m = models.MLP(**hp.discriminator_params)
            m.load_state_dict(ck["state_dict"])
            torch.optim.Adagrad(m.parameters(), lr=0.01).load_state_dict(ck["optimizer"])
    # every scalar, stage by stage, against the GanTrainer-driven loop
    for stage in fused:
        names = [(s["name"], s["step"]) for s in fused[stage]]
        assert names == [(s["name"], s["step"]) for s in modular[stage]], stage
        for a, b in zip(fused[stage], modular[stage]):
            if "acc" in a["name"] or "spoofing" in a["name"]:
                # frame counts: a sigmoid output within rounding of 0.5 may land on the other side
                assert abs(a["value"] - b["value"]) <= 5e-3, (stage, a, b)
            else:
                assert abs(a["value"] - b["value"]) <= TOL * max(abs(b["value"]), 1e-2), (stage, a, b)
    names = {stage: sorted({s["name"] for s in v}) for stage, v in fused.items()}
    assert "train spoofing rate" in names["gan"] and "E(mge)" in names["gan"]
    assert "train discriminator loss" not in names["baseline"] and "train mcd metric" in names["baseline"]
    assert "train mge loss" not in names["gan_d_warmup"] and "Real train acc" in names["gan_d_warmup"]
    assert [s["step"] for s in fused["gan"]][0] == 3                    # --restart_epoch=2: epochs 3 and 4


def test_lstm_generator_takes_the_gantrainer_path(dev, tmp_path, capsys):
    from gantts_b200 import train
    root = str(tmp_path)
    xd, yd = H.write_vc_data(os.path.join(root, "data"))

    def run(hp, name):
        torch.manual_seed(0)
        logdir = os.path.join(root, "log", name)
        assert train.main(["--hparams=nepoch=1", "--w_d=1", "--checkpoint-dir=%s/%s" % (root, name),
                           "--log-event-path=%s" % logdir, xd, yd], hp=hp) == 0
        with open(os.path.join(logdir, "scalars.jsonl")) as f:
            return [json.loads(line)["name"] for line in f]

    lstm_hp = H.vc_hp(generator="LSTMRNN", generator_params={"in_dim": None, "out_dim": None, "num_hidden": 1,
                                                             "hidden_dim": 16, "bidirectional": True, "dropout": 0.0})
    lstm_names = run(lstm_hp, "lstm")
    assert "Training step: GanTrainer" in capsys.readouterr().out
    assert lstm_names == run(H.vc_hp(), "mlp")
    assert "Training step: FusedGanStep" in capsys.readouterr().out
