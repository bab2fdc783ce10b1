"""Time the fused GAN step (FusedGanStep: one C call per mini-batch) against the modular GanTrainer (Python autograd
over the native ops) on the generators the fused step runs, each with its MLP discriminator.

Workloads (full-length batches; mse_w = 0, mge_w = 1 unless stated):
  vc            hparams.vc with adversarial training: In2OutHighwayNet 177 -> 512 x 3 -> 177 (static 59), D 59 -> 256 ->
                256 -> 1, dropout 0.5, Adagrad lr 0.01 wd 0, B = 20 x T = 1000, w_d = 1
  cfg1          the same generator without a discriminator: B = 8 x T = 200, w_d = 0, mse_w = mge_w = 1
  tts_acoustic  SRURNN 425 -> 6 x 512 bidirectional ReLU -> 187 (dropout 0.2, rnn_dropout 0.2), D 483 -> 256 x 3 -> 1
                conditioned on x with dropout 0.5, Adagrad lr 0.01 wd 0, B = 20 x T = 1000, w_d = 1
  tts_duration  SRURNN 416 -> 6 x 512 bidirectional ReLU -> 5 (one static stream), D 421 -> 256 x 3 -> 1 conditioned,
                Adam lr 1e-3 betas (0.5, 0.9), B = 32 x T = 128, w_d = 1
  cfg3          In2OutRNNHighwayNet 177 -> 177 (static 59, 3 x 512 bidirectional LSTM, LSTM dropout 0.5), D 59 -> 256 ->
                256 -> 1 with dropout 0.5, Adagrad lr 0.01 wd 0, B = 16 x T = 2000, w_d = 1

The two paths alternate in one process, round by round, each round timed with CUDA events after a warm-up; the GPU's
name, power limit and maximum SM clock are queried in the same run (nvidia-smi, read-only).  Needs a CUDA device.

--stage d_warmup and --spoof time the features of the five-stage recipe (train_gan.sh) instead of the modular path: in
one process, round by round, the full fused step ("fused"), with --stage d_warmup the discriminator warm-up step
(FusedGanStep.step(update_g=False): "fused_d_only"), and with --spoof the full step that also counts the spoofing rate of
a reference discriminator (train.py:549-558: "fused_spoof").  The reference discriminator has D's class and shape on the
adversarial columns alone (train.py:779-781), so with --rnn-d it is an LSTMRNN too.

--rnn-d replaces the MLP discriminator of vc and tts_acoustic by a recurrent one, LSTMRNN(n, 1, 2, 256,
bidirectional=True, dropout=0.5, last_sigmoid=True) with n = 59 (vc) or 425 + 58 conditioning + adversarial inputs
(tts_acoustic), and times the fused step against the modular path as above.

--dump-outputs DIR: after the timed loop, DIR/<workload>/ receives what the fused path's caller holds after its last
step, as float32 .npy files: the loss vector, y_hat, y_hat_static, both flat gradient buffers and every updated
parameter of both models.  Two builds run with the same arguments can then be compared array by array.

    python tools/time_fused_step.py [--workload vc|cfg1|tts_acoustic|tts_duration|cfg3|all] [--rounds R] [--steps K]
                                    [--warmup W] [--json OUT] [--dump-outputs DIR] [--stage adversarial|d_warmup]
                                    [--spoof] [--rnn-d]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

WINDOWS = [(0, 0, np.array([1.0])), (1, 1, np.array([-0.5, 0.0, 0.5])), (1, 1, np.array([1.0, -2.0, 1.0]))]
ADAGRAD = dict(optimizer="Adagrad", okw=dict(lr=0.01, weight_decay=0.0))
# kind, batch, loss weights, optimiser and the default rounds / steps per round / warm-up steps
WORKLOADS = {
    "vc": dict(kind="highway", B=20, T=1000, w_d=1.0, mse_w=0.0, mge_w=1.0, runs=(5, 20, 10), **ADAGRAD),
    "cfg1": dict(kind="highway", B=8, T=200, w_d=0.0, mse_w=1.0, mge_w=1.0, runs=(5, 20, 10), **ADAGRAD),
    "tts_acoustic": dict(kind="sru", B=20, T=1000, w_d=1.0, mse_w=0.0, mge_w=1.0, runs=(5, 10, 5), in_dim=425,
                         out_dim=187, n_adv=58, **ADAGRAD),
    "tts_duration": dict(kind="sru", B=32, T=128, w_d=1.0, mse_w=0.0, mge_w=1.0, runs=(5, 10, 5), in_dim=416,
                         out_dim=5, n_adv=5, optimizer="Adam",
                         okw=dict(lr=1e-3, betas=(0.5, 0.9), weight_decay=0.0, eps=1e-8)),
    "cfg3": dict(kind="rnn_highway", B=16, T=2000, w_d=1.0, mse_w=0.0, mge_w=1.0, runs=(5, 5, 3), **ADAGRAD),
}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    line = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else ""
    parts = [s.strip() for s in line.split(",")] if line else []
    return {"name": parts[0] if parts else torch.cuda.get_device_name(0),
            "power_limit": parts[1] if len(parts) > 1 else None,
            "sm_clock_max": parts[2] if len(parts) > 2 else None}


def hparams(name):
    from gantts_b200 import step as gstep
    if name == "tts_acoustic":
        return gstep.HParams(dict(gstep.TTS_ACOUSTIC, discriminator_linguistic_condition=True))
    if name == "tts_duration":
        return gstep.HParams(windows=WINDOWS[:1], stream_sizes=[5], has_dynamic_features=[False],
                             adversarial_streams=[True], mask_nth_mgc_for_adv_loss=0,
                             discriminator_linguistic_condition=True)
    return gstep.HParams(windows=WINDOWS, stream_sizes=[177], has_dynamic_features=[True], adversarial_streams=[True],
                         mask_nth_mgc_for_adv_loss=0, discriminator_linguistic_condition=False)


def models(w, dev, rnn_d=False):
    import gantts_b200
    M = gantts_b200.models
    torch.manual_seed(1234)
    if w["kind"] == "highway":
        mg = M.In2OutHighwayNet(in_dim=177, out_dim=177, static_dim=59, num_hidden=3, hidden_dim=512, dropout=0.5)
        md = M.MLP(59, 1, 2, 256, dropout=0.5, last_sigmoid=True)
    elif w["kind"] == "sru":
        mg = M.SRURNN(in_dim=w["in_dim"], out_dim=w["out_dim"], num_hidden=6, hidden_dim=512, bidirectional=True,
                      dropout=0.2, use_relu=1, rnn_dropout=0.2)
        md = M.MLP(w["in_dim"] + w["n_adv"], 1, 3, 256, dropout=0.5, last_sigmoid=True)
    else:
        mg = M.In2OutRNNHighwayNet(in_dim=177, out_dim=177, static_dim=59, num_hidden=3, hidden_dim=512,
                                   bidirectional=True, dropout=0.5)
        md = M.MLP(59, 1, 2, 256, dropout=0.5, last_sigmoid=True)
    if rnn_d:
        torch.manual_seed(4321)
        md = M.LSTMRNN(md.layers[0].weight.shape[1], 1, 2, 256, bidirectional=True, dropout=0.5, last_sigmoid=True)
    return mg.to(dev).train(), md.to(dev).train()


def reference_discriminator(md, n_adv, dev):
    """The spoofing-rate discriminator: D's class and shape (train.py:779-781 builds it from hp.discriminator like D) on
    the n_adv adversarial columns alone, since train.py:554-555 feeds it no conditioning."""
    import gantts_b200
    M = gantts_b200.models
    torch.manual_seed(99)
    if isinstance(md, M._LSTMNet):
        rnn = getattr(md, md._rnn_attr)
        ref_d = type(md)(n_adv, 1, rnn.num_layers, rnn.hidden_size, bidirectional=rnn.bidirectional, dropout=rnn.dropout,
                         last_sigmoid=True)
    else:
        ref_d = M.MLP(n_adv, 1, len(md.layers), md.layers[0].weight.shape[0], dropout=md.dropout_p, last_sigmoid=True)
    return ref_d.to(dev)


def dump(out_dir, fs, mg, md):
    os.makedirs(out_dir, exist_ok=True)
    arrays = {"losses": fs.losses, "y_hat": fs.y_hat, "y_hat_static": fs.y_hat_static,
              "grad_g": fs.grad_buffer(0), "grad_d": fs.grad_buffer(1)}
    for pre, m in (("g.", mg), ("d.", md)):
        arrays.update({pre + k: v for k, v in m.state_dict().items()})
    for k, t in arrays.items():
        np.save(os.path.join(out_dir, k + ".npy"), t.detach().float().cpu().numpy())


def run(name, w, rounds, steps, warmup, dev, dump_dir=None, stage="adversarial", spoof=False, rnn_d=False):
    from gantts_b200 import fused, step as gstep
    from oracle import nnmnkwii_port as nnp
    B, T = w["B"], w["T"]
    hp = hparams(name)
    in_dim = w.get("in_dim", 177)
    g = torch.Generator().manual_seed(7)
    x = torch.randn(B, T, in_dim, generator=g).to(dev)
    y = torch.randn(B, T, w.get("out_dim", 177), generator=g).to(dev)
    lengths = torch.full((B,), T, dtype=torch.int64, device=dev)
    adv_w = 1.0 if w["w_d"] > 0 else 0.0
    kw = dict(w_d=w["w_d"], mse_w=w["mse_w"], mge_w=w["mge_w"], optimizer=w["optimizer"], optimizer_params=w["okw"])
    mg, md = models(w, dev, rnn_d)
    fs = fused.FusedGanStep(mg, md, hp, B, T, seed=1, **kw)
    steps_of = {"fused": lambda: fs.step(x, y, lengths, adv_w=adv_w)}
    if stage == "d_warmup":
        steps_of["fused_d_only"] = lambda: fs.step(x, y, lengths, adv_w=adv_w, update_g=False)
    if spoof:
        ref_d = reference_discriminator(md, len(fused.adversarial_columns(hp)), dev)
        fs_spoof = fused.FusedGanStep(*models(w, dev, rnn_d), hp, B, T, seed=2, reference_discriminator=ref_d, **kw)
        steps_of["fused_spoof"] = lambda: fs_spoof.step(x, y, lengths, adv_w=adv_w)
    if len(steps_of) == 1:
        tr = gstep.GanTrainer(*models(w, dev, rnn_d), hp, **kw)
        R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(hp.windows, T)).to(dev)
        steps_of["modular"] = lambda: tr.step(x, y, lengths, R, adv_w=adv_w)
    for fn in steps_of.values():
        for _ in range(warmup):
            fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in steps_of}
    for _ in range(rounds):
        for k, fn in steps_of.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(steps):
                fn()
            b.record()
            b.synchronize()
            ms[k].append(a.elapsed_time(b) / steps)
    if dump_dir:
        dump(os.path.join(dump_dir, name), fs, mg, md)
    out = {"workload": name, "B": B, "T": T, "rounds": rounds, "steps_per_round": steps,
           "discriminator": type(md).__name__}
    for k, v in ms.items():
        med = float(np.median(v))
        out[k] = {"ms_per_step_median": round(med, 4), "ms_per_step_min": round(min(v), 4),
                  "ms_per_step_max": round(max(v), 4), "frames_per_s": round(B * T / med * 1e3, 1)}
    for k in ms:
        if k != "fused":
            out["ratio_%s_vs_fused" % k] = round(out[k]["ms_per_step_median"] / out["fused"]["ms_per_step_median"], 3)
    if "modular" in ms:
        out["speedup_fused_vs_modular"] = round(out["modular"]["ms_per_step_median"] / out["fused"]["ms_per_step_median"], 3)
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--workload", choices=list(WORKLOADS) + ["all"], default="all")
    ap.add_argument("--rounds", type=int, default=None, help="default: per workload (5)")
    ap.add_argument("--steps", type=int, default=None, help="steps per round; default: per workload (20, 10 or 5)")
    ap.add_argument("--warmup", type=int, default=None, help="default: per workload (10, 5 or 3)")
    ap.add_argument("--json", default=None, help="also write the results to this file")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the fused path's outputs after the timed loop to DIR/<workload>/*.npy")
    ap.add_argument("--stage", choices=("adversarial", "d_warmup"), default="adversarial",
                    help="d_warmup: also time the discriminator warm-up step (update_g=False)")
    ap.add_argument("--spoof", action="store_true",
                    help="also time the full step with the spoofing-rate count of a reference discriminator")
    ap.add_argument("--rnn-d", action="store_true",
                    help="vc / tts_acoustic with an LSTMRNN discriminator (2 x 256 bidirectional) instead of the MLP")
    args = ap.parse_args()
    if args.rnn_d and args.workload not in ("vc", "tts_acoustic"):
        sys.exit("time_fused_step.py: --rnn-d times the vc and tts_acoustic workloads")
    if args.stage == "d_warmup" or args.spoof:
        ok = [k for k, w in WORKLOADS.items() if w["w_d"] > 0]
        if args.workload not in ok:
            sys.exit("time_fused_step.py: --stage d_warmup / --spoof need a workload with a discriminator: %s" % ok)
    if not torch.cuda.is_available():
        sys.exit("time_fused_step.py: needs a CUDA device (there is no CPU path to time)")
    import __graft_entry__
    __graft_entry__.build()
    dev = torch.device("cuda:0")
    res = {"gpu": gpu_info(), "results": []}
    for name in (list(WORKLOADS) if args.workload == "all" else [args.workload]):
        w = WORKLOADS[name]
        rounds, steps, warmup = [d if a is None else a for a, d in zip((args.rounds, args.steps, args.warmup), w["runs"])]
        r = run(name, w, rounds, steps, warmup, dev, args.dump_outputs, args.stage, args.spoof, args.rnn_d)
        print(json.dumps(r), flush=True)
        res["results"].append(r)
    print(json.dumps({"gpu": res["gpu"]}))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
