"""Time the fused GAN step (FusedGanStep: one C call per mini-batch) against the modular GanTrainer (Python autograd
over the native ops) on the SRURNN generator of hparams `tts_acoustic` and `tts_duration`.

Workloads (conditioned discriminator, generator dropout 0.2 / rnn_dropout 0.2, discriminator dropout 0.5, full-length
batches, w_d = 1, mse_w = 0, mge_w = 1):
  tts_acoustic  SRURNN 425 -> 6 x 512 bidirectional ReLU -> 187, D 483 -> 256 x 3 -> 1, Adagrad lr 0.01,
                B = 20 x T = 1000
  tts_duration  SRURNN 416 -> 6 x 512 bidirectional ReLU -> 5 (one static stream), D 421 -> 256 x 3 -> 1,
                Adam lr 1e-3 betas (0.5, 0.9), B = 32 x T = 128

The two paths alternate in one process, round by round, each round timed with CUDA events after a warm-up; the GPU's
name, power limit and maximum SM clock are queried in the same run (nvidia-smi, read-only).  Needs a CUDA device.

    python tools/time_sru_step.py [--rounds 5] [--steps 10] [--warmup 5] [--json OUT]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.time_vc_step import gpu_info  # noqa: E402

WINDOWS = [(0, 0, np.array([1.0])), (1, 1, np.array([-0.5, 0.0, 0.5])), (1, 1, np.array([1.0, -2.0, 1.0]))]
WORKLOADS = {
    "tts_acoustic": dict(B=20, T=1000, in_dim=425, out_dim=187, n_adv=58, optimizer="Adagrad",
                         okw=dict(lr=0.01, weight_decay=0.0)),
    "tts_duration": dict(B=32, T=128, in_dim=416, out_dim=5, n_adv=5, optimizer="Adam",
                         okw=dict(lr=1e-3, betas=(0.5, 0.9), weight_decay=0.0, eps=1e-8)),
}


def hparams(name):
    from gantts_b200 import step as gstep
    if name == "tts_acoustic":
        return gstep.HParams(dict(gstep.TTS_ACOUSTIC, discriminator_linguistic_condition=True))
    return gstep.HParams(windows=WINDOWS[:1], stream_sizes=[5], has_dynamic_features=[False], adversarial_streams=[True],
                         mask_nth_mgc_for_adv_loss=0, discriminator_linguistic_condition=True)


def run(name, w, rounds, steps, warmup, dev):
    import gantts_b200
    from gantts_b200 import fused, step as gstep
    from oracle import nnmnkwii_port as nnp
    B, T = w["B"], w["T"]
    hp = hparams(name)

    def models():
        torch.manual_seed(1234)
        mg = gantts_b200.models.SRURNN(in_dim=w["in_dim"], out_dim=w["out_dim"], num_hidden=6, hidden_dim=512,
                                       bidirectional=True, dropout=0.2, use_relu=1, rnn_dropout=0.2)
        md = gantts_b200.models.MLP(w["in_dim"] + w["n_adv"], 1, 3, 256, dropout=0.5, last_sigmoid=True)
        return mg.to(dev).train(), md.to(dev).train()
    g = torch.Generator().manual_seed(7)
    x = torch.randn(B, T, w["in_dim"], generator=g).to(dev)
    y = torch.randn(B, T, w["out_dim"], generator=g).to(dev)
    lengths = torch.full((B,), T, dtype=torch.int64, device=dev)
    kw = dict(w_d=1.0, mse_w=0.0, mge_w=1.0, optimizer=w["optimizer"])
    fs = fused.FusedGanStep(*models(), hp, B, T, seed=1, optimizer_params=w["okw"], **kw)
    tr = gstep.GanTrainer(*models(), hp, optimizer_params=w["okw"], **kw)
    R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(hp.windows, T)).to(dev)
    steps_of = {"fused": lambda: fs.step(x, y, lengths),
                "modular": lambda: tr.step(x, y, lengths, R)}
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
    out = {"workload": name, "B": B, "T": T, "rounds": rounds, "steps_per_round": steps}
    for k, v in ms.items():
        med = float(np.median(v))
        out[k] = {"ms_per_step_median": round(med, 3), "ms_per_step_min": round(min(v), 3),
                  "ms_per_step_max": round(max(v), 3), "frames_per_s": round(B * T / med * 1e3, 1)}
    out["speedup_fused_vs_modular"] = round(out["modular"]["ms_per_step_median"] / out["fused"]["ms_per_step_median"], 3)
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--workload", choices=sorted(WORKLOADS) + ["all"], default="all")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--json", default=None, help="also write the results to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_sru_step.py: needs a CUDA device (there is no CPU path to time)")
    import __graft_entry__
    __graft_entry__.build()
    dev = torch.device("cuda:0")
    res = {"gpu": gpu_info(), "results": []}
    for name in (sorted(WORKLOADS) if args.workload == "all" else [args.workload]):
        r = run(name, WORKLOADS[name], args.rounds, args.steps, args.warmup, dev)
        print(json.dumps(r), flush=True)
        res["results"].append(r)
    print(json.dumps({"gpu": res["gpu"]}))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
