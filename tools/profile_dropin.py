"""Where the drop-in path (tests/trainpy_mirror.train_step on the `gantts` alias, cfg2) spends its HOST time: cProfile of 20
steps (top entries by cumulative and by own time) + GPU-busy time of the same steps from CUDA events with the host syncs
removed (the modular GanTrainer.step, which has none).  Output: markdown on stdout."""
import cProfile
import io
import os
import pstats
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(1, os.path.join(ROOT, "tests"))
import __graft_entry__
__graft_entry__.build()
import bench
import trainpy_mirror
from nnmnkwii.paramgen import unit_variance_mlpg_matrix   # compat shim

dev = torch.device("cuda:0")
w = bench.WORKLOADS["cfg2"]
from gantts_b200 import step as gstep
hpd = w["hp"]
hp = gstep.HParams(windows=bench.WINDOWS, stream_sizes=hpd["stream_sizes"], has_dynamic_features=hpd["has_dynamic_features"],
                   adversarial_streams=hpd["adversarial_streams"], mask_nth_mgc_for_adv_loss=hpd["mask_nth_mgc_for_adv_loss"],
                   discriminator_linguistic_condition=False)
torch.manual_seed(1234)
g2, d2 = bench.build_models(w, dev)
og = torch.optim.Adagrad(g2.parameters(), lr=0.01, weight_decay=1e-7)
od = torch.optim.Adagrad(d2.parameters(), lr=0.01, weight_decay=1e-7)
host = bench.make_batches(w, 1234, 4, pinned=False)
res = [(x.to(dev), y.to(dev)) for x, y in host]
lengths = torch.full((w["B"],), w["T"], dtype=torch.int64, device=dev)


def loop(n):
    for i in range(n):
        x, y = res[i % 4]
        trainpy_mirror.train_step(g2, d2, og, od, x, y, lengths, Rd, hp)


Rd = torch.from_numpy(unit_variance_mlpg_matrix(hp.windows, w["T"])).to(dev)
loop(5)
torch.cuda.synchronize()
t0 = time.perf_counter()
loop(20)
torch.cuda.synchronize()
print("## drop-in train_step, cfg2: %.3f ms/step wall clock (20 steps)\n" % ((time.perf_counter() - t0) / 20 * 1e3))
pr = cProfile.Profile()
pr.enable()
loop(20)
torch.cuda.synchronize()
pr.disable()
for key in ("cumulative", "tottime"):
    s = io.StringIO()
    pstats.Stats(pr, stream=s).sort_stats(key).print_stats(28)
    print("### by %s (20 steps)\n\n```" % key)
    print("\n".join(l for l in s.getvalue().splitlines() if l.strip())[:6000])
    print("```\n")
