"""Same-box library bar for the recurrent generators (SURVEY.md 2.2 K8): torch-CUDA nn.LSTM (cuDNN) forward + backward at
the BASELINE cfg3 / cfg5 shapes next to gantts_b200.rnn.lstm_forward on the same weights and inputs.  CUDA events,
3 warm-ups + 5 timed iterations.  Prints one markdown table."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import __graft_entry__
__graft_entry__.build()
from gantts_b200 import rnn

dev = torch.device("cuda:0")
torch.manual_seed(0)


def timeit(fn, warm=3, iters=5):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def case(name, B, T, I, H, layers):
    lstm = torch.nn.LSTM(I, H, layers, batch_first=True, bidirectional=True).to(dev)
    x = torch.randn(B, T, I, device=dev, requires_grad=True)
    g = torch.randn(B, T, 2 * H, device=dev)
    lens = [T] * B

    def cudnn_fwd():
        with torch.no_grad():
            lstm(x)

    def cudnn_fb():
        y, _ = lstm(x)
        y.backward(g)

    def cudnn_tf32_fb():
        torch.backends.cudnn.allow_tf32 = True
        y, _ = lstm(x)
        y.backward(g)

    def ours_fwd():
        with torch.no_grad():
            rnn.lstm_forward(lstm, x, lens, False)

    def ours_fb():
        rnn.lstm_forward(lstm, x, lens, True).backward(g)

    torch.backends.cudnn.allow_tf32 = False
    a, b = timeit(cudnn_fwd), timeit(cudnn_fb)
    c = timeit(cudnn_tf32_fb)
    torch.backends.cudnn.allow_tf32 = False
    d, e = timeit(ours_fwd), timeit(ours_fb)
    flops = 2.0 * B * T * sum(2 * 4 * H * ((I if k == 0 else 2 * H) + H) for k in range(layers))
    print("| %s | B=%d T=%d %d->%dx%d bi | %.1f | %.1f | %.1f | %.1f | %.1f | %.2f | %.1f |" % (
        name, B, T, I, layers, H, a, b, c, d, e, e / b, 3 * flops / (e * 1e-3) / 1e12), flush=True)


print("| config | shape | cuDNN fp32 fwd ms | cuDNN fp32 fwd+bwd ms | cuDNN TF32 fwd+bwd ms | ours fwd ms | ours fwd+bwd ms | "
      "ours / cuDNN fp32 | ours TF/s (3x fwd flops) |")
print("|---|---|---|---|---|---|---|---|---|")
case("cfg3", 16, 2000, 177, 512, 3)
case("cfg5", 64, 1500, 425, 512, 3)
case("small", 8, 300, 177, 512, 3)
