"""Micro-timing of gantts_mlp_fwd/bwd (CUDA events) for the cfg2 generator and discriminator shapes."""
import os, sys, ctypes
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import __graft_entry__
__graft_entry__.build()
from gantts_b200 import ops, _lib
dev = torch.device("cuda:0")
torch.manual_seed(0)

def run(M, dims, p, last_act, tag):
    Ws = [(torch.randn(o, i) / i ** 0.5).to(dev).requires_grad_(True) for i, o in zip(dims[:-1], dims[1:])]
    bs = [torch.zeros(o, device=dev, requires_grad=True) for o in dims[1:]]
    x = torch.rand(M, dims[0], device=dev)
    g = torch.randn(M, dims[-1], device=dev)
    def f():
        y = ops.mlp_stack(x, Ws, bs, p=p, training=p > 0, last_act=last_act, seed=5)
        return y
    for _ in range(40):
        y = f(); y.backward(g)
    torch.cuda.synchronize()
    e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    n = 20
    tf = tb = 0.0
    for _ in range(n):
        e[0].record(); y = f(); e[1].record(); y.backward(g); e[2].record()
        torch.cuda.synchronize()
        tf += e[0].elapsed_time(e[1]); tb += e[1].elapsed_time(e[2])
    lib = _lib.load()
    lib.gantts_profile_enable(1)
    for _ in range(n):
        y = f()
    torch.cuda.synchronize()
    ms, wk, cnt = (ctypes.c_double * 8)(), (ctypes.c_double * 8)(), (ctypes.c_longlong * 8)()
    lib.gantts_profile_collect(ms, wk, cnt)
    msf, cf = ms[0], cnt[0]
    for _ in range(n):
        y = f(); y.backward(g)
    torch.cuda.synchronize()
    ms2, wk2, cnt2 = (ctypes.c_double * 8)(), (ctypes.c_double * 8)(), (ctypes.c_longlong * 8)()
    lib.gantts_profile_collect(ms2, wk2, cnt2)
    lib.gantts_profile_enable(0)
    print("   gemm-only [%s]:" % tag, flush=True); print("    fwd KK %.1f us (%d launches/iter); fwd+bwd KK %.1f us MN %.1f us" % (
        msf / n * 1e3, cf // n, ms2[0] / n * 1e3, ms2[1] / n * 1e3), flush=True)
    fl = 2.0 * M * sum(a * b for a, b in zip(dims[:-1], dims[1:]))
    print("%-28s fwd %.1f us (%.0f TF alg)  bwd %.1f us (%.0f TF alg)" % (
        tag, tf / n * 1e3, fl / (tf / n * 1e-3) / 1e12,
        tb / n * 1e3, 2 * fl / (tb / n * 1e-3) / 1e12), flush=True)

run(32000, [425, 512, 512, 512, 187], 0.0, _lib.ACT_NONE, "G 425-512x3-187 p=0")
run(32000, [425, 512, 512, 512, 187], 0.5, _lib.ACT_NONE, "G 425-512x3-187 p=.5")
run(32000, [425, 512, 512, 512, 187], 0.0, _lib.ACT_NONE, "G 425-512x3-187 p=0")
run(64000, [58, 256, 256, 256, 1], 0.5, _lib.ACT_SIGMOID, "D 58-256x3-1 2M rows p=.5")
run(64000, [58, 256, 256, 256, 1], 0.0, _lib.ACT_SIGMOID, "D 58-256x3-1 2M rows p=0")
