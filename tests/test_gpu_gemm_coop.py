"""Cooperative tiles of the bf16x3 GEMM (both MMA warpgroups of a CTA on one tile, 64 rows each; the default) against the
ping-pong schedule (one warpgroup per tile, tiles in turn, GANTTS_B200_GEMM_COOP=0), for every launch of an MLP stack:
K-major forward and input-gradient launches with all three epilogues, and the weight gradients.

Each output element is the same MMAs in the same order either way (k ascending, hi*hi, hi*lo, lo*hi per K = 16 step), so
the forward output, input gradient, weight and bias gradients must agree bit for bit -- dropout and derivative codes
included: on the cfg2 step's shapes (G 425-512-512-512-187 over 32 000 frames, D 58-256-256-256-1 over the 64 000
real|fake rows) and on row counts that leave partial tiles and uneven reduction splits."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

G_DIMS = [425, 512, 512, 512, 187]
D_DIMS = [58, 256, 256, 256, 1]
SHAPES = [("G", 32000), ("D", 64000), ("G", 31999), ("D", 777), ("G", 4097), ("D", 130)]


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__
    __graft_entry__.build()
    return torch.device("cuda:0")


def run_stack(dev, net, M):
    from gantts_b200 import ops, _lib
    dims, act = (G_DIMS, _lib.ACT_NONE) if net == "G" else (D_DIMS, _lib.ACT_SIGMOID)
    torch.manual_seed(M)
    Ws = [(torch.randn(o, i) / np.sqrt(i)).to(dev).requires_grad_(True) for i, o in zip(dims[:-1], dims[1:])]
    bs = [(torch.randn(o) * 0.1).to(dev).requires_grad_(True) for o in dims[1:]]
    x = torch.randn(M, dims[0], device=dev, requires_grad=True)
    y = ops.mlp_stack(x, Ws, bs, p=0.5, training=True, seed=M, last_act=act)
    y.backward(torch.randn_like(y))
    torch.cuda.synchronize()
    return [y.detach(), x.grad] + [w.grad for w in Ws] + [b.grad for b in bs]


def assert_bitwise(a_outs, b_outs):
    for i, (a, b) in enumerate(zip(a_outs, b_outs)):
        assert torch.equal(a, b), "output %d differs (max |d| %g)" % (i, float((a - b).abs().max()))


@pytest.mark.parametrize("net,M", SHAPES)
def test_coop_tiles_match_ping_pong_bitwise(dev, monkeypatch, net, M):
    monkeypatch.setenv("GANTTS_B200_GEMM_COOP", "1")
    coop = run_stack(dev, net, M)
    monkeypatch.setenv("GANTTS_B200_GEMM_COOP", "0")
    assert_bitwise(coop, run_stack(dev, net, M))

