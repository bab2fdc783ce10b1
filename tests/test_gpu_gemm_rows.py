"""An output row of the bf16x3 GEMM does not depend on how many rows the launch covers, for every launch of an MLP
stack that produces it: K-major forward and input-gradient launches with all three epilogues, the staged fp32 stores
of unaligned rows (y_hat ld 187, the input gradient ld 58) included.

Each output element is the same MMAs in the same order whichever tile and warpgroup it falls in (k ascending, hi*hi,
hi*lo, lo*hi per K = 16 step), and dropout and derivative codes are keyed by the global row.  So the first M' rows of
an M-row run -- forward output, and input gradient under the same upstream gradient rows -- must equal an M'-row run
on those rows bit for bit: on the cfg2 step's shapes (G 425-512-512-512-187 over 32 000 frames, D 58-256-256-256-1
over the 64 000 real|fake rows) and on row counts that leave partial tiles.  Weight and bias gradients are left out:
their split-K plan depends on the row count."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

G_DIMS = [425, 512, 512, 512, 187]
D_DIMS = [58, 256, 256, 256, 1]
SHAPES = [("G", 32000), ("D", 64000), ("G", 31999), ("D", 777), ("G", 4097), ("D", 130)]
# (net, M, M') for every M' < M of the same net in SHAPES
PAIRS = [(net, M, m) for net, M in SHAPES for n, m in SHAPES if n == net and m < M]


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__
    __graft_entry__.build()
    return torch.device("cuda:0")


def run_stack(dev, net, M, seed, rows=None):
    """Forward and backward of the stack over the first `rows` (default: all) of M input and upstream-gradient rows
    drawn on the CPU from `seed`, which also keys the dropout."""
    from gantts_b200 import ops, _lib
    dims, act = (G_DIMS, _lib.ACT_NONE) if net == "G" else (D_DIMS, _lib.ACT_SIGMOID)
    torch.manual_seed(seed)
    Ws = [(torch.randn(o, i) / np.sqrt(i)).to(dev).requires_grad_(True) for i, o in zip(dims[:-1], dims[1:])]
    bs = [(torch.randn(o) * 0.1).to(dev).requires_grad_(True) for o in dims[1:]]
    x = torch.randn(M, dims[0])[:rows].to(dev).requires_grad_(True)
    g = torch.randn(M, dims[-1])[:rows].to(dev)
    y = ops.mlp_stack(x, Ws, bs, p=0.5, training=True, seed=seed, last_act=act)
    y.backward(g)
    torch.cuda.synchronize()
    return [y.detach(), x.grad] + [w.grad for w in Ws] + [b.grad for b in bs]


def assert_bitwise(a_outs, b_outs):
    for i, (a, b) in enumerate(zip(a_outs, b_outs)):
        assert torch.equal(a, b), "output %d differs (max |d| %g)" % (i, float((a - b).abs().max()))


@pytest.mark.parametrize("net,M,rows", PAIRS)
def test_row_bits_do_not_depend_on_launch_rows(dev, net, M, rows):
    full = run_stack(dev, net, M, seed=M)
    part = run_stack(dev, net, M, seed=M, rows=rows)
    assert_bitwise([full[0][:rows], full[1][:rows]], part[:2])
