"""The planes epilogue of the K-major bf16x3 GEMM leaves through TMA stores that clip each warp's 16-row x 32-column
box at the launch's last row and at the plane pitch.  These cases put every kind of edge under those boxes: row counts
that end inside a warp's 16 rows, a tile's 128 rows and the cfg2 step's 32 000 (1, 127, 129, 31 995), hidden widths
with a partial column tile or a pitch tail (64, 187 -> pitch 192, 256, 512), dropout on and off, and a row window that
starts inside a tile.

An MLP [40, N, N, 24] runs two planes-forward launches (hidden layers of width N, with derivative codes) and one
planes-backward launch (the hidden gradient of width N) whose outputs only reach y and the input gradient through the
next GEMM.  Both must be bit-identical to the same rows inside a 32 000-row run (dropout is keyed by the global row),
and match the exact-fp32 per-layer engine (engine="simt") within the tensor-core tolerance of 1e-4."""
import functools

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

FULL = 32000
ROWS = [1, 127, 129, FULL - 5]
WIDTHS = [64, 187, 256, 512]
DIMS_IN, DIMS_OUT = 40, 24
SEED = 424242


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__
    __graft_entry__.build()
    return torch.device("cuda:0")


@functools.lru_cache(maxsize=None)
def problem(N):
    """Weights, biases, FULL input rows and upstream-gradient rows on the CPU."""
    g = torch.Generator().manual_seed(N)
    dims = [DIMS_IN, N, N, DIMS_OUT]
    Ws = [torch.randn(o, i, generator=g) / np.sqrt(i) for i, o in zip(dims[:-1], dims[1:])]
    bs = [torch.randn(o, generator=g) * 0.1 for o in dims[1:]]
    x = torch.randn(FULL, DIMS_IN, generator=g)
    gy = torch.randn(FULL, DIMS_OUT, generator=g)
    return Ws, bs, x, gy


def run(dev, N, p, lo, hi, slope=0.01, engine="tc"):
    """y and the input gradient of rows [lo, hi) run alone, through the fused stack (tc) or layer by layer (simt)."""
    from gantts_b200 import ops, _lib
    Ws, bs, x, gy = problem(N)
    Ws = [w.to(dev).requires_grad_(True) for w in Ws]
    bs = [b.to(dev).requires_grad_(True) for b in bs]
    xs = x[lo:hi].to(dev).requires_grad_(True)
    if engine == "tc":
        y = ops.mlp_stack(xs, Ws, bs, p=p, training=p > 0, seed=SEED, slope=slope)
    else:
        lib = _lib.load()
        h = xs
        for l in range(2):
            h = ops.linear_act(h, Ws[l], bs[l], _lib.ACT_LEAKY_DROPOUT, p=p, training=p > 0, engine="simt",
                               seed=lib.gantts_mlp_layer_seed(SEED, l), slope=slope)
        y = ops.linear_act(h, Ws[2], bs[2], _lib.ACT_NONE, engine="simt")
    y.backward(gy[lo:hi].to(dev))
    torch.cuda.synchronize()
    return y.detach(), xs.grad


@functools.lru_cache(maxsize=None)
def full_run(dev, N, p):
    return run(dev, N, p, 0, FULL)


def rel_err(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


@pytest.mark.parametrize("p", [0.0, 0.5])
@pytest.mark.parametrize("N", WIDTHS)
@pytest.mark.parametrize("rows", ROWS)
def test_planes_rows_alone_match_full_run(dev, rows, N, p):
    fy, fgx = full_run(dev, N, p)
    y, gx = run(dev, N, p, 0, rows)
    assert torch.equal(y, fy[:rows]), "y differs (max |d| %g)" % float((y - fy[:rows]).abs().max())
    assert torch.equal(gx, fgx[:rows]), "gx differs (max |d| %g)" % float((gx - fgx[:rows]).abs().max())


@pytest.mark.parametrize("N", WIDTHS)
@pytest.mark.parametrize("lo,hi", [(129, 4129), (FULL - 300, FULL - 1)])
def test_planes_row_window_matches_full_run(dev, N, lo, hi):
    """Rows [lo, hi) as a launch of their own: every tile and box boundary moves against the full run's (no dropout,
    whose keys would follow the window's own row numbers)."""
    fy, fgx = full_run(dev, N, 0.0)
    y, gx = run(dev, N, 0.0, lo, hi)
    assert torch.equal(y, fy[lo:hi]) and torch.equal(gx, fgx[lo:hi])


@pytest.mark.parametrize("p", [0.0, 0.5])
@pytest.mark.parametrize("N", WIDTHS)
@pytest.mark.parametrize("rows", [127, 129])
def test_planes_match_simt(dev, rows, N, p):
    """slope 1 keeps pre-activations within rounding of zero from landing on different sides of the kink in the two
    engines (test_gpu_parity.py explains)."""
    y, gx = run(dev, N, p, 0, rows, slope=1.0)
    ry, rgx = run(dev, N, p, 0, rows, slope=1.0, engine="simt")
    assert rel_err(y, ry) < 1e-4 and rel_err(gx, rgx) < 1e-4, (rel_err(y, ry), rel_err(gx, rgx))
