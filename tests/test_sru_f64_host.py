"""Pins tests/sru_f64.py, the float64 reference of the SRU scan kernels, without a GPU:
  * the restatement equals the SRU layer of oracle/gantts_port.py (sru_layer_forward) run in float64, output and every
    gradient, for k = 3 and 4, one and two directions, all three activations, with and without the output mask;
  * its length-exact forward is, row by row, the padded forward of that row alone at T = its length;
  * the GPU case matrix reaches every chunk tail, the 128-thread block edges and every kind of length;
  * gantts_sru_fwd and gantts_sru_bwd refuse a B * columns their launch cannot count, before any device work.
"""
import pytest
import torch

import sru_f64 as ref
from sru_f64 import CASES
from oracle import gantts_port as gp

TOL = 1e-12
FAKE = 1 << 20          # placeholder device pointer: the argument checks never dereference it


def _rel(a, b):
    a, b = a.detach(), b.detach()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-300))


def _layer(B, T, n_in, d, bidir, seed, p):
    g = torch.Generator().manual_seed(seed)
    dirs = 2 if bidir else 1
    ncols = dirs * d
    k = 3 if n_in == ncols else 4
    x = torch.randn(B, T, n_in, generator=g, dtype=torch.float64)
    W = (torch.rand(n_in, ncols * k, generator=g, dtype=torch.float64) * 2 - 1) * (3.0 / n_in) ** 0.5
    bias = (torch.rand(2 * ncols, generator=g, dtype=torch.float64) * 2 - 1) * 0.5
    mask = (torch.rand(B, ncols, generator=g, dtype=torch.float64) >= p).double() / (1 - p) if p else None
    dh = torch.randn(B, T, ncols, generator=g, dtype=torch.float64)
    return k, x, W, bias, mask, dh


@pytest.mark.parametrize("act", [0, 1, 2])
@pytest.mark.parametrize("bidir", [False, True])
@pytest.mark.parametrize("k", [3, 4])
@pytest.mark.parametrize("p", [0.0, 0.3])
def test_restatement_equals_oracle_layer_float64(k, bidir, act, p):
    B, T, d = 3, 11, 5
    ncols = d * (2 if bidir else 1)
    n_in = ncols if k == 3 else 7
    kk, x, W, bias, mask, dh = _layer(B, T, n_in, d, bidir, 10 * k + 2 * bidir + act, p)
    assert kk == k
    dirs = 2 if bidir else 1

    # the oracle: x (T, B, n_in), bias [dir][f | r][d]
    xo, Wo, bo = (t.clone().requires_grad_(True) for t in (x, W, bias))
    bport = torch.stack([bo[:ncols].view(dirs, d), bo[ncols:].view(dirs, d)], 1).reshape(-1)
    ho = gp.sru_layer_forward(xo.transpose(0, 1), Wo, bport, bidirectional=bidir, use_tanh=act == 1,
                              use_relu=act == 2, mask_h=mask).transpose(0, 1)
    ho.backward(dh)

    # the restatement at the C contract: u = x W, the highway input x when k == 3
    xr, Wr, br = (t.clone().requires_grad_(True) for t in (x, W, bias))
    u = xr @ Wr
    h, c = ref.sru_f64(u, xr if k == 3 else None, br, mask, d, bidir, act)
    h.backward(dh)
    assert _rel(h, ho.detach()) < TOL
    for name, a, b in (("x", xr, xo), ("W", Wr, Wo), ("bias", br, bo)):
        assert _rel(a.grad, b.grad) < TOL, name

    # the scan's own backward: du / dx / dbias_part map back to the same gradients
    du, dx, part = ref.sru_f64_bwd(u.detach(), x if k == 3 else None, bias, mask, d, bidir, act, dh)
    assert _rel(part.sum(0), br.grad) < TOL
    gx = du @ W.t() + (dx if k == 3 else 0)
    assert _rel(gx, xr.grad) < TOL
    assert _rel(torch.einsum("bti,btj->ij", x, du), Wr.grad) < TOL
    # the ReLU pattern of the cell states themselves gives the same gradients
    du2, dx2, part2 = ref.sru_f64_bwd(u.detach(), x if k == 3 else None, bias, mask, d, bidir, act, dh, c_relu=c)
    assert torch.equal(du2, du) and torch.equal(part2, part) and (k == 4 or torch.equal(dx2, dx))


def test_relu_pattern_comes_from_the_given_cells():
    """With c_relu the forward value is still max(c, 0); the derivative is the given pattern's, so flipping the sign of
    one cell state of the pattern changes the gradient of that frame and of every earlier one."""
    B, T, d = 1, 6, 1
    g = torch.Generator().manual_seed(4)
    u = torch.randn(B, T, 4, generator=g, dtype=torch.float64)
    bias = torch.zeros(2, dtype=torch.float64)
    dh = torch.ones(B, T, 1, dtype=torch.float64)
    h, c = ref.sru_f64(u, None, bias, None, d, False, 2)
    flipped = c.clone()
    flipped[0, 3, 0] = -flipped[0, 3, 0]
    h2, _ = ref.sru_f64(u, None, bias, None, d, False, 2, c_relu=flipped)
    assert torch.equal(h, h2)
    du, _, _ = ref.sru_f64_bwd(u, None, bias, None, d, False, 2, dh, c_relu=c)
    du2, _, _ = ref.sru_f64_bwd(u, None, bias, None, d, False, 2, dh, c_relu=flipped)
    diff = (du - du2).abs().view(T, 4).sum(1)
    assert bool((diff[:4] > 0).all()) and bool((diff[4:] == 0).all())


@pytest.mark.parametrize("k,bidir,act", [(4, 1, 2), (3, 1, 1), (4, 0, 0), (3, 0, 2)])
def test_length_exact_forward_is_each_row_alone(k, bidir, act):
    B, T, d = 6, 13, 3
    ncols = d * (2 if bidir else 1)
    lengths = [13, 1, 0, -2, 20, 7]
    g = torch.Generator().manual_seed(9)
    u = torch.randn(B, T, ncols * k, generator=g, dtype=torch.float64)
    x = torch.randn(B, T, ncols, generator=g, dtype=torch.float64) if k == 3 else None
    bias = torch.randn(2 * ncols, generator=g, dtype=torch.float64) * 0.5
    h, c = ref.sru_f64(u, x, bias, None, d, bidir, act, lengths=lengths)
    hp, _ = ref.sru_f64(u, x, bias, None, d, bidir, act)
    assert torch.equal(ref.sru_f64(u, x, bias, None, d, bidir, act, lengths=[T] * B)[0], hp)
    for b, n in enumerate(lengths):
        L = min(max(n, 0), T)
        assert bool((h[b, L:] == 0).all()) and bool((c[b, L:] == 0).all())
        if L:
            alone, _ = ref.sru_f64(u[b:b + 1, :L], x[b:b + 1, :L] if k == 3 else None, bias, None, d, bidir, act)
            assert _rel(h[b:b + 1, :L], alone) < 1e-14, (b, n)     # the same arithmetic on a batch of one row
    # the reverse direction starts at L - 1: a row shorter than T differs from the padded scan there
    if bidir:
        assert not torch.equal(h[5, :7, d:], hp[5, :7, d:])
    assert torch.equal(h[5, :7, :d], hp[5, :7, :d])


# ---------------------------------------------------------------------------------------------- the GPU matrix
def test_gpu_case_matrix_reaches_every_edge():
    ids = [c[0] for c in CASES]
    assert len(set(ids)) == len(ids)
    Ts = {T for _, B, T, d, k, bidir, act, p in CASES}
    assert {T % ref.SRU_UNR for T in Ts} == set(range(ref.SRU_UNR))
    assert {1, 8, 9, 15, 16, 17, 1000} <= Ts
    ncols = {B * d * (2 if bidir else 1) for _, B, T, d, k, bidir, act, p in CASES}
    assert {1, 127, 128, 129} <= ncols
    # several blocks, the last one partial
    assert any(n > 2 * ref.SRU_THREADS and n % ref.SRU_THREADS for n in ncols)
    # the full cross of k x direction count x activation x mask at a shape with a chunk tail
    cross = {(k, bidir, act, p > 0) for _, B, T, d, k, bidir, act, p in CASES if T % ref.SRU_UNR}
    assert len(cross) == 2 * 2 * 3 * 2
    # every variant sees a tail in both directions
    for k in (3, 4):
        assert {T % ref.SRU_UNR for _, B, T, d, kk, bidir, act, p in CASES if kk == k and bidir} == set(range(8))
    assert ("B4-T200-d512-k4-bi-relu-mask0.2", 4, 200, 512, 4, 1, 2, 0.2) in CASES
    assert ("B4-T200-d512-k3-bi-relu-mask0.2", 4, 200, 512, 3, 1, 2, 0.2) in CASES
    # lengths of 0, 1, T, below 0 and above T
    kinds = set()
    for i, (_, B, T, *rest) in enumerate(CASES):
        lens = ref.case_lengths(B, T, i)
        assert len(lens) == B
        kinds |= {"0" if n == 0 else "1" if n == 1 else "T" if n == T else "<0" if n < 0 else ">T" if n > T else "mid"
                  for n in lens}
    assert {"0", "1", "T", "<0", ">T", "mid"} <= kinds


def test_case_inputs_reach_both_sides_of_every_gate():
    u, x, bias, mask, dh = ref.case_inputs(3, 17, 8, 3, 1, 0.3, 1)
    assert u.shape == (3, 17, 48) and x.shape == (3, 17, 16) and mask.shape == (3, 16) and dh.shape == (3, 17, 16)
    assert bool((mask == 0).any()) and bool(torch.allclose(mask[mask != 0], torch.tensor(1 / 0.7)))
    assert float(bias.min()) < 0 < float(bias.max())
    _, x4, _, m4, _ = ref.case_inputs(2, 5, 4, 4, 0, 0.0, 2)
    assert x4 is None and m4 is None


# ---------------------------------------------------------------------------------------------- argument rules
@pytest.fixture(scope="module")
def lib():
    import __graft_entry__
    __graft_entry__.build()
    from gantts_b200 import _lib
    return _lib.load()


@pytest.mark.parametrize("B,d,bidir,refused", [
    (1 << 20, 1 << 10, 0, False),          # B * columns = 2^30: the largest accepted
    (1 << 20, 1 << 10, 1, True),           # 2^31: overflows the launch's int count
    ((1 << 20) + 1, 1 << 10, 0, True),
    (1 << 22, 1 << 10, 1, True),           # 2^33: wraps to 0 in int
])
def test_sru_fwd_bwd_refuse_too_many_columns(lib, B, d, bidir, refused):
    from gantts_b200 import _lib
    if not refused:
        # an accepted shape gets past the rule; the null output pointer is the next one refused, still before any launch
        rc = lib.gantts_sru_fwd(FAKE, None, FAKE, None, None, FAKE, B, 1, d, 4, bidir, 2, None)
        assert rc == _lib.GANTTS_E_BADARG and "sru_fwd: null output" in lib.gantts_last_error_string().decode()
        rc = lib.gantts_sru_bwd(FAKE, None, FAKE, None, FAKE, FAKE, None, None, FAKE, B, 1, d, 4, bidir, 2, None)
        assert rc == _lib.GANTTS_E_BADARG and "sru_bwd: null pointer" in lib.gantts_last_error_string().decode()
        return
    needle = "sru: B = %d and d = %d must be >= 1 with B * columns <= 2^30" % (B, d)
    rc = lib.gantts_sru_fwd(FAKE, None, FAKE, None, FAKE, FAKE, B, 4, d, 4, bidir, 2, None)
    assert rc == _lib.GANTTS_E_BADARG
    assert needle in lib.gantts_last_error_string().decode()
    rc = lib.gantts_sru_bwd(FAKE, FAKE, FAKE, None, FAKE, FAKE, FAKE, FAKE, FAKE, B, 4, d, 3, bidir, 1, None)
    assert rc == _lib.GANTTS_E_BADARG
    assert needle in lib.gantts_last_error_string().decode()
    # gantts_sru_fwd_lengths keeps its own rule of the same wording
    rc = lib.gantts_sru_fwd_lengths(FAKE, None, FAKE, FAKE, FAKE, B, 4, d, 4, bidir, 2, None)
    assert rc == _lib.GANTTS_E_BADARG
    assert "B * columns <= 2^30" in lib.gantts_last_error_string().decode()


def test_sru_fwd_bwd_shape_rules_still_hold(lib):
    from gantts_b200 import _lib
    for kw, needle in ((dict(B=0), "sru: bad shape"), (dict(k=5), "sru: bad shape"), (dict(act=3), "bad activation 3")):
        a = dict(B=2, T=4, d=8, k=4, act=2)
        a.update(kw)
        rc = lib.gantts_sru_fwd(FAKE, None, FAKE, None, FAKE, FAKE, a["B"], a["T"], a["d"], a["k"], 1, a["act"], None)
        assert rc == _lib.GANTTS_E_BADARG and needle in lib.gantts_last_error_string().decode(), kw
    rc = lib.gantts_sru_fwd(FAKE, None, FAKE, None, FAKE, FAKE, 2, 4, 8, 3, 1, 2, None)   # k = 3 without x
    assert rc == _lib.GANTTS_E_BADARG and "sru: null pointer" in lib.gantts_last_error_string().decode()
