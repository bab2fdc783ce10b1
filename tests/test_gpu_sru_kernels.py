"""The SRU scan kernels (csrc/sru.cu) against the float64 restatement of tests/sru_f64.py, at the C API:
gantts_sru_fwd, gantts_sru_bwd and gantts_sru_fwd_lengths through ctypes, as gantts_b200/rnn.py calls them; then
SRUCell / SRU on both GEMM engines against the same restatement.

Every output is filled with NaN before a call; dx is prefilled with random values and dx_after - dx_before must be the
highway gradient (the backward adds into dx).  Errors are max|got - ref| over max|ref| per (sequence, direction), so a
short sequence cannot hide behind a long one.  The length-exact forward must be exactly 0.0 from each length on, equal
gantts_sru_fwd bit for bit when every length is T, and give each row bit for bit what a one-row gantts_sru_fwd gives at
T = its length.  Row b of a B-row launch must equal the same row launched alone (one thread per (b, column)), and two
identical calls must give identical results.  ReLU's derivative pattern comes from the device's saved c (see
tests/sru_f64.py).

Bars, fp32 scan against float64: 5e-6, as for the LSTM kernels, for h, c, du, dx and dbias (whose error is taken over the
largest sum of |du| it adds, see _per_sequence_bias); 2e-5 for the length-exact h, whose single-column rows of 1 to 9
frames (B = 127, d = 1) have so few values that their largest |h| can sit far below the u and x it is computed from
(h = r g(c) + (1 - r) x' cancels).  The worst errors over the whole matrix on an NVIDIA H100 80GB HBM3 (700 W): h 4.1e-7,
c 3.3e-7, du 5.0e-7, dx 3.2e-7, dbias 3.1e-7, length-exact h 1.8e-6 -- a few fp32 roundings, not growing with T up to
1000; the bars leave a factor of 10.
"""
import pytest
import torch

import sru_f64 as ref
from sru_f64 import CASES

pytestmark = pytest.mark.gpu

TOL = {"h": 5e-6, "c": 5e-6, "du": 5e-6, "dx": 5e-6, "dbias": 5e-6, "h_len": 2e-5}
LAYER_TOL = {"simt": 2e-5, "tc": 1e-4}          # tests/test_gpu_parity.py's engine bars


def _lib():
    import __graft_entry__
    __graft_entry__.build()
    from gantts_b200 import _lib as L
    return L


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _ptr(t):
    return t.data_ptr() if t is not None else None


def _dev(t):
    return t.cuda().contiguous() if t is not None else None


def _nan(*shape):
    return torch.full(shape, float("nan"), device="cuda")


class Scan(object):
    """The three C calls on device tensors, every output NaN-poisoned before its call."""

    def __init__(self, L, d, k, bidir, act):
        self.L, self.lib = L, L.load()
        self.d, self.k, self.bidir, self.act = d, k, bidir, act
        self.ncols = d * (2 if bidir else 1)

    def _check(self, rc):
        assert rc == 0, self.lib.gantts_last_error_string().decode()

    def fwd(self, u, x, bias, mask):
        B, T, _ = u.shape
        h, c = _nan(B, T, self.ncols), _nan(B, T, self.ncols)
        self._check(self.lib.gantts_sru_fwd(_ptr(u), _ptr(x), _ptr(bias), _ptr(mask), h.data_ptr(), c.data_ptr(),
                                            B, T, self.d, self.k, self.bidir, self.act, _stream()))
        torch.cuda.synchronize()
        return h, c

    def bwd(self, u, x, bias, mask, c, dh, dx0):
        B, T, _ = u.shape
        du, part = _nan(*u.shape), _nan(B, 2 * self.ncols)
        dx = dx0.clone() if self.k == 3 else None
        self._check(self.lib.gantts_sru_bwd(_ptr(u), _ptr(x), _ptr(bias), _ptr(mask), c.data_ptr(), dh.data_ptr(),
                                            du.data_ptr(), _ptr(dx), part.data_ptr(), B, T, self.d, self.k, self.bidir,
                                            self.act, _stream()))
        torch.cuda.synchronize()
        return du, dx, part

    def fwd_lengths(self, u, x, bias, lengths):
        B, T, _ = u.shape
        h = _nan(B, T, self.ncols)
        lens = torch.tensor(lengths, dtype=torch.int64, device="cuda")
        self._check(self.lib.gantts_sru_fwd_lengths(_ptr(u), _ptr(x), _ptr(bias), lens.data_ptr(), h.data_ptr(), B, T,
                                                    self.d, self.k, self.bidir, self.act, _stream()))
        torch.cuda.synchronize()
        return h


def _err(got, exp):
    got, exp = got.double(), exp.double()
    return float((got - exp).abs().max() / exp.abs().max().clamp_min(1e-30))


def _worst(a, b):
    return float("nan") if a != a or b != b else max(a, b)


def _per_sequence(got, exp, frames, d, dirs, width):
    """Worst error of got [B][T][ncols * width] over (sequence, direction), each on its first frames[b] frames."""
    w = 0.0
    for b, n in enumerate(frames):
        if n > 0:
            for di in range(dirs):
                sl = slice(di * d * width, (di + 1) * d * width)
                w = _worst(w, _err(got[b, :n, sl], exp[b, :n, sl]))
    return w


def _per_sequence_bias(got, exp, scale, d, dirs):
    """dbias_part [B][2*ncols] per (sequence, direction), over the largest sum of |du| over T among its sums: a sum over
    the frames can cancel to far below its terms, and an fp32 sum is only as exact as the terms it adds."""
    ncols = d * dirs
    w = 0.0
    for b in range(got.shape[0]):
        for di in range(dirs):
            idx = list(range(di * d, (di + 1) * d)) + list(range(ncols + di * d, ncols + (di + 1) * d))
            e = float((got[b, idx].double() - exp[b, idx]).abs().max() / scale[b, idx].max().clamp_min(1e-30))
            w = _worst(w, e)
    return w


def run_case(L, i, case):
    cid, B, T, d, k, bidir, act, p = case
    dirs = 2 if bidir else 1
    row = {"id": cid, "problems": [], "errors": {}}
    u, x, bias, mask, dh = ref.case_inputs(B, T, d, k, bidir, p, 1000 + i)
    dx0 = torch.randn(B, T, d * dirs, generator=torch.Generator().manual_seed(2000 + i))
    ud, xd, bd, md, dhd, dx0d = (_dev(t) for t in (u, x, bias, mask, dh, dx0))
    s = Scan(L, d, k, bidir, act)

    # padded forward and backward against float64
    h, c = s.fwd(ud, xd, bd, md)
    du, dx, part = s.bwd(ud, xd, bd, md, c, dhd, dx0d)
    h, c, du, part = h.cpu(), c.cpu(), du.cpu(), part.cpu()
    dxg = dx.cpu().double() - dx0.double() if k == 3 else None
    f64 = lambda t: t.double() if t is not None else None
    h64, c64 = ref.sru_f64(f64(u), f64(x), f64(bias), f64(mask), d, bidir, act)
    du64, dx64, part64 = ref.sru_f64_bwd(u, x, bias, mask, d, bidir, act, dh, c_relu=c)
    full = [T] * B
    e = row["errors"]
    e["h"] = _per_sequence(h, h64, full, d, dirs, 1)
    e["c"] = _per_sequence(c, c64, full, d, dirs, 1)
    e["du"] = _per_sequence(du, du64, full, d, dirs, k)
    if k == 3:
        e["dx"] = _per_sequence(dxg, dx64, full, d, dirs, 1)
    du64v = du64.abs().view(B, T, d * dirs, k)
    e["dbias"] = _per_sequence_bias(part, part64, torch.cat([du64v[..., 1].sum(1), du64v[..., 2].sum(1)], 1), d, dirs)

    # length-exact forward: against float64, exact zeros from each length on
    lens = ref.case_lengths(B, T, i)
    clamped = [min(max(n, 0), T) for n in lens]
    hl = s.fwd_lengths(ud, xd, bd, lens).cpu()
    hl64, _ = ref.sru_f64(f64(u), f64(x), f64(bias), None, d, bidir, act, lengths=lens)
    e["h_len"] = _per_sequence(hl, hl64, clamped, d, dirs, 1)
    if not bool(torch.isfinite(hl).all()) or not all(bool((hl[b, n:] == 0).all()) for b, n in enumerate(clamped)):
        row["problems"].append("length-exact h not finite, or not exactly 0 from a length on")

    for kk, v in e.items():
        if not v <= TOL[kk]:
            row["problems"].append("%s error %.3g > %.0e" % (kk, v, TOL[kk]))

    # bit for bit: every length T is gantts_sru_fwd without a mask; each row is a one-row gantts_sru_fwd at T = L
    h_nomask, _ = s.fwd(ud, xd, bd, None)
    if not torch.equal(s.fwd_lengths(ud, xd, bd, full), h_nomask):
        row["problems"].append("lengths all T differ from gantts_sru_fwd")
    for b, n in enumerate(clamped):
        if n > 0:
            sub = lambda t: t[b:b + 1, :n].contiguous() if t is not None else None
            alone, _ = s.fwd(sub(ud), sub(xd), bd, None)
            if not torch.equal(hl[b:b + 1, :n], alone.cpu()):
                row["problems"].append("length-exact row %d (L = %d) differs from a one-row forward" % (b, n))

    # bit for bit: a row launched alone, and a repeated call
    hd, cd = s.fwd(ud, xd, bd, md)
    rep = s.bwd(ud, xd, bd, md, cd, dhd, dx0d)
    if not (torch.equal(hd.cpu(), h) and torch.equal(cd.cpu(), c) and torch.equal(rep[0].cpu(), du)
            and torch.equal(rep[2].cpu(), part) and (k == 4 or torch.equal(rep[1], dx))):
        row["problems"].append("a repeated call differs")
    for b in range(B):
        r = lambda t: t[b:b + 1].contiguous() if t is not None else None
        h1, c1 = s.fwd(r(ud), r(xd), bd, r(md))
        du1, dx1, part1 = s.bwd(r(ud), r(xd), bd, r(md), c1, r(dhd), r(dx0d))
        if not (torch.equal(h1.cpu(), h[b:b + 1]) and torch.equal(c1.cpu(), c[b:b + 1])
                and torch.equal(du1.cpu(), du[b:b + 1]) and torch.equal(part1.cpu(), part[b:b + 1])
                and (k == 4 or torch.equal(dx1, dx[b:b + 1]))):
            row["problems"].append("row %d launched alone differs" % b)
    return row


@pytest.fixture(scope="module")
def matrix():
    L = _lib()
    return [run_case(L, i, case) for i, case in enumerate(CASES)]


def test_matrix_vs_float64(matrix):
    worst = {}
    print("\nSRU scans vs float64 (%s)" % torch.cuda.get_device_name(0))
    for r in matrix:
        for kk, v in r["errors"].items():
            worst[kk] = _worst(worst.get(kk, 0.0), v)
        print("%-36s %s%s" % (r["id"], " ".join("%s %.2e" % kv for kv in r["errors"].items()),
                              "  <-- " + "; ".join(r["problems"]) if r["problems"] else ""))
    print("worst per tensor: " + " ".join("%s %.3e (bar %.0e)" % (kk, worst[kk], TOL[kk]) for kk in TOL))
    failures = ["%s: %s" % (r["id"], "; ".join(r["problems"])) for r in matrix if r["problems"]]
    assert not failures, "\n".join(failures)


# ------------------------------------------------------------------------------------------------ layer level
def _act_flags(act):
    return dict(use_tanh=int(act == 1), use_relu=int(act == 2))


def _cell_f64(x, W, bias, mask_x, mask_h, d, bidir, act, k, c_relu):
    """One SRUCell in train mode: u = (x * mask_x) W, the highway input the unmasked x (k == 3)."""
    xin = x * mask_x.unsqueeze(1) if mask_x is not None else x
    h, _ = ref.sru_f64(xin @ W, x if k == 3 else None, bias, mask_h, d, bidir, act, c_relu=c_relu)
    return h


@pytest.mark.parametrize("engine", ["simt", "tc"])
@pytest.mark.parametrize("n_in,d,bidir,act", [(16, 8, True, 0), (20, 8, True, 0), (12, 12, False, 1), (10, 12, False, 2),
                                              (24, 12, True, 2), (9, 16, True, 1)])
def test_sru_cell_vs_float64(engine, n_in, d, bidir, act):
    """SRUCell in train mode (rnn_dropout 0.25 on the GEMM input, dropout 0.3 on g(c_t)), masks regenerated from the
    seeds the cell draws: the output and the gradients of x, weight and bias."""
    from gantts_b200 import rnn, ops
    _lib()
    dev = torch.device("cuda:0")
    torch.manual_seed(61 + n_in + act)
    B, T = 3, 19
    cell = rnn.SRUCell(n_in, d, dropout=0.3, rnn_dropout=0.25, bidirectional=bidir, **_act_flags(act))
    cell.bias.data.uniform_(-0.5, 0.5)
    k, ncols = cell.k, d * (2 if bidir else 1)
    x = torch.randn(B, T, n_in)
    g = torch.randn(B, T, ncols)
    cell.to(dev).train()
    s_x, s_h = ops.peek_seeds(2)
    xg = x.to(dev).requires_grad_(True)
    yg = cell(xg, engine=engine)
    c_dev = yg.grad_fn.saved_tensors[4].cpu()                # the scan's saved cell states
    yg.backward(g.to(dev))
    mask_x = ops.dropout_mask(B, n_in, 0.25, s_x, dev).cpu().double()
    mask_h = ops.dropout_mask(B, ncols, 0.3, s_h, dev).cpu().double()
    assert 0 < float((mask_x == 0).float().mean()) < 1 and 0 < float((mask_h == 0).float().mean()) < 1
    xr = x.double().requires_grad_(True)
    Wr = cell.weight.detach().cpu().double().requires_grad_(True)
    br = cell.bias.detach().cpu().double().requires_grad_(True)
    yr = _cell_f64(xr, Wr, br, mask_x, mask_h, d, bidir, act, k, c_dev)
    yr.backward(g.double())
    errs = {"y": _err(yg.detach().cpu(), yr.detach()), "gx": _err(xg.grad.cpu(), xr.grad),
            "gW": _err(cell.weight.grad.cpu(), Wr.grad), "gb": _err(cell.bias.grad.cpu(), br.grad)}
    assert max(errs.values()) < LAYER_TOL[engine], (k, errs)


@pytest.mark.parametrize("engine", ["simt", "tc"])
@pytest.mark.parametrize("act", [0, 1])
def test_sru_stack_vs_float64(engine, act):
    """SRU: 3 bidirectional layers (k = 4, then k = 3 twice) in train mode, dropout 0.3 on every layer but the last,
    rnn_dropout 0.2, T = 21: the output and the gradients of x and of every layer's weight and bias."""
    from gantts_b200 import rnn, ops
    _lib()
    dev = torch.device("cuda:0")
    torch.manual_seed(71 + act)
    B, T, n_in, d = 4, 21, 10, 6
    m = rnn.SRU(n_in, d, num_layers=3, dropout=0.3, rnn_dropout=0.2, bidirectional=True, **_act_flags(act))
    for cell in m.rnn_lst:
        cell.bias.data.uniform_(-0.5, 0.5)
    assert [cell.k for cell in m.rnn_lst] == [4, 3, 3]
    x = torch.randn(B, T, n_in)
    g = torch.randn(B, T, 2 * d)
    m.to(dev).train()
    seeds = ops.peek_seeds(5)                              # per layer: rnn_dropout, then dropout below the top
    xg = x.to(dev).requires_grad_(True)
    yg = m(xg, engine=engine)
    yg.backward(g.to(dev))
    xr = x.double().requires_grad_(True)
    h, params, si = xr, [], 0
    for li, cell in enumerate(m.rnn_lst):
        W = cell.weight.detach().cpu().double().requires_grad_(True)
        b = cell.bias.detach().cpu().double().requires_grad_(True)
        params.append((cell, W, b))
        mx = ops.dropout_mask(B, cell.n_in, 0.2, seeds[si], dev).cpu().double()
        si += 1
        mh = None
        if li + 1 < len(m.rnn_lst):
            mh = ops.dropout_mask(B, 2 * d, 0.3, seeds[si], dev).cpu().double()
            si += 1
        h = _cell_f64(h, W, b, mx, mh, d, True, act, cell.k, None)
    h.backward(g.double())
    errs = {"y": _err(yg.detach().cpu(), h.detach()), "gx": _err(xg.grad.cpu(), xr.grad)}
    for li, (cell, W, b) in enumerate(params):
        errs["gW%d" % li] = _err(cell.weight.grad.cpu(), W.grad)
        errs["gb%d" % li] = _err(cell.bias.grad.cpu(), b.grad)
    assert max(errs.values()) < LAYER_TOL[engine], errs
