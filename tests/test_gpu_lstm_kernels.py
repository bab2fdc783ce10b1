"""The LSTM recurrence kernels (csrc/lstm.cu) against the float64 restatement of tests/lstm_f64.py, at the C API:
gantts_lstm_layer_fwd, gantts_lstm_layer_bwd and gantts_lstm_hprev through ctypes, as gantts_b200/rnn.py calls them.

Every output is filled with NaN before a call.  h and dxproj must then be written on every frame and be exactly 0.0
beyond each length; gates and cells are compared on valid frames; hprev must be bit-exact.  Errors are max|got - ref|
over max|ref| per (sequence, direction), so a short sequence cannot hide behind a long one.  The case matrix reaches
every kernel body lstm_run chooses (tests/test_lstm_f64_host.py pins that at 132 SMs).

Bars, fp32 FFMA recurrence against float64: 5e-6 for every tensor.  The worst errors over the whole matrix, register and
shared-memory kernels, on an NVIDIA H100 80GB HBM3 (132 SMs, 700 W): h 3.9e-7, gates 4.6e-7, cells 2.8e-7, dxproj 4.1e-7 --
a few fp32 roundings, not growing with T up to 200; the bars leave a factor of 10.
"""
import pytest
import torch

import lstm_f64 as ref
from lstm_f64 import CASES

pytestmark = pytest.mark.gpu

TOL = {"h": 5e-6, "gates": 5e-6, "cells": 5e-6, "dxproj": 5e-6}


def _lib():
    import __graft_entry__
    __graft_entry__.build()
    from gantts_b200 import _lib as L
    return L


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _inputs(B, T, H, ndir, seed):
    g = torch.Generator().manual_seed(seed)
    xproj = torch.randn(B, T, ndir * 4 * H, generator=g)
    k = 1.0 / H ** 0.5                                     # nn.LSTM's initialisation range
    W_hh = (torch.rand(ndir, 4 * H, H, generator=g) * 2 - 1) * k
    dh = torch.randn(B, T, ndir * H, generator=g)          # nonzero beyond the lengths too: must be ignored
    return xproj, W_hh, dh


class Layer(object):
    """One layer's buffers on the device and the three C calls, every output NaN-poisoned before its call."""

    def __init__(self, L, xproj, W_hh, lengths):
        self.L, self.lib = L, L.load()
        self.B, self.T, _ = xproj.shape
        self.ndir, _, self.H = W_hh.shape
        dev = torch.device("cuda:0")
        self.xproj, self.W_hh = xproj.to(dev).contiguous(), W_hh.to(dev).contiguous()
        self.lens = torch.tensor(lengths, dtype=torch.int64, device=dev)
        self.bar = torch.zeros(self.lib.gantts_lstm_workspace_bytes(), dtype=torch.uint8, device=dev)
        B, T, H, nd = self.B, self.T, self.H, self.ndir
        self.h = torch.empty(B, T, nd * H, device=dev)
        self.gates = torch.empty(nd, B, T, 4 * H, device=dev)
        self.cells = torch.empty(nd, B, T, H, device=dev)
        self.dxproj = torch.empty(B, T, nd * 4 * H, device=dev)

    def fwd(self, B=None, H=None, ndir=None):
        for t in (self.h, self.gates, self.cells):
            t.fill_(float("nan"))
        rc = self.lib.gantts_lstm_layer_fwd(self.xproj.data_ptr(), self.W_hh.data_ptr(), self.lens.data_ptr(),
                                            self.h.data_ptr(), self.gates.data_ptr(), self.cells.data_ptr(),
                                            B or self.B, self.T, H or self.H, ndir or self.ndir, self.bar.data_ptr(),
                                            self.bar.numel(), _stream())
        torch.cuda.synchronize()
        return rc

    def bwd(self, dh, B=None, H=None, ndir=None):
        dh = dh.to(self.h.device).contiguous()
        self.dxproj.fill_(float("nan"))
        rc = self.lib.gantts_lstm_layer_bwd(dh.data_ptr(), self.W_hh.data_ptr(), self.lens.data_ptr(),
                                            self.gates.data_ptr(), self.cells.data_ptr(), self.dxproj.data_ptr(),
                                            B or self.B, self.T, H or self.H, ndir or self.ndir, self.bar.data_ptr(),
                                            self.bar.numel(), _stream())
        torch.cuda.synchronize()
        return rc

    def hprev(self, h, d, ndir=None):
        h = h.to(self.h.device).contiguous()
        out = torch.full((self.B, self.T, self.H), float("nan"), device=self.h.device)
        rc = self.lib.gantts_lstm_hprev(h.data_ptr(), self.lens.data_ptr(), out.data_ptr(), self.B, self.T, self.H,
                                        ndir or self.ndir, d, _stream())
        torch.cuda.synchronize()
        return rc, out.cpu()

    def error(self):
        return self.lib.gantts_last_error_string().decode()


def _err(got, exp):
    got, exp = got.double(), exp.double()
    return float((got - exp).abs().max() / exp.abs().max().clamp_min(1e-30))


def _per_sequence_errors(lengths, H, ndir, got, exp):
    """Worst error per tensor of `got` over the (sequence, direction) pairs, each on its valid frames."""
    part = {"h": lambda t, b, n, d: t[b, :n, d * H:(d + 1) * H],
            "gates": lambda t, b, n, d: t[d, b, :n],
            "cells": lambda t, b, n, d: t[d, b, :n],
            "dxproj": lambda t, b, n, d: t[b, :n, d * 4 * H:(d + 1) * 4 * H]}
    worst = {k: 0.0 for k in got}
    for b, n in enumerate(lengths):
        for d in range(ndir):
            for k in got:
                e_ = _err(part[k](got[k], b, n, d), part[k](exp[k], b, n, d))
                worst[k] = float("nan") if e_ != e_ or worst[k] != worst[k] else max(worst[k], e_)
    return worst


def _zero_beyond(t, lengths):
    """True when t [B][T][...] is finite everywhere and exactly 0.0 on every frame at or beyond each length."""
    if not bool(torch.isfinite(t).all()):
        return False
    return all(bool((t[b, n:] == 0).all()) for b, n in enumerate(lengths))


def run_case(L, case, sms):
    """One case of the matrix: a report row {id, variant, errors, problems}."""
    cid, B, T, H, ndir, lengths = case
    seed = 1000 + CASES.index(case)
    xproj, W_hh, dh = _inputs(B, T, H, ndir, seed)
    row = {"id": cid, "variant": ref.variant(H, ndir, sms), "problems": []}
    layer = Layer(L, xproj, W_hh, lengths)
    fwd_plan, bwd_plan = ref.plan(H, ndir, sms, False), ref.plan(H, ndir, sms, True)
    rc = layer.fwd()
    if fwd_plan[2] is not None:
        if rc == 0 or fwd_plan[2] not in layer.error():
            row["problems"].append("forward not refused for %s: rc %d, %r" % (fwd_plan[2], rc, layer.error()))
        return row
    if rc != 0:
        row["problems"].append("forward failed: %s" % layer.error())
        return row
    got = {"h": layer.h.cpu(), "gates": layer.gates.cpu(), "cells": layer.cells.cpu()}
    h64, g64, c64 = ref.lstm_layer_f64(xproj.double(), W_hh.double(), lengths)
    exp = {"h": h64, "gates": g64, "cells": c64}
    rc = layer.bwd(dh)
    if bwd_plan[2] is not None:
        if rc == 0 or bwd_plan[2] not in layer.error():
            row["problems"].append("backward not refused for %s: rc %d, %r" % (bwd_plan[2], rc, layer.error()))
    else:
        if rc != 0:
            row["problems"].append("backward failed: %s" % layer.error())
            return row
        got["dxproj"] = layer.dxproj.cpu()
        exp["dxproj"] = ref.lstm_layer_dxproj_f64(xproj, W_hh, lengths, dh)
        if not _zero_beyond(got["dxproj"], lengths):
            row["problems"].append("dxproj not finite, or not exactly 0 beyond a length")
    if not _zero_beyond(got["h"], lengths):
        row["problems"].append("h not finite, or not exactly 0 beyond a length")
    errs = _per_sequence_errors(lengths, H, ndir, got, exp)
    row["errors"] = errs
    for k, e in errs.items():
        if not e <= TOL[k]:
            row["problems"].append("%s error %.3g > %.0e" % (k, e, TOL[k]))
    # hprev: a gather of an arbitrary h (nonzero beyond the lengths, where the copy must give 0), bit for bit
    hr = torch.randn(B, T, ndir * H, generator=torch.Generator().manual_seed(seed + 1))
    for d in range(ndir):
        rc, hp = layer.hprev(hr, d)
        if rc != 0 or not torch.equal(hp, ref.lstm_hprev(hr, lengths, H, ndir, d)):
            row["problems"].append("hprev of direction %d differs (rc %d)" % (d, rc))
    return row


def run_matrix():
    """A report row for every case."""
    L = _lib()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return [run_case(L, case, sms) for case in CASES]


def report(title, rows):
    worst = {}
    print("\n%s (%s, %d SMs)" % (title, torch.cuda.get_device_name(0), torch.cuda.get_device_properties(0).multi_processor_count))
    print("%-40s %-56s %s" % ("case", "forward / backward kernel", "errors"))
    for r in rows:
        errs = r.get("errors", {})
        for k, e in errs.items():
            w = worst.get(k, 0.0)
            worst[k] = float("nan") if e != e or w != w else max(w, e)
        print("%-40s %-56s %s%s" % (r["id"], r["variant"], " ".join("%s %.2e" % kv for kv in errs.items()),
                                   "  <-- " + "; ".join(r["problems"]) if r["problems"] else ""))
    print("worst per tensor: " + " ".join("%s %.3e (bar %.0e)" % (k, worst[k], TOL[k]) for k in TOL if k in worst))
    return worst


def _failures(rows):
    return ["%s: %s" % (r["id"], "; ".join(r["problems"])) for r in rows if r["problems"]]


# ------------------------------------------------------------------------------------------------- the matrix
def test_matrix_vs_float64():
    rows = run_matrix()
    report("LSTM recurrence vs float64", rows)
    assert not _failures(rows), "\n".join(_failures(rows))


def test_repeated_calls_are_bit_identical():
    L = _lib()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for H, ndir, B in ((12, 2, 33), (260, 1, 17), (516, 1, 17), (528, 2, 20)):
        T, lengths = 6, ref.case_lengths("unsorted", B, 6, 7)
        xproj, W_hh, dh = _inputs(B, T, H, ndir, 77)
        layer = Layer(L, xproj, W_hh, lengths)
        runs = []
        for _ in range(2):
            assert layer.fwd() == 0, layer.error()
            assert layer.bwd(dh) == 0, layer.error()
            runs.append([t.cpu() for t in (layer.h, layer.gates, layer.cells, layer.dxproj)])
        for a, b in zip(*runs):
            assert torch.equal(a.nan_to_num(7.0), b.nan_to_num(7.0)), (H, ndir, ref.variant(H, ndir, sms))


# --------------------------------------------------------------------------------------------------- refusals
def test_hs16_forward_vs_float64_and_backward_refused():
    """The smallest bidirectional H whose backward does not fit (532 at 132 SMs: 16 units per CTA, 290 KB of shared
    memory): the forward still runs and matches, the backward is refused with the limit named and leaves the device
    usable."""
    L = _lib()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    H = ref.first_untrainable(2, sms)
    assert ref.pick_hs(H, 2, sms)[0] == 16 or ref.plan(H, 2, sms, True)[0] == "lstm_bwd_kernel<8>"
    B, T, lengths = 5, 6, [6, 1, 4, 6, 3]
    xproj, W_hh, dh = _inputs(B, T, H, 2, 5)
    layer = Layer(L, xproj, W_hh, lengths)
    assert layer.fwd() == 0, layer.error()
    h64, g64, c64 = ref.lstm_layer_f64(xproj.double(), W_hh.double(), lengths)
    assert _zero_beyond(layer.h.cpu(), lengths)
    got = {"h": layer.h.cpu(), "gates": layer.gates.cpu(), "cells": layer.cells.cpu()}
    errs = _per_sequence_errors(lengths, H, 2, got, {"h": h64, "gates": g64, "cells": c64})
    assert all(e <= TOL[k] for k, e in errs.items()), errs
    assert layer.bwd(dh) == 3                              # GANTTS_E_UNSUPPORTED
    msg = layer.error()
    assert "shared memory" in msg and "227 KB" in msg and "backward" in msg, msg
    assert bool(torch.isnan(layer.dxproj).all())           # refused before any launch
    lib = L.load()
    assert lib.gantts_lstm_layer_supported(H, 2, 0) == 0
    assert lib.gantts_lstm_layer_supported(H, 2, 1) == 3 and "shared memory" in layer.error()
    assert lib.gantts_lstm_layer_supported(H - 4, 2, 1) == 0
    small = Layer(L, *_inputs(3, 4, 8, 2, 6)[:2], [4, 2, 3])
    assert small.fwd() == 0 and small.bwd(torch.randn(3, 4, 16)) == 0, small.error()


def test_host_argument_refusals():
    L = _lib()
    xproj, W_hh, dh = _inputs(4, 3, 8, 2, 9)
    layer = Layer(L, xproj, W_hh, [3, 3, 2, 1])
    for kw, what in ((dict(B=129), "batch 129"), (dict(H=6), "multiple of 4"), (dict(ndir=3), "ndir"),
                     (dict(B=-1), "batch -1")):
        assert layer.fwd(**kw) == 1, kw                     # GANTTS_E_BADARG
        assert what in layer.error(), (kw, layer.error())
        assert bool(torch.isnan(layer.h).all())
        assert layer.bwd(dh, **kw) == 1, kw
        assert what in layer.error(), (kw, layer.error())
    for d, nd in ((1, 1), (2, 2), (-1, 2)):
        rc, out = layer.hprev(torch.zeros(4, 3, 16), d, ndir=nd)
        assert rc == 1 and "lstm_hprev" in layer.error() and bool(torch.isnan(out).all()), (d, nd)
    lib = L.load()
    assert lib.gantts_lstm_layer_supported(6, 1, 0) == 1 and lib.gantts_lstm_layer_supported(8, 3, 1) == 1


def test_lstmrnn_refuses_an_untrainable_layer_before_its_forward():
    """LSTMRNN with gradients on: refused at the forward, naming the limit; without gradients (evaluation, the spoof
    count) the same model runs its forward."""
    import gantts_b200
    _lib()
    dev = torch.device("cuda:0")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    H = ref.first_untrainable(2, sms)
    m = gantts_b200.models.LSTMRNN(in_dim=6, out_dim=1, num_hidden=1, hidden_dim=H, bidirectional=True,
                                   last_sigmoid=True).to(dev).train()
    x = torch.randn(2, 5, 6, device=dev)
    with pytest.raises(RuntimeError, match="shared memory"):
        m(x, [5, 3])
    with torch.no_grad():
        y = m(x, [5, 3])
    assert y.shape == (2, 5, 1) and bool(torch.isfinite(y).all())
    ok = gantts_b200.models.LSTMRNN(in_dim=6, out_dim=1, num_hidden=1, hidden_dim=H - 4, bidirectional=True,
                                    last_sigmoid=True).to(dev).train()
    ok(x, [5, 3]).sum().backward()
    assert all(bool(torch.isfinite(p.grad).all()) for p in ok.parameters())


@pytest.mark.parametrize("where", ["generator", "discriminator"])
def test_fused_step_refuses_an_untrainable_lstm_at_construction(where):
    import gantts_b200
    from gantts_b200 import fused
    from fused_step_helpers import step_hp
    _lib()
    dev = torch.device("cuda:0")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    bad = ref.first_untrainable(2, sms)
    M = gantts_b200.models
    mg = M.In2OutRNNHighwayNet(in_dim=24, out_dim=24, static_dim=8, num_hidden=1,
                               hidden_dim=bad if where == "generator" else 12, bidirectional=True, dropout=0.0).to(dev)
    md = M.LSTMRNN(in_dim=8, out_dim=1, num_hidden=1, hidden_dim=bad if where == "discriminator" else 12,
                   bidirectional=True, last_sigmoid=True).to(dev)
    ohp = dict(stream_sizes=[24], has_dynamic_features=[True], adversarial_streams=[True], mask_nth_mgc_for_adv_loss=0,
               num_windows=3, discriminator_linguistic_condition=False)
    with pytest.raises(RuntimeError, match="shared memory"):
        fused.FusedGanStep(mg, md, step_hp(ohp), 2, 10, seed=1)

