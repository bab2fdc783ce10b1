"""Pins tests/lstm_f64.py, the float64 reference of the LSTM recurrence kernels, without a GPU:
  * the layer restatement equals torch.nn.LSTM in float64 on pack_padded_sequence / pad_packed_sequence, outputs and
    every gradient (dxproj mapped back to dW_ih, db, dW_hh through hprev, and to dx);
  * the mirror of the kernel choice in csrc/lstm.cu, and that the GPU case matrix reaches every kernel body at 132 SMs.
"""
import pytest
import torch
from torch.nn.utils.rnn import pack_padded_sequence, pad_packed_sequence

import lstm_f64 as ref
from lstm_f64 import CASES

TOL = 1e-12


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-300))


def _torch_lstm(I, H, layers, bidir, seed):
    torch.manual_seed(seed)
    return torch.nn.LSTM(I, H, layers, batch_first=True, bidirectional=bidir).double()


def _layer_weights(lstm, k):
    sfx = ["", "_reverse"][:2 if lstm.bidirectional else 1]
    W_ih = [getattr(lstm, "weight_ih_l%d%s" % (k, s)) for s in sfx]
    W_hh = torch.stack([getattr(lstm, "weight_hh_l%d%s" % (k, s)) for s in sfx], 0)
    bias = [getattr(lstm, "bias_ih_l%d%s" % (k, s)) + getattr(lstm, "bias_hh_l%d%s" % (k, s)) for s in sfx]
    return W_ih, W_hh, bias


def _restated_stack(lstm, x, lengths, dh):
    """The stack through lstm_f64 with the hand mapping of rnn._LSTMLayer.backward: forward layer by layer, then top down
    dxproj (autograd through the float64 loop) -> dx, dW_ih, db (= db_ih = db_hh), dW_hh (through hprev)."""
    ndir = 2 if lstm.bidirectional else 1
    H = lstm.hidden_size
    ins, hs = [x], []
    with torch.no_grad():
        for k in range(lstm.num_layers):
            W_ih, W_hh, bias = _layer_weights(lstm, k)
            xproj = torch.cat([ins[-1] @ W_ih[d].t() + bias[d] for d in range(ndir)], 2)
            h, _, _ = ref.lstm_layer_f64(xproj, W_hh, lengths)
            hs.append(h)
            ins.append(h)
    grads, g = {}, dh
    for k in reversed(range(lstm.num_layers)):
        W_ih, W_hh, bias = _layer_weights(lstm, k)
        inp = ins[k].detach()
        with torch.no_grad():
            xproj = torch.cat([inp @ W_ih[d].t() + bias[d] for d in range(ndir)], 2)
        dxp = ref.lstm_layer_dxproj_f64(xproj, W_hh, lengths, g)
        dx = torch.zeros_like(inp)
        for d, s in enumerate(["", "_reverse"][:ndir]):
            dd = dxp[:, :, d * 4 * H:(d + 1) * 4 * H]
            hprev = ref.lstm_hprev(hs[k], lengths, H, ndir, d)
            grads["weight_ih_l%d%s" % (k, s)] = torch.einsum("btg,bti->gi", dd, inp)
            grads["weight_hh_l%d%s" % (k, s)] = torch.einsum("btg,bth->gh", dd, hprev)
            grads["bias_ih_l%d%s" % (k, s)] = grads["bias_hh_l%d%s" % (k, s)] = dd.sum((0, 1))
            dx = dx + dd @ W_ih[d].detach()
        g = dx
    return hs[-1], g, grads


@pytest.mark.parametrize("B,T,I,H,layers,bidir,lengths", [
    (4, 9, 5, 6, 1, False, [9, 7, 3, 1]),
    (4, 9, 5, 6, 1, True, [9, 7, 3, 1]),
    (5, 8, 3, 4, 1, True, [2, 8, 1, 5, 8]),           # unsorted, with length-1 sequences
    (3, 1, 4, 5, 1, True, [1, 1, 1]),                  # T = 1
    (1, 6, 3, 7, 1, False, [6]),
    (4, 7, 5, 6, 2, True, [7, 1, 4, 6]),               # two chained layers
    (3, 6, 4, 3, 2, False, [6, 5, 2]),
])
def test_restatement_equals_torch_lstm_float64(B, T, I, H, layers, bidir, lengths):
    lstm = _torch_lstm(I, H, layers, bidir, seed=B * 100 + T)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(B, T, I, generator=g, dtype=torch.float64)
    dh = torch.randn(B, T, (2 if bidir else 1) * H, generator=g, dtype=torch.float64)
    for b, n in enumerate(lengths):
        x[b, n:] = 0.0

    xl = x.clone().requires_grad_(True)
    packed = pack_padded_sequence(xl, torch.tensor(lengths), batch_first=True, enforce_sorted=False)
    out, _ = lstm(packed)
    y, _ = pad_packed_sequence(out, batch_first=True, total_length=T)
    lstm.zero_grad()
    y.backward(dh)

    h, dx, grads = _restated_stack(lstm, x, lengths, dh)
    assert _rel(h, y.detach()) < TOL
    for b, n in enumerate(lengths):
        assert bool((h[b, n:] == 0).all())
    assert _rel(dx, xl.grad) < TOL
    for name, p in lstm.named_parameters():
        assert _rel(grads[name], p.grad) < TOL, name


def test_restatement_tape_matches_the_cell_equations():
    """gates are (i, f, g, o) after activation and cells the c of each valid frame; both zero beyond a length."""
    B, T, H, lengths = 3, 5, 4, [5, 2, 3]
    g = torch.Generator().manual_seed(1)
    xproj = torch.randn(B, T, 2 * 4 * H, generator=g, dtype=torch.float64)
    W_hh = torch.randn(2, 4 * H, H, generator=g, dtype=torch.float64) * 0.3
    h, gates, cells = ref.lstm_layer_f64(xproj, W_hh, lengths)
    for b, n in enumerate(lengths):
        for d in range(2):
            order = range(n) if d == 0 else range(n - 1, -1, -1)
            hp, cp = torch.zeros(H, dtype=torch.float64), torch.zeros(H, dtype=torch.float64)
            for t in order:
                pre = xproj[b, t, d * 4 * H:(d + 1) * 4 * H] + W_hh[d] @ hp
                i, f, gg, o = pre[:H].sigmoid(), pre[H:2 * H].sigmoid(), pre[2 * H:3 * H].tanh(), pre[3 * H:].sigmoid()
                cp = f * cp + i * gg
                hp = o * cp.tanh()
                assert torch.allclose(gates[d, b, t], torch.cat([i, f, gg, o]), rtol=0, atol=1e-15)
                assert torch.allclose(cells[d, b, t], cp, rtol=0, atol=1e-15)
                assert torch.allclose(h[b, t, d * H:(d + 1) * H], hp, rtol=0, atol=1e-15)
            assert bool((gates[d, b, n:] == 0).all()) and bool((cells[d, b, n:] == 0).all())


def test_hprev_gather():
    h = torch.arange(2 * 4 * 6, dtype=torch.float32).view(2, 4, 6) + 1
    hp0 = ref.lstm_hprev(h, [4, 2], 3, 2, 0)
    hp1 = ref.lstm_hprev(h, [4, 2], 3, 2, 1)
    assert torch.equal(hp0[0], torch.cat([torch.zeros(1, 3), h[0, :3, :3]]))
    assert torch.equal(hp1[0], torch.cat([h[0, 1:, 3:], torch.zeros(1, 3)]))
    assert torch.equal(hp0[1], torch.cat([torch.zeros(1, 3), h[1, :1, :3], torch.zeros(2, 3)]))
    assert torch.equal(hp1[1], torch.cat([h[1, 1:2, 3:], torch.zeros(3, 3)]))


# ------------------------------------------------------------------------------------------- kernel choice
def test_kernel_choice_at_132_sms():
    """The thresholds of the variant table in DESIGN.md (H100 SXM, 132 SMs)."""
    v = lambda H, nd: ref.variant(H, nd, 132)
    assert v(256, 2) == "lstm_fwd_reg_kernel<32> / lstm_bwd_reg_kernel<4>"
    assert v(260, 2) == "lstm_fwd_reg_kernel<64> / lstm_bwd_reg_kernel<8>"
    assert v(512, 2) == v(512, 1) == "lstm_fwd_reg_kernel<64> / lstm_bwd_reg_kernel<8>"
    assert v(516, 2) == v(528, 2) == v(580, 1) == "lstm_fwd_kernel<8> / lstm_bwd_kernel<8>"
    assert v(532, 2).startswith("lstm_fwd_kernel<16> / refused (lstm_bwd_kernel<16>: shared memory")
    assert v(584, 1).startswith("lstm_fwd_kernel<8> / refused (lstm_bwd_kernel<8>: shared memory")
    assert ref.plan(532, 2, 132, True)[1] == 290304                       # (32 (4H + 4) + 4352) * 4 B
    assert ref.first_untrainable(2, 132) == 532 and ref.first_untrainable(1, 132) == 584
    assert ref.pick_hs(1056, 1, 132) == (8, 132) and ref.pick_hs(1060, 1, 132) == (16, 67)
    assert ref.plan(684, 2, 132, False)[2] is None and ref.plan(688, 2, 132, False)[2] == "shared memory"
    assert ref.plan(1056, 1, 132, False)[2] is None and ref.plan(1060, 1, 132, False)[2] == "shared memory"


def test_kernel_choice_moves_with_the_sm_count():
    """On a 114-SM H100 a bidirectional H = 512 layer (cfg3, cfg5) gets 16 units per CTA, whose backward is refused."""
    assert ref.variant(512, 2, 114).startswith("lstm_fwd_kernel<16> / refused (lstm_bwd_kernel<16>: shared memory")
    assert ref.first_untrainable(2, 114) == 460
    assert ref.variant(456, 2, 114) == "lstm_fwd_reg_kernel<64> / lstm_bwd_reg_kernel<8>"


def test_gpu_case_matrix_reaches_every_kernel_at_132_sms():
    ids = [c[0] for c in CASES]
    assert len(set(ids)) == len(ids)
    reached = {ref.variant(H, nd, 132) for _, B, T, H, nd, lens in CASES}
    assert reached >= {"lstm_fwd_reg_kernel<32> / lstm_bwd_reg_kernel<4>",
                       "lstm_fwd_reg_kernel<64> / lstm_bwd_reg_kernel<8>",
                       "lstm_fwd_kernel<8> / lstm_bwd_kernel<8>"}
    # every matrix case trains at 132 SMs; HS = 16 (forward only) is test_hs16_forward_vs_float64_and_backward_refused's
    assert all(ref.trainable(H, nd, 132) for _, B, T, H, nd, lens in CASES)
    # the lower edge of KR = 64 (H % 8 == 4: half of the last CTA's slice empty) and the batch edges
    assert {(260, 1), (260, 2), (516, 1), (516, 2)} <= {(H, nd) for _, B, T, H, nd, lens in CASES}
    assert {1, 16, 17, 33, 128} <= {B for _, B, T, H, nd, lens in CASES}
    # the shared-memory kernels at their largest batch, on a full and a partial last slice
    assert {(516, 128), (528, 128)} <= {(H, B) for _, B, T, H, nd, lens in CASES}
    assert any(T == 1 for _, B, T, H, nd, lens in CASES)
    for _, B, T, H, nd, lens in CASES:
        assert len(lens) == B and all(1 <= n <= T for n in lens) and max(lens) == T
    assert any(1 in lens and sorted(lens) != lens and sorted(lens, reverse=True) != lens for *_, lens in CASES)
    assert ("spoof-count-max-B128-T64-H256-bi", 128, 64, 256, 2) in [c[:5] for c in CASES]
    assert ("cfg3-width-B16-T200-H512-bi", 16, 200, 512, 2) in [c[:5] for c in CASES]
