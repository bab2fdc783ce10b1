"""Plain float64 restatement of one LSTM layer at the contract of gantts_lstm_layer_fwd / _bwd and gantts_lstm_hprev
(include/gantts_b200.h), a mirror of which recurrence kernel csrc/lstm.cu launches for a shape, and the case
matrix tests/test_gpu_lstm_kernels.py runs.

The layer: xproj [B][T][ndir*4H] (x W_ih^T + b_ih + b_hh, direction-major columns), W_hh [ndir][4H][H], lengths [B].
Sequence b runs for t < lengths[b]; direction 1 starts at t = lengths[b] - 1 (pack_padded_sequence semantics).  There is
no hand-written backward here: dxproj is torch.autograd through the float64 loop.
"""
import numpy as np
import torch

# csrc/lstm.cu
LSTM_THREADS = 256
LSTM_BC = 16
LSTM_MAX_B = 128
SMEM_LIMIT = 227 * 1024
F32 = 4


def lstm_layer_f64(xproj, W_hh, lengths):
    """-> h [B][T][ndir*H] (zero beyond each length), gates [ndir][B][T][4H] (i, f, g, o after activation) and
    cells [ndir][B][T][H], both zero beyond each length.  Differentiable with respect to xproj and W_hh."""
    B, T, _ = xproj.shape
    ndir, G4, H = W_hh.shape
    lens = torch.as_tensor([int(v) for v in lengths], dtype=torch.int64)
    hs, gs, cs = [], [], []
    for d in range(ndir):
        h = xproj.new_zeros(B, H)
        c = xproj.new_zeros(B, H)
        h_t, g_t, c_t = [None] * T, [None] * T, [None] * T
        for t in (range(T) if d == 0 else range(T - 1, -1, -1)):
            valid = (lens > t).view(B, 1)
            pre = xproj[:, t, d * G4:(d + 1) * G4] + h @ W_hh[d].t()
            i = torch.sigmoid(pre[:, :H])
            f = torch.sigmoid(pre[:, H:2 * H])
            g = torch.tanh(pre[:, 2 * H:3 * H])
            o = torch.sigmoid(pre[:, 3 * H:])
            c_new = f * c + i * g
            h_new = o * torch.tanh(c_new)
            # the state only advances on valid frames: the reverse direction meets zeros until t = lengths[b] - 1
            c = torch.where(valid, c_new, c)
            h = torch.where(valid, h_new, h)
            zero = torch.zeros_like(h_new)
            h_t[t] = torch.where(valid, h_new, zero)
            c_t[t] = torch.where(valid, c_new, zero)
            g_t[t] = torch.where(valid, torch.cat([i, f, g, o], 1), torch.zeros_like(pre))
        hs.append(torch.stack(h_t, 1))
        gs.append(torch.stack(g_t, 1))
        cs.append(torch.stack(c_t, 1))
    return torch.cat(hs, 2), torch.stack(gs, 0), torch.stack(cs, 0)


def lstm_layer_dxproj_f64(xproj, W_hh, lengths, dh):
    """dL/dxproj for dL/dh = dh, by autograd through lstm_layer_f64 (xproj is the leaf; dh beyond a length is ignored)."""
    xp = xproj.detach().to(torch.float64).requires_grad_(True)
    h, _, _ = lstm_layer_f64(xp, W_hh.detach().to(torch.float64), lengths)
    return torch.autograd.grad(h, xp, dh.to(torch.float64))[0]


def lstm_hprev(h, lengths, H, ndir, d):
    """The values gantts_lstm_hprev copies: hprev[b][t] = h[b][t - 1 (d = 0) | t + 1 (d = 1)][d*H:(d+1)*H], zero at each
    sequence's first step and beyond its length.  An index gather, so bit-exact in any dtype."""
    B, T, _ = h.shape
    out = h.new_zeros(B, T, H)
    for b, n in enumerate(int(v) for v in lengths):
        src = h[b, :, d * H:(d + 1) * H]
        if d == 0:
            out[b, 1:n] = src[0:n - 1]
        else:
            out[b, 0:n - 1] = src[1:n]
    return out


# ----------------------------------------------------------------------------------------- kernel choice (lstm.cu)
def pick_hs(H, ndir, sms):
    """lstm_pick_hs: (hidden units per CTA, CTAs per direction); HS = 0 when neither 8 nor 16 fits one wave."""
    for hs in (8, 16):
        s = -(-H // hs)
        if s * ndir <= sms:
            return hs, s
    return 0, 0


def plan(H, ndir, sms, bwd):
    """lstm_plan / lstm_run: (kernel name, dynamic shared memory in bytes, refusal or None)."""
    hs, _ = pick_hs(H, ndir, sms)
    if hs == 0:
        return None, 0, "one wave"
    if hs == 8 and H <= 512:
        if not bwd:
            KR = 32 if H <= 256 else 64
            return "lstm_fwd_reg_kernel<%d>" % KR, (LSTM_BC * 8 * KR + 8 * LSTM_BC * 32 + LSTM_MAX_B * 8) * F32, None
        RPT = 4 if 4 * H <= 4 * LSTM_THREADS else 8
        return "lstm_bwd_reg_kernel<%d>" % RPT, (LSTM_BC * RPT * LSTM_THREADS + 8 * 64 + 2 * LSTM_MAX_B * 8) * F32, None
    if not bwd:
        smem = (4 * hs * (H + 4) + LSTM_BC * H + LSTM_BC * 4 * hs + LSTM_MAX_B * hs) * F32
    else:
        smem = (hs * (4 * H + 4) + LSTM_BC * (4 * H + 4) + LSTM_THREADS + 2 * LSTM_MAX_B * hs) * F32
    name = "lstm_%s_kernel<%d>" % ("bwd" if bwd else "fwd", hs)
    return name, smem, ("shared memory" if smem > SMEM_LIMIT else None)


def variant(H, ndir, sms):
    """'forward kernel / backward kernel' of a layer; a refused launch reads 'refused (<kernel>: <limit>)'."""
    out = []
    for bwd in (False, True):
        name, smem, why = plan(H, ndir, sms, bwd)
        out.append(name if why is None else "refused (%s: %s)" % (name, why))
    return " / ".join(out)


def trainable(H, ndir, sms):
    return all(plan(H, ndir, sms, bwd)[2] is None for bwd in (False, True))


def first_untrainable(ndir, sms):
    """The smallest H (a multiple of 4) whose forward runs but whose backward is refused."""
    H = 4
    while trainable(H, ndir, sms) or plan(H, ndir, sms, False)[2] is not None:
        H += 4
        assert H <= 4096
    return H


H_LIST = (4, 12, 256, 260, 512, 516, 528)


def case_lengths(kind, B, T, seed):
    if kind in ("full", "T=1"):
        return [T] * B
    if kind == "desc":
        return [max(1, T - (b * T) // B) for b in range(B)]
    # unsorted ragged: the full length, two sequences of length 1, the rest anywhere in [1, T]
    rng = np.random.RandomState(seed)
    lens = [T, 1, 1] + [int(v) for v in rng.randint(1, T + 1, max(B - 3, 0))]
    lens = lens[:B]
    rng.shuffle(lens)
    return lens


def _cases():
    """(id, B, T, H, ndir, lengths) of the GPU case matrix (tests/test_gpu_lstm_kernels.py)"""
    cases = []
    for H in H_LIST:
        T = 23 if H < 256 else 7          # the float64 loop runs on the CPU: short where H is large
        for ndir in (1, 2):
            shapes = [(1, T, "full"), (17, T, "desc"), (33, T, "unsorted"), (16, 1, "T=1")]
            if H in (12, 260, 516, 528):
                shapes.append((128, T, "unsorted"))
            for B, Tc, kind in shapes:
                cases.append(("H%d-%s-B%d-T%d-%s" % (H, "bi" if ndir == 2 else "uni", B, Tc, kind), B, Tc, H, ndir, kind))
    cases.append(("spoof-count-max-B128-T64-H256-bi", 128, 64, 256, 2, "unsorted"))
    cases.append(("cfg3-width-B16-T200-H512-bi", 16, 200, 512, 2, "desc"))
    return [(cid, B, T, H, ndir, case_lengths(kind, B, T, i)) for i, (cid, B, T, H, ndir, kind) in enumerate(cases)]


CASES = _cases()
