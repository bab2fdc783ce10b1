"""Plain float64 restatement of the SRU v1 scan at the contract of gantts_sru_fwd / gantts_sru_bwd /
gantts_sru_fwd_lengths (include/gantts_b200.h), and the case matrix tests/test_gpu_sru_kernels.py runs.

The scan: u [B][T][ncols*k] with k fastest (candidate, forget, reset[, highway]), ncols = d * (bidir ? 2 : 1); x [B][T]
[ncols] is the highway input when k == 3; bias [2*ncols] = forget | reset; mask_h [B][ncols] (already scaled) multiplies
g(c_t); act 0 / 1 / 2 = identity / tanh / ReLU.  Columns [0, d) run forward in time, [d, 2d) backward:
    f = sigmoid(u_1 + b_f), r = sigmoid(u_2 + b_r), c_t = f c_{t-1} + (1 - f) u_0, h_t = r g(c_t) m + (1 - r) x'_t
with x' = x (k == 3) or u_3 (k == 4).  There is no hand-written backward here: du, dx and the bias gradient are
torch.autograd through the float64 loop.

ReLU kink: a cell within rounding of 0 can fall on either side of it in fp32, and the other branch then carries through dc
to every earlier frame.  So the backward takes ReLU's derivative pattern from the device's saved c when one is given (the
forward value stays the float64 max(c, 0), which differs from it by at most |c|).
"""
import numpy as np
import torch

SRU_UNR = 8            # csrc/sru.cu: steps per chunk of the scans
SRU_THREADS = 128      # threads per block: one per (batch row, column)


def _act(c, act, pattern):
    if act == 1:
        return torch.tanh(c)
    if act == 2:
        if pattern is None:
            return torch.relu(c)
        # the value of max(c, 0), the derivative of the given pattern
        return torch.relu(c).detach() + (c - c.detach()) * pattern
    return c


def sru_f64(u, x, bias, mask_h, d, bidir, act, c_relu=None, lengths=None):
    """-> h, c [B][T][ncols] of the scan; differentiable with respect to u, x and bias.  c_relu: [B][T][ncols] cell
    states whose sign gives ReLU's derivative (the device's saved c), or None.  lengths: None for the padded scan of
    gantts_sru_fwd; else the length-exact scan of gantts_sru_fwd_lengths (sequence b over L = clamp(lengths[b], 0, T)
    frames, the reverse direction starting at L - 1 with a zero cell, h and c 0 from L on)."""
    B, T, ku = u.shape
    dirs = 2 if bidir else 1
    ncols = d * dirs
    k = ku // ncols
    uu = u.view(B, T, ncols, k)
    L = torch.full((B,), T, dtype=torch.int64) if lengths is None else \
        torch.as_tensor([min(max(int(v), 0), T) for v in lengths], dtype=torch.int64)
    hs, cs = [], []
    for di in range(dirs):
        cols = slice(di * d, (di + 1) * d)
        bf, br = bias[cols], bias[ncols:][cols]
        m = mask_h[:, cols] if mask_h is not None else None
        c = u.new_zeros(B, d)
        h_t, c_t = [None] * T, [None] * T
        for t in (range(T) if di == 0 else range(T - 1, -1, -1)):
            valid = (L > t).view(B, 1)
            g = uu[:, t, cols]
            f = torch.sigmoid(g[..., 1] + bf)
            r = torch.sigmoid(g[..., 2] + br)
            c_new = f * c + (1 - f) * g[..., 0]
            xp = x[:, t, cols] if k == 3 else g[..., 3]
            pat = (c_relu[:, t, cols] > 0).to(u.dtype) if (c_relu is not None and act == 2) else None
            val = _act(c_new, act, pat)
            h_new = r * (val * m if m is not None else val) + (1 - r) * xp
            # the state only advances on valid frames: the reverse direction meets zeros until t = L - 1
            c = torch.where(valid, c_new, c)
            zero = torch.zeros_like(h_new)
            h_t[t] = torch.where(valid, h_new, zero)
            c_t[t] = torch.where(valid, c_new, zero)
        hs.append(torch.stack(h_t, 1))
        cs.append(torch.stack(c_t, 1))
    return torch.cat(hs, 2), torch.cat(cs, 2)


def sru_f64_bwd(u, x, bias, mask_h, d, bidir, act, dh, c_relu=None):
    """(du [B][T][ncols*k], dx [B][T][ncols] (k == 3, else None), dbias_part [B][2*ncols]) for dL/dh = dh by autograd
    through sru_f64.  dx is the highway term the kernel ADDS to its dx; dbias_part[b] = (sum_t du[b, t, col*k + 1],
    sum_t du[b, t, col*k + 2])."""
    B, T, ku = u.shape
    ncols = d * (2 if bidir else 1)
    k = ku // ncols
    u64 = u.detach().to(torch.float64).requires_grad_(True)
    x64 = x.detach().to(torch.float64).requires_grad_(True) if k == 3 else None
    m64 = mask_h.detach().to(torch.float64) if mask_h is not None else None
    cr = c_relu.detach().to(torch.float64) if c_relu is not None else None
    h, _ = sru_f64(u64, x64, bias.detach().to(torch.float64), m64, d, bidir, act, cr)
    leaves = [u64] + ([x64] if k == 3 else [])
    grads = torch.autograd.grad(h, leaves, dh.to(torch.float64))
    du = grads[0]
    dx = grads[1] if k == 3 else None
    duv = du.view(B, T, ncols, k)
    part = torch.cat([duv[..., 1].sum(1), duv[..., 2].sum(1)], 1)
    return du, dx, part


# ------------------------------------------------------------------------------------------------- the case matrix
SPECIAL_LENGTHS = ("T", 1, 0, -1, "T+3", "T/2")


def case_lengths(B, T, i):
    """Lengths for the length-exact forward: rows cycle through T, 1, 0, a negative one, one above T and T / 2 (shifted
    by the case index i), the rest anywhere in [0, T]."""
    rng = np.random.RandomState(100 + i)
    out = []
    for b in range(B):
        if b < len(SPECIAL_LENGTHS):
            s = SPECIAL_LENGTHS[(b + i) % len(SPECIAL_LENGTHS)]
            out.append({"T": T, "T+3": T + 3, "T/2": T // 2}.get(s, s))
        else:
            out.append(int(rng.randint(0, T + 1)))
    return out


def _cases():
    """(id, B, T, d, k, bidir, act, mask_p) of the GPU matrix"""
    cases = []
    # the full cross at a small shape with a chunk tail (17 = 2 * 8 + 1)
    for k in (3, 4):
        for bidir in (0, 1):
            for act in (0, 1, 2):
                for p in (0.0, 0.3):
                    cases.append((3, 17, 8, k, bidir, act, p))
    # every residue of T mod 8, T = 1, and a long scan, on one variant per k
    for T in (1, 2, 3, 4, 5, 6, 7, 8, 9, 15, 16, 17, 63, 64, 65, 1000):
        cases.append((2, T, 4, 4, 1, 2, 0.3))
        cases.append((2, T, 4, 3, 1, 1, 0.0))
    # B * ncols across the 128-thread block edges, and several blocks whose last one is partial
    for B, d, bidir, k, act in ((1, 1, 0, 4, 0), (127, 1, 0, 3, 2), (1, 127, 0, 4, 1), (2, 32, 1, 4, 2),
                                (1, 64, 1, 3, 0), (3, 43, 0, 3, 1), (129, 1, 0, 4, 2), (5, 37, 1, 3, 2),
                                (3, 100, 1, 4, 1)):
        cases.append((B, 9, d, k, bidir, act, 0.3))
    # the tts_acoustic layer: 512 bidirectional ReLU units (dropout 0.2), layer 0 (k = 4) and the layers above (k = 3)
    for k in (4, 3):
        cases.append((4, 200, 512, k, 1, 2, 0.2))
    out = []
    for B, T, d, k, bidir, act, p in cases:
        cid = "B%d-T%d-d%d-k%d-%s-%s%s" % (B, T, d, k, "bi" if bidir else "uni", ("id", "tanh", "relu")[act],
                                            "-mask%g" % p if p else "")
        out.append((cid, B, T, d, k, bidir, act, p))
    return out


CASES = _cases()


def case_inputs(B, T, d, k, bidir, p, seed):
    """u, x (k == 3, else None), bias, mask_h (p > 0, else None), dh: float32 on the CPU.  Forget / reset
    pre-activations spread over both sides of 0; dh nonzero everywhere."""
    g = torch.Generator().manual_seed(seed)
    ncols = d * (2 if bidir else 1)
    u = torch.randn(B, T, ncols * k, generator=g)
    x = torch.randn(B, T, ncols, generator=g) if k == 3 else None
    bias = (torch.rand(2 * ncols, generator=g) * 2 - 1) * 0.5
    mask = None
    if p > 0:
        keep = torch.rand(B, ncols, generator=g) >= p
        mask = keep.float() / (1 - p)
    dh = torch.randn(B, T, ncols, generator=g)
    return u, x, bias, mask, dh
