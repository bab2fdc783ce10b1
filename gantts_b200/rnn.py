"""nn.LSTM replacement on the native kernels: input projections of all time steps as one tensor-core
GEMM, the recurrence in gantts_lstm_layer_fwd/bwd (persistent cooperative kernel), packed-sequence
semantics of reference gantts/models.py:101-112,182-187,205-210 (pack_padded_sequence ->
nn.LSTM -> pad_packed_sequence) without packing: outputs beyond each length are zero, the reverse
direction starts at the last valid frame."""
import ctypes

import torch

from . import _lib
from . import config
from . import ops


class _LSTMLayer(torch.autograd.Function):
    """One (bi)directional LSTM layer.  W_ih: [ndir*4H, I] (direction-stacked), W_hh: [ndir, 4H, H],
    bias: [ndir*4H] (= b_ih + b_hh)."""

    @staticmethod
    def forward(ctx, x, lengths, W_ih, W_hh, bias, engine):
        ops.require_cuda(x, W_ih, W_hh, bias)
        lib = _lib.load()
        B, T, I = x.shape
        ndir, G4, H = W_hh.shape
        x2 = x.contiguous().view(B * T, I)
        W_ih, W_hh, bias = W_ih.contiguous(), W_hh.contiguous(), bias.contiguous()
        dev = x.device
        xproj = torch.empty(B * T, ndir * G4, dtype=torch.float32, device=dev)
        ws = ops.workspace(lib.gantts_linear_workspace_bytes(B * T, ndir * G4, I, engine), dev)
        _lib.check(lib.gantts_linear_fwd(x2.data_ptr(), I, W_ih.data_ptr(), bias.data_ptr(), xproj.data_ptr(),
                                         ndir * G4, B * T, ndir * G4, I, _lib.ACT_NONE, 0.0, 0.0, 0, engine,
                                         ws.data_ptr(), ws.numel(), ops._stream()))
        h = torch.empty(B, T, ndir * H, dtype=torch.float32, device=dev)
        gates = torch.zeros(ndir, B, T, G4, dtype=torch.float32, device=dev)
        cells = torch.zeros(ndir, B, T, H, dtype=torch.float32, device=dev)
        bar = ops.workspace(lib.gantts_lstm_workspace_bytes(), dev, "lstm_bar")
        _lib.check(lib.gantts_lstm_layer_fwd(xproj.data_ptr(), W_hh.data_ptr(), lengths.data_ptr(), h.data_ptr(),
                                             gates.data_ptr(), cells.data_ptr(), B, T, H, ndir, bar.data_ptr(),
                                             bar.numel(), ops._stream()))
        ctx.save_for_backward(x2, lengths, W_ih, W_hh, h, gates, cells)
        ctx.engine, ctx.dims = engine, (B, T, I, H, ndir, bias is not None)
        return h

    @staticmethod
    def backward(ctx, dh):
        lib = _lib.load()
        x2, lengths, W_ih, W_hh, h, gates, cells = ctx.saved_tensors
        B, T, I, H, ndir, _ = ctx.dims
        G4, dev, eng = 4 * H, dh.device, ctx.engine
        dh = dh.contiguous()
        dxproj = torch.empty(B * T, ndir * G4, dtype=torch.float32, device=dev)
        bar = ops.workspace(lib.gantts_lstm_workspace_bytes(), dev, "lstm_bar")
        _lib.check(lib.gantts_lstm_layer_bwd(dh.data_ptr(), W_hh.data_ptr(), lengths.data_ptr(), gates.data_ptr(),
                                             cells.data_ptr(), dxproj.data_ptr(), B, T, H, ndir, bar.data_ptr(),
                                             bar.numel(), ops._stream()))
        M = B * T
        need_gx = ctx.needs_input_grad[0]
        gx = torch.empty(M, I, dtype=torch.float32, device=dev) if need_gx else None
        gW_ih = torch.empty_like(W_ih)
        gb = torch.empty(ndir * G4, dtype=torch.float32, device=dev)
        gz = torch.empty(M, ndir * G4, dtype=torch.float32, device=dev)
        ws = ops.workspace(lib.gantts_linear_workspace_bytes(M, ndir * G4, max(I, H), eng), dev)
        # dx, dW_ih, dbias from the direction-stacked projection (act NONE: gz = dxproj)
        _lib.check(lib.gantts_linear_bwd(dxproj.data_ptr(), ndir * G4, dxproj.data_ptr(), ndir * G4, x2.data_ptr(), I,
                                         W_ih.data_ptr(), gz.data_ptr(), gx.data_ptr() if gx is not None else None, I,
                                         gW_ih.data_ptr(), gb.data_ptr(), M, ndir * G4, I, _lib.ACT_NONE, 0.0, 0.0, 0,
                                         eng, ws.data_ptr(), ws.numel(), ops._stream()))
        # dW_hh[dir] = dxproj_dir^T h_prev
        gW_hh = torch.empty_like(W_hh)
        hprev = torch.empty(M, H, dtype=torch.float32, device=dev)
        gzd = torch.empty(M, G4, dtype=torch.float32, device=dev)
        for d in range(ndir):
            _lib.check(lib.gantts_lstm_hprev(h.data_ptr(), lengths.data_ptr(), hprev.data_ptr(), B, T, H, ndir, d,
                                             ops._stream()))
            dxd = dxproj[:, d * G4:(d + 1) * G4]
            _lib.check(lib.gantts_linear_bwd(dxd.data_ptr(), ndir * G4, dxd.data_ptr(), ndir * G4, hprev.data_ptr(), H,
                                             W_hh[d].data_ptr(), gzd.data_ptr(), None, H, gW_hh[d].data_ptr(), None,
                                             M, G4, H, _lib.ACT_NONE, 0.0, 0.0, 0, eng, ws.data_ptr(), ws.numel(),
                                             ops._stream()))
        return (gx.view(B, T, I) if gx is not None else None), None, gW_ih, gW_hh, gb, None


class _Dropout(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, p, seed):
        ops.require_cuda(x)
        lib = _lib.load()
        x = x.contiguous()
        y = torch.empty_like(x)
        cols = x.shape[-1]
        _lib.check(lib.gantts_dropout(x.data_ptr(), y.data_ptr(), x.numel() // cols, cols, p, seed, ops._stream()))
        ctx.cfg = (p, seed)
        return y

    @staticmethod
    def backward(ctx, gy):
        lib = _lib.load()
        p, seed = ctx.cfg
        gy = gy.contiguous()
        gx = torch.empty_like(gy)
        cols = gy.shape[-1]
        _lib.check(lib.gantts_dropout(gy.data_ptr(), gx.data_ptr(), gy.numel() // cols, cols, p, seed, ops._stream()))
        return gx, None, None


def lengths_tensor(lengths, B, T, device):
    """Accepts what the reference passes as `lengths` (list of ints / 0-d tensors, LongTensor, None)."""
    if lengths is None:
        return torch.full((B,), T, dtype=torch.int64, device=device)
    if torch.is_tensor(lengths):
        return lengths.to(device=device, dtype=torch.int64).contiguous().view(-1)
    return torch.tensor([int(v) for v in lengths], dtype=torch.int64, device=device)


def lstm_forward(lstm, x, lengths, training, engine=None):
    """Run the weights of a torch ``nn.LSTM`` (batch_first) through the native kernels.
    x: (B, T, I) CUDA; returns (B, T_out, dirs*H) with T_out = max(lengths) like pad_packed_sequence."""
    if not lstm.batch_first:
        raise RuntimeError("gantts_b200: only batch_first LSTMs are supported")
    eng = config.engine_id(engine)
    B, T, _ = x.shape
    lens = lengths_tensor(lengths, B, T, x.device)
    ndir = 2 if lstm.bidirectional else 1
    if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in lstm.parameters())):
        # a layer whose backward this device cannot run is refused before its forward, not in loss.backward()
        _lib.check(_lib.load().gantts_lstm_layer_supported(lstm.hidden_size, ndir, 1))
    h = x
    for k in range(lstm.num_layers):
        sfx = ["", "_reverse"][:ndir]
        W_ih = torch.cat([getattr(lstm, "weight_ih_l%d%s" % (k, s)) for s in sfx], 0)
        W_hh = torch.stack([getattr(lstm, "weight_hh_l%d%s" % (k, s)) for s in sfx], 0)
        bias = torch.cat([getattr(lstm, "bias_ih_l%d%s" % (k, s)) + getattr(lstm, "bias_hh_l%d%s" % (k, s))
                          for s in sfx], 0)
        h = _LSTMLayer.apply(h, lens, W_ih, W_hh, bias, eng)
        if training and lstm.dropout > 0 and k + 1 < lstm.num_layers:
            h = _Dropout.apply(h, float(lstm.dropout), ops.draw_seed())
    # pad_packed_sequence returns max(lengths) frames.  The reference always passes HOST lengths
    # (cpu_sorted_lengths, train.py:503): those are honoured.  A CUDA lengths tensor keeps the padded length
    # (reading its maximum would be a host synchronisation per forward; in train.py's batches it equals T).
    if lengths is not None and not (torch.is_tensor(lengths) and lengths.is_cuda):
        t_out = int(max(int(v) for v in lengths))
        if t_out < T:
            h = h[:, :t_out]
    return h


# ------------------------------------------------------------------------------------ SRU
class _SRUScan(torch.autograd.Function):
    """h, = SRU v1 scan over u = x W (see csrc/sru.cu).  u: (B,T,ncols*k); x_hw: (B,T,ncols) or None."""

    @staticmethod
    def forward(ctx, u, x_hw, bias, mask_h, d, k, bidir, act):
        ops.require_cuda(u, bias)
        lib = _lib.load()
        B, T, _ = u.shape
        ncols = d * (2 if bidir else 1)
        u = u.contiguous()
        xh = x_hw.contiguous() if x_hw is not None else None
        mh = mask_h.contiguous() if mask_h is not None else None
        h = torch.empty(B, T, ncols, dtype=torch.float32, device=u.device)
        c = torch.empty(B, T, ncols, dtype=torch.float32, device=u.device)
        _lib.check(lib.gantts_sru_fwd(u.data_ptr(), xh.data_ptr() if xh is not None else None, bias.data_ptr(),
                                      mh.data_ptr() if mh is not None else None, h.data_ptr(), c.data_ptr(),
                                      B, T, d, k, int(bidir), act, ops._stream()))
        ctx.save_for_backward(u, xh if xh is not None else u.new_empty(0), bias,
                              mh if mh is not None else u.new_empty(0), c)
        ctx.cfg = (d, k, bidir, act, xh is not None, mh is not None)
        return h

    @staticmethod
    def backward(ctx, dh):
        lib = _lib.load()
        u, xh, bias, mh, c = ctx.saved_tensors
        d, k, bidir, act, has_x, has_m = ctx.cfg
        B, T, _ = u.shape
        ncols = d * (2 if bidir else 1)
        dh = dh.contiguous()
        du = torch.empty_like(u)
        dx = torch.zeros(B, T, ncols, dtype=torch.float32, device=u.device) if has_x else None
        part = torch.empty(B, 2 * ncols, dtype=torch.float32, device=u.device)
        _lib.check(lib.gantts_sru_bwd(u.data_ptr(), xh.data_ptr() if has_x else None, bias.data_ptr(),
                                      mh.data_ptr() if has_m else None, c.data_ptr(), dh.data_ptr(), du.data_ptr(),
                                      dx.data_ptr() if has_x else None, part.data_ptr(), B, T, d, k, int(bidir), act,
                                      ops._stream()))
        return du, dx, part.sum(0), None, None, None, None, None


class SRUCell(torch.nn.Module):
    """Parameters of one SRU layer with the shapes/initialisation of the upstream 2017 implementation:
    weight (n_in, dirs*n_out*k), bias (dirs*n_out*2); k = 3 when n_in == dirs*n_out else 4."""

    def __init__(self, n_in, n_out, dropout=0.0, rnn_dropout=0.0, bidirectional=False, use_tanh=1, use_relu=0):
        super(SRUCell, self).__init__()
        self.n_in, self.n_out, self.bidirectional = n_in, n_out, bidirectional
        self.dropout, self.rnn_dropout = dropout, rnn_dropout
        self.activation_type = 2 if use_relu else (1 if use_tanh else 0)
        out_size = n_out * 2 if bidirectional else n_out
        self.k = 4 if n_in != out_size else 3
        self.weight = torch.nn.Parameter(torch.empty(n_in, out_size * self.k))
        self.bias = torch.nn.Parameter(torch.zeros(out_size * 2))
        val_range = (3.0 / n_in) ** 0.5
        torch.nn.init.uniform_(self.weight, -val_range, val_range)

    def forward(self, x, engine=None, lengths=None):
        """x: (B, T, n_in) -> (B, T, dirs*n_out).  lengths: None (every sequence runs over the padded T, like the
        upstream SRU), or int64 CUDA (B,) in eval mode: sequence b runs over its own lengths[b] frames, its reverse
        direction starts at lengths[b] - 1, and h is 0 beyond (gantts_sru_fwd_lengths; forward only)."""
        B, T, _ = x.shape
        ncols = self.n_out * (2 if self.bidirectional else 1)
        if lengths is not None:
            return self._forward_lengths(x, lengths, engine)
        # upstream cuda_functional.SRUCell.forward: only the GEMM input is masked (u = (input * mask_x) @ W); the
        # highway term (1 - r) * x of SRU_Compute receives the UNMASKED input.
        x_in = x
        if self.training and self.rnn_dropout > 0:        # variational: one mask per sequence, shared over time
            ones = torch.ones(B, 1, self.n_in, device=x.device)
            x = x_in * _Dropout.apply(ones, float(self.rnn_dropout), ops.draw_seed())
        u = ops.linear_act(x, self.weight.t().contiguous(), None, _lib.ACT_NONE, engine=engine)
        mask_h = None
        if self.training and self.dropout > 0:
            mask_h = _Dropout.apply(torch.ones(B, ncols, device=x.device), float(self.dropout), ops.draw_seed())
        x_hw = x_in if self.k == 3 else None
        return _SRUScan.apply(u, x_hw, self.bias, mask_h, self.n_out, self.k, self.bidirectional,
                              self.activation_type)


    def _forward_lengths(self, x, lengths, engine):
        if self.training or torch.is_grad_enabled() and (x.requires_grad or self.weight.requires_grad):
            raise RuntimeError("gantts_b200: the SRU forward with lengths is eval-only and has no backward: call it in "
                               "eval mode under torch.no_grad()")
        if not (torch.is_tensor(lengths) and lengths.is_cuda and lengths.dtype == torch.int64):
            raise RuntimeError("gantts_b200: the SRU forward with lengths needs int64 CUDA lengths")
        lib = _lib.load()
        B, T, _ = x.shape
        ncols = self.n_out * (2 if self.bidirectional else 1)
        u = ops.linear_act(x, self.weight.t().contiguous(), None, _lib.ACT_NONE, engine=engine).contiguous()
        xh = x.contiguous() if self.k == 3 else None
        h = torch.empty(B, T, ncols, dtype=torch.float32, device=x.device)
        _lib.check(lib.gantts_sru_fwd_lengths(u.data_ptr(), xh.data_ptr() if xh is not None else None,
                                              self.bias.data_ptr(), lengths.contiguous().data_ptr(), h.data_ptr(),
                                              B, T, self.n_out, self.k, int(self.bidirectional),
                                              self.activation_type, ops._stream()))
        return h


class SRU(torch.nn.Module):
    """Stack of SRU layers (``rnn_lst``) like upstream ``cuda_functional.SRU``; batch-first here."""

    def __init__(self, input_size, hidden_size, num_layers=2, dropout=0.0, rnn_dropout=0.0, bidirectional=False,
                 use_tanh=1, use_relu=0):
        super(SRU, self).__init__()
        self.rnn_lst = torch.nn.ModuleList()
        out_size = hidden_size * 2 if bidirectional else hidden_size
        for i in range(num_layers):
            self.rnn_lst.append(SRUCell(input_size if i == 0 else out_size, hidden_size,
                                        dropout=dropout if i + 1 != num_layers else 0.0, rnn_dropout=rnn_dropout,
                                        bidirectional=bidirectional, use_tanh=use_tanh, use_relu=use_relu))

    def forward(self, x, engine=None, lengths=None):
        """lengths: see SRUCell.forward (None: the padded semantics of the reference's SRURNN, used in training)."""
        for cell in self.rnn_lst:
            x = cell(x, engine=engine, lengths=lengths)
        return x
