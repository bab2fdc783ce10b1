"""CPU restatement of one mini-batch of reference train_loop (train.py:528-580) with a recurrent discriminator (LSTMRNN, or
GRURNN -- also an nn.LSTM --, with last_sigmoid=True; train.py:774 builds the class hp.discriminator names), composed from
the pinned functions of oracle/gantts_port.py.  TEST INFRASTRUCTURE, pinned to tests/golden/rnn_d.npz by
test_rnn_d_host.py.

The discriminator is one single-layer CPU torch nn.LSTM per layer on packed sequences (pack_padded_sequence /
pad_packed_sequence as models.py:182-187,205-210), with nn.LSTM's inter-layer dropout replaced by injected multipliers, then
hidden2out and the sigmoid.  With all-ones masks it is the reference's multi-layer nn.LSTM.  Every forward receives
`lengths` like train.py:261,265,307 pass them.

gan_step follows oracle/gantts_port.gan_step line by line (one zero_grad, y_hat_static not detached in the discriminator
update, the discriminator stepped before the adversarial forward); update_g = False is the discriminator warm-up
(train.py --discriminator-warmup, :696), reported like tests/dwarmup_oracle.py reports it.
"""
import numpy as np
import torch

from oracle import gantts_port as gp

KINDS = ("weight_ih", "weight_hh", "bias_ih", "bias_hh")


class RnnDiscriminator(object):
    """LSTMRNN / GRURNN(last_sigmoid=True) from a state_dict whose stack lives under `prefix` ("lstm" or "gru").  ``named``
    maps the model's parameter names to leaf tensors in model.parameters() order."""

    def __init__(self, sd, prefix, num_layers, hidden, bidir):
        self.sfx = ["", "_reverse"][:2 if bidir else 1]
        self.nh = hidden * len(self.sfx)
        self.named, self.layers = {}, []
        for k in range(num_layers):
            n_in = np.asarray(sd["%s.weight_ih_l%d" % (prefix, k)]).shape[1]
            m = torch.nn.LSTM(n_in, hidden, 1, batch_first=True, bidirectional=bidir)
            with torch.no_grad():
                for s in self.sfx:
                    for n in KINDS:
                        key = "%s.%s_l%d%s" % (prefix, n, k, s)
                        getattr(m, "%s_l0%s" % (n, s)).copy_(torch.as_tensor(np.asarray(sd[key])))
                        self.named[key] = getattr(m, "%s_l0%s" % (n, s))
            self.layers.append(m)
        for n in ("weight", "bias"):
            self.named["hidden2out." + n] = torch.as_tensor(np.asarray(sd["hidden2out." + n])).clone().float() \
                .requires_grad_(True)

    def params(self):
        return list(self.named.values())

    def forward(self, x, lengths, masks=None):
        """sigmoid(hidden2out(LSTM(x))) on packed sequences; masks[k] ([B * T][ndir H] multipliers) scales the output of
        layer k < num_layers - 1, None = no dropout."""
        h = x
        for k, m in enumerate(self.layers):
            packed = torch.nn.utils.rnn.pack_padded_sequence(h, [int(v) for v in lengths], batch_first=True)
            out, _ = m(packed)
            h, _ = torch.nn.utils.rnn.pad_packed_sequence(out, batch_first=True, total_length=x.size(1))
            if masks is not None and k + 1 < len(self.layers):
                h = h * masks[k].view_as(h)
        return torch.sigmoid(torch.nn.functional.linear(h, self.named["hidden2out.weight"], self.named["hidden2out.bias"]))


def gan_step(g_forward, g_params, g_sum, d, d_sum, x, y, lengths, R, hp, w_d=1.0, mse_w=0.0, mge_w=1.0, adv_w=1.0,
             training=True, lr=0.01, weight_decay=1e-7, update=True, update_g=True, d_masks=None, d_opt=None, g_opt=None):
    """oracle/gantts_port.gan_step with the recurrent discriminator `d` (a RnnDiscriminator, stepped in place with Adagrad
    state d_sum or the stepper d_opt).  ``d_masks`` = {"real": [...], "fake": [...], "adv": [...]} holds the inter-layer
    multipliers of the three discriminator forwards (None: no dropout).  Returns (dict of floats, y_hat, y_hat_static)."""
    y_static = gp.get_static_features(y, hp["num_windows"], hp["stream_sizes"], hp["has_dynamic_features"])
    mask = gp.sequence_mask(lengths, x.size(1)).unsqueeze(-1)
    d_params = d.params()
    for p in list(g_params) + d_params:
        p.grad = None
    y_hat, y_hat_static = g_forward()
    out = {}
    T = mask.sum().item()
    cond = hp.get("discriminator_linguistic_condition", False)
    dm = d_masks or {}
    real_in = gp.get_selected_static_stream(y_static, hp)
    fake_in = gp.get_selected_static_stream(y_hat_static if update_g else y_hat_static.detach(), hp)
    if cond:
        real_in = torch.cat((x, real_in), -1)
        fake_in = torch.cat((x, fake_in), -1)
    D_real = d.forward(real_in, lengths, dm.get("real"))
    out["real_correct"] = ((D_real > 0.5).float() * mask).sum().item()
    D_fake = d.forward(fake_in, lengths, dm.get("fake"))
    out["fake_correct"] = ((D_fake < 0.5).float() * mask).sum().item()
    loss_real, loss_fake = gp.bce_real(D_real, mask, T), gp.bce_fake(D_fake, mask, T)
    loss_d = loss_real + loss_fake
    if update:
        loss_d.backward(retain_graph=True)
        dg = [p.grad for p in d_params]
        out["d_grad_norm"] = float(gp.clip_grad_norm(dg, 1.0))
        if d_opt is not None:
            d_opt(d_params, dg)
        else:
            gp.adagrad_step(d_params, dg, d_sum, lr, weight_decay)
    out.update(loss_d=loss_d.item(), loss_fake_d=loss_fake.item(), loss_real_d=loss_real.item())
    loss_mge = gp.masked_mse(y_hat_static, y_static, mask=mask)
    loss_mse = gp.masked_mse(y_hat, y, mask=mask)
    if adv_w > 0 and update_g:
        fake_in = gp.get_selected_static_stream(y_hat_static, hp)
        if cond:
            fake_in = torch.cat((x, fake_in), -1)
        loss_adv = gp.bce_real(d.forward(fake_in, lengths, dm.get("adv")), mask, T)
    else:
        loss_adv, adv_w = y.new_zeros(()), 0.0
    loss_g = (mse_w * loss_mse + mge_w * loss_mge) + adv_w * loss_adv
    if update and update_g:
        loss_g.backward()
        g_params = list(g_params)
        gg = [p.grad if p.grad is not None else torch.zeros_like(p) for p in g_params]
        out["g_grad_norm"] = float(gp.clip_grad_norm(gg, 1.0))
        if g_opt is not None:
            g_opt(g_params, gg)
        else:
            gp.adagrad_step(g_params, gg, g_sum, lr, weight_decay)
    elif update:
        out["g_grad_norm"] = 0.0
    out.update(loss_mse=loss_mse.item(), loss_mge=loss_mge.item(), loss_adv=float(loss_adv.detach()),
               loss_g=float(loss_g.detach()), frames=T)
    return out, y_hat.detach(), y_hat_static.detach()
