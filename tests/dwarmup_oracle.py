"""CPU restatement of the discriminator warm-up step and of the spoofing-rate count, composed from the pinned functions of
oracle/gantts_port.py.  TEST INFRASTRUCTURE, pinned to tests/golden/dwarmup.npz by test_dwarmup_host.py.

d_only_step: one mini-batch of reference train_loop (train.py:528-566) with update_g = False (--discriminator-warmup,
:696): apply_generator, update_discriminator (:245-279), and NOT update_generator.  It reports the loss slots the fused
step reports for such a step: the D losses, counts and gradient norm as in the full step, the forward values of MSE /
MGE, loss_adv = 0, loss_g = mse_w loss_mse + mge_w loss_mge, g_grad_norm = 0.

spoof_count: train.py:549-558, the frames of y_hat_static the frozen reference discriminator takes for natural (D_ref in
eval mode, :445; no linguistic conditioning, :554-555).
"""
import torch

from oracle import gantts_port as gp


def d_only_step(g_forward, d_layers, d_sum, x, y, lengths, hp, mse_w=0.0, mge_w=1.0, dropout_d=0.0, lr=0.01,
                weight_decay=1e-7, d_masks=None, d_opt=None):
    """``g_forward()`` -> (y_hat, y_hat_static) of apply_generator; ``d_layers`` [(W, b), ...] requiring grad, stepped in
    place with Adagrad (state ``d_sum``) or the stepper ``d_opt``.  Returns (dict of floats, y_hat, y_hat_static)."""
    y_static = gp.get_static_features(y, hp["num_windows"], hp["stream_sizes"], hp["has_dynamic_features"])
    mask = gp.sequence_mask(lengths, x.size(1)).unsqueeze(-1)
    d_params = [t for pair in d_layers for t in pair]
    for p in d_params:
        p.grad = None
    with torch.no_grad():          # the generator is not stepped: its gradient from loss_d is never used
        y_hat, y_hat_static = g_forward()
    T = mask.sum().item()
    dm = d_masks or {}
    real_in = gp.get_selected_static_stream(y_static, hp)
    fake_in = gp.get_selected_static_stream(y_hat_static, hp)
    if hp.get("discriminator_linguistic_condition", False):
        real_in = torch.cat((x, real_in), -1)
        fake_in = torch.cat((x, fake_in), -1)
    D_real = gp.mlp_forward(real_in, d_layers, dropout_d, True, last_sigmoid=True, masks=dm.get("real"))
    D_fake = gp.mlp_forward(fake_in, d_layers, dropout_d, True, last_sigmoid=True, masks=dm.get("fake"))
    out = {"real_correct": ((D_real > 0.5).float() * mask).sum().item(),
           "fake_correct": ((D_fake < 0.5).float() * mask).sum().item()}
    loss_real, loss_fake = gp.bce_real(D_real, mask, T), gp.bce_fake(D_fake, mask, T)
    loss_d = loss_real + loss_fake
    loss_d.backward()
    dg = [p.grad for p in d_params]
    out["d_grad_norm"] = float(gp.clip_grad_norm(dg, 1.0))
    if d_opt is not None:
        d_opt(d_params, dg)
    else:
        gp.adagrad_step(d_params, dg, d_sum, lr, weight_decay)
    with torch.no_grad():
        loss_mge = gp.masked_mse(y_hat_static, y_static, mask=mask)
        loss_mse = gp.masked_mse(y_hat, y, mask=mask)
    out.update(loss_d=loss_d.item(), loss_fake_d=loss_fake.item(), loss_real_d=loss_real.item(),
               loss_mse=loss_mse.item(), loss_mge=loss_mge.item(), loss_adv=0.0,
               loss_g=float(mse_w * loss_mse + mge_w * loss_mge), g_grad_norm=0.0, frames=T)
    return out, y_hat.detach(), y_hat_static.detach()


def spoof_count(ref_layers, y_hat_static, mask, hp):
    """``((D_ref(get_selected_static_stream(y_hat_static)) > 0.5).float() * mask).sum()`` (train.py:549-558)."""
    with torch.no_grad():
        return ((reference_output(ref_layers, y_hat_static, hp) > 0.5).float() * mask).sum().item()


def reference_output(ref_layers, y_hat_static, hp):
    """D_ref's output on the adversarial columns of y_hat_static, dropout off."""
    with torch.no_grad():
        return gp.mlp_forward(gp.get_selected_static_stream(y_hat_static, hp), ref_layers, last_sigmoid=True)
