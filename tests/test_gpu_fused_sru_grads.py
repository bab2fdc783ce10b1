"""The fused GAN step's SRURNN generator gradients, tensor by tensor, against the oracle's autograd.

Phases 1 and 2 of the step leave the raw generator gradients (before clipping and the optimiser) in grad_buffer(0), in
model_g.parameters() order.  Each parameter's slice is compared with the gradient the oracle (GeneratorOracle("sru") in
gp.gan_step, fed the step's own dropout masks) deposits on it: the fake term of loss_d plus loss_g, as in the reference's
train loop.  A gradient norm or a first Adagrad step (about lr * sign(g) per weight) cannot see an error in one tensor
that is small next to the whole generator; this can: one layer's bias gradient (sru_bias_reduce_kernel), its split-K dW,
or the highway gradient one layer leaves for the one below.

The shapes have chunk tails (T = 9, 37: the scans run 8 steps per chunk) and B * columns = 5 * 32 = 160 threads, two
128-thread blocks, the last one partial.  The oracle's discriminator takes the product's weights after its step in phase
2, so that the adversarial term compares the generators alone (see fused_step_helpers.adv_loss_with).  The oracle is
fp32; the bar is the fused step's 2e-4.  The worst error over the 16 cases on an NVIDIA H100 80GB HBM3 (700 W) was 1.6e-5
(layer 1's bias gradient; y_hat 9.2e-6), a factor of 12 below it.
"""
import pytest
import torch

from conftest import WINDOWS, TTS_HP, rel_err
from fused_step_helpers import (d_masks, dev, generator_oracle, make_batch, npy, ragged_lengths,  # noqa: F401
                                sd_numpy, sru_masks, sru_models, step_hp)
from oracle import gantts_port as gp
from oracle import nnmnkwii_port as nnp

ACOUSTIC_HP = dict(TTS_HP, discriminator_linguistic_condition=True)
TOL = 2e-4


@pytest.mark.gpu
@pytest.mark.parametrize("mse_w", [0.0, 1.0])
@pytest.mark.parametrize("relu", [True, False])
@pytest.mark.parametrize("k0", [4, 3])
@pytest.mark.parametrize("T", [9, 37])
def test_fused_sru_generator_gradients_per_tensor(dev, T, k0, relu, mse_w):
    """3 bidirectional SRU layers of 16 (layer 0 with k = k0, the others k = 3), dropout 0.2 / rnn_dropout 0.2, D with
    dropout 0.5 conditioned on x.  mse_w = 0 takes the MLPG adjoint that writes the operand planes directly, 1 the fp32
    one."""
    from gantts_b200 import fused
    B, hidden, d_hidden, p_d = 5, 16, 32, 0.5
    nc = 2 * hidden
    in_dim = nc if k0 == 3 else 20
    mg, md = sru_models(400 + T + k0 + 2 * relu, in_dim, 187, 3, hidden, True, relu, 0.2, 0.2, d_hidden, 3, p_d, 58)
    assert [c.k for c in mg.gru.rnn_lst] == [k0, 3, 3] and B * nc == 160
    gen = generator_oracle(mg)
    d_layers = gp.discriminator_layers(sd_numpy(md))
    mg.to(dev).train(), md.to(dev).train()
    fs = fused.FusedGanStep(mg, md, step_hp(ACOUSTIC_HP), B, T, w_d=1.0, mse_w=mse_w, mge_w=1.0, weight_decay=0.0,
                            seed=70 + T)
    lens = ragged_lengths(B, T, 80 + T)
    x, y = make_batch(B, T, in_dim, 187, lens, 90 + T)
    xd, yd, ld = x.to(dev), y.to(dev), torch.LongTensor(lens).to(dev)
    fs.cfg.adv_w, fs._step, fs.cfg.opt_step = 1.0, 1, 1
    for ph in (1, 2):                                  # up to the generator's gradients; no clip, no optimiser step
        fs._call(ph, xd, yd, ld, 0.0, fs._seed)
    fs.last_seed = fs._seed
    gb = fs.grad_buffer(0).cpu()
    stepped_d = [q.detach().cpu() for q in md.parameters()]

    def d_take_product_step(params, grads):
        with torch.no_grad():
            for q, v in zip(params, stepped_d):
                q.copy_(v)
    seen = {}

    def g_record(params, grads):
        seen["grads"] = [g.clone() for g in grads]

    R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, T))
    gm, dm = sru_masks(fs, mg, B, dev), d_masks(fs, B * T, [d_hidden] * 3, p_d, dev)
    ref, yh_ref, _ = gp.gan_step(lambda: gen.forward(x, R, lens, ACOUSTIC_HP, masks=gm), gen.params(), None, d_layers,
                                 None, x, y, lens, R, ACOUSTIC_HP, w_d=1.0, mse_w=mse_w, mge_w=1.0, adv_w=1.0,
                                 dropout_d=p_d, training=True, weight_decay=0.0, d_masks=dm,
                                 d_opt=d_take_product_step, g_opt=g_record)
    # gan_step hands its optimiser the clipped gradients: undo clip_grad_norm's factor
    total = torch.tensor(ref["g_grad_norm"], dtype=torch.float32)
    coef = torch.clamp(1.0 / (total + 1e-6), max=1.0)
    want = {n: g / coef for n, g in zip(gen.named, seen["grads"])}

    errs = {"y_hat": rel_err(npy(fs.y_hat), yh_ref.numpy())}
    off = 0
    for n, q in mg.named_parameters():
        k = q.numel()
        errs[n] = rel_err(gb[off:off + k].view(q.shape).numpy(), want[n].numpy())
        off += k
    assert off == gb.numel() and len(errs) == 1 + 2 * 4
    print("\nT %d k0 %d %s mse_w %g: " % (T, k0, "relu" if relu else "tanh", mse_w)
          + " ".join("%s %.2e" % kv for kv in errs.items()))
    assert max(errs.values()) < TOL, errs
