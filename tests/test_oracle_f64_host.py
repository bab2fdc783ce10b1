"""The oracle in float64, the reference the fused step's per-tensor gradient tests compare against (CPU only).

GeneratorOracle / DiscriminatorOracle / discriminator_layers take dtype=torch.float64 and unit_variance_mlpg_matrix
dtype=np.float64; the defaults stay float32 and give the bits test_oracle_golden.py pins.  For every generator kind
(MLP, In2OutHighwayNet, In2OutRNNHighwayNet, SRURNN) and every discriminator kind (MLP, LSTMRNN and GRURNN, uni- and
bidirectional), on tiny ragged batches with dropout masks injected:

* torch.autograd.gradcheck passes on the float64 forwards;
* the gradients gan_step hands its optimisers (clip_grad_norm undone) are the derivatives of the losses it reports: D's of
  loss_d, G's of loss_d + loss_g, by central differences along a random direction;
* the float64 oracle agrees with the float32 one to fp32 rounding: losses, y_hat_static and every gradient (to the
  rounding of its model's whole gradient).
"""
import numpy as np
import pytest
import torch

from conftest import WINDOWS, rel_err
from fused_step_helpers import build, generator_oracle, make_models, sd_numpy
from oracle import gantts_port as gp
from oracle import nnmnkwii_port as nnp

B, T = 3, 7
GENERATORS = ["mlp", "highway", "rnn_highway", "sru"]
DISCRIMINATORS = [  # (class, bidirectional, conditioned on x)
    ("MLP", False, False), ("LSTMRNN", False, True), ("LSTMRNN", True, False), ("GRURNN", False, False),
    ("GRURNN", True, True)]
F32_TOL = 1e-5


def keep(rows, cols, p, g):
    """A dropout multiplier {0, 1/(1-p)} as the product draws them (float32)."""
    return (torch.rand(rows, cols, generator=g) >= p).float() / (1.0 - p)


def models(g_kind, d_spec):
    """(model_g, model_d, oracle hparams, d_in, d_out) on the host."""
    d_cls, bidir, cond = d_spec
    seed = 300 + GENERATORS.index(g_kind) * 10 + DISCRIMINATORS.index(d_spec)
    if d_cls == "MLP":
        mg, md, ohp, d_in, d_out, _, _, _ = build(g_kind, seed)
        return mg, md, ohp, d_in, d_out
    mg, md, ohp, d_in = make_models(g_kind, seed, cond, d_layers=2, d_hidden=8, bidir=bidir, p_d=0.5,
                                    gru=d_cls == "GRURNN")
    return mg, md, ohp, d_in, 187 if g_kind in ("mlp", "sru") else d_in


def masks(g_kind, mg, md, seed):
    """Keep masks for the generator and for the three discriminator forwards (real, fake, adv) of a (B, T) batch."""
    g = torch.Generator().manual_seed(seed)
    M = B * T
    if g_kind in ("mlp", "highway"):
        gm = [keep(M, l.weight.shape[0], 0.5, g) for l in (mg.layers if g_kind == "mlp" else mg.H)]
    elif g_kind == "rnn_highway":
        lm = mg.lstm
        gm = [keep(M, 2 * lm.hidden_size, 0.3, g) for _ in range(lm.num_layers - 1)]
    else:
        cells = list(mg.gru.rnn_lst)
        gm = [(keep(B, c.n_in, 0.2, g), keep(B, 2 * c.n_out, 0.2, g) if i + 1 < len(cells) else None)
              for i, c in enumerate(cells)]
    if hasattr(md, "last_linear"):
        widths = [l.weight.shape[0] for l in md.layers]
        dm = {k: [keep(M, w, 0.5, g) for w in widths] for k in ("real", "fake", "adv")}
    else:
        lstm = getattr(md, md._rnn_attr)
        nh = lstm.hidden_size * (2 if lstm.bidirectional else 1)
        dm = {k: [keep(M, nh, 0.5, g) for _ in range(lstm.num_layers - 1)] for k in ("real", "fake", "adv")}
    return gm, dm


def setup(g_kind, d_spec, dtype):
    mg, md, ohp, d_in, d_out = models(g_kind, d_spec)
    lens = [T, 5, 4]
    g = torch.Generator().manual_seed(7)
    x, y = torch.randn(B, T, d_in, generator=g), torch.randn(B, T, d_out, generator=g)
    for b, n in enumerate(lens):
        x[b, n:] = 0
        y[b, n:] = 0
    npdt = np.float64 if dtype == torch.float64 else np.float32
    R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, T, npdt))
    gen = generator_oracle(mg, dtype)
    d = gp.DiscriminatorOracle(sd_numpy(md), dtype)
    gm, dm = masks(g_kind, mg, md, 11)
    return gen, d, ohp, x.to(dtype), y.to(dtype), lens, R, gm, dm


def gan_step_grads(gen, d, ohp, x, y, lens, R, gm, dm):
    """(losses, y_hat_static, D's raw gradients, G's raw gradients) of one gan_step that leaves both models unstepped."""
    seen = {}
    out, _, ys = gp.gan_step(lambda: gen.forward(x, R, lens, ohp, masks=gm), gen.params(), None, d, None, x, y, lens, R,
                             ohp, mse_w=0.5, weight_decay=0.0, d_masks=dm,
                             d_opt=lambda p, g: seen.__setitem__("d", [v.clone() for v in g]),
                             g_opt=lambda p, g: seen.__setitem__("g", [v.clone() for v in g]))
    unclip = lambda grads, norm: [v / min(1.0 / (norm + 1e-6), 1.0) for v in grads]
    return out, ys, unclip(seen["d"], out["d_grad_norm"]), unclip(seen["g"], out["g_grad_norm"])


def reported_losses(gen, d, ohp, x, y, lens, R, gm, dm):
    """(loss_d, loss_d + loss_g) gan_step reports without updating anything."""
    with torch.no_grad():
        out, _, _ = gp.gan_step(lambda: gen.forward(x, R, lens, ohp, masks=gm), gen.params(), None, d, None, x, y,
                                lens, R, ohp, mse_w=0.5, update=False, d_masks=dm)
    return out["loss_d"], out["loss_d"] + out["loss_g"]


CASES = [(g, d) for g in GENERATORS for d in DISCRIMINATORS]
IDS = ["%s-%s%s%s" % (g, d[0], "-bi" if d[1] else "", "-cond" if d[2] else "") for g, d in CASES]


def test_mlpg_matrix_dtypes():
    """The float64 R is the matrix the float32 one is rounded from; the default stays float32."""
    r32, r64 = nnp.unit_variance_mlpg_matrix(WINDOWS, 11), nnp.unit_variance_mlpg_matrix(WINDOWS, 11, np.float64)
    assert r32.dtype == np.float32 and r64.dtype == np.float64
    assert np.array_equal(r64.astype(np.float32), r32)


@pytest.mark.parametrize("g_kind,d_spec", CASES, ids=IDS)
def test_f64_forwards_pass_gradcheck(g_kind, d_spec):
    """gradcheck of the generator's outputs with respect to its parameters, and of D's output with respect to its
    parameters and its input.  gradcheck perturbs its (dense) inputs in place, so the closures read the oracles' own
    parameter tensors."""
    gen, d, ohp, x, y, lens, R, gm, dm = setup(g_kind, d_spec, torch.float64)
    assert all(p.dtype == torch.float64 for p in gen.params() + d.params())

    def g_out(*params):
        y_hat, y_hat_static = gen.forward(x, R, lens, ohp, masks=gm)
        return (y_hat_static,) if g_kind == "rnn_highway" else (y_hat, y_hat_static)
    assert torch.autograd.gradcheck(g_out, tuple(gen.params()), fast_mode=True)
    n_in = d.params()[0].shape[1]
    d_in = torch.rand(B, T, n_in, dtype=torch.float64, generator=torch.Generator().manual_seed(5)).requires_grad_(True)
    assert torch.autograd.gradcheck(lambda v, *params: d.forward(v, lens, dm["real"]), (d_in,) + tuple(d.params()),
                                    fast_mode=True)


@pytest.mark.parametrize("g_kind,d_spec", CASES, ids=IDS)
def test_gan_step_gradients_are_the_derivatives_of_its_losses(g_kind, d_spec):
    """D's gradients are d loss_d / d theta_D and G's d (loss_d + loss_g) / d theta_G (train.py accumulates the fake term
    of loss_d on G before its step): central differences of the losses gan_step reports along a random direction."""
    gen, d, ohp, x, y, lens, R, gm, dm = setup(g_kind, d_spec, torch.float64)
    args = (gen, d, ohp, x, y, lens, R, gm, dm)
    _, _, gd, gg = gan_step_grads(*args)
    eps = 1e-6
    g = torch.Generator().manual_seed(3)
    for which, params, grads in ((0, d.params(), gd), (1, gen.params(), gg)):
        v = [torch.randn(p.shape, dtype=p.dtype, generator=g) for p in params]
        analytic = sum(float((a * b).sum()) for a, b in zip(grads, v))
        ends = []
        for sign in (1.0, -1.0):
            with torch.no_grad():
                for p, u in zip(params, v):
                    p.add_(u, alpha=sign * eps)
            ends.append(reported_losses(*args)[which])
            with torch.no_grad():
                for p, u in zip(params, v):
                    p.sub_(u, alpha=sign * eps)
        numeric = (ends[0] - ends[1]) / (2 * eps)
        assert abs(numeric - analytic) <= 1e-5 * max(abs(analytic), 1e-3), ("DG"[which], numeric, analytic)


@pytest.mark.parametrize("g_kind,d_spec", CASES, ids=IDS)
def test_f64_oracle_agrees_with_f32(g_kind, d_spec):
    """The same gan_step in float64 and float32: losses, y_hat_static and every raw gradient to fp32 rounding."""
    o64, ys64, d64, g64 = gan_step_grads(*setup(g_kind, d_spec, torch.float64))
    o32, ys32, d32, g32 = gan_step_grads(*setup(g_kind, d_spec, torch.float32))
    assert ys64.dtype == torch.float64 and ys32.dtype == torch.float32
    for k in ("loss_d", "loss_mse", "loss_mge", "loss_adv", "loss_g", "d_grad_norm", "g_grad_norm"):
        assert abs(o64[k] - o32[k]) <= F32_TOL * abs(o64[k]), (k, o64[k], o32[k])
    assert rel_err(ys32.numpy(), ys64.numpy()) < F32_TOL
    # each tensor to fp32 rounding of its model's gradient: a bias of the output unit is a sum over the frames whose
    # terms nearly cancel, so its own magnitude is no measure of the rounding in it
    for tag, a, b in (("D", d64, d32), ("G", g64, g32)):
        scale = max(float(u.abs().max()) for u in a)
        for i, (u, v) in enumerate(zip(a, b)):
            err = float((v.double() - u).abs().max()) / scale
            assert err < F32_TOL, (tag, i, err)
