"""The fused GAN step's raw gradients, tensor by tensor, against the float64 oracle's autograd, for every generator and
discriminator it trains.

A loss, a global gradient norm or a first Adagrad step (about lr * sign(g) per weight) cannot see an error in one tensor:
a gradient off by a constant factor moves every weight by the same lr * sign(g), a flipped sign moves it by 2 lr, which
is within the weight check's 0.0201, and the norm only sees a tensor that carries a real share of it.  A bias vector, a
gate, one layer's split-K dW or one half of the stacked real|fake pass does not.  So each test runs the step phase by
phase (fused_step_helpers.split_step):

* after phase 1 grad_buffer(1) holds D's raw gradients (the real and fake BCE terms of loss_d);
* after phase 2 grad_buffer(0) holds G's raw gradients (the fake term of loss_d plus loss_g, as the reference's train loop
  accumulates them before clip_grad_norm);

and compares each parameter's slice of the flat buffer, in parameters() order, with the gradient the oracle's gan_step
deposits on that parameter in float64: every parameter, input and R in float64, the step's own dropout masks injected,
clip_grad_norm's coefficient undone with the oracle's own norms.  The oracle's discriminator takes the product's weights
after its step, so that the adversarial term compares the generators alone (see fused_step_helpers.adv_loss_with).  The
slices must tile the buffer exactly.  Every error is printed (-s).

The bar is the fused step's 2e-4 of the tensor's largest element, for every tensor, y_hat and y_hat_static, with two
exceptions:

* The bias of D's single output unit (last_linear.bias / hidden2out.bias) is a sum over the frames whose real and fake
  terms nearly cancel, so its own value is no measure of its rounding (fp32 summation left it 4.6e-4 of its value on
  one In2OutRNNHighwayNet case).  Its error is taken relative to the sum of the absolute values of those per-frame
  terms (output_bias_terms), computed in float64.
* At the two production sizes (cfg2, cfg1) the LeakyReLU hidden layers' tensors (KINKED) have their own bar, KINK_TOL.
  The product's bf16x3 GEMMs carry about 16 significant bits per operand, so a few of the millions of
  pre-activations land on the other side of the kink than in float64 (test_leaky_kink_flip_count_is_bounded), and
  each such element swaps a derivative 1 <-> 0.01 for one frame.  At 4 x 200 frames that one frame is a large share of
  a weight gradient: the float64 oracle itself, with its weights rounded to a bf16 hi + lo pair, moves these tensors
  by up to 5.6e-2 at cfg1 and leaves the gate and the output layers within 4e-6.  Every tensor not below a kink keeps
  2e-4 at these sizes, and every case at the small sizes keeps 2e-4 for all its tensors.

The MLP-discriminator cases put the full-length utterance last (batch(longest_last=True)), so that the last rows of each
half of the stacked real | fake pass, the tails of the backward's row tiles, are valid frames and not padding.

On an NVIDIA H100 80GB HBM3 at its 700 W power limit, the worst error of any tensor held to 2e-4, over the 40 cases,
was 1.9e-5 (the GRURNN discriminator's gru.weight_hh_l1, a factor of 10 below the bar); D's output bias stayed within
2.8e-7 of its per-frame terms; the worst of the kinked tensors was 4.4e-2 at cfg1 (G's H.2.weight; bar 1.5e-1) and
2.2e-3 at cfg2 (G's layers.2.weight; bar 1e-2).  The module takes about 30 s of wall time there, 7.6 s of it the cfg2
case's float64 reference at B = 32.

Each of these changes to the library, one at a time, fails this module and passes the older fused-step modules
(test_gpu_fused_highway, _rnn_highway, _sru, _rnn_d, test_gpu_step_streams, _real_half, test_gpu_dwarmup_spoof,
test_gpu_opt_per_model) except where noted:

* D's first hidden-layer bias gradient scaled by 1.001: 28 of the 40 cases fail;
* the real half's last partial 64-row tile dropped from D's first-layer weight-gradient launch: 11 cases fail (and
  test_gpu_step_real_half's oracle comparison, 5 tests of test_gpu_dwarmup_spoof, 2 of test_gpu_opt_per_model);
* the highway gate's T.bias gradient scaled by 1.001: 5 cases fail (and 1 of 9 of test_gpu_fused_highway);
* bias_hh of the LSTM discriminator's first reverse direction scaled by 1.001: 6 cases fail.

test_gpu_fused_ragged, run under the first two only, passes the first and fails its ragged-epoch test under the second.
"""
import re
import time

import numpy as np
import pytest
import torch

from conftest import WINDOWS, rel_err
from fused_step_helpers import (build, d_lstm_masks, d_masks, dev, g_masks, generator_oracle, make_batch,  # noqa: F401
                                make_models, npy, ragged_lengths, rhw_models, sd_numpy, split_step, sru_models, step_hp,
                                tts_ohp)
from oracle import gantts_port as gp
from oracle import nnmnkwii_port as nnp

TOL = 2e-4
# A delta window two frames wide takes the FIR and combine MLPG kernels; the reference's windows the substitution ones.
FIR_WINDOWS = [WINDOWS[0], (2, 2, np.array([-0.2, -0.1, 0.0, 0.1, 0.2])), WINDOWS[2]]
# the weight and bias gradients of a LeakyReLU hidden layer (MLP "layers.i", In2OutHighwayNet "H.i"; not last_linear)
KINKED = re.compile(r"^[DG] (layers|H)\.\d+\.")
KINK_TOL = {"cfg2": 1e-2, "cfg1": 1.5e-1}
WORST = {"strict": (0.0, None), "kinked": (0.0, None)}


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    if WORST["strict"][1] is not None:
        print("\nworst error on %s: %.2e (%s); of the kinked tensors at production size %.2e (%s)"
              % ((torch.cuda.get_device_name(0),) + WORST["strict"] + WORST["kinked"]))


def _kind(mg):
    return {"MLP": "mlp", "In2OutHighwayNet": "highway", "In2OutRNNHighwayNet": "rnn_highway",
            "SRURNN": "sru"}[type(mg).__name__]


def _widths(layers):
    return [int(l.weight.shape[0]) for l in layers]


def step_masks(fs, mg, md, b, t, dev):
    """The generator's and the discriminator's keep masks of the step's last call, of shape (b, t)."""
    kind = _kind(mg)
    g_hidden = _widths(mg.layers if kind == "mlp" else mg.H) if kind in ("mlp", "highway") else None
    gm = g_masks(kind, fs, mg, b, t, g_hidden, dev)
    if hasattr(md, "last_linear"):
        return gm, d_masks(fs, b * t, _widths(md.layers), md.dropout_p, dev)
    return gm, d_lstm_masks(fs, md, b * t, dev)


def per_tensor(tag, buf, model, want, scales=None):
    """The error of each parameter's slice of the flat gradient buffer `buf` against want[name]: rel_err, or for the
    tensors named in `scales` max |delta| / scales[name]."""
    errs, off = {}, 0
    for n, q in model.named_parameters():
        k = q.numel()
        got, ref = buf[off:off + k].view(q.shape).numpy().astype(np.float64), want[n].numpy()
        if scales and n in scales:
            errs["%s %s" % (tag, n)] = float(np.abs(got - ref).max() / scales[n])
        else:
            errs["%s %s" % (tag, n)] = rel_err(got, ref)
        off += k
    assert off == buf.numel() and len(errs) == len(want), (tag, off, buf.numel(), sorted(want))
    return errs


def output_bias_terms(d_sd, x, y, ys, lens, ohp, dm):
    """sum |dL/dz| over the frames of D's output unit in the stacked real | fake pass, divided by the frames: the sum of
    the absolute values of the per-frame terms whose sum is the output bias's gradient (real frames (D - 1) / T, fake
    frames D / T), in float64, from D's weights before its step.  The real and fake terms nearly cancel, so this, not the
    bias gradient itself, is the scale of its rounding."""
    d = gp.DiscriminatorOracle(d_sd, torch.float64)
    y_static = gp.get_static_features(y, ohp["num_windows"], ohp["stream_sizes"], ohp["has_dynamic_features"])
    real_in, fake_in = (gp.get_selected_static_stream(v, ohp) for v in (y_static, ys))
    if ohp["discriminator_linguistic_condition"]:
        real_in, fake_in = torch.cat((x, real_in), -1), torch.cat((x, fake_in), -1)
    mask = gp.sequence_mask(lens, x.size(1)).unsqueeze(-1).double()
    with torch.no_grad():
        d_real, d_fake = d.forward(real_in, lens, dm["real"]), d.forward(fake_in, lens, dm["fake"])
        return float((((1 - d_real).abs() + d_fake.abs()) * mask).sum() / mask.sum())


def unclipped(oracle, grads, norm, scale):
    """{name: raw gradient} of the gradients gan_step handed its optimiser, clip_grad_norm's coefficient undone."""
    coef = min(1.0 / (norm + 1e-6), 1.0)
    return {n: g * (scale / coef) for n, g in zip(oracle.named, grads)}


def step_vs_f64(fs, mg, md, ohp, x, y, lens, dev, tag, update_g=True, frames=None, kink_tol=None):
    """One training step of `fs` on the host batch (x, y, lens) against the float64 oracle; asserts and returns the
    errors.  update_g=False is the D-only warm-up step (only D's tensors are compared).  frames: the normaliser the
    caller passes, as one rank of several does; each raw gradient is then the reference's times sum(lens) / frames.
    kink_tol: the bar of the LeakyReLU hidden layers' tensors (KINKED) at production sizes; every other tensor keeps
    TOL."""
    b, t = int(x.shape[0]), int(x.shape[1])
    gen = generator_oracle(mg, torch.float64)
    d_sd = sd_numpy(md)
    d = gp.DiscriminatorOracle(d_sd, torch.float64)
    raw = {}

    def snapshot(ph):
        raw[ph] = fs.grad_buffer(1 if ph == 1 else 0).cpu()
    split_step(fs, x.to(dev), y.to(dev), torch.LongTensor(lens).to(dev), update_g=update_g, phases=(1, 2, 4),
               between=snapshot, frames=frames)
    stepped_d = {n: q.detach().cpu().double() for n, q in md.named_parameters()}
    seen = {}

    def d_take_product_step(params, grads):
        seen["d"] = [g.clone() for g in grads]
        with torch.no_grad():
            for n, q in zip(d.named, params):
                q.copy_(stepped_d[n])

    def g_record(params, grads):
        seen["g"] = [g.clone() for g in grads]

    R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(fs.hp.windows, t, np.float64))
    gm, dm = step_masks(fs, mg, md, b, t, dev)
    x64, y64 = x.double(), y.double()
    ref, yh_ref, ys_ref = gp.gan_step(lambda: gen.forward(x64, R, lens, ohp, masks=gm), gen.params(), None, d, None,
                                      x64, y64, lens, R, ohp, w_d=1.0, mse_w=fs.cfg.mse_w, mge_w=1.0, adv_w=1.0,
                                      training=True, weight_decay=0.0, update_g=update_g, d_masks=dm,
                                      d_opt=d_take_product_step, g_opt=g_record)
    scale = 1.0 if frames is None else sum(lens) / float(frames)
    errs = {"y_hat_static": rel_err(npy(fs.y_hat_static), ys_ref.numpy())}
    if _kind(mg) != "rnn_highway":                     # In2OutRNNHighwayNet's first output is its input (models.py:118)
        errs["y_hat"] = rel_err(npy(fs.y_hat), yh_ref.numpy())
    out_bias = [n for n, q in md.named_parameters() if q.numel() == 1]
    assert out_bias == [n for n, _ in md.named_parameters()][-1:], out_bias
    bias_scale = scale * output_bias_terms(d_sd, x64, y64, ys_ref, lens, ohp, dm)
    errs.update(per_tensor("D", raw[1], md, unclipped(d, seen["d"], ref["d_grad_norm"], scale),
                           {out_bias[0]: bias_scale}))
    if update_g:
        errs.update(per_tensor("G", raw[2], mg, unclipped(gen, seen["g"], ref["g_grad_norm"], scale)))
    print("\n%s (%d x %d): " % (tag, b, t) + " ".join("%s %.2e" % kv for kv in errs.items()))
    bars = {n: kink_tol if kink_tol is not None and KINKED.match(n) else TOL for n in errs}
    for n, e in errs.items():
        key = "kinked" if bars[n] != TOL else "strict"
        if e > WORST[key][0]:
            WORST[key] = (e, "%s, %s" % (tag, n))
    bad = {n: e for n, e in errs.items() if not e < bars[n]}
    assert not bad, (tag, bad)
    return errs


def new_step(mg, md, ohp, B, T, dev, mse_w=0.0, seed=0, windows=None):
    from gantts_b200 import fused
    hp = step_hp(ohp)
    if windows is not None:
        hp["windows"] = windows
    mg.to(dev).train(), md.to(dev).train()
    return fused.FusedGanStep(mg, md, hp, B, T, w_d=1.0, mse_w=mse_w, mge_w=1.0, weight_decay=0.0, seed=seed)


def batch(B, T, d_in, d_out, seed, full=False, positive=False, longest_last=False):
    """(x, y, lengths) of B utterances padded to T: the first one full length (the last one with longest_last, so that
    the last rows of each half of the stacked discriminator pass, the tails of its row tiles, are valid frames; the
    recurrent oracles pack sequences and need the lengths in descending order)."""
    lens = [T] * B if full else ragged_lengths(B, T, seed)
    if longest_last:
        lens = lens[::-1]
    x, y = make_batch(B, T, d_in, d_out, lens, seed + 1)
    return (x.abs() if positive else x), y, lens


def tts_mlp_models(seed, cond, d_in=20, g_hidden=32, g_layers=2, d_hidden=16, d_layers=2, p=0.5):
    """MLP G d_in -> g_hidden x g_layers -> 187 and MLP D (58 adversarial columns, + d_in when conditioned on x) ->
    d_hidden x d_layers -> 1, both with dropout p, on the TTS layout (mask_nth_mgc_for_adv_loss = 2)."""
    import gantts_b200
    M = gantts_b200.models
    torch.manual_seed(seed)
    mg = M.MLP(d_in, 187, g_layers, g_hidden, dropout=p, last_sigmoid=False)
    md = M.MLP(58 + (d_in if cond else 0), 1, d_layers, d_hidden, dropout=p, last_sigmoid=True)
    return mg, md, tts_ohp(cond)


@pytest.mark.gpu
@pytest.mark.parametrize("mse_w", [0.0, 1.0])
@pytest.mark.parametrize("cond", [False, True])
def test_mlp_generator_gradients_per_tensor(dev, cond, mse_w):
    """MLP G 20-32-32-187 and MLP D 58-16-16-1 (78 inputs conditioned on x), dropout 0.5.  mse_w = 0 takes the MLPG
    adjoint that writes the operand planes directly, 1 the fp32 one."""
    mg, md, ohp = tts_mlp_models(100 + 2 * cond + int(mse_w), cond)
    fs = new_step(mg, md, ohp, 3, 45, dev, mse_w=mse_w, seed=11)
    x, y, lens = batch(3, 45, 20, 187, 12 + cond, positive=True, longest_last=True)
    step_vs_f64(fs, mg, md, ohp, x, y, lens, dev, "mlp cond %d mse_w %g" % (cond, mse_w))


@pytest.mark.gpu
def test_shaped_calls_gradients_per_tensor(dev):
    """A step at the configured (3, 337), then steps of (1, 5) and (2, 129) on the same FusedGanStep: row counts off every
    GEMM-tile and GEMV row-block boundary, with valid frames in each half's last rows, after a larger call has filled the
    workspace."""
    mg, md, ohp = tts_mlp_models(110, True)
    fs = new_step(mg, md, ohp, 3, 337, dev, mse_w=1.0, seed=13)
    for i, (b, t) in enumerate([(3, 337), (1, 5), (2, 129)]):
        x, y, lens = batch(b, t, 20, 187, 30 + i, positive=True, longest_last=True)
        step_vs_f64(fs, mg, md, ohp, x, y, lens, dev, "shaped call %d" % i)


@pytest.mark.gpu
def test_cfg2_gradients_per_tensor(dev):
    """The bench's cfg2: MLP G 425-512-512-512-187 and MLP D 58-256-256-256-1, dropout 0.5, full-length utterances of
    T = 1000: the side-stream weight-gradient branch and the split-K plans at production size."""
    B, T = 32, 1000
    mg, md, ohp = tts_mlp_models(120, False, d_in=425, g_hidden=512, g_layers=3, d_hidden=256, d_layers=3)
    fs = new_step(mg, md, ohp, B, T, dev, seed=15)
    x, y, lens = batch(B, T, 425, 187, 40, full=True)
    x.uniform_()
    t0 = time.time()
    step_vs_f64(fs, mg, md, ohp, x, y, lens, dev, "cfg2", kink_tol=KINK_TOL["cfg2"])
    print("cfg2 (B = %d): %.1f s with the float64 reference" % (B, time.time() - t0))


def vc_highway_models(seed, S, hidden, layers, d_hidden, d_layers, p=0.5):
    import gantts_b200
    M = gantts_b200.models
    torch.manual_seed(seed)
    mg = M.In2OutHighwayNet(in_dim=3 * S, out_dim=3 * S, static_dim=S, num_hidden=layers, hidden_dim=hidden, dropout=p)
    md = M.MLP(S, 1, d_layers, d_hidden, dropout=p, last_sigmoid=True)
    ohp = dict(stream_sizes=[3 * S], has_dynamic_features=[True], adversarial_streams=[True],
               mask_nth_mgc_for_adv_loss=0, num_windows=3, discriminator_linguistic_condition=False)
    return mg, md, ohp


@pytest.mark.gpu
@pytest.mark.parametrize("family", ["substitution", "fir"])
def test_highway_generator_gradients_per_tensor(dev, family):
    """In2OutHighwayNet 27-24-24-27 (S = 9), MLP D 9-16-16-1, dropout 0.5, with the reference's windows (the
    substitution MLPG kernels) and a 5-tap delta window (the FIR and combine kernels).  The gate's T.weight / T.bias come
    first in the buffer."""
    mg, md, ohp = vc_highway_models(130 + (family == "fir"), 9, 24, 2, 16, 2)
    assert [n for n, _ in mg.named_parameters()][:2] == ["T.weight", "T.bias"]
    fs = new_step(mg, md, ohp, 4, 41, dev, mse_w=1.0, seed=17, windows=FIR_WINDOWS if family == "fir" else None)
    x, y, lens = batch(4, 41, 27, 27, 50, longest_last=True)
    step_vs_f64(fs, mg, md, ohp, x, y, lens, dev, "highway " + family)


@pytest.mark.gpu
def test_highway_generator_cfg1_size_gradients_per_tensor(dev):
    """In2OutHighwayNet 177-512x3-177 (S = 59) and MLP D 59-256-256-1, dropout 0.5, at 4 x 200."""
    mg, md, ohp = vc_highway_models(140, 59, 512, 3, 256, 2)
    fs = new_step(mg, md, ohp, 4, 200, dev, seed=19)
    x, y, lens = batch(4, 200, 177, 177, 60, longest_last=True)
    step_vs_f64(fs, mg, md, ohp, x, y, lens, dev, "highway cfg1", kink_tol=KINK_TOL["cfg1"])


@pytest.mark.gpu
@pytest.mark.parametrize("T", [9, 37])
def test_rnn_highway_generator_gradients_per_tensor(dev, T):
    """In2OutRNNHighwayNet 24 -> 2 bidirectional LSTM layers of 12, dropout 0.3 -> 24 (S = 8), MLP D 8-32-32-1."""
    mg, md = rhw_models(150 + T, 8, 2, 12, True, 0.3, 32, 2, 0.5)
    ohp = dict(stream_sizes=[24], has_dynamic_features=[True], adversarial_streams=[True],
               mask_nth_mgc_for_adv_loss=0, num_windows=3, discriminator_linguistic_condition=False)
    fs = new_step(mg, md, ohp, 5, T, dev, seed=21)
    x, y, lens = batch(5, T, 24, 24, 70 + T)
    step_vs_f64(fs, mg, md, ohp, x, y, lens, dev, "rnn_highway T %d" % T)


@pytest.mark.gpu
@pytest.mark.parametrize("mse_w", [0.0, 1.0])
@pytest.mark.parametrize("relu", [True, False])
@pytest.mark.parametrize("k0", [4, 3])
@pytest.mark.parametrize("T", [9, 37])
def test_fused_sru_generator_gradients_per_tensor(dev, T, k0, relu, mse_w):
    """3 bidirectional SRU layers of 16 (layer 0 with k = k0, the others k = 3), dropout 0.2 / rnn_dropout 0.2, D
    32-32-32 with dropout 0.5 conditioned on x.  T = 9 and 37 leave chunk tails (the scans run 8 steps per chunk), and
    B * columns = 5 * 32 = 160 threads are two 128-thread blocks, the last one partial."""
    B, hidden, d_hidden, p_d = 5, 16, 32, 0.5
    nc = 2 * hidden
    in_dim = nc if k0 == 3 else 20
    mg, md = sru_models(400 + T + k0 + 2 * relu, in_dim, 187, 3, hidden, True, relu, 0.2, 0.2, d_hidden, 3, p_d, 58)
    assert [c.k for c in mg.gru.rnn_lst] == [k0, 3, 3] and B * nc == 160
    ohp = tts_ohp(True)
    fs = new_step(mg, md, ohp, B, T, dev, mse_w=mse_w, seed=70 + T)
    lens = ragged_lengths(B, T, 80 + T)
    x, y = make_batch(B, T, in_dim, 187, lens, 90 + T)
    step_vs_f64(fs, mg, md, ohp, x, y, lens, dev, "sru T %d k0 %d %s mse_w %g" % (T, k0, "relu" if relu else "tanh",
                                                                               mse_w))


@pytest.mark.gpu
@pytest.mark.parametrize("cond", [False, True])
@pytest.mark.parametrize("bidir", [False, True])
@pytest.mark.parametrize("gru", [False, True])
def test_recurrent_discriminator_gradients_per_tensor(dev, gru, bidir, cond):
    """MLP G 20-24-24-187 and an LSTMRNN (GRURNN: the same nn.LSTM under .gru) D of 2 layers of 12, LSTM dropout 0.5:
    every weight_ih / weight_hh / bias_ih / bias_hh slot (and its _reverse) and hidden2out."""
    mg, md, ohp, d_in = make_models("mlp", 160 + 4 * gru + 2 * bidir + cond, cond, d_layers=2, d_hidden=12,
                                    bidir=bidir, p_d=0.5, gru=gru)
    fs = new_step(mg, md, ohp, 3, 40, dev, seed=23)
    x, y, lens = batch(3, 40, d_in, 187, 80, positive=True)
    step_vs_f64(fs, mg, md, ohp, x, y, lens, dev, "%s D bidir %d cond %d" % ("GRURNN" if gru else "LSTMRNN", bidir,
                                                                              cond))


@pytest.mark.gpu
@pytest.mark.parametrize("d_kind", ["mlp", "lstm"])
@pytest.mark.parametrize("g_kind", ["mlp", "highway"])
def test_d_only_step_gradients_per_tensor(dev, g_kind, d_kind):
    """The D-only warm-up step (GANTTS_STEP_D_ONLY): D's tensors against gan_step(..., update_g=False)."""
    if d_kind == "mlp":
        mg, md, ohp = (tts_mlp_models(170, False) if g_kind == "mlp" else vc_highway_models(171, 9, 24, 2, 16, 2))
        d_in = 20 if g_kind == "mlp" else 27
    else:
        mg, md, ohp, d_in = make_models(g_kind, 172, False, d_layers=2, d_hidden=12, bidir=True, p_d=0.5)
    d_out = 187 if g_kind == "mlp" else d_in
    fs = new_step(mg, md, ohp, 3, 40, dev, mse_w=0.5, seed=25)
    x, y, lens = batch(3, 40, d_in, d_out, 90, positive=g_kind == "mlp")
    g0 = [q.detach().clone() for q in mg.parameters()]
    step_vs_f64(fs, mg, md, ohp, x, y, lens, dev, "D-only %s G %s D" % (g_kind, d_kind), update_g=False)
    assert all(torch.equal(a, q) for a, q in zip(g0, mg.parameters()))


@pytest.mark.gpu
def test_caller_frames_gradients_per_tensor(dev):
    """frames given by the caller as twice the local count, as one rank of two passes it: every raw gradient is the
    reference's at that normaliser, half of the single-process one."""
    mg, md, ohp = tts_mlp_models(180, True)
    fs = new_step(mg, md, ohp, 3, 45, dev, mse_w=1.0, seed=27)
    x, y, lens = batch(3, 45, 20, 187, 100, positive=True, longest_last=True)
    step_vs_f64(fs, mg, md, ohp, x, y, lens, dev, "frames 2 x local", frames=2 * sum(lens))
