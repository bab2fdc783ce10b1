"""Phase 1 of the fused GAN step runs the real half of the stacked discriminator pass (gather, forward, BCE terms and the
input-gradient chain of rows [0, M)) on the library's branch stream, beside the generator's forward, and the fake half on
the caller's stream; D's weight gradients read both halves after them.  These tests step twin models, one read on a
non-default caller stream straight after each call and one synchronised after every call, and compare them bit for bit:
losses, y_hat_static, parameters and optimiser state.  The shapes put M = B * T off every boundary of the split: (3, 337)
is not a multiple of a 128-row GEMM tile or of the GEMV tail's row blocks, (1, 5) is less than one tile.  A small step is
also checked against the oracle's restatement of train.py's step.
"""
import pytest
import torch

from conftest import TTS_HP, WINDOWS, rel_err
from fused_step_helpers import build, dev, fused, make_batch, npy, ragged_lengths, split_step, tts_ohp  # noqa: F401
from oracle import gantts_port as gp
from oracle import nnmnkwii_port as nnp
from test_gpu_step_streams import assert_same, record

B, T = 3, 337
# (b, t, update_g): the capacity, less than one GEMM tile, a D-only step, the capacity again
SEQUENCE = [(3, 337, True), (1, 5, True), (2, 129, False), (3, 337, True)]
KINDS = ["mlp", "mlp_cond", "highway"]


def models(kind, seed):
    """(model_g, model_d, oracle hparams, d_in, d_out) on the host: an MLP or In2OutHighwayNet generator, an MLP D."""
    import gantts_b200
    if kind == "mlp_cond":
        torch.manual_seed(seed)
        mg = gantts_b200.models.MLP(20, 187, 2, 32, dropout=0.5, last_sigmoid=False)
        md = gantts_b200.models.MLP(20 + 58, 1, 2, 16, dropout=0.5, last_sigmoid=True)
        return mg, md, tts_ohp(True), 20, 187
    mg, md, hp, d_in, d_out, _, _, _ = build(kind, seed)
    return mg, md, hp, d_in, d_out


def setup(kind, dev, seed=3):
    mg, md, hp, d_in, d_out = models(kind, seed)
    mg.to(dev), md.to(dev)
    fs = fused(mg, md, hp, B, T, seed=17)
    batches = []
    for i, (b, t, _) in enumerate(SEQUENCE):
        lens = ragged_lengths(b, t, 50 + i)
        x, y = make_batch(b, t, d_in, d_out, lens, 60 + i)
        batches.append((x.to(dev), y.to(dev), torch.LongTensor(lens).to(dev)))
    return fs, mg, md, batches


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_shaped_steps_complete_on_the_callers_stream(dev, kind):
    """Shaped training and D-only steps issued on a non-default stream and read on it with no synchronisation equal bit
    for bit the steps of a twin synchronised after every call."""
    fs, mg, md, batches = setup(kind, dev)
    caller = torch.cuda.Stream(device=dev)
    caller.wait_stream(torch.cuda.current_stream(dev))
    got = []
    with torch.cuda.stream(caller):
        for (x, y, lengths), (_, _, update_g) in zip(batches, SEQUENCE):
            fs.step(x, y, lengths, update_g=update_g)
            got.append(record(fs, mg, md))
    torch.cuda.synchronize()
    fs2, mg2, md2, batches2 = setup(kind, dev)
    for i, ((x, y, lengths), (_, _, update_g)) in enumerate(zip(batches2, SEQUENCE)):
        fs2.step(x, y, lengths, update_g=update_g)
        torch.cuda.synchronize()
        assert_same(got[i], record(fs2, mg2, md2), "%s step %d" % (kind, i))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_phase_split_shaped_steps_equal_one_call(dev, kind):
    """The same shaped steps, each split into the discriminator phase and then the generator and finishing phases,
    equal bit for bit the steps made as one call."""
    fs, mg, md, batches = setup(kind, dev)
    full = []
    for (x, y, lengths), (_, _, update_g) in zip(batches, SEQUENCE):
        fs.step(x, y, lengths, update_g=update_g)
        full.append(record(fs, mg, md))
    fs2, mg2, md2, batches2 = setup(kind, dev)
    for i, ((x, y, lengths), (_, _, update_g)) in enumerate(zip(batches2, SEQUENCE)):
        split_step(fs2, x, y, lengths, update_g=update_g)
        assert_same(full[i], record(fs2, mg2, md2), "%s step %d" % (kind, i))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_shaped_step_captured_in_a_graph(dev, kind):
    """A shaped training step captured in a CUDA graph and replayed computes bit for bit the same step made eagerly."""
    fs, mg, md, batches = setup(kind, dev)
    fs.step(*batches[0])
    torch.cuda.synchronize()
    fs2, mg2, md2, batches2 = setup(kind, dev)
    fs2.step(*batches2[0])
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fs2.step(*batches2[1])
    graph.replay()
    torch.cuda.synchronize()
    fs.step(*batches[1])
    torch.cuda.synchronize()
    assert_same(record(fs, mg, md), record(fs2, mg2, md2), "%s graph replay" % kind)


@pytest.mark.gpu
def test_small_step_matches_the_oracle(dev):
    """One step of a small dropout-free MLP pair with a ragged batch of M = 3 * 37 rows against the oracle's restatement
    of train.py's step: losses, y_hat, y_hat_static."""
    import gantts_b200
    from gantts_b200 import step as gstep
    from gantts_b200 import fused as F
    torch.manual_seed(4)
    mg = gantts_b200.models.MLP(20, 187, 2, 32, dropout=0.0, last_sigmoid=False)
    md = gantts_b200.models.MLP(58, 1, 2, 16, dropout=0.0, last_sigmoid=True)
    names = ["layers.0", "layers.1", "last_linear"]
    layers = lambda m: [(m.state_dict()[n + ".weight"].clone(), m.state_dict()[n + ".bias"].clone()) for n in names]
    state = gp.GanStepState(layers(mg), layers(md))
    b, t = 3, 37
    lens = ragged_lengths(b, t, 9)
    x, y = make_batch(b, t, 20, 187, lens, 10)
    mg.to(dev), md.to(dev)
    fs = F.FusedGanStep(mg, md, gstep.HParams(gstep.TTS_ACOUSTIC, discriminator_linguistic_condition=False), b, t)
    ng = len(list(mg.parameters()))
    with torch.no_grad():
        for s, v in zip(state.g_sum + state.d_sum, fs._sums[:ng] + fs._sums[ng:]):
            s.copy_(v.cpu())
    R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, t))
    ref, yh_ref, ys_ref = gp.gan_step_mlp(state, x, y, lens, R, TTS_HP)
    fs.step(x.to(dev), y.to(dev), torch.LongTensor(lens).to(dev), frames=sum(lens))
    got = fs.loss_dict()
    errs = {k: abs(got[k] - ref[k]) / abs(ref[k]) for k in ("loss_d", "loss_mge", "loss_adv", "loss_g")}
    errs["y_hat"] = rel_err(npy(fs.y_hat), yh_ref.numpy())
    errs["y_hat_static"] = rel_err(npy(fs.y_hat_static), ys_ref.numpy())
    assert max(errs.values()) < 2e-4, errs
    assert got["real_correct"] == ref["real_correct"] and got["fake_correct"] == ref["fake_correct"]
