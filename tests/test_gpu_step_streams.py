"""The fused GAN step runs the MLP stacks' weight gradients on the library's side stream, beside the input-gradient chain,
and joins it back before each call returns.  The caller's stream is the whole contract: these tests read every result on
that stream straight after the call and compare it bit for bit with a twin model stepped under a device synchronise after
every call, with the phases split the way a data-parallel caller splits them, and with a second run of the same steps.

Shapes: the bench's cfg2 (MLP G 425-512-512-512-187, MLP D 58-256-256-256-1, B=32 x T=1000), and a small ragged one
whose stacks have three layers (one gradient buffer per layer on the concurrent path).
"""
import pytest
import torch

from conftest import TTS_HP
from fused_step_helpers import build, dev, fused, make_batch, ragged_lengths, split_step  # noqa: F401

SHAPES = ["cfg2", "small"]


def models(shape, seed):
    """(model_g, model_d, oracle hparams, d_in, d_out, B, T, lengths) on the host."""
    import gantts_b200
    if shape == "cfg2":
        torch.manual_seed(seed)
        mg = gantts_b200.models.MLP(425, 187, 3, 512, dropout=0.5, last_sigmoid=False)
        md = gantts_b200.models.MLP(58, 1, 3, 256, dropout=0.5, last_sigmoid=True)
        return mg, md, TTS_HP, 425, 187, 32, 1000, [1000] * 32
    mg, md, hp, d_in, d_out, _, _, _ = build("mlp", seed)
    return mg, md, hp, d_in, d_out, 3, 40, ragged_lengths(3, 40, seed)


def setup(shape, dev, seed=5):
    mg, md, hp, d_in, d_out, B, T, lens = models(shape, seed)
    mg.to(dev), md.to(dev)
    fs = fused(mg, md, hp, B, T, seed=11)
    batches = []
    for i in range(3):
        x, y = make_batch(B, T, d_in, d_out, lens, 40 + i)
        batches.append((x.to(dev), y.to(dev)))
    return fs, mg, md, batches, torch.LongTensor(lens).to(dev)


def record(fs, mg, md):
    """Copies, enqueued on the current stream, of what a caller reads after a step."""
    return ([fs.losses.clone(), fs.y_hat_static.clone(), fs.grad_buffer(0).clone(), fs.grad_buffer(1).clone()] +
            [p.detach().clone() for p in list(mg.parameters()) + list(md.parameters())] +
            [s.clone() for s in fs._sums + fs._sqs])


def assert_same(a, b, what):
    assert len(a) == len(b)
    for i, (u, v) in enumerate(zip(a, b)):
        assert torch.equal(u, v), (what, i)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", SHAPES)
def test_results_complete_on_the_callers_stream(dev, shape):
    """Steps issued on a non-default stream and read on it right after each call, with no synchronisation, equal bit for
    bit the steps of an identically seeded twin synchronised after every call."""
    fs, mg, md, batches, lengths = setup(shape, dev)
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    got = []
    with torch.cuda.stream(side):
        for i in range(3):
            fs.step(*batches[i], lengths)
            got.append(record(fs, mg, md))
    torch.cuda.synchronize()

    fs2, mg2, md2, batches2, lengths2 = setup(shape, dev)
    for i in range(3):
        fs2.step(*batches2[i], lengths2)
        torch.cuda.synchronize()
        assert_same(got[i], record(fs2, mg2, md2), "step %d" % i)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", SHAPES)
def test_phase_split_calls_equal_one_call(dev, shape):
    """Three training steps, a D-only step and a training step, each as one native call, equal bit for bit the same steps
    each split into the discriminator phase and then the generator and finishing phases."""
    plan = [True, True, True, False, True]
    fs, mg, md, batches, lengths = setup(shape, dev)
    full = []
    for i, update_g in enumerate(plan):
        fs.step(*batches[i % 3], lengths, update_g=update_g)
        full.append(record(fs, mg, md))
    fs2, mg2, md2, batches2, lengths2 = setup(shape, dev)
    for i, update_g in enumerate(plan):
        split_step(fs2, *batches2[i % 3], lengths2, update_g=update_g)
        assert_same(full[i], record(fs2, mg2, md2), "step %d (update_g=%s)" % (i, update_g))


@pytest.mark.gpu
def test_repeated_runs_are_identical(dev):
    """Two runs of five cfg2 steps from the same state give identical losses, parameters and optimiser state."""
    runs = []
    for _ in range(2):
        fs, mg, md, batches, lengths = setup("cfg2", dev)
        for i in range(5):
            fs.step(*batches[i % 3], lengths)
        runs.append(record(fs, mg, md))
        del fs
    assert_same(runs[0], runs[1], "run")


@pytest.mark.gpu
@pytest.mark.parametrize("shape", SHAPES)
def test_step_captured_in_a_graph(dev, shape):
    """A training step captured in a CUDA graph (the side stream forks from and joins the capturing stream through events)
    and replayed computes bit for bit what the same step computes eagerly."""
    fs, mg, md, batches, lengths = setup(shape, dev)
    fs.step(*batches[0], lengths)
    torch.cuda.synchronize()
    fs2, mg2, md2, batches2, lengths2 = setup(shape, dev)
    fs2.step(*batches2[0], lengths2)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fs2.step(*batches2[1], lengths2)
    graph.replay()
    torch.cuda.synchronize()
    fs.step(*batches[1], lengths)
    torch.cuda.synchronize()
    assert_same(record(fs, mg, md), record(fs2, mg2, md2), "graph replay")
