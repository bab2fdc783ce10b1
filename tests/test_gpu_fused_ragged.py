"""FusedGanStep on mini-batches of their own shape (b, t) within the configured capacity (B, T), as train.py's collate_fn
makes them (each batch padded to its own max_len, a short last batch), and the MLPG table built on the device.

Checkers: a chain of steps each built for exactly the call's shape, with the state handed over through state_dict and the
same seeds (bit for bit); the oracle port of train.py's step with R built per batch max_len, and GanTrainer, at the
tolerances of the other fused-step modules (2e-4 relative); the host table builder (bit for bit).
"""
import numpy as np
import pytest
import torch

from conftest import TTS_HP, WINDOWS, rel_err
from fused_step_helpers import build, dev, fused, make_batch, npy, ragged_lengths, step_hp  # noqa: F401
from oracle import gantts_port as gp
from oracle import nnmnkwii_port as nnp

TOL = 2e-4
B, T = 3, 40
# (b, t, kind of step): full shape, t - 7, b < B with t not a multiple of 32, the smallest batch, full shape again.  With
# Adam the D-only step leaves n_g != n_d, so the next training step runs as phases 1|2 then 4.
SEQUENCE = [(3, 40, "train"), (3, 33, "d_only"), (2, 29, "train"), (1, 5, "eval"), (3, 40, "train")]


def reference_discriminator(hp, seed):
    import gantts_b200
    from gantts_b200 import fused as F
    torch.manual_seed(seed)
    n_adv = len(F.adversarial_columns(step_hp(hp)))
    return gantts_b200.models.MLP(n_adv, 1, 1, 8, dropout=0.0, last_sigmoid=True)


def run(fs, x, y, lens, what):
    lengths = torch.LongTensor(lens).to(x.device)
    if what == "eval":
        fs.step(x, y, lengths, train=False)
    else:
        fs.step(x, y, lengths, train=True, update_g=what == "train")


def record(fs, mg, md):
    return ([fs.losses.clone(), fs.y_hat.clone(), fs.y_hat_static.clone(), fs.spoof_count.clone()] +
            [p.detach().clone() for p in list(mg.parameters()) + list(md.parameters())] +
            [s.clone() for s in fs._sums + fs._sqs])


@pytest.mark.gpu
@pytest.mark.parametrize("kind,optimizer,mse_w", [("mlp", "Adagrad", 0.0), ("mlp", "Adam", 0.5), ("highway", "Adam", 0.0),
                                                  ("sru", "Adagrad", 0.0), ("rnn_highway", "Adam", 0.0)])
def test_shaped_calls_equal_exactly_sized_steps(dev, kind, optimizer, mse_w):
    """One step of capacity (B, T) running the shape sequence computes bit for bit what a chain of steps built for each
    shape computes: losses, y_hat, y_hat_static, the spoof count, both models' parameters and optimiser state."""
    results = []
    for capacity in (True, False):
        mg, md, hp, d_in, d_out, _, _, _ = build(kind, 7)
        ref = reference_discriminator(hp, 8)
        mg.to(dev), md.to(dev), ref.to(dev)
        fs, sd, out = None, None, []
        for i, (b, t, what) in enumerate(SEQUENCE):
            lens = ragged_lengths(b, t, 20 + i)
            x, y = make_batch(b, t, d_in, d_out, lens, 30 + i)
            if capacity:
                fs = fs or fused(mg, md, hp, B, T, optimizer, mse_w=mse_w, seed=10, reference_discriminator=ref)
            else:
                fs = fused(mg, md, hp, b, t, optimizer, mse_w=mse_w, seed=10, reference_discriminator=ref)
                if sd is not None:
                    fs.load_state_dict(sd)
            run(fs, x.to(dev), y.to(dev), lens, what)
            assert tuple(fs.y_hat.shape[:2]) == (b, t) and tuple(fs.y_hat_static.shape[:2]) == (b, t)
            out.append(record(fs, mg, md))
            sd = fs.state_dict()
        results.append((out, sd))
    (cap, sd_cap), (exact, sd_exact) = results
    for i, (a, e) in enumerate(zip(cap, exact)):
        assert len(a) == len(e)
        for j, (u, v) in enumerate(zip(a, e)):
            assert torch.equal(u, v), (kind, optimizer, SEQUENCE[i], j)
    assert sd_cap["step"] == sd_exact["step"] and sd_cap["seed"] == sd_exact["seed"]
    for key in ("optimizer_g", "optimizer_d"):
        assert float(sd_cap[key]["state"][0]["step"]) == float(sd_exact[key]["state"][0]["step"])


@pytest.mark.gpu
def test_outputs_at_the_configured_shape_are_the_buffers(dev):
    mg, md, hp, d_in, d_out, _, _, _ = build("mlp", 3)
    mg.to(dev), md.to(dev)
    fs = fused(mg, md, hp, B, T)
    y_hat, y_hat_static = fs.y_hat, fs.y_hat_static
    for b, t in ((2, 17), (B, T)):
        lens = ragged_lengths(b, t, 1)
        x, y = make_batch(b, t, d_in, d_out, lens, 2)
        fs.step(x.to(dev), y.to(dev), torch.LongTensor(lens).to(dev))
    assert fs.y_hat is y_hat and fs.y_hat_static is y_hat_static


@pytest.mark.gpu
def test_shapes_beyond_the_capacity_are_refused(dev):
    mg, md, hp, d_in, d_out, _, _, _ = build("mlp", 3)
    mg.to(dev), md.to(dev)
    fs = fused(mg, md, hp, B, T)
    for b, t in ((B + 1, T), (B, T + 1)):
        x, y = torch.zeros(b, t, d_in, device=dev), torch.zeros(b, t, d_out, device=dev)
        with pytest.raises(RuntimeError, match="exceeds the configured"):
            fs.step(x, y, torch.full((b,), t, dtype=torch.int64, device=dev))
    x, y = torch.zeros(2, 10, d_in, device=dev), torch.zeros(2, 10, d_out, device=dev)
    with pytest.raises(RuntimeError, match="lengths must have shape"):
        fs.step(x, y, torch.full((3,), 10, dtype=torch.int64, device=dev))


@pytest.mark.gpu
def test_gradient_buffers_stay_put_across_shapes(dev):
    """grad_buffer(0 / 1) are the same memory before and after steps of different shapes (the data-parallel path
    all-reduces these views between the phases of a call)."""
    mg, md, hp, d_in, d_out, _, _, _ = build("sru", 4)
    mg.to(dev), md.to(dev)
    fs = fused(mg, md, hp, B, T, "Adam")
    before = [fs.grad_buffer(i).data_ptr() for i in (0, 1)]
    sizes = [fs.grad_buffer(i).numel() for i in (0, 1)]
    for i, (b, t, what) in enumerate(SEQUENCE):
        lens = ragged_lengths(b, t, i)
        x, y = make_batch(b, t, d_in, d_out, lens, i)
        run(fs, x.to(dev), y.to(dev), lens, what)
    fs._grad_views = {}                 # ask the library again
    assert [fs.grad_buffer(i).data_ptr() for i in (0, 1)] == before
    assert [fs.grad_buffer(i).numel() for i in (0, 1)] == sizes
    assert fs.grad_buffer(0).abs().sum().item() > 0


def collate_epoch(n_utt, B, d_in, d_out, seed, lo=20, hi=70):
    """One epoch of train.py's collate_fn batches (train.py:145-155): lengths seeded, sorted descending, each batch padded
    to its own max_len, the last batch short."""
    rng = np.random.RandomState(seed)
    lens_all = sorted((int(v) for v in rng.randint(lo, hi, n_utt)), reverse=True)
    batches = []
    for i in range(0, n_utt, B):
        lens = lens_all[i:i + B]
        x, y = make_batch(len(lens), lens[0], d_in, d_out, lens, seed + i)
        batches.append((x, y, lens))
    return batches


def mlp_pair(seed):
    import gantts_b200
    torch.manual_seed(seed)
    mg = gantts_b200.models.MLP(20, 187, 2, 32, dropout=0.0, last_sigmoid=False)
    md = gantts_b200.models.MLP(58, 1, 2, 16, dropout=0.0, last_sigmoid=True)
    return mg, md


def layers_of(m):
    ps = [p.detach().cpu() for p in m.parameters()]
    return list(zip(ps[0::2], ps[1::2]))


LOSS_KEYS = ("loss_d", "loss_fake_d", "loss_real_d", "loss_mge", "loss_mse", "loss_adv", "loss_g", "d_grad_norm",
             "g_grad_norm")


@pytest.mark.gpu
def test_ragged_epoch_matches_the_reference_step(dev):
    """A collate_fn epoch (4 batches of 3 and a last batch of 2, each padded to its own max_len) through one FusedGanStep
    of capacity (3, 70): every batch against the oracle port of train.py's step with R built for that batch's max_len,
    from the product's weights and Adagrad state.  Padding a batch to the capacity T instead changes y_hat_static."""
    from gantts_b200 import step as gstep
    from gantts_b200 import fused as F
    batches = collate_epoch(14, 3, 20, 187, 5)
    assert len(batches) == 5 and len(batches[-1][2]) == 2
    Tcap = 70
    mg, md = mlp_pair(11)
    mg.to(dev), md.to(dev)
    hp_dev = gstep.HParams(gstep.TTS_ACOUSTIC, discriminator_linguistic_condition=False)
    fs = F.FusedGanStep(mg, md, hp_dev, 3, Tcap)
    ng = len(list(mg.parameters()))
    for x, y, lens in batches:
        state = gp.GanStepState(layers_of(mg), layers_of(md))
        with torch.no_grad():
            for s, v in zip(state.g_sum + state.d_sum, fs._sums[:ng] + fs._sums[ng:]):
                s.copy_(v.cpu())
        R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, x.shape[1]))
        ref, yh_ref, ys_ref = gp.gan_step_mlp(state, x, y, lens, R, TTS_HP)
        fs.step(x.to(dev), y.to(dev), torch.LongTensor(lens).to(dev), frames=sum(lens))
        got = fs.loss_dict()
        errs = {k: abs(got[k] - ref[k]) / abs(ref[k]) for k in LOSS_KEYS}
        errs["y_hat"] = rel_err(npy(fs.y_hat), yh_ref.numpy())
        errs["y_hat_static"] = rel_err(npy(fs.y_hat_static), ys_ref.numpy())
        assert max(errs.values()) < TOL, (x.shape, errs)
        assert got["real_correct"] == ref["real_correct"] and got["fake_correct"] == ref["fake_correct"]
        assert got["frames"] == float(sum(lens))

    # the same first batch padded to the capacity T: the MLPG solves over 70 frames, the valid frames change
    x, y, lens = batches[0]
    t = x.shape[1]
    assert t < Tcap
    outs = []
    for pad in (0, Tcap - t):
        mg, md = mlp_pair(11)
        mg.to(dev), md.to(dev)
        fs = F.FusedGanStep(mg, md, hp_dev, 3, Tcap)
        xp = torch.nn.functional.pad(x, (0, 0, 0, pad))
        yp = torch.nn.functional.pad(y, (0, 0, 0, pad))
        fs.step(xp.to(dev), yp.to(dev), torch.LongTensor(lens).to(dev), train=False)
        outs.append(npy(fs.y_hat_static)[:, :t])
    assert rel_err(outs[1], outs[0]) > 1e-3, rel_err(outs[1], outs[0])


@pytest.mark.gpu
def test_ragged_epoch_matches_gan_trainer(dev):
    """The same collate_fn epoch through FusedGanStep (capacity (3, 70)) and GanTrainer (R per batch max_len), test
    phase from the same weights: every loss, count and output agrees at 2e-4."""
    from gantts_b200 import step as gstep
    from gantts_b200 import fused as F
    batches = collate_epoch(14, 3, 20, 187, 6)
    hp_dev = gstep.HParams(gstep.TTS_ACOUSTIC, discriminator_linguistic_condition=False)
    mg, md = mlp_pair(12)
    mg.to(dev).eval(), md.to(dev).eval()
    fs = F.FusedGanStep(mg, md, hp_dev, 3, 70)
    tr = gstep.GanTrainer(mg, md, hp_dev)
    for x, y, lens in batches:
        x, y, lengths = x.to(dev), y.to(dev), torch.LongTensor(lens).to(dev)
        R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, x.shape[1])).to(dev)
        out, yh, ys = tr.step(x, y, lengths, R, train=False)
        fs.step(x, y, lengths)
        got = fs.loss_dict()
        for k in ("loss_d", "loss_fake_d", "loss_real_d", "loss_mge", "loss_mse", "loss_adv", "loss_g"):
            assert abs(got[k] - float(out[k])) <= TOL * abs(float(out[k])), (k, got[k], float(out[k]))
        for k in ("real_correct", "fake_correct", "frames"):
            assert got[k] == float(out[k]), k
        assert rel_err(npy(fs.y_hat_static), npy(ys)) < TOL
        assert rel_err(npy(fs.y_hat), npy(yh)) < TOL


WINDOW_SETS = {
    "hparams": WINDOWS,
    "two": WINDOWS[:2],
    "static": WINDOWS[:1],
    "backward_difference": [(0, 0, np.array([1.0])), (1, 0, np.array([-1.0, 1.0]))],
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(WINDOW_SETS))
def test_device_table_equals_the_host_table(dev, name):
    """ops.mlpg_table_device is bit for bit ops.mlpg_table_full_host for every T in 1..2100."""
    from gantts_b200 import ops
    windows = WINDOW_SETS[name]
    bad = []
    for Tn in range(1, 2101):
        host = ops.mlpg_table_full_host(windows, Tn)
        got = ops.mlpg_table_device(windows, Tn, dev).cpu().numpy()
        if not np.array_equal(host.view(np.int32), got.view(np.int32)):
            bad.append(Tn)
    assert not bad, (name, bad[:10], len(bad))
