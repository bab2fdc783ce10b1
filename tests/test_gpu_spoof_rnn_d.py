"""The spoofing-rate count (train.py:549-558) with a recurrent reference discriminator on the GPU: FusedGanStep and
GanTrainer with reference_discriminator = LSTMRNN / GRURNN (train.py:779-781 builds it from hp.discriminator like D), run by
gantts_spoof_count_lstm.

Checker: the oracle's spoof_count on a DiscriminatorOracle (pinned to the reference by test_spoof_rnn_host.py) on the
product's own pre-update y_hat_static.  The count is an integer, but a frame whose D_ref lies within rounding of 0.5 may
fall on either side: the counts may differ by at most the number of valid frames whose CPU |D_ref - 0.5| is below
TIE_BAND.  The band is 1e-5: on an NVIDIA H100 80GB HBM3 (700 W) the count's own D_ref output, read back from its
workspace, differed from the CPU's by at most 3.6e-6 (median 1.3e-6 or less) over every case below, and the frames
whose side differed all lay within 6e-8 of 0.5 (the median frame, which `centre` puts on 0.5).  Every check prints how
many frames fall inside the band.  GRURNN vs LSTMRNN, shaped calls and the step's outputs with and without a count are
compared bit for bit.
"""
import pytest
import torch

from conftest import WINDOWS
from fused_step_helpers import (assert_equal_lists, dev, make_batch, make_models, ragged_lengths, sd_numpy,  # noqa: F401
                                snapshot, step_hp)
from oracle import gantts_port as gp
from oracle import nnmnkwii_port as nnp

TIE_BAND = 1e-5


def ref_discriminator(n_adv, layers, hidden, bidir, dev, seed, gru=False):
    """A reference discriminator with inter-layer dropout 0.5 (it must run with dropout off) left in train mode."""
    import gantts_b200
    torch.manual_seed(seed)
    cls = gantts_b200.models.GRURNN if gru else gantts_b200.models.LSTMRNN
    return cls(n_adv, 1, layers, hidden, bidirectional=bidir, dropout=0.5, last_sigmoid=True).to(dev).train()


def centre(ref_d, ys, lens, ohp):
    """Scale and shift ref_d's hidden2out so that its outputs on ys fall on both sides of 0.5."""
    with torch.no_grad():
        ref_d.hidden2out.weight.mul_(10.0)
        ref_d.hidden2out.bias.zero_()
        z = torch.logit(gp.reference_output(gp.DiscriminatorOracle(sd_numpy(ref_d)), ys, lens, ohp))
        mask = gp.sequence_mask(lens, ys.size(1)).unsqueeze(-1)
        ref_d.hidden2out.bias.fill_(-float(z[mask > 0].median()))


def check_count(got, ref_d, ys, lens, ohp, what):
    """got == the restatement's count on ys, up to the valid frames whose CPU |D_ref - 0.5| < TIE_BAND."""
    o = gp.DiscriminatorOracle(sd_numpy(ref_d))
    mask = gp.sequence_mask(lens, ys.size(1)).unsqueeze(-1)
    want = gp.spoof_count(o, ys, lens, mask, ohp)
    close = float(((gp.reference_output(o, ys, lens, ohp) - 0.5).abs() < TIE_BAND).float().mul(mask).sum())
    print("spoof count %s: got %g, restatement %g, %g frame(s) within %g of 0.5" % (what, float(got), want, close,
                                                                                   TIE_BAND))
    assert abs(float(got) - want) <= close, (what, float(got), want, close)
    return want


def models(kind, seed, d_kind):
    """(generator, discriminator, ohp, d_in, d_out, n_adv): the generator of fused_step_helpers.make_models with its
    LSTMRNN D (d_kind "lstm": 2 x 12 bidirectional, dropout 0.5), or an MLP D (d_kind "mlp": 2 x 16, dropout 0.5)."""
    import gantts_b200
    mg, md, ohp, d_in = make_models(kind, seed, False)
    n_adv = md.lstm.input_size
    if d_kind == "mlp":
        torch.manual_seed(seed + 1)
        md = gantts_b200.models.MLP(n_adv, 1, 2, 16, dropout=0.5, last_sigmoid=True)
    d_out = mg.hidden2out.weight.shape[0] if hasattr(mg, "hidden2out") else mg.last_linear.weight.shape[0]
    return mg, md, ohp, d_in, d_out, n_adv


def batch(B, T, d_in, d_out, seed, dev):
    lens = ragged_lengths(B, T, seed)
    x, y = make_batch(B, T, d_in, d_out, lens, seed + 1)
    return lens, x.abs().to(dev), y.to(dev), torch.LongTensor(lens).to(dev)


# generator, discriminator, reference D layers, bidirectional
CASES = [("mlp", "mlp", 1, False), ("highway", "mlp", 2, True), ("sru", "mlp", 3, True), ("rnn_highway", "mlp", 2, False),
         ("mlp", "lstm", 2, True), ("highway", "lstm", 3, False), ("sru", "lstm", 1, True), ("rnn_highway", "lstm", 2, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,d_kind,layers,bidir", CASES)
def test_spoof_count_rnn_fused_and_gan_trainer_match_restatement(dev, kind, d_kind, layers, bidir):
    """eval -> D-only -> full -> eval steps of FusedGanStep, then training, D-only and eval steps of GanTrainer, with an
    LSTMRNN reference D (12 units per direction, dropout 0.5 left on in train mode), B = 4 x T = 60 ragged: every count
    equals the restatement's on the step's own pre-update y_hat_static, within the tie band."""
    from gantts_b200 import fused, step as gstep
    B, T = 4, 60
    mg, md, ohp, d_in, d_out, n_adv = models(kind, 80 + layers + 2 * bidir, d_kind)
    mg.to(dev).eval(), md.to(dev).eval()
    ref_d = ref_discriminator(n_adv, layers, 12, bidir, dev, 81)
    lens, x, y, ld = batch(B, T, d_in, d_out, 82, dev)
    plain = fused.FusedGanStep(mg, md, step_hp(ohp), B, T, seed=83)
    plain.step(x, y, ld)
    centre(ref_d, plain.y_hat_static.cpu(), lens, ohp)
    r0 = snapshot(*ref_d.parameters())
    fs = fused.FusedGanStep(mg, md, step_hp(ohp), B, T, seed=83, reference_discriminator=ref_d)
    for i, (train, update_g) in enumerate(((False, True), (True, False), (True, True), (False, True))):
        mg.train(train), md.train(train)
        fs.step(x, y, ld, update_g=update_g)
        got = fs.loss_dict()
        want = check_count(got["spoof_count"], ref_d, fs.y_hat_static.cpu(), lens, ohp, "fused %d" % i)
        if i == 0:
            assert 0 < want < sum(lens)                        # the reference D's outputs straddle 0.5
        assert float(fs.spoof_count) == got["spoof_count"]
    assert ref_d.training
    assert_equal_lists(r0, snapshot(*ref_d.parameters()), "reference D")
    R = torch.from_numpy(nnp.unit_variance_mlpg_matrix(WINDOWS, T)).to(dev)
    tr = gstep.GanTrainer(mg, md, step_hp(ohp), w_d=1.0, reference_discriminator=ref_d)
    assert not ref_d.training                                   # train.py:445
    for i, (train, update_g) in enumerate(((True, True), (True, False), (False, True))):
        mg.train(train), md.train(train)
        out, _, ys = tr.step(x, y, lens, R, train=train, update_g=update_g)
        check_count(out["spoof_count"], ref_d, ys.detach().cpu(), lens, ohp, "GanTrainer %d" % i)
    assert_equal_lists(r0, snapshot(*ref_d.parameters()), "reference D")


@pytest.mark.gpu
def test_spoof_count_rnn_vc_full_width(dev):
    """vc at full width: In2OutHighwayNet 177 -> 512 x 3 -> 177 with an MLP D, B = 20 x T = 1000, reference D
    LSTMRNN(59, 1, 2, 256, bidirectional=True); a training step and an eval step."""
    from gantts_b200 import fused
    import gantts_b200
    B, T = 20, 1000
    mg, _, ohp, d_in = make_models("highway", 90, False, full=True)
    torch.manual_seed(91)
    md = gantts_b200.models.MLP(59, 1, 2, 256, dropout=0.5, last_sigmoid=True)
    mg.to(dev).eval(), md.to(dev).eval()
    ref_d = ref_discriminator(59, 2, 256, True, dev, 92)
    lens, x, y, ld = batch(B, T, d_in, d_in, 93, dev)
    plain = fused.FusedGanStep(mg, md, step_hp(ohp), B, T, seed=94)
    plain.step(x, y, ld)
    centre(ref_d, plain.y_hat_static.cpu(), lens, ohp)
    fs = fused.FusedGanStep(mg, md, step_hp(ohp), B, T, seed=94, reference_discriminator=ref_d)
    for i, train in enumerate((True, False)):
        mg.train(train), md.train(train)
        fs.step(x, y, ld)
        want = check_count(fs.loss_dict()["spoof_count"], ref_d, fs.y_hat_static.cpu(), lens, ohp, "vc full %d" % i)
        assert 0 < want < sum(lens)


@pytest.mark.gpu
def test_grurnn_reference_equals_lstmrnn_reference_bit_for_bit(dev):
    """A GRURNN reference D (an nn.LSTM stored as .gru) gives exactly the count of an LSTMRNN one with the same weights,
    and neither changes anything else the step computes."""
    from gantts_b200 import fused
    B, T = 3, 40
    runs = []
    for gru in (False, True):
        mg, md, ohp, d_in, d_out, n_adv = models("highway", 100, "lstm")
        mg.to(dev).train(), md.to(dev).train()
        ref_d = ref_discriminator(n_adv, 2, 8, True, dev, 101, gru=gru)
        if gru:
            with torch.no_grad():
                for p, q in zip(ref_d.parameters(), runs[0][0]):
                    p.copy_(q)
        fs = fused.FusedGanStep(mg, md, step_hp(ohp), B, T, seed=102, reference_discriminator=ref_d)
        counts = []
        for it in range(3):
            mg.train(it < 2), md.train(it < 2)
            fs.step(*batch(B, T, d_in, d_out, 103 + it, dev)[1:], update_g=it != 0)
            counts.append(fs.spoof_count.clone())
        runs.append((snapshot(*ref_d.parameters()), counts + [fs.losses.clone(), fs.y_hat_static.clone()]
                     + snapshot(*mg.parameters(), *md.parameters())))
    assert_equal_lists(runs[0][1], runs[1][1], "GRURNN vs LSTMRNN reference")


@pytest.mark.gpu
def test_spoof_count_rnn_shaped_calls_equal_exactly_sized_steps(dev):
    """A step built for (B, T) = (4, 40) runs the shapes (4, 40) -> (4, 33) -> (2, 29) -> (1, 5) with exactly the count and
    the results of steps built for each shape, bit for bit."""
    from gantts_b200 import fused
    B, T = 4, 40
    shapes = [((B, T), True), ((B, T - 7), True), ((2, 29), False), ((1, 5), True)]
    mg, md, ohp, d_in, d_out, n_adv = models("mlp", 110, "lstm")
    mg.to(dev).train(), md.to(dev).train()
    ref_d = ref_discriminator(n_adv, 2, 8, True, dev, 111)
    cap = fused.FusedGanStep(mg, md, step_hp(ohp), B, T, seed=112, reference_discriminator=ref_d)
    for i, ((b, t), update_g) in enumerate(shapes):
        tg, td = models("mlp", 110, "lstm")[:2]
        tg.to(dev).train(), td.to(dev).train()
        with torch.no_grad():
            for p, q in zip(list(tg.parameters()) + list(td.parameters()), list(mg.parameters()) + list(md.parameters())):
                p.copy_(q)
        ex = fused.FusedGanStep(tg, td, step_hp(ohp), b, t, seed=112, reference_discriminator=ref_d)
        ex.load_state_dict(cap.state_dict())
        x, y, ld = batch(b, t, d_in, d_out, 113 + i, dev)[1:]
        cap.step(x, y, ld, update_g=update_g)
        ex.step(x, y, ld, update_g=update_g)
        assert torch.equal(cap.spoof_count, ex.spoof_count), i
        assert torch.equal(cap.losses, ex.losses), i
        assert torch.equal(cap.y_hat_static, ex.y_hat_static) and torch.equal(cap.y_hat, ex.y_hat), i
        assert_equal_lists(snapshot(*tg.parameters(), *td.parameters()), snapshot(*mg.parameters(), *md.parameters()),
                           "parameters %d" % i)
        assert_equal_lists(ex._sums, cap._sums, "optimiser state %d" % i)


@pytest.mark.gpu
def test_reference_discriminator_untouched_and_step_unchanged(dev):
    """The reference D's parameters and training flag are unchanged by the count, and a step with the count computes
    exactly what a step without a reference D computes: losses, outputs, both models and the optimiser state."""
    from gantts_b200 import fused
    B, T = 3, 40
    runs = []
    for with_ref in (False, True):
        mg, md, ohp, d_in, d_out, n_adv = models("rnn_highway", 120, "lstm")
        mg.to(dev).train(), md.to(dev).train()
        ref_d = ref_discriminator(n_adv, 3, 8, False, dev, 121) if with_ref else None
        r0 = snapshot(*ref_d.parameters()) if with_ref else []
        fs = fused.FusedGanStep(mg, md, step_hp(ohp), B, T, seed=122, reference_discriminator=ref_d)
        for it, update_g in enumerate((False, True, True)):
            fs.step(*batch(B, T, d_in, d_out, 123 + it, dev)[1:], update_g=update_g)
        mg.eval(), md.eval()
        fs.step(*batch(B, T, d_in, d_out, 130, dev)[1:])
        if with_ref:
            assert ref_d.training
            assert_equal_lists(r0, snapshot(*ref_d.parameters()), "reference D")
            assert "spoof_count" in fs.loss_dict()
        runs.append([fs.losses.clone(), fs.y_hat.clone(), fs.y_hat_static.clone(), fs.grad_buffer(0).clone(),
                     fs.grad_buffer(1).clone()] + snapshot(*mg.parameters(), *md.parameters()) + fs._sums)
    assert_equal_lists(runs[0], runs[1], "with vs without a reference D")


@pytest.mark.gpu
def test_recurrent_reference_discriminator_refusals(dev):
    """A conditioned recurrent reference D is refused by both paths citing train.py:549-555; FusedGanStep refuses a
    recurrent reference D for B > 128 at construction."""
    from gantts_b200 import fused, step as gstep
    mg, md, ohp, d_in, d_out, n_adv = models("mlp", 140, "mlp")
    mg.to(dev).train(), md.to(dev).train()
    cond = ref_discriminator(d_in + n_adv, 2, 8, True, dev, 141)
    with pytest.raises(RuntimeError, match="train.py:549-555"):
        fused.FusedGanStep(mg, md, step_hp(ohp), 2, 16, reference_discriminator=cond)
    with pytest.raises(RuntimeError, match="train.py:549-555"):
        gstep.GanTrainer(mg, md, step_hp(ohp), reference_discriminator=cond)
    ref_d = ref_discriminator(n_adv, 2, 8, True, dev, 142)
    with pytest.raises(RuntimeError, match="LSTM_MAX_B = 128"):
        fused.FusedGanStep(mg, md, step_hp(ohp), 129, 8, reference_discriminator=ref_d)
    assert fused.FusedGanStep(mg, md, step_hp(ohp), 128, 8, reference_discriminator=ref_d)._ref_ws.numel() > 0
