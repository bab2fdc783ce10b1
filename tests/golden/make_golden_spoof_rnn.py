"""Generate tests/golden/spoof_rnn.npz by running the UNMODIFIED reference (r9y9/gantts @ fb1e75f, imported read-only from
the checkout GANTTS_REFERENCE_ROOT points at, through oracle.reference_loader) on seeded inputs:

    GANTTS_REFERENCE_ROOT=/path/to/gantts python tests/golden/make_golden_spoof_rnn.py

The spoofing-rate count of the adversarial stage (train.py:549-558) with a recurrent reference discriminator: train.py:779-781
builds it from hp.discriminator like D, so with hp.discriminator = "LSTMRNN" or "GRURNN" it is one of those.  The count
comes from the reference's own spoof block (make_golden_dwarmup.spoof_block); the helpers and conventions are those of
make_golden.py, which writes the other golden files.
"""
import os
import sys

import numpy as np
import torch
from torch import optim

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)

from oracle import reference_loader  # noqa: E402
from make_golden import lengths_desc, npy, state_arrays  # noqa: E402
from make_golden_dwarmup import spoof_block  # noqa: E402


def gen_spoof_rnn(ref, out):
    """Per case: `vc` (toy width) or `tts_acoustic` unconditioned, with an LSTMRNN or a GRURNN reference discriminator (2
    layers of 8 units, bidirectional, dropout 0.5) put in eval mode the way train_loop does (:445).  An MLP generator and an
    MLP discriminator train over two mini-batches with ragged lengths sorted descending: a discriminator warm-up step
    (update_generator not called, train.py:696) and then a full step (train.py:541-575).  Each batch runs the spoof block
    on the generator output of its step; before the first one the reference discriminator's last logit is centred on that
    batch so that its outputs fall on both sides of 0.5.  Stored per batch: x, y, lengths, y_hat_static, the reference
    discriminator's output on it and the count."""
    tr, hparams, M = ref.train, ref.hparams, ref.models
    from oracle.nnmnkwii_port import unit_variance_mlpg_matrix
    block = spoof_block(ref)
    B, T = 3, 16
    cases = [("vc", hparams.vc, 27, 27, 9), ("tts", hparams.tts_acoustic, 20, 187, 58)]
    for name, hp, d_in, d_out, n_adv in cases:
        for ref_cls in ("LSTMRNN", "GRURNN"):
            rng = np.random.default_rng(31)
            tag = "%s_%s_" % (name, ref_cls.lower())
            saved = (hp.stream_sizes, hp.discriminator_linguistic_condition)
            if hp is hparams.vc:
                hp.stream_sizes = [27]                # 9 static dims x 3 windows (hparams.py:27 with order 9)
            hp.discriminator_linguistic_condition = False
            tr.hp = hp
            torch.manual_seed(37)
            g = M.MLP(in_dim=d_in, out_dim=d_out, num_hidden=2, hidden_dim=24, dropout=0.0, last_sigmoid=False)
            d = M.MLP(in_dim=n_adv, out_dim=1, num_hidden=2, hidden_dim=16, dropout=0.0, last_sigmoid=True)
            ref_d = getattr(M, ref_cls)(in_dim=n_adv, out_dim=1, num_hidden=2, hidden_dim=8, bidirectional=True,
                                        dropout=0.5, last_sigmoid=True)
            ref_d.eval()                              # train.py:445
            g.train(), d.train()
            state_arrays(g, tag + "g0_", out)
            og = optim.Adagrad(g.parameters(), lr=0.01, weight_decay=1e-7)
            od = optim.Adagrad(d.parameters(), lr=0.01, weight_decay=1e-7)
            R = torch.from_numpy(unit_variance_mlpg_matrix(hp.windows, T))
            for it in range(2):
                lens = lengths_desc(rng, B, T)
                x = torch.randn(B, T, d_in) if hp is hparams.vc else torch.rand(B, T, d_in) * 0.98 + 0.01
                y = torch.randn(B, T, d_out)
                for b, n in enumerate(lens):
                    x[b, n:] = 0
                    y[b, n:] = 0
                lengths = torch.LongTensor(lens)
                y_static = ref.multistream.get_static_features(y, len(hp.windows), hp.stream_sizes,
                                                               hp.has_dynamic_features)
                mask = ref.seqloss.sequence_mask(lengths).unsqueeze(-1)
                og.zero_grad(), od.zero_grad()
                y_hat, y_hat_static = tr.apply_generator(g, x, R, lens)
                if it == 0:
                    with torch.no_grad():
                        ref_d.hidden2out.weight.mul_(10.0)
                        ref_d.hidden2out.bias.zero_()
                        z = torch.logit(ref_d(tr.get_selected_static_stream(y_hat_static), lengths=lens))
                        ref_d.hidden2out.bias.fill_(-float(z[mask > 0].median()))
                    state_arrays(ref_d, tag + "ref_", out)
                ns = dict(vars(tr), reference_discriminator=ref_d, y_hat_static=y_hat_static, cpu_sorted_lengths=lens,
                          mask=mask, regard_fake_as_natural=0)
                exec(block, ns)
                with torch.no_grad():
                    target = ref_d(tr.get_selected_static_stream(y_hat_static), lengths=lens)
                tr.update_discriminator(d, od, x, y_static, y_hat_static, lens, mask, "train")
                if it == 1:
                    tr.update_generator(g, d, og, x, y, y_hat, y_static, y_hat_static, 1.0, lens, mask, "train",
                                        mse_w=0.0, mge_w=1.0)
                p = "%sit%d_" % (tag, it)
                out[p + "x"], out[p + "y"], out[p + "lengths"] = npy(x), npy(y), np.array(lens)
                out[p + "y_hat_static"], out[p + "target"] = npy(y_hat_static), npy(target)
                out[p + "spoof"] = np.float64(ns["regard_fake_as_natural"])
            hp.stream_sizes, hp.discriminator_linguistic_condition = saved


def main():
    ref = reference_loader.load()
    torch.manual_seed(1234)
    torch.set_num_threads(1)
    d = {}
    gen_spoof_rnn(ref, d)
    np.savez_compressed(os.path.join(HERE, "spoof_rnn.npz"), **d)
    print("spoof_rnn", os.path.getsize(os.path.join(HERE, "spoof_rnn.npz")))


if __name__ == "__main__":
    main()
