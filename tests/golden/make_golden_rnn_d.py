"""Generate tests/golden/rnn_d.npz by running the UNMODIFIED reference (r9y9/gantts @ fb1e75f, imported read-only from
the checkout GANTTS_REFERENCE_ROOT points at, through oracle.reference_loader) on seeded inputs:

    GANTTS_REFERENCE_ROOT=/path/to/gantts python tests/golden/make_golden_rnn_d.py

GAN steps with a recurrent discriminator (hp.discriminator = "LSTMRNN" or "GRURNN", last_sigmoid=True; train.py:774)
through the reference's own apply_generator / update_discriminator / update_generator (train.py:336-355, 245-279,
282-320), and one discriminator warm-up case (update_generator not called, train.py:696).  The cases of one hparams set
share their mini-batches and initial generator, and only the final state is kept, so that the file stays small.  The
helpers and conventions are those of make_golden.py, which writes the other golden files.
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
from make_golden import _run_ref_step, lengths_desc, npy, state_arrays  # noqa: E402

LOSS_KEYS = ("loss_d", "loss_fake_d", "loss_real_d", "loss_mse", "loss_mge", "loss_adv", "loss_g",
             "real_correct", "fake_correct")

# tag: (hparams name, discriminator class, bidirectional D, conditioned D, update_g, optimisers)
CASES = {
    "lstm_uni": ("tts_acoustic", "LSTMRNN", False, False, True, ("adagrad", "adam")),
    "lstm_bi_cond": ("tts_acoustic", "LSTMRNN", True, True, True, ("adagrad", "adam")),
    "gru_bi": ("tts_acoustic", "GRURNN", True, False, True, ("adagrad", "adam")),
    "hw_lstm_bi": ("vc", "LSTMRNN", True, False, True, ("adagrad", "adam")),
    "lstm_bi_d_only": ("tts_acoustic", "LSTMRNN", True, False, False, ("adagrad",)),
}
B, T = 3, 12
G_SEED, D_SEED = 43, 47


def make_generator(M, hp_name):
    """The generator of an hparams set, initialised from G_SEED: an MLP 20 -> 8 -> 187 on tts_acoustic, an
    In2OutHighwayNet 27 -> 8 -> 27 (static 9) on vc."""
    torch.manual_seed(G_SEED)
    if hp_name == "vc":
        return M.In2OutHighwayNet(in_dim=27, out_dim=27, static_dim=9, num_hidden=1, hidden_dim=8, dropout=0.0)
    return M.MLP(in_dim=20, out_dim=187, num_hidden=1, hidden_dim=8, dropout=0.0, last_sigmoid=False)


def gen_rnn_d(ref, out):
    """Per hparams set (`tts_acoustic`; `vc` at toy width) two mini-batches with ragged lengths sorted descending and one
    initial generator, shared by its cases (stored once as `<hp>_it<k>_x|y|lengths` and `<hp>_g0_*`).  Each case runs
    both mini-batches from that generator and a recurrent discriminator initialised from D_SEED (2 layers of 4 units per
    direction), dropout 0, with Adagrad (hparams.py:223-227) and Adam (0.5, 0.9) (hparams.py:125-130), the D-only case
    with Adagrad.  Stored per mini-batch: losses and counts; after the second one: y_hat_static, the weights of both models
    and the discriminator optimiser's state (the generator's optimiser is pinned by the other golden files, and its
    weights here)."""
    tr, hparams, M = ref.train, ref.hparams, ref.models
    from oracle.nnmnkwii_port import unit_variance_mlpg_matrix
    data = {}
    for hp_name, d_in, d_out in (("tts_acoustic", 20, 187), ("vc", 27, 27)):
        rng = np.random.default_rng(23)
        torch.manual_seed(29)
        data[hp_name] = []
        for it in range(2):
            lens = lengths_desc(rng, B, T)
            x = torch.randn(B, T, d_in) if hp_name == "vc" else torch.rand(B, T, d_in) * 0.98 + 0.01
            y = torch.randn(B, T, d_out)
            for b, n in enumerate(lens):
                x[b, n:] = 0
                y[b, n:] = 0
            data[hp_name].append((x, y, lens))
            p = "%s_it%d_" % (hp_name, it)
            out[p + "x"], out[p + "y"], out[p + "lengths"] = npy(x), npy(y), np.array(lens)
        state_arrays(make_generator(M, hp_name), hp_name + "_g0_", out)
    for name, (hp_name, d_cls, bidir, cond, update_g, opts) in CASES.items():
        hp = getattr(hparams, hp_name)
        n_adv, d_in = (9, 27) if hp_name == "vc" else (58, 20)
        for opt_name in opts:
            tag = "%s_%s_" % (name, opt_name)
            saved = (hp.stream_sizes, hp.discriminator_linguistic_condition)
            if hp is hparams.vc:
                hp.stream_sizes = [27]                # 9 static dims x 3 windows (hparams.py:27 with order 9)
            hp.discriminator_linguistic_condition = cond
            tr.hp = hp
            g = make_generator(M, hp_name)
            torch.manual_seed(D_SEED)
            d = getattr(M, d_cls)(in_dim=n_adv + (d_in if cond else 0), out_dim=1, num_hidden=2, hidden_dim=4,
                                  bidirectional=bidir, dropout=0.0, last_sigmoid=True)
            g.train(), d.train()
            state_arrays(d, tag + "d0_", out)
            if opt_name == "adam":
                og = optim.Adam(g.parameters(), lr=1e-3, betas=(0.5, 0.9), weight_decay=0)
                od = optim.Adam(d.parameters(), lr=1e-3, betas=(0.5, 0.9), weight_decay=0)
            else:
                og = optim.Adagrad(g.parameters(), lr=0.01, weight_decay=1e-7)
                od = optim.Adagrad(d.parameters(), lr=0.01, weight_decay=1e-7)
            R = torch.from_numpy(unit_variance_mlpg_matrix(hp.windows, T))
            for it, (x, y, lens) in enumerate(data[hp_name]):
                if update_g:
                    res, y_hat, y_hat_static = _run_ref_step(ref, tr, hp, g, d, og, od, x, y, lens, R, 1.0, 0.0, 1.0)
                else:
                    lengths = torch.LongTensor(lens)
                    y_static = ref.multistream.get_static_features(y, len(hp.windows), hp.stream_sizes,
                                                                   hp.has_dynamic_features)
                    mask = ref.seqloss.sequence_mask(lengths).unsqueeze(-1)
                    og.zero_grad(), od.zero_grad()
                    y_hat, y_hat_static = tr.apply_generator(g, x, R, lens)
                    ld, lf, lr_, rc, fc = tr.update_discriminator(d, od, x, y_static, y_hat_static, lens, mask, "train")
                    res = dict(loss_d=ld, loss_fake_d=lf, loss_real_d=lr_, real_correct=rc, fake_correct=fc)
                p = "%sit%d_" % (tag, it)
                out[p + "losses"] = np.array([float(res.get(k, np.nan)) for k in LOSS_KEYS], dtype=np.float64)
            out[tag + "y_hat_static"] = npy(y_hat_static)
            state_arrays(g, tag + "g_", out)
            state_arrays(d, tag + "d_", out)
            for i, q in enumerate(d.parameters()):
                for k, v in od.state[q].items():
                    out["%sdopt%d_%s" % (tag, i, k)] = npy(v) if torch.is_tensor(v) else np.float64(v)
            hp.stream_sizes, hp.discriminator_linguistic_condition = saved


def main():
    ref = reference_loader.load()
    torch.manual_seed(1234)
    torch.set_num_threads(1)
    d = {}
    gen_rnn_d(ref, d)
    np.savez_compressed(os.path.join(HERE, "rnn_d.npz"), **d)
    print("rnn_d", os.path.getsize(os.path.join(HERE, "rnn_d.npz")))


if __name__ == "__main__":
    main()
