"""Generate tests/golden/dwarmup.npz by running the UNMODIFIED reference (r9y9/gantts @ fb1e75f, imported read-only from
the checkout GANTTS_REFERENCE_ROOT points at, through oracle.reference_loader) on seeded inputs:

    GANTTS_REFERENCE_ROOT=/path/to/gantts python tests/golden/make_golden_dwarmup.py

The vectors of the discriminator warm-up (train.py --discriminator-warmup) and of the spoofing-rate count of the
adversarial stage (train.py:549-558), through the reference's own apply_generator / update_discriminator and its own
spoof block; the helpers and conventions are those of make_golden.py, which writes the other golden files.
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


def spoof_block(ref):
    """The spoofing-rate block of reference train_loop (train.py:549-558, ``if reference_discriminator is not None:``
    after apply_generator), compiled out of the file unmodified; executed in a namespace holding the train module's
    globals and the loop's locals, it adds the count to ``regard_fake_as_natural``."""
    import ast
    path = os.path.join(reference_loader.REFERENCE_ROOT, "train.py")
    tree = ast.parse(open(path).read(), path)
    loop = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "train_loop"]
    assert len(loop) == 1
    blocks = [n for n in ast.walk(loop[0]) if isinstance(n, ast.If) and ast.unparse(n.test) == "reference_discriminator is not None"
              and any(isinstance(s, ast.AugAssign) and getattr(s.target, "id", "") == "regard_fake_as_natural"
                      for s in ast.walk(n))]
    assert len(blocks) == 1
    return compile(ast.Module(body=blocks, type_ignores=[]), path, "exec")


def gen_dwarmup(ref, out):
    """The discriminator warm-up of the reference (train_gan.sh stages 3-4, --discriminator-warmup: train.py:696
    update_g = False): apply_generator (train.py:336-355) and update_discriminator (:245-279) alone, update_generator not
    called, two consecutive mini-batches with ragged lengths and dropout 0; MLP G + MLP D on `vc` (toy width) and on
    `tts_acoustic` unconditioned, each with Adagrad (hparams.py:223-227) and with Adam (0.5, 0.9) (hparams.py:125-130).
    Every batch also runs the spoofing-rate block of train_loop (:549-558) with a reference discriminator built with
    dropout 0.5 and put in eval mode the way train_loop does (:445)."""
    tr, hparams, M = ref.train, ref.hparams, ref.models
    from oracle.nnmnkwii_port import unit_variance_mlpg_matrix
    block = spoof_block(ref)
    rng = np.random.default_rng(17)
    B, T = 3, 16
    cases = [("vc", hparams.vc, 27, 27, 9), ("tts", hparams.tts_acoustic, 20, 187, 58)]
    for name, hp, d_in, d_out, n_adv in cases:
        for opt_name in ("adagrad", "adam"):
            tag = "%s_%s_" % (name, opt_name)
            saved = (hp.stream_sizes, hp.discriminator_linguistic_condition)
            if hp is hparams.vc:
                hp.stream_sizes = [27]                # 9 static dims x 3 windows (hparams.py:27 with order 9)
            hp.discriminator_linguistic_condition = False
            tr.hp = hp
            torch.manual_seed(41)
            g = M.MLP(in_dim=d_in, out_dim=d_out, num_hidden=2, hidden_dim=24, dropout=0.0, last_sigmoid=False)
            d = M.MLP(in_dim=n_adv, out_dim=1, num_hidden=2, hidden_dim=16, dropout=0.0, last_sigmoid=True)
            ref_d = M.MLP(in_dim=n_adv, out_dim=1, num_hidden=2, hidden_dim=16, dropout=0.5, last_sigmoid=True)
            ref_d.eval()                              # train.py:445
            g.train(), d.train()
            for pre, m in (("g0_", g), ("d0_", d)):
                state_arrays(m, tag + pre, out)
            if opt_name == "adam":
                og = optim.Adam(g.parameters(), lr=1e-3, betas=(0.5, 0.9), weight_decay=0)
                od = optim.Adam(d.parameters(), lr=1e-3, betas=(0.5, 0.9), weight_decay=0)
            else:
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
                    # centre the reference D's logits on this batch so that its outputs fall on both sides of 0.5
                    with torch.no_grad():
                        ref_d.last_linear.weight.mul_(10.0)
                        ref_d.last_linear.bias.zero_()
                        z = torch.logit(ref_d(tr.get_selected_static_stream(y_hat_static), lengths=lens))
                        ref_d.last_linear.bias.fill_(-float(z[mask > 0].median()))
                    state_arrays(ref_d, tag + "ref_", out)
                ns = dict(vars(tr), reference_discriminator=ref_d, y_hat_static=y_hat_static, cpu_sorted_lengths=lens,
                          mask=mask, regard_fake_as_natural=0)
                exec(block, ns)
                ld, lf, lr_, rc, fc = tr.update_discriminator(d, od, x, y_static, y_hat_static, lens, mask, "train")
                p = "%sit%d_" % (tag, it)
                out[p + "x"], out[p + "y"], out[p + "lengths"] = npy(x), npy(y), np.array(lens)
                out[p + "y_hat"], out[p + "y_hat_static"] = npy(y_hat), npy(y_hat_static)
                out[p + "losses"] = np.array([ld, lf, lr_, rc, fc], dtype=np.float64)
                out[p + "spoof"] = np.float64(ns["regard_fake_as_natural"])
                state_arrays(g, p + "g_", out)
                state_arrays(d, p + "d_", out)
                for i, q in enumerate(d.parameters()):
                    for k, v in od.state[q].items():
                        out["%sdopt%d_%s" % (p, i, k)] = npy(v) if torch.is_tensor(v) else np.float64(v)
            hp.stream_sizes, hp.discriminator_linguistic_condition = saved


def main():
    ref = reference_loader.load()
    torch.manual_seed(1234)
    torch.set_num_threads(1)
    d = {}
    gen_dwarmup(ref, d)
    np.savez_compressed(os.path.join(HERE, "dwarmup.npz"), **d)
    print("dwarmup", os.path.getsize(os.path.join(HERE, "dwarmup.npz")))


if __name__ == "__main__":
    main()
