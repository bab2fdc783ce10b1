"""Helpers shared by the fused-generator test modules (test_gpu_fused_highway.py, test_gpu_fused_sru.py,
test_gpu_fused_rnn_highway.py): batches, the step's discriminator masks, the oracle's re-sync between steps, the
comparisons, and host-only gantts_gan_step_t configurations for the configuration-rule tests."""
import numpy as np
import pytest
import torch

from conftest import WINDOWS
from oracle import gantts_port as gp

FAKE = 1 << 20          # placeholder device pointer: the configuration check and the workspace layout never dereference it


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__
    __graft_entry__.build()
    return torch.device("cuda:0")


def npy(t):
    return t.detach().cpu().numpy()


def step_hp(ohp):
    """gantts_b200.step.HParams of an oracle hparams dict."""
    from gantts_b200 import step as gstep
    return gstep.HParams(windows=WINDOWS[:ohp["num_windows"]], stream_sizes=ohp["stream_sizes"],
                         has_dynamic_features=ohp["has_dynamic_features"],
                         adversarial_streams=ohp["adversarial_streams"],
                         mask_nth_mgc_for_adv_loss=ohp["mask_nth_mgc_for_adv_loss"],
                         discriminator_linguistic_condition=ohp["discriminator_linguistic_condition"])


def ragged_lengths(B, T, seed):
    rng = np.random.RandomState(seed)
    return sorted([T] + [int(v) for v in rng.randint(T // 2, T, B - 1)], reverse=True)


def make_batch(B, T, d_in, d_out, lens, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, T, d_in, generator=g)
    y = torch.randn(B, T, d_out, generator=g)
    for b, n in enumerate(lens):
        x[b, n:] = 0
        y[b, n:] = 0
    return x, y


def sd_numpy(m):
    return {k: v.detach().cpu().numpy() for k, v in m.state_dict().items()}


def d_masks(fs, M, d_hidden, p, dev):
    """The discriminator's keep masks of the last training step (gantts_gan_step_seed: 1 = stacked real|fake, 2 = adv)."""
    from gantts_b200 import ops, _lib
    lib = _lib.load()
    s = fs.last_seed
    stacked = ops.mlp_dropout_masks(2 * M, d_hidden, p, lib.gantts_gan_step_seed(s, 1), dev)
    return {"real": [m[:M].cpu() for m in stacked], "fake": [m[M:].cpu() for m in stacked],
            "adv": [m.cpu() for m in ops.mlp_dropout_masks(M, d_hidden, p, lib.gantts_gan_step_seed(s, 2), dev)]}


def adv_loss_with(md, x, ys_ref, lens, ohp, adv_masks):
    """loss_adv of the oracle's y_hat_static through the PRODUCT's updated discriminator.  The adversarial forward runs
    after the discriminator's first Adagrad / Adam step, which moves every weight by about lr * sign(g): a weight whose
    gradient is within rounding of zero lands 2 lr apart in the two implementations, and at the conditioned D's 483
    inputs those few weights move loss_adv by a few 1e-4.  With the product's D on both sides the comparison isolates
    the generator's output and the loss arithmetic."""
    ps = list(md.parameters())
    layers = [(w.detach().cpu(), b.detach().cpu()) for w, b in zip(ps[0::2], ps[1::2])]
    fake_in = gp.get_selected_static_stream(ys_ref, ohp)
    if ohp["discriminator_linguistic_condition"]:
        fake_in = torch.cat((x, fake_in), -1)
    mask = gp.sequence_mask(lens, x.size(1)).unsqueeze(-1)
    D = gp.mlp_forward(fake_in, layers, last_sigmoid=True, masks=adv_masks)
    return float(gp.bce_real(D, mask, mask.sum().item()))


def loss_errors(got, ref, keys):
    return {k: abs(float(got[k]) - ref[k]) / max(abs(ref[k]), 1e-12) for k in keys}


def check_weights(model, named, tag, median=5e-6):
    """Every parameter of `model` against the oracle tensor of the same name: median |delta| below `median` and max
    <= 0.0201 (a first Adagrad / Adam step moves a weight by lr * sign(g))."""
    for k, v in model.named_parameters():
        d = np.abs(npy(v) - named[k].detach().numpy())
        assert np.median(d) < median and d.max() <= 0.0201, (tag, k, np.median(d), d.max())


def resync_oracle(fs, mg, md, gen, d_params, d_sums, g_opt=None, d_opt=None):
    """Start the oracle's next step from the product's weights and optimiser state: gen.named (keyed like
    mg.named_parameters()) with gen.sums or the Adam stepper g_opt in gen.named's order; d_params with d_sums or d_opt."""
    sd = fs.state_dict()
    order = list(gen.named)
    names = [n for n, _ in mg.named_parameters()]
    with torch.no_grad():
        for n, q in mg.named_parameters():
            gen.named[n].copy_(q.detach().cpu())
        for r, q in zip(d_params, md.parameters()):
            r.copy_(q.detach().cpu())
        for key, idx, sums, opt in (("optimizer_g", [order.index(n) for n in names], gen.sums, g_opt),
                                    ("optimizer_d", range(len(d_params)), d_sums, d_opt)):
            st = sd[key]["state"]
            for i, j in enumerate(idx):
                if opt is None:
                    sums[j].copy_(st[i]["sum"].cpu())
                else:
                    opt.m[j].copy_(st[i]["exp_avg"].cpu())
                    opt.v[j].copy_(st[i]["exp_avg_sq"].cpu())


def step_config(g_dims, d_dims, streams, static_cols, adv_cols, conditioned=False):
    """A gantts_gan_step_t with an MLP generator g_dims and discriminator d_dims, Adagrad, w_d = 1, B = 2 x T = 16 and no
    tensor tables yet (fill_tables); the caller adds its generator's shape block."""
    from gantts_b200 import _lib
    c = _lib.GanStepT()
    c.B, c.T = 2, 16
    for m, dims, act in ((c.g, g_dims, _lib.ACT_NONE), (c.d, d_dims, _lib.ACT_SIGMOID)):
        m.num_layers = len(dims) - 1
        for i, v in enumerate(dims):
            m.dims[i] = v
        m.last_act = act
    c.streams = _lib.make_streams(streams)
    c.windows = _lib.make_windows(WINDOWS)
    c.mlpg_table = FAKE
    c.n_static = c.n_static_cols = len(static_cols)
    for i, v in enumerate(static_cols):
        c.static_cols[i] = v
    c.n_adv = len(adv_cols)
    for i, v in enumerate(adv_cols):
        c.adv_cols[i] = v
    c.d_conditioned = int(conditioned)
    c.w_d, c.mge_w, c.adv_w, c.max_norm, c.lr_g, c.lr_d, c.eps = 1.0, 1.0, 1.0, 1.0, 0.01, 0.01, 1e-10
    c.optimizer = _lib.OPT_ADAGRAD
    return c


def fill_tables(c, n_g):
    """Placeholder tensors and Adagrad state for n_g generator tensors and the discriminator's 2 per layer."""
    for tab, n in ((c.g_tensors, n_g), (c.d_tensors, 2 * c.d.num_layers)):
        tab.n = n
        for i in range(n):
            tab.param[i] = tab.state[i] = FAKE
    return c


def use_adam(c, missing=()):
    """Switch c to Adam with exp_avg_sq for every tensor but the generator tensors in `missing`."""
    from gantts_b200 import _lib
    c.optimizer, c.beta1, c.beta2 = _lib.OPT_ADAM, 0.5, 0.9
    for tab in (c.g_tensors, c.d_tensors):
        for i in range(tab.n):
            tab.state2[i] = FAKE
    for i in missing:
        c.g_tensors.state2[i] = None


def config_checker():
    """(ws, err, rejected): the workspace size gantts_gan_step_workspace_bytes gives a config (0 = rejected), the last
    error message, and rejected(make, mutate, needle) asserting that mutate(make()) is rejected with `needle` in it."""
    import ctypes
    import __graft_entry__
    __graft_entry__.build()
    from gantts_b200 import _lib
    lib = _lib.load()
    ws = lambda c: lib.gantts_gan_step_workspace_bytes(ctypes.byref(c))
    err = lambda: lib.gantts_last_error_string().decode()

    def rejected(make, mutate, needle):
        c = make()
        mutate(c)
        assert ws(c) == 0 and needle in err(), (needle, err())
    return ws, err, rejected
