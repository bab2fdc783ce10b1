"""CPU-only tests of the discriminator's own optimiser (reference train.py:796-799 builds optimizer_g and optimizer_d from
their own hparams):

* the host-only rules of gantts_gan_step_t.d_opt that gantts_gan_step_workspace_bytes applies (placeholder device
  pointers: the checks run before anything touches the device) -- a zero-filled block keeps every configuration's
  acceptance and workspace exactly as they were before the block existed, mixed kinds need exp_avg_sq only for the Adam
  model, and each rule on the block is refused with its message;
* the ctypes mirror of the block against the C compiler's view of the header;
* gantts_b200.optim.OptimizerState (what FusedGanStep.opt_g / opt_d are) against torch.optim: param_groups as
  exp_lr_scheduler (train.py:323-333) writes them, state_dict / load_state_dict in both directions.
"""
import ctypes
import os
import subprocess

import pytest
import torch

from conftest import ROOT
from fused_step_helpers import (FAKE, TTS_STREAMS, _rhw_step_config, _rnn_d_config, _sru_step_config, _vc_step_config,
                                config_checker, fill_tables, step_config, use_adam)

# gantts_gan_step_workspace_bytes of these configurations before gantts_gan_step_t had the d_opt block (every one
# accepted; the same with Adagrad and with Adam on both models)
PARENT_WORKSPACE = {"mlp": 1495552, "highway": 1860352, "sru": 1831168, "rnn_highway": 2227968, "rnn_d": 1539840}


def _mlp_config():
    c = step_config([20, 32, 187], [58, 16, 1], TTS_STREAMS, list(range(60)) + [180, 183, 184], list(range(2, 60)))
    return fill_tables(c, 4)


def _configs():
    return {"mlp": _mlp_config, "highway": _vc_step_config, "sru": _sru_step_config, "rnn_highway": _rhw_step_config,
            "rnn_d": _rnn_d_config}


def _own(c, kind, beta1=0.5, beta2=0.9, eps=1e-8, opt_step=1):
    o = c.d_opt
    o.own, o.optimizer, o.beta1, o.beta2, o.eps, o.opt_step = 1, kind, beta1, beta2, eps, opt_step


@pytest.mark.parametrize("name", sorted(PARENT_WORKSPACE))
def test_zero_d_block_keeps_acceptance_and_workspace(name):
    """A zero-filled d_opt (every configuration built without it) is accepted with the workspace it had before the block
    existed, under Adagrad and under Adam; an own block repeating the top-level fields changes nothing either."""
    from gantts_b200 import _lib
    ws, err, _ = config_checker()
    make = _configs()[name]
    for adam in (False, True):
        c = make()
        if adam:
            use_adam(c)
        assert bytes(c.d_opt) == bytes(_lib.OptimizerT())
        assert ws(c) == PARENT_WORKSPACE[name], (name, adam, err())
        _own(c, c.optimizer, c.beta1, c.beta2, c.eps, 1)
        assert ws(c) == PARENT_WORKSPACE[name], (name, adam, err())


def test_mixed_kinds_need_exp_avg_sq_only_for_adam():
    """Adam G + Adagrad D and Adagrad G + Adam D are accepted with exp_avg_sq for the Adam model alone (the workspace does
    not depend on the optimisers); a missing exp_avg_sq of the Adam model is refused, naming that model."""
    from gantts_b200 import _lib
    ws, err, rejected = config_checker()
    base = PARENT_WORKSPACE["mlp"]

    def adam_g_adagrad_d():
        c = _mlp_config()
        c.optimizer, c.beta1, c.beta2 = _lib.OPT_ADAM, 0.5, 0.9
        for i in range(c.g_tensors.n):
            c.g_tensors.state2[i] = FAKE
        _own(c, _lib.OPT_ADAGRAD, 0.0, 0.0, 1e-10, 0)          # Adagrad reads neither betas nor the step number
        return c

    def adagrad_g_adam_d():
        c = _mlp_config()
        for i in range(c.d_tensors.n):
            c.d_tensors.state2[i] = FAKE
        _own(c, _lib.OPT_ADAM, 0.5, 0.9, 1e-8, 3)
        return c
    assert ws(adam_g_adagrad_d()) == base, err()
    assert ws(adagrad_g_adam_d()) == base, err()
    rejected(adam_g_adagrad_d, lambda c: c.g_tensors.state2.__setitem__(1, None),
             "Adam needs exp_avg_sq for generator tensor 1")
    rejected(adagrad_g_adam_d, lambda c: c.d_tensors.state2.__setitem__(2, None),
             "Adam needs exp_avg_sq for discriminator tensor 2")
    # with a zero block D follows G's kind: G Adagrad -> D needs no exp_avg_sq, G Adam -> it does
    c = _mlp_config()
    assert ws(c) == base
    c = adam_g_adagrad_d()
    c.d_opt = _lib.OptimizerT()
    assert ws(c) == 0 and "Adam needs exp_avg_sq for discriminator tensor 0" in err()


def test_d_block_rules_are_refused_with_their_message():
    from gantts_b200 import _lib
    ws, err, rejected = config_checker()

    def make():
        c = _mlp_config()
        for i in range(c.d_tensors.n):
            c.d_tensors.state2[i] = FAKE
        _own(c, _lib.OPT_ADAM, 0.5, 0.9, 1e-8, 1)
        return c
    assert ws(make()) > 0, err()
    rejected(make, lambda c: setattr(c.d_opt, "own", 2), "d_opt.own must be 0")
    rejected(make, lambda c: setattr(c.d_opt, "own", -1), "d_opt.own must be 0")
    rejected(make, lambda c: setattr(c.d_opt, "optimizer", 2), "unknown discriminator optimizer 2")
    rejected(make, lambda c: setattr(c.d_opt, "optimizer", -1), "unknown discriminator optimizer -1")
    rejected(make, lambda c: setattr(c.d_opt, "beta1", 1.0), "discriminator Adam betas out of range")
    rejected(make, lambda c: setattr(c.d_opt, "beta2", -0.1), "discriminator Adam betas out of range")
    rejected(make, lambda c: setattr(c.d_opt, "opt_step", 0), "discriminator Adam needs d_opt.opt_step >= 1")
    rejected(make, lambda c: setattr(c.d_opt, "opt_step", -5), "discriminator Adam needs d_opt.opt_step >= 1")
    # Adagrad reads neither: out-of-range betas and step 0 are accepted
    c = make()
    c.d_opt.optimizer, c.d_opt.beta1, c.d_opt.opt_step = _lib.OPT_ADAGRAD, 7.0, 0
    assert ws(c) > 0, err()
    # an own block is read whatever the top-level optimiser says; the top-level rules still hold for the generator
    rejected(make, lambda c: setattr(c, "optimizer", 5), "unknown optimizer 5")


def test_optimizer_block_layout_matches_header(tmp_path):
    """ctypes OptimizerT and GanStepT.d_opt against the C compiler: sizes and offsets; the block sits right before
    opt_step (opt_step and d_lstm stay the struct's last two fields)."""
    from gantts_b200 import _lib
    names = [f for f, _ in _lib.GanStepT._fields_]
    assert names[-3:] == ["d_opt", "opt_step", "d_lstm"]
    lines = ['  printf(" %zu", sizeof(gantts_optimizer_t));\n', '  printf(" %zu", offsetof(gantts_gan_step_t, d_opt));\n']
    want = [ctypes.sizeof(_lib.OptimizerT), _lib.GanStepT.d_opt.offset]
    for f, _ in _lib.OptimizerT._fields_:
        lines.append('  printf(" %%zu", offsetof(gantts_optimizer_t, %s));\n' % f)
        want.append(getattr(_lib.OptimizerT, f).offset)
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "gantts_b200.h"\nint main(void) {\n' + "".join(lines) +
                   "  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got == want


# ---- OptimizerState (host side; the tensors may live anywhere)
def exp_lr_scheduler(optimizer, epoch, nepoch, init_lr=0.0001, lr_decay_epoch=100):
    """Reference train.py:323-333 (the print left out): lr = init_lr * 0.1^(epoch // lr_decay_epoch) into every group."""
    lr = init_lr * (0.1 ** (epoch // lr_decay_epoch))
    for param_group in optimizer.param_groups:
        param_group['lr'] = lr
    return optimizer


def _state(kind, params, **hyper):
    from gantts_b200.optim import OptimizerState
    st = [torch.zeros_like(p) for p in params]
    st2 = [torch.zeros_like(p) for p in params] if kind == "Adam" else []
    return OptimizerState(kind, params, st, st2, **hyper)


def test_param_groups_are_the_hyper_parameters():
    params = [torch.zeros(3, 2), torch.zeros(3)]
    o = _state("Adam", params, lr=1e-3, betas=(0.5, 0.9))
    g = o.param_groups[0]
    assert len(o.param_groups) == 1 and len(g["params"]) == 2 and all(a is b for a, b in zip(g["params"], params))
    assert (g["lr"], g["betas"], g["eps"], g["weight_decay"]) == (1e-3, (0.5, 0.9), 1e-8, 0.0)
    for epoch, k in ((0, 0), (99, 0), (100, 1), (250, 2)):
        want = 1e-3 * (0.1 ** k)
        exp_lr_scheduler(o, epoch, 300, init_lr=1e-3, lr_decay_epoch=100)
        assert o.lr == want and o.param_groups[0]["lr"] == want
    o.weight_decay, o.eps, o.betas = 0.1, 1e-6, [0.8, 0.99]
    assert (g["weight_decay"], g["eps"], g["betas"]) == (0.1, 1e-6, (0.8, 0.99))
    a = _state("Adagrad", params)
    assert (a.lr, a.eps, a.weight_decay) == (0.01, 1e-10, 0.0)
    with pytest.raises(AttributeError):
        a.betas
    with pytest.raises(TypeError):
        _state("Adagrad", params, betas=(0.5, 0.9))
    with pytest.raises(RuntimeError, match="amsgrad=True is not implemented"):
        _state("Adam", params, amsgrad=True)
    with pytest.raises(RuntimeError, match="lr_decay=0.5 is not implemented"):
        _state("Adagrad", params, lr_decay=0.5)
    with pytest.raises(RuntimeError, match="no native optimiser 'SGD'"):
        _state("SGD", params)


@pytest.mark.parametrize("kind", ["Adagrad", "Adam"])
def test_state_dict_round_trips_through_torch_optim(kind):
    """Our state_dict loads into torch.optim.<kind> and torch's comes back, with every group field and the step; a
    torch.optim.Adam that has not stepped (empty state) loads as fresh state."""
    torch.manual_seed(3)
    params = [torch.randn(4, 3), torch.randn(4)]
    hyper = dict(lr=0.02, weight_decay=0.001, eps=1e-7) if kind == "Adagrad" else \
        dict(lr=2e-3, betas=(0.5, 0.9), weight_decay=0.01, eps=1e-7)
    o = _state(kind, params, **hyper)
    for ts in (o._state, o._state2):
        for t in ts:
            t.uniform_(0.0, 1.0)
    o.steps = 5
    ref = [p.clone().requires_grad_(True) for p in params]
    topt = getattr(torch.optim, kind)(ref, lr=1.0)
    topt.load_state_dict(o.state_dict())
    tg = topt.param_groups[0]
    for k, v in hyper.items():
        assert tg[k] == v, k
    keys = ("sum",) if kind == "Adagrad" else ("exp_avg", "exp_avg_sq")
    for i, p in enumerate(ref):
        assert float(topt.state[p]["step"]) == 5.0
        for k, ts in zip(keys, (o._state, o._state2)):
            assert torch.equal(topt.state[p][k], ts[i])
    # torch steps once, ours takes its state back
    for p in ref:
        p.grad = torch.ones_like(p)
    tg["lr"] = 0.5
    topt.step()
    back = _state(kind, params)
    back.load_state_dict(topt.state_dict())
    assert back.steps == 6 and back.lr == 0.5 and back.weight_decay == hyper["weight_decay"] and back.eps == hyper["eps"]
    if kind == "Adam":
        assert back.betas == (0.5, 0.9)
    for i, p in enumerate(ref):
        for k, ts in zip(keys, (back._state, back._state2)):
            assert torch.equal(topt.state[p][k], ts[i])
    if kind == "Adam":
        fresh = torch.optim.Adam([p.clone() for p in params], lr=3e-3, betas=(0.6, 0.95))
        back.load_state_dict(fresh.state_dict())
        assert back.steps == 0 and back.lr == 3e-3 and back.betas == (0.6, 0.95)
        assert all(not t.any() for t in back._state + back._state2)


def test_load_state_dict_refuses_what_the_native_step_does_not_do():
    params = [torch.zeros(2)]
    o = _state("Adam", params)
    sd = o.state_dict()
    sd["param_groups"][0]["amsgrad"] = True
    with pytest.raises(RuntimeError, match="amsgrad=True"):
        o.load_state_dict(sd)
    sd = torch.optim.Adam([torch.zeros(2, requires_grad=True)], decoupled_weight_decay=True).state_dict()
    with pytest.raises(RuntimeError, match="decoupled_weight_decay=True"):
        o.load_state_dict(sd)
    a = _state("Adagrad", params)
    with pytest.raises(RuntimeError, match="has no 'sum'"):
        a.load_state_dict({"state": {0: {"step": torch.tensor(1.0), "exp_avg": torch.zeros(2), "exp_avg_sq": torch.zeros(2)}},
                           "param_groups": [{"lr": 0.1, "params": [0]}]})
    with pytest.raises(RuntimeError, match="2 parameters, this optimiser 1"):
        a.load_state_dict(torch.optim.Adagrad([torch.zeros(2, requires_grad=True), torch.zeros(2, requires_grad=True)]).state_dict())
