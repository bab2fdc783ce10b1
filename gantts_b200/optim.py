"""clip_grad_norm_(params, max_norm) + torch.optim.Adagrad.step() / torch.optim.Adam.step() as ONE native pass
(gantts_grad_sumsq + gantts_clip_adagrad_step / gantts_clip_adam_step), replacing reference
train.py:275-276,317-318 (optimisers of hparams.py:223-227,240-244,125-130)."""
import ctypes

import torch

from . import _lib
from . import ops


# torch.optim's param_groups entries of the two optimisers hparams.py uses, with their defaults, in torch's key order
GROUP_DEFAULTS = {
    "Adagrad": dict(lr=0.01, lr_decay=0, eps=1e-10, weight_decay=0.0, initial_accumulator_value=0, foreach=None,
                    maximize=False, differentiable=False, fused=None),
    "Adam": dict(lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, amsgrad=False, maximize=False, foreach=None,
                 capturable=False, differentiable=False, fused=None),
}
STATE_KEYS = {"Adagrad": ("sum",), "Adam": ("exp_avg", "exp_avg_sq")}
# group settings of torch.optim the native update does not implement: (key, value the native update implements)
_FIXED = (("lr_decay", 0), ("amsgrad", False), ("maximize", False), ("decoupled_weight_decay", False))


def _check_fixed(group, kind, who):
    for k, want in _FIXED:
        if k in group and group[k] != want:
            raise RuntimeError("%s: %s=%r is not implemented by the native %s step" % (who, k, group[k], kind))


def _group_value(key, v):
    if key in ("lr", "eps", "weight_decay"):
        return float(v)
    if key == "betas":
        return (float(v[0]), float(v[1]))
    return v


class OptimizerState(object):
    """One model's optimiser as reference train.py sees it: ``param_groups`` (a single group, read by every step, so
    exp_lr_scheduler of train.py:323-333 can set ``param_groups[0]["lr"]``), ``state_dict()`` and ``load_state_dict()``
    in the layout of torch.optim.Adagrad / torch.optim.Adam (save_checkpoint / load_checkpoint of train.py:162-171,
    :651-658 exchange files with those classes).  ``state`` / ``state2`` are the per-parameter state tensors (Adagrad:
    sum; Adam: exp_avg, exp_avg_sq), updated in place by whoever steps the model; ``steps`` counts its steps.  ``.lr``,
    ``.weight_decay``, ``.eps`` and (Adam) ``.betas`` read and write the group."""

    def __init__(self, kind, params, state, state2, **hyper):
        if kind not in GROUP_DEFAULTS:
            raise RuntimeError("gantts_b200: no native optimiser %r (Adagrad and Adam are the ones hparams.py uses)" % kind)
        group = dict(GROUP_DEFAULTS[kind])
        for k, v in hyper.items():
            if k not in group:
                raise TypeError("%s got an unexpected hyper-parameter %r" % (kind, k))
            group[k] = _group_value(k, v)
        _check_fixed(group, kind, type(self).__name__)
        group["params"] = list(params)
        self.kind = kind
        self.param_groups = [group]
        self._state, self._state2 = list(state), list(state2)
        self.steps = 0

    def _hyper(self, key):
        if key not in self.param_groups[0]:
            raise AttributeError("%s (%s) has no %s" % (type(self).__name__, self.kind, key))
        return self.param_groups[0][key]

    def _set_hyper(self, key, v):
        if key not in self.param_groups[0]:
            raise AttributeError("%s (%s) has no %s" % (type(self).__name__, self.kind, key))
        self.param_groups[0][key] = _group_value(key, v)

    lr = property(lambda self: self._hyper("lr"), lambda self, v: self._set_hyper("lr", v))
    weight_decay = property(lambda self: self._hyper("weight_decay"), lambda self, v: self._set_hyper("weight_decay", v))
    eps = property(lambda self: self._hyper("eps"), lambda self, v: self._set_hyper("eps", v))
    betas = property(lambda self: self._hyper("betas"), lambda self, v: self._set_hyper("betas", v))

    def state_dict(self):
        keys = STATE_KEYS[self.kind]
        tensors = [self._state] + ([self._state2] if len(keys) > 1 else [])
        state = {}
        for i in range(len(self._state)):
            e = {"step": torch.tensor(float(self.steps))}
            for k, ts in zip(keys, tensors):
                e[k] = ts[i].detach().clone()
            state[i] = e
        group = {k: v for k, v in self.param_groups[0].items() if k != "params"}
        group["params"] = list(range(len(self._state)))
        return {"state": state, "param_groups": [group]}

    def load_state_dict(self, sd):
        """State and every group field of a state_dict in torch.optim layout (ours or torch.optim's own).  An empty
        ``state`` (a torch.optim.Adam that has not stepped) is fresh state; a missing ``step`` keeps ``steps``."""
        name = type(self).__name__
        groups = sd.get("param_groups") or [{}]
        if len(groups) != 1:
            raise RuntimeError("%s.load_state_dict: %d parameter groups, the native step has one" % (name, len(groups)))
        grp = groups[0]
        _check_fixed(grp, self.kind, name + ".load_state_dict")
        if "params" in grp and len(grp["params"]) != len(self._state):
            raise RuntimeError("%s.load_state_dict: the state_dict has %d parameters, this optimiser %d"
                               % (name, len(grp["params"]), len(self._state)))
        st = sd["state"]
        keys = STATE_KEYS[self.kind]
        tensors = [self._state] + ([self._state2] if len(keys) > 1 else [])
        if not st:
            for ts in tensors:
                for t in ts:
                    t.zero_()
            self.steps = 0
        for i in range(len(self._state) if st else 0):
            e = st.get(i, st.get(str(i)))
            if e is None:
                raise RuntimeError("%s.load_state_dict: no state for parameter %d" % (name, i))
            for k, ts in zip(keys, tensors):
                if k not in e:
                    raise RuntimeError("%s.load_state_dict: parameter %d has no %r (a %s state_dict?)"
                                       % (name, i, k, "Adam" if self.kind == "Adagrad" else "Adagrad"))
                ts[i].copy_(e[k])
            if "step" in e:
                self.steps = int(float(e["step"]))
        for k in self.param_groups[0]:
            if k != "params" and k in grp:
                self._set_hyper(k, grp[k])


class _ClipOptimizer(object):
    """Flat-buffer optimiser base: ``.grad`` of every parameter is a view into ``flat_grad`` (one buffer => one
    NCCL all-reduce per model under data parallelism); global-norm clipping precedes the update."""

    def __init__(self, params, max_norm=1.0):
        self.params = [p for p in params]
        if not self.params:
            raise RuntimeError("%s: empty parameter list" % type(self).__name__)
        for p in self.params:
            ops.require_cuda(p)
            if not p.is_contiguous():
                raise RuntimeError("%s: parameters must be contiguous" % type(self).__name__)
        self.max_norm = float(max_norm)
        dev = self.params[0].device
        self.total = sum(p.numel() for p in self.params)
        self.flat_grad = torch.zeros(self.total, dtype=torch.float32, device=dev)
        self.sumsq = torch.zeros(1, dtype=torch.float32, device=dev)
        self._grads = self._views(self.flat_grad)
        for p, g in zip(self.params, self._grads):
            p.grad = g
        n = len(self.params)
        self._n = n
        self._sizes = (ctypes.c_int64 * n)(*[p.numel() for p in self.params])
        self._ws = torch.empty(_lib.load().gantts_optim_workspace_bytes(), dtype=torch.uint8, device=dev)
        self.steps = 0

    def _views(self, flat):
        out, off = [], 0
        for p in self.params:
            n = p.numel()
            out.append(flat[off:off + n].view_as(p))
            off += n
        return out

    def _ptrs(self, tensors):
        return (ctypes.c_void_p * self._n)(*[t.data_ptr() for t in tensors])

    def zero_grad(self):
        self.flat_grad.zero_()
        for p, g in zip(self.params, self._grads):
            if p.grad is not g:
                p.grad = g

    def _sumsq(self):
        lib = _lib.load()
        for p, g in zip(self.params, self._grads):
            if p.grad is not g:
                raise RuntimeError("%s: .grad was re-bound; use zero_grad() of this optimizer" % type(self).__name__)
        _lib.check(lib.gantts_grad_sumsq(self._ptrs(self._grads), self._sizes, self._n, self.sumsq.data_ptr(),
                                         self._ws.data_ptr(), self._ws.numel(), ops._stream()))

    def grad_norm(self):
        """Device tensor: total gradient norm seen by the last step (before clipping)."""
        return self.sumsq.sqrt()


class ClipAdagrad(_ClipOptimizer, OptimizerState):
    """Adagrad (lr_decay=0, initial_accumulator_value=0, eps=1e-10) preceded by global-norm clipping."""

    def __init__(self, params, lr=0.01, weight_decay=0.0, max_norm=1.0, eps=1e-10):
        _ClipOptimizer.__init__(self, params, max_norm)
        self.flat_sum = torch.zeros_like(self.flat_grad)
        self._sums = self._views(self.flat_sum)
        OptimizerState.__init__(self, "Adagrad", self.params, self._sums, [], lr=lr, weight_decay=weight_decay, eps=eps)

    def step(self):
        lib = _lib.load()
        g = self.param_groups[0]
        self._sumsq()
        _lib.check(lib.gantts_clip_adagrad_step(self._ptrs(self.params), self._ptrs(self._grads),
                                                self._ptrs(self._sums), self._sizes, self._n,
                                                self.sumsq.data_ptr(), self.max_norm, float(g["lr"]),
                                                float(g["weight_decay"]), float(g["eps"]), ops._stream()))
        self.steps += 1

    def load_state_dict(self, sd):
        if "state" in sd:
            OptimizerState.load_state_dict(self, sd)
        else:                                   # round-1 layout
            for s, v in zip(self._sums, sd["sum"]):
                s.copy_(v)
            self.steps = int(sd.get("steps", 0))


class ClipAdam(_ClipOptimizer, OptimizerState):
    """torch.optim.Adam (amsgrad off) preceded by global-norm clipping: the duration model's optimiser
    (reference hparams.py:125-130: lr 1e-3, betas (0.5, 0.9), weight_decay 0)."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), weight_decay=0.0, max_norm=1.0, eps=1e-8):
        _ClipOptimizer.__init__(self, params, max_norm)
        self.flat_m, self.flat_v = torch.zeros_like(self.flat_grad), torch.zeros_like(self.flat_grad)
        self._m, self._v = self._views(self.flat_m), self._views(self.flat_v)
        OptimizerState.__init__(self, "Adam", self.params, self._m, self._v, lr=lr, betas=betas,
                                weight_decay=weight_decay, eps=eps)

    def step(self):
        lib = _lib.load()
        g = self.param_groups[0]
        b1, b2 = g["betas"]
        self._sumsq()
        self.steps += 1
        _lib.check(lib.gantts_clip_adam_step(self._ptrs(self.params), self._ptrs(self._grads), self._ptrs(self._m),
                                             self._ptrs(self._v), self._sizes, self._n, self.sumsq.data_ptr(),
                                             self.max_norm, float(g["lr"]), float(b1), float(b2),
                                             float(g["weight_decay"]), float(g["eps"]), self.steps, ops._stream()))


def make_optimizer(name, params, **kw):
    """``getattr(optim, hp.optimizer_g)(params, **hp.optimizer_g_params)`` of reference train.py:784-789 for the
    native classes."""
    if name == "Adagrad":
        return ClipAdagrad(params, **kw)
    if name == "Adam":
        return ClipAdam(params, **kw)
    raise RuntimeError("gantts_b200: no native optimiser %r (Adagrad and Adam are the ones hparams.py uses)" % name)
