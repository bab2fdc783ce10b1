"""Device-side epoch log of the training loop (reference train.py:531-595 per batch, :597-637 per phase).

``EpochLog.add`` enqueues one batch (gantts_epoch_log_add: the batch's objective distortions and its flagged losses,
correct counts and spoof count folded into an fp64 record on the device); ``EpochLog.read`` does the phase's one
synchronising read and returns the scalars train.py logs, under train.py's names.  Per batch nothing comes back to the
host, where train.py reads the losses and counts with ``.item()`` and pulls both (B, T, D) tensors for
compute_distortions."""
import ctypes

import numpy as np
import torch

from . import _lib
from . import multistream
from . import ops
from .fused import LOSS_NAMES

# compute_distortions' keys per hp.name (train.py:411-428), in its dict order, and their record slots
METRIC_NAMES = {"acoustic": ("mcd", "bap_mcd", "f0_rmse", "vuv_err"), "duration": ("dur_rmse",), "vc": ("mcd",)}
_METRIC_SLOT = {"mcd": 0, "bap_mcd": 1, "f0_rmse": 2, "vuv_err": 3, "dur_rmse": 4}
# train.py's running_loss keys (:476-480) for the step's loss scalars, in the order of its log loop (:610-616)
_LOSS_KEYS = (("mse", "loss_mse"), ("mge", "loss_mge"), ("discriminator", "loss_d"), ("loss_real_d", "loss_real_d"),
              ("loss_fake_d", "loss_fake_d"), ("loss_adv", "loss_adv"), ("generator", "loss_g"))


def log_config(hp):
    """(gantts_epoch_log_t, static columns) of hp: the static-column map of the fused step and the column groups of
    gantts_b200/metrics.py for hp.name acoustic / duration / vc."""
    nw = len(hp.windows)
    scols = multistream.static_feature_columns(nw, hp.stream_sizes, hp.has_dynamic_features,
                                               [True] * len(hp.stream_sizes))
    if len(scols) > _lib.MAX_COLS:
        raise RuntimeError("EpochLog: %d static columns (at most %d)" % (len(scols), _lib.MAX_COLS))
    c = _lib.EpochLogT()
    c.n_static = len(scols)
    for i, v in enumerate(scols):
        c.static_cols[i] = int(v)
    D = len(scols)
    if hp.name == "acoustic":
        s_mgc, s_lf0, s_vuv, s_bap = [int(v) for v in multistream.get_static_stream_sizes(
            hp.stream_sizes, hp.has_dynamic_features, nw)]
        c.kind = _lib.METRIC_ACOUSTIC
        c.cols = _lib.DistortionColsT(1, s_mgc - 1, s_mgc + s_lf0 + s_vuv, s_bap, s_mgc, s_mgc + s_lf0, 1, 0, 0)
    elif hp.name == "duration":
        c.kind = _lib.METRIC_DURATION
        c.cols = _lib.DistortionColsT(0, 0, 0, 0, -1, -1, 0, 0, D)
    elif hp.name == "vc":
        c.kind = _lib.METRIC_VC
        c.cols = _lib.DistortionColsT(0, D, 0, 0, -1, -1, 0, 0, 0)
    else:
        raise RuntimeError("EpochLog: unknown hparams name %r (acoustic, duration and vc are)" % (hp.name,))
    return c, [int(v) for v in scols]


class EpochLog(object):
    def __init__(self, hp, Y_data_mean, Y_data_std, device):
        """Y_data_mean / Y_data_std: the static+dynamic-domain statistics the loader scales y with (numpy or tensor);
        the log de-normalises each static column with the entry of the column it is read from, as train.py:358-380
        and metrics.py do."""
        lib = _lib.load()
        self.hp, self.device = hp, torch.device(device)
        self.cfg, scols = log_config(hp)
        nbytes = lib.gantts_epoch_log_workspace_bytes(ctypes.byref(self.cfg))
        if nbytes == 0:
            raise RuntimeError("gantts_b200 epoch_log config rejected: %s" % lib.gantts_last_error_string().decode())
        Ym, Ys = (np.asarray(v.cpu() if torch.is_tensor(v) else v, dtype=np.float64).reshape(-1)
                  for v in (Y_data_mean, Y_data_std))
        self.mean = torch.as_tensor(Ym[scols].astype(np.float32), device=self.device)
        self.std = torch.as_tensor(Ys[scols].astype(np.float32), device=self.device)
        self._ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        self.record = torch.zeros(_lib.LOG_SLOTS, dtype=torch.float64, device=self.device)
        self.metric_names = METRIC_NAMES[hp.name]
        self._flags = None

    def reset(self):
        """Zero the record on the current stream (a new phase)."""
        _lib.check(_lib.load().gantts_epoch_log_reset(self.record.data_ptr(), ops._stream()))
        self._flags = None

    def add(self, losses12, y, y_hat_static, lengths, update_d, update_g, spoof=None):
        """Fold one batch: losses12 the step's 12 loss scalars (fused.LOSS_NAMES order, CUDA float32), y the step's
        input (b, t, static + dynamic), y_hat_static (b, t, n_static) with any batch / time strides, lengths CUDA int64
        (b,), spoof the reference discriminator's count (CUDA float32 scalar) or None.  Enqueue-only."""
        key = (bool(update_d), bool(update_g), spoof is not None)
        if self._flags is None:
            self._flags = key
        elif self._flags != key:
            raise RuntimeError("EpochLog: every batch of a phase is logged with the same update_d / update_g / spoof")
        ops.require_cuda(losses12, y, y_hat_static, spoof)
        if losses12.numel() != len(LOSS_NAMES) or not losses12.is_contiguous():
            raise RuntimeError("EpochLog: losses12 must be a contiguous vector of %d scalars" % len(LOSS_NAMES))
        if y.dim() != 3 or y_hat_static.dim() != 3 or tuple(y.shape[:2]) != tuple(y_hat_static.shape[:2]):
            raise RuntimeError("EpochLog: y and y_hat_static must be (b, t, .) of the same b, t")
        if y.stride(2) != 1 or y_hat_static.stride(2) != 1 or y_hat_static.shape[2] != self.cfg.n_static:
            raise RuntimeError("EpochLog: y and y_hat_static need unit column stride and y_hat_static %d columns"
                               % self.cfg.n_static)
        b, t = int(y.shape[0]), int(y.shape[1])
        if not lengths.is_cuda or lengths.dtype != torch.int64 or tuple(lengths.shape) != (b,):
            raise RuntimeError("EpochLog: lengths must be a CUDA int64 tensor of shape (b,) = (%d,)" % b)
        flags = ((_lib.LOG_UPDATE_D if update_d else 0) | (_lib.LOG_UPDATE_G if update_g else 0) |
                 (_lib.LOG_SPOOF if spoof is not None else 0))
        lib = _lib.load()
        _lib.check(lib.gantts_epoch_log_add(
            ctypes.byref(self.cfg), flags, losses12.data_ptr(), spoof.data_ptr() if spoof is not None else None,
            y.data_ptr(), y.stride(0), y.stride(1), int(y.shape[2]), y_hat_static.data_ptr(), y_hat_static.stride(0),
            y_hat_static.stride(1), lengths.data_ptr(), b, t, self.mean.data_ptr(), self.std.data_ptr(),
            self.record.data_ptr(), self._ws.data_ptr(), self._ws.numel(), ops._stream()))

    def read(self, phase, mse_w=0.0, mge_w=1.0):
        """The phase's one synchronising read: the dict of scalars train.py:597-637 logs for `phase` under the
        update_d / update_g / reference-D settings the batches were added with, in its order.  ``self.sums`` then holds
        the raw sums (N, total_num_frames, every loss name, spoof_count and the metric sums)."""
        r = self.record.tolist()
        update_d, update_g, spoof = self._flags or (False, False, False)
        N, frames = r[_lib.LOG_N], r[_lib.LOG_FRAMES]
        loss = dict(zip(LOSS_NAMES, r[_lib.LOG_LOSSES:_lib.LOG_LOSSES + len(LOSS_NAMES)]))
        metrics = {k: r[_lib.LOG_METRICS + _METRIC_SLOT[k]] for k in self.metric_names}
        self.sums = dict(N=N, total_num_frames=frames, spoof_count=r[_lib.LOG_SPOOFED], **loss)
        self.sums.update({"metric " + k: v for k, v in metrics.items()})
        out = {}
        if update_d and update_g and phase == "train":
            e_mge = (mse_w * loss["loss_mse"] + mge_w * loss["loss_mge"]) / N
            e_adv = loss["loss_adv"] / N
            out["E(mge)"], out["E(adv)"] = e_mge, e_adv
            out["MGE/ADV loss weight"] = e_mge / e_adv
        enabled = {"mse": update_g, "mge": update_g, "discriminator": update_d, "loss_real_d": update_d,
                   "loss_fake_d": update_d, "loss_adv": update_g and update_d, "generator": update_g}
        for ty, name in _LOSS_KEYS:
            if enabled[ty]:
                out["%s %s loss" % (phase, ty)] = loss[name] / N
        if update_g:
            for k, v in metrics.items():
                out["%s %s metric" % (phase, k)] = v / N
        if update_d:
            out["Real %s acc" % phase] = loss["real_correct"] / frames
            out["Fake %s acc" % phase] = loss["fake_correct"] / frames
        if spoof:
            out["%s spoofing rate" % phase] = r[_lib.LOG_SPOOFED] / frames
        return out
