# coding: utf-8
"""Trainining script for GAN-based TTS and VC models.

usage: train.py [options] <inputs_dir> <outputs_dir>

options:
    --hparams_name=<name>       Name of hyper params [default: vc].
    --hparams=<parmas>          Hyper parameters to be overrided [default: ].
    --checkpoint-dir=<dir>      Where to save models [default: checkpoints].
    --checkpoint-g=<name>       Load generator from checkpoint if given.
    --checkpoint-d=<name>       Load discriminator from checkpoint if given.
    --checkpoint-r=<name>       Load reference model to compute spoofing rate.
    --max_files=<N>             Max num files to be collected. [default: -1]
    --discriminator-warmup      Warmup discriminator.
    --w_d=<f>                   Adversarial (ADV) loss weight [default: 1.0].
    --mse_w=<f>                 Mean squared error (MSE) loss weight [default: 0.0].
    --mge_w=<f>                 Minimum generation error (MGE) loss weight [default: 1.0].
    --restart_epoch=<N>         Restart epoch [default: -1].
    --reset_optimizers          Reset optimizers, otherwise restored from checkpoint.
    --log-event-path=<name>     Log event path.
    --disable-slack             Disable slack message.
    -h, --help                  Show this help message and exit
"""
# The usage above is the reference train.py's, so each `python train.py ...` line of train_gan.sh runs as
# `python -m gantts_b200.train ...`.  The step is FusedGanStep (one native call per mini-batch) whenever it takes the
# models, else GanTrainer; each phase's logged values accumulate on the device (epochlog.EpochLog) and are read once
# per phase.  Each split's normalised features stay on the device when they fit (DeviceBatches), so a mini-batch is
# one gather kernel rather than a host collate and copy.  --disable-slack is accepted and does nothing.
import json
import os
import sys
import time
from os.path import abspath, exists, join, splitext
from warnings import warn

import numpy as np
import torch
from torch.utils import data as data_utils

from . import models
from . import multistream
from . import ops
from .epochlog import EpochLog
from .fused import LOSS_NAMES, FusedGanStep
from .step import GanTrainer

test_size = 0.112           # train.py:64-66
random_state = 1234
checkpoint_interval = 10


# ---- data (train.py:71-159, 701-770) ----

def train_test_split_files(files, test_size=test_size, random_state=random_state):
    """sklearn's train_test_split(files, test_size=, random_state=) (ShuffleSplit: ceil(test_size n) test items, the
    first ones of RandomState(random_state).permutation(n), the train items next), without needing sklearn."""
    n = len(files)
    n_test = int(np.ceil(test_size * n))
    perm = np.random.RandomState(random_state).permutation(n)
    return [files[i] for i in perm[n_test:]], [files[i] for i in perm[:n_test]]


def npy_files(dirname, train=True, max_files=None, test=False):
    """NPYDataSource.collect_files (train.py:78-90): the sorted .npy files, the last 5 held out, the rest split."""
    files = sorted(join(dirname, d) for d in os.listdir(dirname) if splitext(d)[-1] == ".npy")
    if test:
        return files[len(files) - 5:]
    files = files[:len(files) - 5]
    if max_files is not None and max_files > 0:
        files = files[:max_files]
    train_files, test_files = train_test_split_files(files)
    return train_files if train else test_files


class NpyDataset(object):
    """FileSourceDataset(NPYDataSource) behind a MemoryCacheDataset of cache_size utterances."""

    def __init__(self, files, cache_size=1200):
        self.files, self.cache_size, self.cache = list(files), cache_size, {}

    def __getitem__(self, idx):
        if idx not in self.cache:
            if len(self.cache) >= self.cache_size:
                self.cache.pop(next(iter(self.cache)))
            self.cache[idx] = np.load(self.files[idx])
        return self.cache[idx]

    def __len__(self):
        return len(self.files)


def meanvar(datasets, lengths=None):
    """Per-column mean and variance (float64, ddof 0) over the frames of every utterance of `datasets` in turn, the
    first lengths[i] of utterance i when lengths are given (train.py:725-730: vc's statistics are joint over X then Y)."""
    def frames():
        for ds in datasets:
            for i in range(len(ds)):
                x = np.asarray(ds[i], dtype=np.float64)
                yield x if lengths is None else x[:lengths[i]]
    n, s = 0, 0.0
    for x in frames():
        n, s = n + len(x), s + x.sum(axis=0)
    mean = s / n
    ss = 0.0
    for x in frames():
        ss = ss + ((x - mean) ** 2).sum(axis=0)
    return mean, ss / n


def minmax(dataset):
    mn = mx = None
    for i in range(len(dataset)):
        a, b = dataset[i].min(axis=0), dataset[i].max(axis=0)
        mn, mx = (a, b) if mn is None else (np.minimum(mn, a), np.maximum(mx, b))
    return mn, mx


def minmax_scale_params(data_min, data_max, feature_range=(0.01, 0.99)):
    data_range = data_max - data_min
    scale_ = (feature_range[1] - feature_range[0]) / np.where(data_range == 0, 1.0, data_range)
    return feature_range[0] - data_min * scale_, scale_


class VCDataset(object):
    def __init__(self, X, Y, data_mean, data_std):
        self.X, self.Y, self.data_mean, self.data_std = X, Y, data_mean, data_std

    def __getitem__(self, idx):
        return ((self.X[idx] - self.data_mean) / self.data_std, (self.Y[idx] - self.data_mean) / self.data_std)

    def __len__(self):
        return len(self.X)


class TTSDataset(object):
    def __init__(self, X, Y, X_data_min, X_data_max, Y_data_mean, Y_data_std, hp):
        self.X, self.Y, self.hp = X, Y, hp
        self.X_data_min, self.X_data_scale = minmax_scale_params(X_data_min, X_data_max)
        self.Y_data_mean, self.Y_data_std = Y_data_mean, Y_data_std

    def __getitem__(self, idx):
        x = self.X[idx] * self.X_data_scale + self.X_data_min
        y = (self.Y[idx] - self.Y_data_mean) / self.Y_data_std
        if self.hp.recompute_delta_features:
            y = multistream.recompute_delta_features(y, self.Y_data_mean, self.Y_data_std, self.hp.windows,
                                                     self.hp.stream_sizes, self.hp.has_dynamic_features)
        return x, y

    def __len__(self):
        return len(self.X)


def collate_fn(batch):
    """train.py:145-159 with int64 lengths (np.int is gone from numpy)."""
    input_lengths = np.array([len(x[0]) for x in batch], dtype=np.int64)
    max_len = np.max(input_lengths)
    pad = lambda a: np.pad(a, [(0, max_len - len(a)), (0, 0)], mode="constant", constant_values=0)
    x_batch = torch.from_numpy(np.array([pad(x[0]) for x in batch], dtype=np.float32))
    y_batch = torch.from_numpy(np.array([pad(x[1]) for x in batch], dtype=np.float32))
    return x_batch, y_batch, torch.from_numpy(input_lengths)


def sort_batch(x, y, lengths):
    """train.py:494-501 on the host: the batch sorted by length, descending."""
    sorted_lengths, indices = torch.sort(lengths.view(-1), dim=0, descending=True)
    return x[indices], y[indices], sorted_lengths.long()


def _indices(batch):
    return np.asarray(batch, dtype=np.int64)


def pack_corpus(dataset):
    """Every utterance of `dataset` (pairs of frame arrays) as collate_fn casts it, float32, packed frame after frame:
    (X (N, Dx), Y (N, Dy), lengths int64 per utterance)."""
    xs, ys = [], []
    for i in range(len(dataset)):
        x, y = dataset[i]
        xs.append(np.asarray(x, dtype=np.float32))
        ys.append(np.asarray(y, dtype=np.float32))
    lengths = np.array([len(x) for x in xs], dtype=np.int64)
    return np.concatenate(xs), np.concatenate(ys), lengths


class BatchPlan(object):
    """The host side of DeviceBatches: which utterances make each mini-batch, in which row order.  The batches and the
    draws from the global torch RNG are those of a DataLoader over the dataset with the same batch_size and shuffle,
    because a DataLoader over the indices alone makes them; each batch's rows are sorted by sort_batch's torch.sort."""

    def __init__(self, lengths, batch_size, shuffle):
        self.lengths = np.asarray(lengths, dtype=np.int64)
        self.starts = np.concatenate([[0], np.cumsum(self.lengths)[:-1]]).astype(np.int64)
        self.index_loader = data_utils.DataLoader(range(len(self.lengths)), batch_size=batch_size, shuffle=shuffle,
                                                  collate_fn=_indices)

    def __len__(self):
        return len(self.index_loader)

    def epoch(self):
        """One epoch: (plan int64 (2, rows), bounds).  plan[0] holds each row's first frame in the pack and plan[1]
        its length, batch after batch; batch j is rows bounds[j]:bounds[j + 1]."""
        rows, bounds = [], [0]
        for idx in self.index_loader:
            _, order = torch.sort(torch.from_numpy(self.lengths[idx]), dim=0, descending=True)
            rows.append(idx[order.numpy()])
            bounds.append(bounds[-1] + len(idx))
        rows = np.concatenate(rows) if rows else np.zeros(0, dtype=np.int64)
        return np.stack([self.starts[rows], self.lengths[rows]]), bounds


class DeviceBatches(object):
    """One split's normalised features resident on the device, batched as a DataLoader over `dataset` with collate_fn,
    then sort_batch, batches them, bit for bit and with the same draws from the global torch RNG.  Each utterance is
    normalised once, here, by the dataset's own __getitem__.  Iterating yields (x, y, lengths, host lengths) per batch:
    x, y padded on the device by one gantts_corpus_gather launch, lengths a slice of the epoch's plan, which is copied to
    the device once per epoch.  Nothing is copied per batch and nothing waits for the device."""

    def __init__(self, dataset, batch_size, shuffle, device):
        X, Y, lengths = pack_corpus(dataset)
        self.plan = BatchPlan(lengths, batch_size, shuffle)
        self.X = torch.from_numpy(X).to(device)
        self.Y = torch.from_numpy(Y).to(device)
        self.device = device

    def __len__(self):
        return len(self.plan)

    def __iter__(self):
        plan, bounds = self.plan.epoch()
        # A fresh pinned buffer per epoch: the host allocator does not hand it out again before the copy has read it.
        staged = torch.empty(plan.shape, dtype=torch.int64, pin_memory=True)
        staged.numpy()[...] = plan
        dev = staged.to(self.device, non_blocking=True)
        for j in range(len(bounds) - 1):
            s, e = bounds[j], bounds[j + 1]
            lengths = dev[1, s:e]
            x, y = ops.corpus_gather(self.X, self.Y, dev[0, s:e], lengths, int(plan[1, s]))
            yield x, y, lengths, plan[1, s:e].tolist()


def device_corpus_budget():
    """Bytes the resident corpus may take on the current CUDA device: half of its free memory (0 without CUDA)."""
    if not torch.cuda.is_available():
        return 0
    return torch.cuda.mem_get_info()[0] // 2


def load_data(hp, inputs_dir, outputs_dir, max_files):
    """Datasets, statistics (saved to data_dir under the reference's names), derived dims and the two loaders
    (train.py:701-770).  Returns (loaders, Y_data_mean, Y_data_std, longest utterance of either split).

    The loaders are DeviceBatches when both splits fit in device_corpus_budget() and every utterance has a frame, else
    train.py's DataLoaders; both give the same batches from the same RNG draws."""
    data_dir = abspath(join(inputs_dir, os.pardir))
    assert data_dir == abspath(join(outputs_dir, os.pardir))
    X, Y, utt_lengths = {}, {}, {}
    for phase in ("train", "test"):
        train = phase == "train"
        X[phase] = NpyDataset(npy_files(inputs_dir, train=train, max_files=max_files), hp.cache_size)
        Y[phase] = NpyDataset(npy_files(outputs_dir, train=train, max_files=max_files), hp.cache_size)
        x_lengths = np.array([len(x) for x in (X[phase][i] for i in range(len(X[phase])))])
        y_lengths = np.array([len(y) for y in (Y[phase][i] for i in range(len(Y[phase])))])
        assert np.allclose(x_lengths, y_lengths)
        utt_lengths[phase] = x_lengths
        print("Size of dataset for {}: {}".format(phase, len(X[phase])))
    longest = int(max(int(v.max()) for v in utt_lengths.values() if len(v)))
    if hp.name == "vc":
        # joint mean / var over the valid frames of X, then Y (train.py:725-730)
        data_mean, data_var = meanvar([X["train"], Y["train"]], utt_lengths["train"])
        data_std = np.sqrt(data_var)
        np.save(join(data_dir, "data_mean"), data_mean)
        np.save(join(data_dir, "data_var"), data_var)
        if hp.generator_params["in_dim"] is None:
            hp.generator_params["in_dim"] = data_mean.shape[-1]
        if hp.generator_params["out_dim"] is None:
            hp.generator_params["out_dim"] = data_mean.shape[-1]
        make = lambda p: VCDataset(X[p], Y[p], data_mean, data_std)
        Y_mean, Y_std = data_mean, data_std
    else:
        ty = "acoustic" if hp.name == "acoustic" else "duration"
        X_data_min, X_data_max = minmax(X["train"])
        Y_data_mean, Y_data_var = meanvar([Y["train"]])
        Y_data_std = np.sqrt(Y_data_var)
        np.save(join(data_dir, "X_{}_data_min".format(ty)), X_data_min)
        np.save(join(data_dir, "X_{}_data_max".format(ty)), X_data_max)
        np.save(join(data_dir, "Y_{}_data_mean".format(ty)), Y_data_mean)
        np.save(join(data_dir, "Y_{}_data_var".format(ty)), Y_data_var)
        derive_tts_dims(hp, X_data_min.shape[-1], Y_data_mean.shape[-1])
        make = lambda p: TTSDataset(X[p], Y[p], X_data_min, X_data_max, Y_data_mean, Y_data_std, hp)
        Y_mean, Y_std = Y_data_mean, Y_data_std
    frames = sum(int(v.sum()) for v in utt_lengths.values())
    widths = [(X[p][0].shape[-1], Y[p][0].shape[-1]) for p in ("train", "test") if len(X[p])][0]
    corpus_mb = frames * sum(widths) * 4 / 2**20
    # A batch whose utterances all have 0 frames pads to t = 0, which collate_fn returns and the gather refuses.
    empty = any(len(v) and v.min() < 1 for v in utt_lengths.values())
    budget = 0 if empty else device_corpus_budget()
    if all(len(X[p]) for p in ("train", "test")) and frames * sum(widths) * 4 <= budget:
        device = torch.device("cuda", torch.cuda.current_device())
        loaders = {p: DeviceBatches(make(p), hp.batch_size, p == "train", device) for p in ("train", "test")}
        print("Data loader: device corpus on {}, {} frames x ({} + {}) float32 columns = {:.1f} MB".format(
            device, frames, widths[0], widths[1], corpus_mb))
    else:
        loaders = {p: data_utils.DataLoader(make(p), batch_size=hp.batch_size, num_workers=hp.num_workers,
                                            pin_memory=hp.pin_memory, shuffle=(p == "train"), collate_fn=collate_fn)
                   for p in ("train", "test")}
        if empty:
            print("Data loader: host DataLoader (an utterance has no frames)")
        else:
            print("Data loader: host DataLoader, corpus {:.1f} MB, device budget {:.1f} MB".format(corpus_mb,
                                                                                                budget / 2**20))
    return loaders, Y_mean, Y_std, longest


def derive_tts_dims(hp, x_dim, y_dim):
    """in_dim / out_dim of the TTS generator and discriminator left None in hparams.py (train.py:753-768)."""
    if hp.generator_params["in_dim"] is None:
        D = x_dim
        if hp.generator_add_noise:
            D = D + hp.generator_noise_dim
        hp.generator_params["in_dim"] = D
    if hp.generator_params["out_dim"] is None:
        hp.generator_params["out_dim"] = y_dim
    if hp.discriminator_params["in_dim"] is None:
        sizes = multistream.get_static_stream_sizes(hp.stream_sizes, hp.has_dynamic_features, len(hp.windows))
        D = int(np.array(sizes[hp.adversarial_streams]).sum())
        if hp.adversarial_streams[0]:
            D -= hp.mask_nth_mgc_for_adv_loss
        if hp.discriminator_linguistic_condition:
            D = D + x_dim
        hp.discriminator_params["in_dim"] = D


# ---- optimisers and checkpoints (train.py:162-171, 323-333, 651-658) ----

def exp_lr_scheduler(optimizer, epoch, nepoch, init_lr=0.0001, lr_decay_epoch=100):
    """Decay learning rate by a factor of 0.1 every lr_decay_epoch epochs."""
    lr = init_lr * (0.1 ** (epoch // lr_decay_epoch))
    if epoch % lr_decay_epoch == 0:
        print('LR is set to {} at epoch {}'.format(lr, epoch))
    for param_group in optimizer.param_groups:
        param_group['lr'] = lr
    return optimizer


def save_checkpoint(model, optimizer, epoch, checkpoint_dir, name):
    checkpoint_path = join(checkpoint_dir, "checkpoint_epoch{}_{}.pth".format(epoch, name))
    torch.save({"state_dict": model.state_dict(), "optimizer": optimizer.state_dict(), "global_epoch": epoch},
               checkpoint_path)
    print("Saved checkpoint:", checkpoint_path)


def load_checkpoint(model, checkpoint_path):
    """The model's weights; returns the checkpoint (its "optimizer" and "global_epoch" are applied by the caller)."""
    print("Load checkpoint from: {}".format(checkpoint_path))
    checkpoint = torch.load(checkpoint_path, map_location="cpu")
    model.load_state_dict(checkpoint["state_dict"])
    return checkpoint


# ---- the two step paths: each returns (12 loss scalars, y_hat_static, spoof count or None) on the device ----

class FusedPath(object):
    name = "FusedGanStep"

    def __init__(self, fs):
        self.fs, self.opt_g, self.opt_d = fs, fs.opt_g, fs.opt_d

    def step(self, x, y, lengths, cpu_lengths, adv_w, train, update_g):
        losses = self.fs.step(x, y, lengths, adv_w=adv_w, train=train, update_g=update_g)
        return losses, self.fs.y_hat_static, (self.fs.spoof_count if self.fs.ref_d is not None else None)


class ModularPath(object):
    name = "GanTrainer"

    def __init__(self, tr, hp, device):
        from compat.nnmnkwii.paramgen import unit_variance_mlpg_matrix
        self.tr, self.hp, self.device, self.opt_g, self.opt_d = tr, hp, device, tr.opt_g, tr.opt_d
        self._R, self._mlpg_matrix = {}, unit_variance_mlpg_matrix
        self._has_dynamic = bool(np.any(hp.has_dynamic_features))

    def step(self, x, y, lengths, cpu_lengths, adv_w, train, update_g):
        t = int(x.shape[1])
        R = None
        if self._has_dynamic:
            R = self._R.get(t)
            if R is None:
                R = self._R[t] = torch.from_numpy(self._mlpg_matrix(self.hp.windows, t)).to(self.device)
        out, _, y_hat_static = self.tr.step(x, y, cpu_lengths, R, adv_w=adv_w, train=train, update_g=update_g)
        zero = torch.zeros((), dtype=torch.float32, device=self.device)
        losses = torch.stack([out.get(k, zero).float().reshape(()) for k in LOSS_NAMES])
        return losses, y_hat_static.detach(), out.get("spoof_count")


def make_path(model_g, model_d, hp, B, T, w_d, mse_w, mge_w, reference_discriminator, device):
    """FusedGanStep whenever it takes the models, else GanTrainer (the LSTMRNN / GRURNN generators)."""
    kw = dict(w_d=w_d, mse_w=mse_w, mge_w=mge_w, optimizer=hp.optimizer_g, optimizer_params=hp.optimizer_g_params,
              optimizer_d=hp.optimizer_d, optimizer_d_params=hp.optimizer_d_params,
              reference_discriminator=reference_discriminator)
    try:
        path = FusedPath(FusedGanStep(model_g, model_d, hp, B, T, **kw))
    except RuntimeError as e:
        print("FusedGanStep does not take these models ({}); training with GanTrainer".format(e))
        path = ModularPath(GanTrainer(model_g, model_d, hp, **kw), hp, device)
    print("Training step:", path.name)
    return path


# ---- the loop (train.py:435-648) ----

def host_batches(loader, device):
    """The batches of a host DataLoader as DeviceBatches yields them: sorted on the host, copied without blocking."""
    for x, y, lengths in loader:
        x, y, lengths = sort_batch(x, y, lengths)
        cpu_lengths = lengths.tolist()
        yield (x.to(device, non_blocking=True), y.to(device, non_blocking=True),
               lengths.to(device, non_blocking=True), cpu_lengths)


def run_phase(path, loader, log, phase, adv_w, update_d, update_g, device):
    """One phase: every batch (DeviceBatches, or a host DataLoader's through host_batches) stepped and folded into `log`
    on the device.  Nothing here waits for the GPU; the caller reads `log` once."""
    log.reset()
    train = phase == "train"
    batches = loader if isinstance(loader, DeviceBatches) else host_batches(loader, device)
    for x, y, lengths, cpu_lengths in batches:
        losses, y_hat_static, spoof = path.step(x, y, lengths, cpu_lengths, adv_w, train, update_g)
        log.add(losses, y, y_hat_static, lengths, update_d, update_g, spoof)


class ScalarLog(object):
    """log_value of the tensorboard_logger shim, and one JSON line per scalar in <log_event_path>/scalars.jsonl."""

    def __init__(self, log_event_path):
        from compat import tensorboard_logger
        self.tb = tensorboard_logger
        self.tb.configure(log_event_path)
        os.makedirs(log_event_path, exist_ok=True)
        self.path = join(log_event_path, "scalars.jsonl")

    def __call__(self, name, value, step):
        self.tb.log_value(name, value, step)
        with open(self.path, "a") as f:
            f.write(json.dumps({"name": name, "value": float(value), "step": int(step)}) + "\n")


def train_loop(path, models_, loaders, logs, hp, global_epoch, log_value, checkpoint_dir, w_d=0.0, mse_w=0.0,
               mge_w=1.0, update_d=True, update_g=True, device=None):
    model_g, model_d = models_
    E_loss_mge, E_loss_adv = 1, 1
    for global_epoch in range(global_epoch + 1, hp.nepoch + 1):
        if hp.lr_decay_schedule and update_g:
            exp_lr_scheduler(path.opt_g, global_epoch - 1, hp.nepoch, init_lr=hp.optimizer_g_params["lr"],
                             lr_decay_epoch=hp.lr_decay_epoch)
        if hp.lr_decay_schedule and update_d:
            exp_lr_scheduler(path.opt_d, global_epoch - 1, hp.nepoch, init_lr=hp.optimizer_d_params["lr"],
                             lr_decay_epoch=hp.lr_decay_epoch)
        for phase in ("train", "test"):
            for m in (model_g, model_d):
                m.train() if phase == "train" else m.eval()
            adv_w = w_d * float(np.clip(E_loss_mge / E_loss_adv, 0, 1e+3))
            run_phase(path, loaders[phase], logs[phase], phase, adv_w, update_d, update_g, device)
            values = logs[phase].read(phase, mse_w=mse_w, mge_w=mge_w)
            if update_d and update_g and phase == "train":
                E_loss_mge, E_loss_adv = values["E(mge)"], values["E(adv)"]
            for k, v in values.items():
                log_value(k, v, global_epoch)
        if global_epoch % checkpoint_interval == 0:
            save_models(path, models_, update_g, update_d, global_epoch, checkpoint_dir)
    return global_epoch


def save_models(path, models_, update_g, update_d, epoch, checkpoint_dir):
    for model, optimizer, enabled, name in ((models_[0], path.opt_g, update_g, "Generator"),
                                            (models_[1], path.opt_d, update_d, "Discriminator")):
        if enabled:
            save_checkpoint(model, optimizer, epoch, checkpoint_dir, name)


def parse_args(argv=None):
    from compat.docopt import docopt
    return docopt(__doc__, argv=argv)


def main(argv=None, hp=None):
    """The reference train.py's __main__ (:661-859) on the package's step.  ``hp``: the hyper-parameter object to use
    instead of ``getattr(hparams, --hparams_name)`` (``import hparams`` from the caller's path otherwise); --hparams
    is parsed into it either way."""
    args = parse_args(argv)
    print("Command line args:\n", args)
    if hp is None:
        import hparams
        hp = getattr(hparams, args["--hparams_name"])
        hp.parse(args["--hparams"])
        print(hparams.hparams_debug_string(hp))
    else:
        hp.parse(args["--hparams"])
    if hp.generator_add_noise:
        raise SystemExit("gantts_b200.train: hp.generator_add_noise=True (generator noise) is not supported")
    if not torch.cuda.is_available():
        raise SystemExit("gantts_b200.train: needs a CUDA device (there is no CPU path)")
    device = torch.device("cuda")

    inputs_dir, outputs_dir = args["<inputs_dir>"], args["<outputs_dir>"]
    checkpoint_dir = args["--checkpoint-dir"]
    checkpoint_path_d, checkpoint_path_g = args["--checkpoint-d"], args["--checkpoint-g"]
    checkpoint_path_r = args["--checkpoint-r"]
    max_files = int(args["--max_files"])
    w_d, mse_w, mge_w = float(args["--w_d"]), float(args["--mse_w"]), float(args["--mge_w"])
    restart_epoch = int(args["--restart_epoch"])
    reset_optimizers = args["--reset_optimizers"]
    log_event_path = args["--log-event-path"]
    update_d = w_d > 0
    update_g = not args["--discriminator-warmup"]
    if not exists(checkpoint_dir):
        os.makedirs(checkpoint_dir)

    loaders, Y_mean, Y_std, longest = load_data(hp, inputs_dir, outputs_dir, max_files)

    model_g = getattr(models, hp.generator)(**hp.generator_params)
    model_d = getattr(models, hp.discriminator)(**hp.discriminator_params)
    print("Generator:", model_g)
    print("Discriminator:", model_d)
    reference_discriminator = None
    if checkpoint_path_r is not None:
        reference_discriminator = getattr(models, hp.discriminator)(**hp.discriminator_params)
        try:
            load_checkpoint(reference_discriminator, checkpoint_path_r)
        except Exception:
            warn("Invalid cehckpoint for reference discriminator")
            reference_discriminator = None
    global_epoch = 0
    ckpt = {}
    for model, path_, name in ((model_d, checkpoint_path_d, "d"), (model_g, checkpoint_path_g, "g")):
        if path_:
            ckpt[name] = load_checkpoint(model, path_)
            global_epoch = ckpt[name]["global_epoch"]
    model_g, model_d = model_g.to(device), model_d.to(device)
    if reference_discriminator is not None:
        reference_discriminator = reference_discriminator.to(device).eval()

    path = make_path(model_g, model_d, hp, hp.batch_size, longest, w_d, mse_w, mge_w, reference_discriminator, device)
    if not reset_optimizers:
        for name, opt in (("d", path.opt_d), ("g", path.opt_g)):
            if name in ckpt:
                opt.load_state_dict(ckpt[name]["optimizer"])
    if restart_epoch >= 0:
        global_epoch = restart_epoch

    if log_event_path is None:
        log_event_path = "log/run-test" + str(np.random.randint(100000))
    print("Los event path: {}".format(log_event_path))
    log_value = ScalarLog(log_event_path)
    logs = {p: EpochLog(hp, Y_mean, Y_std, device) for p in ("train", "test")}

    print("Start training from epoch {}".format(global_epoch))
    global_epoch = train_loop(path, (model_g, model_d), loaders, logs, hp, global_epoch, log_value, checkpoint_dir,
                              w_d=w_d, mse_w=mse_w, mge_w=mge_w, update_d=update_d, update_g=update_g, device=device)
    save_models(path, (model_g, model_d), update_g, update_d, global_epoch, checkpoint_dir)
    print("Finished!")
    return 0


if __name__ == "__main__":
    since = time.time()
    rc = main()
    print("Elapsed time: {:.1f} min".format((time.time() - since) / 60))
    sys.exit(rc)
