"""Helpers of the training-command tests (test_train_cli_host.py, test_gpu_train_cli.py, test_gpu_epoch_log.py):
hyper-parameter objects shaped like reference hparams.py's, seeded synthetic feature directories, and a restatement of
what train.py:562-637 logs for one phase, fed per batch with host values."""
import copy
import os

import numpy as np

from conftest import WINDOWS


def _HParams():
    from compat.tensorflow.contrib.training import HParams
    return HParams


def vc_hp(order=4, **over):
    """hparams.vc at a tiny size: In2OutHighwayNet and MLP discriminator, every dropout 0, batch 6, no workers."""
    kw = dict(name="vc", order=order, windows=WINDOWS, stream_sizes=[order * 3], has_dynamic_features=[True],
              adversarial_streams=[True], mask_nth_mgc_for_adv_loss=0, generator_add_noise=False,
              generator_noise_dim=200, generator="In2OutHighwayNet",
              generator_params={"in_dim": None, "out_dim": None, "num_hidden": 2, "hidden_dim": 32,
                                "static_dim": order, "dropout": 0.0},
              optimizer_g="Adagrad", optimizer_g_params={"lr": 0.01, "weight_decay": 0},
              discriminator_linguistic_condition=False, discriminator="MLP",
              discriminator_params={"in_dim": order, "out_dim": 1, "num_hidden": 2, "hidden_dim": 16, "dropout": 0.0,
                                    "last_sigmoid": True},
              optimizer_d="Adagrad", optimizer_d_params={"lr": 0.01, "weight_decay": 0},
              nepoch=2, lr_decay_schedule=False, lr_decay_epoch=10, batch_size=6, num_workers=0, pin_memory=True,
              cache_size=1200)
    kw.update(over)
    return _HParams()(**copy.deepcopy(kw))


def tts_acoustic_hp(**over):
    kw = dict(name="acoustic", order=59, windows=WINDOWS, recompute_delta_features=False,
              stream_sizes=[180, 3, 1, 3], has_dynamic_features=[True, True, False, True],
              adversarial_streams=[True, False, False, False], mask_nth_mgc_for_adv_loss=2, generator_add_noise=False,
              generator_noise_dim=200, generator="MLP",
              generator_params={"in_dim": None, "out_dim": None, "num_hidden": 2, "hidden_dim": 32, "dropout": 0.0,
                                "last_sigmoid": False},
              optimizer_g="Adagrad", optimizer_g_params={"lr": 0.01, "weight_decay": 1e-7},
              discriminator_linguistic_condition=True, discriminator="MLP",
              discriminator_params={"in_dim": None, "out_dim": 1, "num_hidden": 2, "hidden_dim": 16, "dropout": 0.0,
                                    "last_sigmoid": True},
              optimizer_d="Adagrad", optimizer_d_params={"lr": 0.01, "weight_decay": 1e-7},
              nepoch=2, lr_decay_schedule=False, lr_decay_epoch=25, batch_size=6, num_workers=0, pin_memory=True,
              cache_size=1200)
    kw.update(over)
    return _HParams()(**copy.deepcopy(kw))


def tts_duration_hp(**over):
    kw = dict(name="duration", windows=WINDOWS[:1], stream_sizes=[5], has_dynamic_features=[False],
              recompute_delta_features=False, adversarial_streams=[True], mask_nth_mgc_for_adv_loss=0,
              generator_add_noise=False, generator_noise_dim=200, generator="MLP",
              generator_params={"in_dim": None, "out_dim": None, "num_hidden": 2, "hidden_dim": 32, "dropout": 0.0,
                                "last_sigmoid": False},
              optimizer_g="Adam", optimizer_g_params={"lr": 1e-3, "betas": (0.5, 0.9), "weight_decay": 0},
              discriminator_linguistic_condition=True, discriminator="MLP",
              discriminator_params={"in_dim": None, "out_dim": 1, "num_hidden": 2, "hidden_dim": 16, "dropout": 0.0,
                                    "last_sigmoid": True},
              optimizer_d="Adam", optimizer_d_params={"lr": 1e-3, "betas": (0.5, 0.9), "weight_decay": 0},
              nepoch=2, lr_decay_schedule=False, lr_decay_epoch=25, batch_size=6, num_workers=0, pin_memory=True,
              cache_size=1200)
    kw.update(over)
    return _HParams()(**copy.deepcopy(kw))


def write_vc_data(root, n_files=30, dim=12, seed=0):
    """root/X and root/Y: n_files time-aligned .npy utterances (float32, 20..60 frames) from a seed."""
    rng = np.random.RandomState(seed)
    xd, yd = os.path.join(root, "X"), os.path.join(root, "Y")
    os.makedirs(xd), os.makedirs(yd)
    for i in range(n_files):
        n = int(rng.randint(20, 61))
        x = rng.randn(n, dim).astype(np.float32)
        y = (0.7 * x + 0.3 * rng.randn(n, dim) + 0.5).astype(np.float32)
        np.save(os.path.join(xd, "utt%03d.npy" % i), x)
        np.save(os.path.join(yd, "utt%03d.npy" % i), y)
    return xd, yd


METRIC_NAMES = {"acoustic": ("mcd", "bap_mcd", "f0_rmse", "vuv_err"), "duration": ("dur_rmse",), "vc": ("mcd",)}


def trainpy_phase_log(batches, phase, update_d, update_g, spoof, mse_w=0.0, mge_w=1.0):
    """What train.py:476-637 logs for a phase whose batches gave `batches`: per batch a dict of the step's host loss
    values (loss_dict()), "lengths" (host list), "distortions" (compute_distortions' dict) and, with a reference D,
    "spoof_count".  Python floats summed in batch order, as train.py does."""
    running_loss = {"generator": 0.0, "mse": 0.0, "mge": 0.0, "loss_real_d": 0.0, "loss_fake_d": 0.0, "loss_adv": 0.0,
                    "discriminator": 0.0}
    running_metrics = {}
    real_correct_count, fake_correct_count, regard_fake_as_natural = 0, 0, 0
    N, total_num_frames = len(batches), 0
    for b in batches:
        total_num_frames += float(sum(b["lengths"]))
        if spoof:
            regard_fake_as_natural += b["spoof_count"]
        if update_d:
            running_loss["discriminator"] += b["loss_d"]
            running_loss["loss_fake_d"] += b["loss_fake_d"]
            running_loss["loss_real_d"] += b["loss_real_d"]
            real_correct_count += b["real_correct"]
            fake_correct_count += b["fake_correct"]
        if update_g:
            running_loss["mse"] += b["loss_mse"]
            running_loss["mge"] += b["loss_mge"]
            running_loss["loss_adv"] += b["loss_adv"]
            running_loss["generator"] += b["loss_g"]
            for k, v in b["distortions"].items():
                running_metrics[k] = running_metrics.get(k, 0.0) + float(v)
    out = {}
    if update_d and update_g and phase == "train":
        E_loss_mge = (mse_w * running_loss["mse"] + mge_w * running_loss["mge"]) / N
        E_loss_adv = running_loss["loss_adv"] / N
        out["E(mge)"], out["E(adv)"], out["MGE/ADV loss weight"] = E_loss_mge, E_loss_adv, E_loss_mge / E_loss_adv
    for ty, enabled in [("mse", update_g), ("mge", update_g), ("discriminator", update_d), ("loss_real_d", update_d),
                        ("loss_fake_d", update_d), ("loss_adv", update_g and update_d), ("generator", update_g)]:
        if enabled:
            out["{} {} loss".format(phase, ty)] = running_loss[ty] / N
    for k, v in running_metrics.items():
        out["{} {} metric".format(phase, k)] = v / N
    if update_d:
        out["Real {} acc".format(phase)] = real_correct_count / total_num_frames
        out["Fake {} acc".format(phase)] = fake_correct_count / total_num_frames
    if spoof:
        out["{} spoofing rate".format(phase)] = regard_fake_as_natural / total_num_frames
    return out
