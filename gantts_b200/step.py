"""The GAN training step of reference train.py (apply_generator :336-355, update_discriminator
:245-279, update_generator :282-320, batch prologue :528-546) on the native ops, without the ~15
host syncs of the original: every loss stays a device scalar until the caller reads it.

Semantics preserved (SURVEY.md 3.2): one zero_grad per step; y_hat_static is NOT detached in the
discriminator update, so the generator also receives the gradient of the fake term; the
discriminator steps before the third D forward used by the adversarial loss; both backwards
accumulate on G before its clip + Adagrad step.
"""
import numpy as np
import torch

from . import multistream
from . import ops
from . import parallel
from .optim import ClipAdagrad, make_optimizer
from .seqloss import sequence_mask


class HParams(dict):
    """Minimal attribute dict with the fields of reference hparams.tts_acoustic the step reads."""
    __getattr__ = dict.__getitem__


TTS_ACOUSTIC = HParams(
    windows=[(0, 0, np.array([1.0])), (1, 1, np.array([-0.5, 0.0, 0.5])), (1, 1, np.array([1.0, -2.0, 1.0]))],
    stream_sizes=[180, 3, 1, 3], has_dynamic_features=[True, True, False, True],
    adversarial_streams=[True, False, False, False], mask_nth_mgc_for_adv_loss=2,
    discriminator_linguistic_condition=False)


def get_selected_static_stream(y_hat_static, hp):
    """reference train.py:232-242 (one gather launch: stream select and mask_nth folded)."""
    sizes = multistream.get_static_stream_sizes(hp.stream_sizes, hp.has_dynamic_features, len(hp.windows))
    cols = multistream.select_stream_columns(sizes, hp.adversarial_streams)
    if hp.mask_nth_mgc_for_adv_loss > 0:
        cols = cols[hp.mask_nth_mgc_for_adv_loss:]
    return ops.gather_cols(y_hat_static, cols)


def apply_generator(model_g, x, R, lengths, hp):
    """reference train.py:336-355 (including the front-padding of a shortened pad_packed_sequence output,
    :346-349 -- a no-op whenever the longest utterance spans the padded length, as in train.py's batches)."""
    if model_g.include_parameter_generation():
        return model_g(x, R, lengths=lengths)
    y_hat = model_g(x, lengths=lengths)
    if y_hat.size(1) != x.size(1):
        y_hat = torch.nn.functional.pad(y_hat.unsqueeze(0), (0, 0, x.size(1) - y_hat.size(-2), 0)).squeeze(0)
    y_hat_static = multistream.multi_stream_mlpg(y_hat, R, hp.stream_sizes, hp.has_dynamic_features)
    return y_hat, y_hat_static


class GanTrainer(object):
    """One-call GAN step over native ops.  ``step`` returns device scalars (no host sync)."""

    def __init__(self, model_g, model_d, hp, w_d=1.0, mse_w=0.0, mge_w=1.0, lr=0.01, weight_decay=1e-7,
                 process_group=None, optimizer="Adagrad", optimizer_params=None, reference_discriminator=None,
                 optimizer_d=None, optimizer_d_params=None):
        """``optimizer`` / ``optimizer_params`` and ``optimizer_d`` / ``optimizer_d_params`` are hp.optimizer_g /
        hp.optimizer_g_params and hp.optimizer_d / hp.optimizer_d_params of reference train.py:796-799: ``opt_g`` and
        ``opt_d`` are ClipAdagrad or ClipAdam with torch.optim's ``param_groups`` / ``state_dict()``, so train.py's
        exp_lr_scheduler, save_checkpoint and load_checkpoint take them as they are.  ``optimizer_d=None`` gives D the
        generator's kind; ``optimizer_d_params=None`` gives D the generator's parameters when the kinds agree, else
        ``lr`` / ``weight_decay`` as the generator would get them.

        ``reference_discriminator``: the frozen discriminator of the adversarial stage (train.py --checkpoint-r);
        every step then returns ``out["spoof_count"]``, the frames of the pre-update y_hat_static it takes for natural
        (train.py:549-558).  It is put in eval mode like train.py:445 does, sees no linguistic conditioning and is
        never updated."""
        from .fused import adversarial_columns, check_reference_discriminator
        self.g, self.d, self.hp = model_g, model_d, hp
        self.ref_d = reference_discriminator
        if reference_discriminator is not None:
            check_reference_discriminator(reference_discriminator, len(adversarial_columns(hp)), "GanTrainer")
            reference_discriminator.eval()
        self.w_d, self.mse_w, self.mge_w = float(w_d), float(mse_w), float(mge_w)
        okw = dict(optimizer_params) if optimizer_params is not None else dict(lr=lr, weight_decay=weight_decay)
        kind_d = optimizer if optimizer_d is None else optimizer_d
        if optimizer_d_params is not None:
            okw_d = dict(optimizer_d_params)
        else:
            okw_d = okw if kind_d == optimizer else dict(lr=lr, weight_decay=weight_decay)
        self.opt_g = make_optimizer(optimizer, model_g.parameters(), **okw)
        self.opt_d = make_optimizer(kind_d, model_d.parameters(), **okw_d) if model_d is not None else None
        self.pg = process_group
        parallel.broadcast_parameters(model_g, group=process_group)
        if model_d is not None:
            parallel.broadcast_parameters(model_d, group=process_group)

    def _allreduce(self, t):
        return parallel.allreduce_sum_(t, self.pg)

    def step(self, x, y, lengths, R, adv_w=1.0, train=True, update_g=True):
        """lengths: CUDA int64 tensor, or what train.py passes (a list of ints / 0-d tensors, sorted descending:
        ``cpu_sorted_lengths``, train.py:503).  The lengths go to the generator and to all three discriminator
        forwards like train.py:542-575 does (recurrent models honour them: packed-sequence semantics).
        ``train=False`` is the "test" phase (train.py:481-486,273,315): no backward, no optimiser step; call
        ``model.eval()`` on the models to switch dropout off as the reference does.
        ``update_g=False`` is the discriminator warm-up step (train.py --discriminator-warmup, :696): update_generator
        is not called, so there is no adversarial forward, no generator backward and no generator step; loss_mse /
        loss_mge are the forward values, loss_adv = 0 and loss_g = mse_w loss_mse + mge_w loss_mge.  Ignored when
        ``train=False``."""
        hp = self.hp
        update_g = update_g or not train
        if not update_g and not (self.w_d > 0 and self.d is not None):
            raise RuntimeError("GanTrainer: update_g=False trains the discriminator alone and needs w_d > 0 and a "
                               "discriminator")
        grad_g = train and update_g
        nw = len(hp.windows)
        if torch.is_tensor(lengths):
            cpu_lengths = lengths
        else:
            cpu_lengths = [int(v) for v in lengths]
            lengths = torch.tensor(cpu_lengths, dtype=torch.int64).to(x.device, non_blocking=True)
        y_static = multistream.get_static_features(y, nw, hp.stream_sizes, hp.has_dynamic_features)   # :528
        mask = sequence_mask(lengths, x.size(1)).unsqueeze(-1)                                        # :535
        self.opt_g.zero_grad()                                                                        # :538
        if self.opt_d is not None:
            self.opt_d.zero_grad()                                                                    # :539
        y_hat_g, y_hat_static_g = apply_generator(self.g, x, R, cpu_lengths, hp)                      # :542
        # The reference back-propagates through the generator TWICE per step: loss_d.backward(retain_graph=True)
        # (train.py:274 -- y_hat_static is not detached, so the discriminator loss deposits gradients on G's parameters)
        # and loss_g.backward() (:316), accumulated in .grad.  Backward is linear in the upstream gradient, so the
        # two are summed HERE, at the generator's outputs, and the generator is traversed once: the losses see leaf
        # copies of (y_hat, y_hat_static), whose .grad collects both contributions.  For the recurrent generators this
        # halves the LSTM backward work of a step (cfg3: 93 -> 47 ms).
        same = y_hat_static_g is y_hat_g
        y_hat = y_hat_g.detach().requires_grad_(grad_g)
        y_hat_static = y_hat if same else y_hat_static_g.detach().requires_grad_(grad_g)
        out = {}
        if self.ref_d is not None:
            # spoofing rate (train.py:549-558): the reference D on the pre-update output, no conditioning, no gradient
            with torch.no_grad():
                target = self.ref_d(get_selected_static_stream(y_hat_static, hp), lengths=cpu_lengths)
                out["spoof_count"] = ops.masked_bce(target, mask, 0)[1]
        # Global number of valid frames (data parallel: normalise by the GLOBAL count, sum grads)
        Tn = self._allreduce(mask.sum().reshape(1))
        if self.w_d > 0 and self.d is not None:
            real_in = get_selected_static_stream(y_static, hp)
            fake_in = get_selected_static_stream(y_hat_static, hp)
            if hp.discriminator_linguistic_condition:
                real_in = torch.cat((x, real_in), -1)
                fake_in = torch.cat((x, fake_in), -1)
            r = ops.masked_bce(self.d(real_in, lengths=cpu_lengths), mask, 0)                         # :261,269
            f = ops.masked_bce(self.d(fake_in, lengths=cpu_lengths), mask, 1)                         # :265,270
            loss_real, loss_fake = r[0] / Tn[0], f[0] / Tn[0]
            loss_d = loss_real + loss_fake
            if train:
                loss_d.backward()                                                                     # :274
                self._allreduce(self.opt_d.flat_grad)
                self.opt_d.step()                                                                     # :275-276
            out.update(loss_d=loss_d.detach(), loss_real_d=loss_real.detach(), loss_fake_d=loss_fake.detach(),
                       real_correct=r[1].detach(), fake_correct=f[1].detach())
        sse_mge = ops._MaskedSSE.apply(y_hat_static, y_static, mask)
        with torch.set_grad_enabled(grad_g and self.mse_w != 0.0):          # a zero weight needs no backward kernel
            sse_mse = ops._MaskedSSE.apply(y_hat, y, mask)
        loss_mge, loss_mse = sse_mge[0] / Tn[0], sse_mse[0] / Tn[0]                                   # :291,294
        if adv_w > 0 and self.w_d > 0 and self.d is not None and update_g:
            fake_in = get_selected_static_stream(y_hat_static, hp)
            if hp.discriminator_linguistic_condition:
                fake_in = torch.cat((x, fake_in), -1)
            a = ops.masked_bce(self.d(fake_in, lengths=cpu_lengths), mask, 0)                         # :307
            loss_adv = a[0] / Tn[0]
        else:
            loss_adv, adv_w = torch.zeros((), device=x.device), 0.0
        loss_g = (self.mse_w * loss_mse + self.mge_w * loss_mge) + adv_w * loss_adv                   # :314
        if grad_g:
            loss_g.backward()                                                                         # :316
            heads, grads = [y_hat_static_g], [y_hat_static.grad]
            if not same and y_hat.grad is not None:
                heads.append(y_hat_g)
                grads.append(y_hat.grad)
            torch.autograd.backward(heads, grads)               # the one pass through MLPG + the generator
            self._allreduce(self.opt_g.flat_grad)
            self.opt_g.step()                                                                         # :317-318
        out.update(loss_mse=loss_mse.detach(), loss_mge=loss_mge.detach(), loss_adv=loss_adv.detach(),
                   loss_g=loss_g.detach(), frames=Tn[0])
        return out, y_hat_g, y_hat_static_g
