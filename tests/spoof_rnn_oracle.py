"""CPU restatement of the spoofing-rate count (train.py:549-558) with a recurrent reference discriminator (LSTMRNN, or
GRURNN -- also an nn.LSTM --, with last_sigmoid=True; train.py:779-781 builds it from hp.discriminator like D), on
tests/rnn_d_oracle.RnnDiscriminator in eval mode (train.py:445: no dropout) and without linguistic conditioning
(:554-555).  TEST INFRASTRUCTURE, pinned to tests/golden/spoof_rnn.npz by test_spoof_rnn_host.py.
"""
import torch

from oracle import gantts_port as gp
from rnn_d_oracle import RnnDiscriminator


def reference_d(sd, prefix, num_layers, hidden, bidir):
    """The reference discriminator from a state_dict whose stack lives under `prefix` ("lstm" or "gru")."""
    return RnnDiscriminator(sd, prefix, num_layers, hidden, bidir)


def reference_output_rnn(ref_d, y_hat_static, lengths, hp):
    """D_ref's output on the adversarial columns of y_hat_static, packed by `lengths`; frames at or beyond a sequence's
    length see h = 0 (pad_packed_sequence)."""
    with torch.no_grad():
        return ref_d.forward(gp.get_selected_static_stream(y_hat_static, hp), lengths, None)


def spoof_count_rnn(ref_d, y_hat_static, lengths, mask, hp):
    """``((D_ref(get_selected_static_stream(y_hat_static), lengths) > 0.5).float() * mask).sum()``."""
    with torch.no_grad():
        return ((reference_output_rnn(ref_d, y_hat_static, lengths, hp) > 0.5).float() * mask).sum().item()
