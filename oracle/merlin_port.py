"""CPU restatement of the frame expansion of reference evaluation_tts.py:200-212 (tts_from_label): the labels with state
durations set, ``nnmnkwii.frontend.merlin.linguistic_features(..., add_frame_features=True, subphone_features="full")``
and the removal of silence frames, for phones whose linguistic rows are already known (the prepared ``X_duration``
rows, silences removed).  TEST INFRASTRUCTURE ONLY.

nnmnkwii is a third-party package the reference does not vendor, so this is written from the definition of Merlin's
``load_labels_with_state_alignment`` "full" block, which nnmnkwii follows: **parity unpinned** against nnmnkwii itself
(tools/check_frame_features.py pins it against a prepared corpus).  It runs the literal per-phone, per-state, per-frame
loop in float64, as nnmnkwii fills its feature matrix, and rounds to float32 as LinguisticSource stores it.
"""
import numpy as np

SUBPHONE_FEATURES = 9


def frame_features(durations):
    """The nine "full" subphone features of one phone with state durations d_1..d_S: (sum d_s, 9) float64."""
    d = [int(v) for v in durations]
    if any(v < 1 for v in d):
        raise ValueError("state durations must be >= 1 (got %s)" % (d,))
    S = len(d)
    phone_duration = sum(d)
    rows = []
    state_duration_base = 0
    for s in range(1, S + 1):
        frame_number = d[s - 1]
        for i in range(frame_number):
            rows.append([
                float(i + 1) / float(frame_number),                                      # fraction through state (fwd)
                float(frame_number - i) / float(frame_number),                           # fraction through state (bwd)
                float(frame_number),                                                     # state length in frames
                float(s),                                                                # state index (fwd)
                float(S + 1 - s),                                                        # state index (bwd)
                float(phone_duration),                                                   # phone length in frames
                float(frame_number) / float(phone_duration),                             # state's share of the phone
                float(phone_duration - i - state_duration_base) / float(phone_duration),  # fraction through phone (bwd)
                float(state_duration_base + i + 1) / float(phone_duration),              # fraction through phone (fwd)
            ])
        state_duration_base += frame_number
    return np.array(rows, dtype=np.float64).reshape(-1, SUBPHONE_FEATURES)


def expand(phone_x, durations):
    """Frame-level features of one utterance: phone_x (P, L) linguistic rows, durations (P, S) state durations.
    Returns (sum of all durations, L + 9) float32: each phone's row repeated over its frames, followed by
    frame_features, in phone order."""
    phone_x = np.asarray(phone_x, dtype=np.float64)
    durations = np.asarray(durations)
    if phone_x.ndim != 2 or durations.ndim != 2 or len(phone_x) != len(durations):
        raise ValueError("expand needs phone_x (P, L) and durations (P, S) of the same P")
    blocks = []
    for row, d in zip(phone_x, durations):
        f = frame_features(d)
        blocks.append(np.concatenate([np.repeat(row[None, :], len(f), axis=0), f], axis=1))
    if not blocks:
        return np.zeros((0, phone_x.shape[1] + SUBPHONE_FEATURES), dtype=np.float32)
    return np.concatenate(blocks).astype(np.float32)
