"""The music-thumbnail cases shared by oracle/make_golden_thumbnail.py and the thumbnail tests: the stubbed-feature cases
(seeded short-term matrices handed to the reference's music_thumbnailing in place of its features) and a generated track
with a planted repeated section."""
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "thumbnail.npz")

# name -> (F, T, short_step, thumb_size, limit_1, limit_2, what is planted in the matrix)
STUB_CASES = {
    "base": (68, 120, 0.5, 10.0, 0, 1, None),
    "f1": (1, 40, 0.5, 2.0, 0, 1, None),
    "f3": (3, 70, 0.5, 10.0, 0, 1, None),
    "f137": (137, 66, 0.5, 5.0, 0, 1, None),
    "limits": (68, 100, 0.5, 10.0, 0.2, 0.8, None),
    "limits_swapped": (68, 90, 0.5, 10.0, 0.7, 0.3, None),
    "limits_negative": (68, 90, 0.5, 5.0, -0.5, -0.1, None),
    "step_025": (68, 130, 0.25, 5.0, 0, 1, None),
    "nan_feature": (68, 80, 0.5, 10.0, 0, 1, "nan"),
    "zero_frame": (68, 80, 0.5, 10.0, 0, 1, "mean"),
    "repeat": (68, 130, 0.5, 10.0, 0, 1, "repeat"),
    "all_masked": (68, 25, 0.5, 10.0, 0, 1, None),
    "one_frame_m1": (68, 1, 0.5, 0.5, 0, 1, None),
    "shorter_than_filter": (68, 12, 0.5, 10.0, 0, 1, None),
    "one_frame": (68, 1, 0.5, 10.0, 0, 1, None),
    "filter_zero": (68, 30, 0.5, 0.2, 0, 1, None),
    "filter_negative": (68, 30, 0.5, -3.0, 0, 1, None),
}


def stub_features(name):
    """The seeded [F, T] short-term matrix of a stubbed case (float64)."""
    F, T, _, _, _, _, plant = STUB_CASES[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    st = rng.normal(size=(F, T)) * rng.choice([1e-3, 1.0, 50.0], size=(F, 1)) + rng.normal(size=(F, 1))
    if plant == "nan":
        st[7, 37] = np.nan
    elif plant == "mean":
        others = np.delete(st, 41, axis=1)
        st[:, 41] = others.mean(axis=1)         # then the frame equals the mean: a zero row after the scaler
    elif plant == "repeat":
        st[:, 95:120] = st[:, 20:45] + 1e-3 * rng.normal(size=(F, 25))
    return st


def planted_track(fs=16000, seconds=60, channels=1):
    """A seeded int16 track of one-second blocks of smoothed noise, each with its own level and colour, in which blocks
    10-21 return exactly at 38-49: the filtered similarity peaks there by a wide margin.  channels=2 adds a second channel
    at half the level."""
    rng = np.random.default_rng(2024)
    blocks = []
    for _ in range(seconds):
        w = rng.normal(size=fs)
        for _ in range(int(rng.integers(0, 4))):
            w = np.cumsum(w) - np.cumsum(w).mean()
            w /= np.abs(w).max()
        blocks.append(w / np.abs(w).max() * rng.uniform(0.05, 0.9))
    blocks[38:50] = blocks[10:22]
    x = (np.concatenate(blocks) * 20000).astype(np.int16)
    if channels == 2:
        x = np.stack([x, x // 2], axis=1)
    return x


def golden():
    """tests/golden/thumbnail.npz (oracle/make_golden_thumbnail.py)."""
    return np.load(GOLDEN)
