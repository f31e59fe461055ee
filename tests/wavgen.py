"""WAV files of every data-chunk flavour, written byte by byte (scipy cannot write 24-bit, extensible headers, extra
chunks or malformed files): the decode tests and oracle/make_golden_pcm.py share this writer, so the golden files are
regenerated from their seeds instead of being stored."""
import struct

import numpy as np

# name -> (B200AA_PCM_* code, format tag, bits per sample)
FORMATS = {"u8": (0, 1, 8), "s16": (1, 1, 16), "s24": (2, 1, 24), "s32": (3, 1, 32), "f32": (4, 3, 32), "f64": (5, 3, 64)}
FLAVOURS = [(name, ch) for name in FORMATS for ch in (1, 2)]          # the 12 (format, channels) flavours
_GUID_TAIL = b"\x00\x00\x10\x00\x80\x00\x00\xaa\x00\x38\x9b\x71"
_RANGE = {"u8": (0, 255), "s16": (-2 ** 15, 2 ** 15 - 1), "s24": (-2 ** 23, 2 ** 23 - 1), "s32": (-2 ** 31, 2 ** 31 - 1)}


def encode(x, name):
    """Raw little-endian data-chunk bytes of samples x ([n] or [n, channels]; for s24 the 24-bit integer values)."""
    x = np.asarray(x)
    if name == "s24":
        v = x.astype("<i4").reshape(-1).view(np.uint8).reshape(-1, 4)
        return v[:, :3].tobytes()
    return np.ascontiguousarray(x).astype({"u8": "u1", "s16": "<i2", "s32": "<i4", "f32": "<f4", "f64": "<f8"}[name]).tobytes()


def chunk(cid, body):
    return cid + struct.pack("<I", len(body)) + body + (b"\x00" if len(body) & 1 else b"")


def fmt_body(fs, channels, tag, bits, extensible=False, block_align=None, bytes_per_s=None):
    ba = channels * bits // 8 if block_align is None else block_align
    bps = fs * ba if bytes_per_s is None else bytes_per_s
    if not extensible:
        return struct.pack("<HHIIHH", tag, channels, fs, bps, ba, bits)
    return (struct.pack("<HHIIHH", 0xFFFE, channels, fs, bps, ba, bits) + struct.pack("<HHI", 22, bits, 0)
            + struct.pack("<I", tag) + _GUID_TAIL)


def wav_bytes(fs, payload, channels, tag, bits, extensible=False, before=(), after=(), data_size=None, riff=b"RIFF",
              block_align=None, bytes_per_s=None, cut=0):
    """A whole file: RIFF header, 'fmt ', the ``before`` chunks ((id, body) pairs), 'data' (declared size ``data_size``,
    default the payload's), the ``after`` chunks; ``cut`` bytes dropped from the end of the file."""
    body = [chunk(b"fmt ", fmt_body(fs, channels, tag, bits, extensible, block_align, bytes_per_s))]
    body += [chunk(cid, b) for cid, b in before]
    size = len(payload) if data_size is None else data_size
    body.append(b"data" + struct.pack("<I", size) + payload + (b"\x00" if len(payload) & 1 else b""))
    body += [chunk(cid, b) for cid, b in after]
    raw = b"WAVE" + b"".join(body)
    out = riff + struct.pack("<I", len(raw)) + raw
    return out[:len(out) - cut] if cut else out


def write(path, fs, x, name, **kw):
    """Write samples x ([n] or [n, channels]) as a `name` WAV file (FORMATS)."""
    x = np.asarray(x)
    channels = 1 if x.ndim == 1 else x.shape[1]
    _, tag, bits = FORMATS[name]
    with open(path, "wb") as f:
        f.write(wav_bytes(fs, encode(x, name), channels, tag, bits, **kw))


def signal(name, channels, n, seed, fs=16000):
    """Seeded audio-like samples of a flavour: two tones and noise at about half of the format's full scale, with the
    two channels different."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / fs
    cols = []
    for c in range(channels):
        f0 = 110.0 * (1 + rng.integers(1, 8)) + 37 * c
        y = 0.3 * np.sin(2 * np.pi * f0 * t) + 0.1 * np.sin(2 * np.pi * 3.1 * f0 * t + c) + 0.08 * rng.standard_normal(n)
        cols.append(y)
    y = np.stack(cols, axis=1) if channels == 2 else cols[0]
    if name in ("f32", "f64"):
        return y.astype(np.float32 if name == "f32" else np.float64)
    lo, hi = _RANGE[name]
    mid, half = (lo + hi + 1) / 2, (hi - lo + 1) / 2
    return np.clip(np.round(mid + half * y), lo, hi).astype(np.int64)


def _f32_bits(u):
    return np.asarray(u, dtype=np.uint32).view(np.float32)


def special_values(name, rng):
    """1-D samples of a format: its edge cases followed by random ones."""
    if name in _RANGE:
        lo, hi = _RANGE[name]
        edges = [lo, lo + 1, -1, 0, 1, hi - 1, hi, (lo + hi) // 2, (lo + hi + 1) // 2]
        if name == "s32":               # odd values above 2^24: float32 rounding, ties included
            edges += [2 ** 24 + 1, 2 ** 24 + 3, -(2 ** 24 + 1), 2 ** 25 + 2, 2 ** 25 + 6, 2 ** 30 + 65, -(2 ** 31 - 65),
                      2 ** 31 - 64, 2 ** 31 - 128]
        edges = [v for v in edges if lo <= v <= hi]
        return np.concatenate([np.array(edges, dtype=np.int64), rng.integers(lo, hi + 1, size=3000)])
    f32 = np.finfo(np.float32)
    sub = _f32_bits([1, 2, 3, 5, 0x7FFFFF, 0x7FFFFE, 0x400001, 0x80000001, 0x80000003, 0x807FFFFF])
    edges32 = np.concatenate([np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 1.0, -1.0, 0.5, 3.0, f32.max, -f32.max,
                                        f32.tiny, -f32.tiny, f32.tiny * 3], dtype=np.float32), sub])
    if name == "f32":
        rand = np.concatenate([rng.standard_normal(1500).astype(np.float32),
                               _f32_bits(rng.integers(1, 2 ** 23, size=500)),                    # subnormals
                               _f32_bits(rng.integers(0, 2 ** 32, size=1000, dtype=np.uint64))])  # any bits, NaNs too
        return np.concatenate([edges32, rand])
    edges64 = np.array([1e39, -1e39, 3.4028235677973366e38, 3.4028235677973362e38, 3.4028236e38, float(f32.max) * 1.5,
                        1 + 2.0 ** -24, 1 + 3 * 2.0 ** -24, -(1 + 2.0 ** -24), 5e-324, -5e-324, 1e-300, 7e-46, 7.006e-46,
                        2.0 ** -150, 2.0 ** -149 * 1.5, 1e-45, -1e-45, 1e308, -np.inf], dtype=np.float64)
    rand = np.concatenate([rng.standard_normal(1500), rng.standard_normal(500) * 1e-40, rng.standard_normal(300) * 1e38,
                           rng.integers(0, 2 ** 63, size=700, dtype=np.uint64).view(np.float64)])
    return np.concatenate([edges32.astype(np.float64), edges64, rand])


def flavour_samples(name, channels, seed):
    rng = np.random.default_rng(seed)
    v = special_values(name, rng)
    if channels == 1:
        return v
    m = 40                                      # every pair of the first 40 values, then random pairs
    head = v[:m]
    left = np.concatenate([np.tile(head, m), v[m:]])
    right = np.concatenate([np.concatenate([np.roll(head, k) for k in range(m)]), rng.permutation(v[m:])])
    return np.stack([left, right], axis=1)
