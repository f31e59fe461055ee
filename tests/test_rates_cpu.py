"""CPU: the per-(fs, window) tables of the short-term kernels across sample rates, run on the host by tests/tables_host.cu.

The sample rate reaches the kernels only through these tables, and their layout changes with it: at 44.1 kHz and above
windows of 600 samples or fewer have mel filters without a single tap, below ~12 kHz the mel filters are long (up to 18
four-tap steps per lane), the chroma lists hold 8 to 10 taps, and below 6 854 Hz the mel bank fails the way the
reference's does (IndexError); just above that rate the last filter ends at bin K - 1, where ``build_pair_blob`` moves a
group's four reads back inside the row (the clamp).  At every specialised window (pair 320 / 480 / 512 / 640 / 800 / 960 / 1024,
solo 400 / 600 / 882, CTA 320 / 400 / 480 / 600 / 640 / 800 / 882), every integer rate from 6 300 to 7 100 Hz and the
common rates from 8 to 192 kHz:

* the status of the mel bank and of the chroma operator is the oracle's exception (IndexError / ValueError / none), and
  the oracle's is the reference's (tests/golden/rates.npz, tests/test_oracle_rates.py);
* ``host_table`` is the oracle's mel bank and chroma operator at every accepted point;
* the pair / solo kernels' blob (``build_pair_blob``) decodes back to the tables (``decode_pair_blob``): walking each
  lane's records as the kernel does, every filter is flushed exactly once, empty ones included, and its taps are exactly
  float32(mel); every four-tap read stays inside the K bins of the row; the chroma lists are exactly float32(chroma
  operator); the DCT rows are float32(DCT);
* every specialised launch fits its shared-memory cap at every accepted point: the pair kernel (kPairCtaCap), the solo
  kernel's feature and chromagram layouts, the CTA kernel at hop w / 2 and at the hops of tests.kernels.RATE_CONFIGS,
  except where its staging is designed to hand a large hop to the generic kernel (CTA_FALLBACK).

Sensitivity (defects planted by hand in ``build_pair_blob``, not committed; each fails the decoder here, at the number of
sweep points given): an empty filter that is not flushed (54), lane lists truncated at LQ = 8 (1 889), chroma lists
truncated at CT = 8 (910), and the clamp moved one bin up (442: the last read lands one past the row) or down (204: the
filter's last tap is dropped).
"""
import subprocess

import numpy as np
import pytest

from oracle import st_oracle as O
from tests import host_exe
from tests.kernels import CTA_FALLBACK, CTA_WINDOWS, FINE, PAIR_WINDOWS, RATE_CONFIGS, RATES, SOLO_WINDOWS, WINDOWS

SWEEP = [(fs, w) for fs in FINE + RATES for w in WINDOWS]
CTA_CAP = 110 * 1024
ST_OK, ST_CHROMA, ST_MEL = 0, -3, -4
EXC = {ST_OK: None, ST_CHROMA: "ValueError", ST_MEL: "IndexError"}


def hops(w):
    return sorted({w // 2} | {s for _, ww, s, _, _ in RATE_CONFIGS if ww == w})


def run_tables(exe, points):
    """{(fs, w): record} of the harness for (fs, window) points."""
    script = "".join("%d %d %d %s\n" % (fs, w, len(hops(w)), " ".join(map(str, hops(w)))) for fs, w in points)
    res = subprocess.run([exe], input=script, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    out, cur = {}, None
    for line in res.stdout.splitlines():
        tag, rest = line[0], line[2:]
        if tag == "T":
            fs, w, mel, chroma, gwords = (int(v) for v in rest.split())
            cur = out[(fs, w)] = dict(mel=mel, chroma=chroma, generic_words=gwords, smem={}, fast=[])
        elif tag == "B":
            cur["layout"] = dict(zip(("words", "lq", "ct", "dct", "mel_rec", "mel_w", "chr"), (int(v) for v in rest.split())))
        elif tag == "W":
            cur["blob"] = np.array(rest.split(), dtype=np.int64).astype(np.int32)
        elif tag == "S":
            kind, nbytes, cap = rest.split()
            cur["smem"][kind] = (int(nbytes), int(cap))
        elif tag == "F":
            cur["fast"].append(tuple(int(v) for v in rest.split()))
    return out


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    return host_exe.build(tmp_path_factory, "tables_host.cu", "-O1")


@pytest.fixture(scope="module")
def tables(harness):
    return run_tables(harness, SWEEP)


@pytest.fixture(scope="module")
def lib():
    from pyaudioanalysis_b200.build import build
    build()
    from pyaudioanalysis_b200 import _lib
    return _lib


def oracle_status(fs, K):
    """(mel, chroma) exception names of the oracle's tables (None: built), and the tables."""
    out = []
    for fn in (O.mel_filterbank, O.chroma_operator):
        try:
            out.append((None, fn(fs, K)))
        except (IndexError, ValueError) as e:
            out.append((type(e).__name__, None))
    return out


def decode_pair_blob(blob, lay, K):
    """Walk the pair blob as the kernel does (csrc/pair_kernel.cuh: rows_to_features).  Returns (mel [40, K], chroma
    [12, K], dct [13, 40]) as float64 sums of the float32 weights, plus the flush count per filter; raises AssertionError on
    a record the kernel would misread (a read past bin K - 1, a flag bit it does not know, a tap never flushed)."""
    LQ, CT = lay["lq"], lay["ct"]
    assert lay["dct"] == 0 and lay["mel_rec"] == (13 * 41 + 3) // 4 * 4, lay
    assert lay["mel_w"] == lay["mel_rec"] + 16 * LQ and lay["mel_w"] % 4 == 0, lay          # float4 loads
    assert lay["chr"] == lay["mel_w"] + 64 * LQ and lay["chr"] % 2 == 0, lay                 # int2 loads
    assert lay["words"] == (lay["chr"] + 32 * CT + 3) // 4 * 4 == blob.size, (lay, blob.size)
    dct = blob[:13 * 41].view(np.float32).reshape(13, 41).astype(np.float64)
    assert not dct[:, 40].any(), "DCT row padding"
    rec = blob[lay["mel_rec"]:lay["mel_w"]].reshape(LQ, 16)
    wts = blob[lay["mel_w"]:lay["chr"]].view(np.float32).reshape(LQ, 16, 4).astype(np.float64)
    assert not (rec & ~0x1ffffff).any(), "record flag bits beyond the flush bit"
    start, fid, flush = rec & 0xffff, (rec >> 16) & 0xff, (rec >> 24) & 1
    assert (start + 4 <= K).all(), "a four-tap read past bin K - 1: start %d, K %d" % (start.max(), K)
    # each step's taps go to the filter the lane flushes next (the kernel's accumulator runs until a flush)
    owner = np.full((LQ, 16), -1)
    nxt = np.full(16, -1)
    for q in range(LQ - 1, -1, -1):
        nxt = np.where(flush[q] == 1, fid[q], nxt)
        owner[q] = nxt
    stray = (owner[:, :, None] < 0) & (wts != 0)
    assert not stray.any(), "taps after a lane's last flush: %d" % stray.sum()
    mel = np.zeros((40, K))
    q, l, j = np.nonzero(wts != 0)
    np.add.at(mel, (owner[q, l], start[q, l] + j), wts[q, l, j])
    assert (fid[flush == 1] < 40).all(), "flush of a filter id >= 40"
    flushes = np.bincount(fid[flush == 1], minlength=40)
    ch = blob[lay["chr"]:lay["chr"] + 32 * CT].reshape(CT, 16, 2)
    cbin, cw = ch[:, :, 0], ch[:, :, 1].copy().view(np.float32).astype(np.float64)
    assert not cw[:, 12:].any(), "chroma weights on lanes 12 .. 15"
    assert ((cbin >= 0) & (cbin < K)).all(), "chroma bin outside the row"
    chroma = np.zeros((12, K))
    t, l = np.nonzero(cw[:, :12] != 0)
    np.add.at(chroma, (l, cbin[t, l]), cw[t, l])
    return mel, chroma, dct[:, :40], flushes


def clamped_groups(mel, K):
    """Four-tap groups of the mel bank whose start lies within three bins of the row's end (build_pair_blob moves them
    back to K - 4)."""
    n = 0
    for row in mel:
        nz = np.nonzero(row)[0]
        if nz.size:
            n += sum(1 for s in range(nz[0], nz[-1] + 1, 4) if s + 4 > K)
    return n


def check_point(fs, w, rec):
    """Everything one (fs, window) record must satisfy; returns its summary (or None where the tables are refused)."""
    K = w // 2
    (mel_exc, mel), (chr_exc, chroma) = oracle_status(fs, K)
    what = "fs=%d w=%d" % (fs, w)
    assert (EXC[rec["mel"]], EXC[rec["chroma"]]) == (mel_exc, chr_exc), what
    if mel_exc or chr_exc:
        assert "blob" not in rec, what
        return None
    lay = rec["layout"]
    dmel, dchroma, ddct, flushes = decode_pair_blob(rec["blob"], lay, K)
    assert (flushes == 1).all(), "%s: flushes per filter %s" % (what, flushes.tolist())
    np.testing.assert_array_equal(dmel, mel.astype(np.float32), err_msg=what + ": decoded mel bank")
    np.testing.assert_array_equal(dchroma, chroma.astype(np.float32), err_msg=what + ": decoded chroma lists")
    np.testing.assert_array_equal(ddct, O.dct_matrix().astype(np.float32), err_msg=what + ": DCT rows")
    empty = int((~mel.any(axis=1)).sum())
    if w in PAIR_WINDOWS:
        nbytes, cap = rec["smem"]["pair"]
        assert nbytes <= cap, "%s: pair kernel %d B > %d B" % (what, nbytes, cap)
    if w in SOLO_WINDOWS:
        for kind in ("solo_features", "solo_chroma"):
            nbytes, cap = rec["smem"][kind]
            assert nbytes <= cap, "%s: %s %d B > %d B" % (what, kind, nbytes, cap)
    return dict(words=lay["words"], lq=lay["lq"], ct=lay["ct"], empty=empty, clamped=clamped_groups(mel, K),
                generic=rec["generic_words"], pair=rec["smem"].get("pair", (0, 0))[0])


def test_tables_across_rates(tables, lib):
    """The whole sweep: statuses, host tables, the pair blob decoded, the specialised launches' caps."""
    summary = {}
    for (fs, w), rec in tables.items():
        s = check_point(fs, w, rec)
        if s is None:
            continue
        summary[(fs, w)] = s
        K = w // 2
        np.testing.assert_allclose(lib.host_table(fs, w, "mel"), O.mel_filterbank(fs, K), rtol=0, atol=1e-15)
        np.testing.assert_allclose(lib.host_table(fs, w, "chroma"), O.chroma_operator(fs, K), rtol=0, atol=1e-15)
    assert len(tables) == len(SWEEP)
    # what the sweep reaches: empty filters at every specialised kind, the clamp, the longest lane lists, refusals
    assert any(s["empty"] for (fs, w), s in summary.items() if w in PAIR_WINDOWS)
    assert any(s["empty"] for (fs, w), s in summary.items() if w in SOLO_WINDOWS)
    assert any(s["clamped"] for s in summary.values())
    assert max(s["lq"] for s in summary.values()) == 18 and max(s["ct"] for s in summary.values()) == 10
    assert any(rec["mel"] == ST_MEL for rec in tables.values())
    for fs, w in [(16000, 800), (48000, 480), (44100, 400), (8000, 800), (7000, 960), (192000, 1024)]:
        print("fs %6d w %4d" % (fs, w), summary[(fs, w)])


def test_refusal_boundary(tables):
    """Per window, the mel bank refuses every rate of the fine sweep below one boundary and accepts every rate from it on;
    the chroma operator accepts all of them."""
    for w in WINDOWS:
        refused = [fs for fs in FINE if tables[(fs, w)]["mel"] == ST_MEL]
        assert refused and refused == list(range(FINE[0], refused[-1] + 1)), (w, refused[:3], refused[-3:])
        assert all(tables[(fs, w)]["chroma"] == ST_OK for fs in FINE), w
        print("w %4d: mel bank refused below %d Hz" % (w, refused[-1] + 1))


def test_largest_tables_fit(tables):
    """The largest blobs of the sweep against the launch footprints the shared-memory budget test
    (tests/smem_budget_host.cu) assumes, and the CTA kernel at every hop of the GPU rate configs."""
    accepted = [r for r in tables.values() if "layout" in r]
    assert max(r["layout"]["words"] for r in accepted) == PAIR_WORDS_MAX
    assert max(r["generic_words"] for r in accepted) == GENERIC_WORDS_MAX
    over = set()
    for (fs, w), rec in tables.items():
        if w not in CTA_WINDOWS or rec["mel"] != ST_OK:
            continue
        for hop, runs, nbytes in rec["fast"]:
            if nbytes > CTA_CAP:
                over.add((w, hop))
    assert over == CTA_FALLBACK, over
    assert all(hop > w for w, hop in over)


# the largest blobs over the sweep (both at 6 854 Hz, window 1024: the lowest accepted rate, the longest mel filters);
# tests/smem_budget_host.cu holds every launch to its cap at these sizes
PAIR_WORDS_MAX, GENERIC_WORDS_MAX = 2232, 1832


def test_rate_configs_reach_their_layouts(harness):
    """The GPU rate configs (tests.kernels.RATE_CONFIGS) reach, through the pair and through the solo kernel, empty mel
    filters, a clamped group and the longest lane lists of the sweep, and the CTA kernel's hand-off at a large hop."""
    recs = run_tables(harness, [(fs, w) for fs, w, _, _, _ in RATE_CONFIGS])
    st = {}
    for fs, w, s, kinds, what in RATE_CONFIGS:
        st[(fs, w)] = check_point(fs, w, recs[(fs, w)])
        assert st[(fs, w)] is not None, (fs, w)
        print("fs %6d w %4d s %4d" % (fs, w, s), st[(fs, w)], what)
    for group in (PAIR_WINDOWS, SOLO_WINDOWS):
        mine = [v for (fs, w), v in st.items() if w in group]
        assert any(v["empty"] for v in mine) and any(v["clamped"] for v in mine), group
    assert max(v["words"] for v in st.values()) == PAIR_WORDS_MAX
    assert max(v["lq"] for v in st.values()) == 18 and max(v["ct"] for v in st.values()) == 10
    assert CTA_FALLBACK <= {(w, s) for _, w, s, _, _ in RATE_CONFIGS}
