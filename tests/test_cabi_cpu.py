"""CPU: the C-ABI library builds, loads and exports every symbol include/b200aa.h declares; host-only
entry points (tables, frame counts) agree with the oracle.  No compute calls (there is no GPU here)."""
import ctypes
import os
import re

import numpy as np
import pytest

from oracle import st_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def L():
    from pyaudioanalysis_b200.build import build
    build()
    from pyaudioanalysis_b200 import _lib
    return _lib


def test_header_symbols_exported(L):
    header = open(os.path.join(ROOT, "include", "b200aa.h")).read()
    declared = set(re.findall(r"\b(b200aa_[a-z_0-9]+)\s*\(", header))
    assert declared, "no declarations found"
    assert declared == set(L.SIGNATURES), (declared ^ set(L.SIGNATURES))
    lib = L.lib()
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.b200aa_abi_version() == 1
    assert b"concatenate" in lib.b200aa_status_string(-2)


@pytest.mark.parametrize("fs,w", [(16000, 800), (44100, 882), (22050, 551), (8000, 400), (48000, 2400), (16000, 16000)])
def test_host_tables_match_oracle(L, fs, w):
    K = w // 2
    np.testing.assert_allclose(L.host_table(fs, w, "mel"), O.mel_filterbank(fs, K), rtol=0, atol=1e-15)
    np.testing.assert_allclose(L.host_table(fs, w, "chroma"), O.chroma_operator(fs, K), rtol=0, atol=1e-15)
    np.testing.assert_allclose(L.host_table(fs, w, "dct"), O.dct_matrix(), rtol=0, atol=1e-15)


def test_table_sparsity_matches_survey(L):
    mel = L.host_table(16000, 800, "mel")
    assert np.count_nonzero(mel) == 323 and np.nonzero(mel.any(axis=0))[0].max() == 171     # SURVEY 8a row 12
    assert np.count_nonzero(L.host_table(16000, 800, "chroma")) == 71                         # row 14
    assert np.count_nonzero(L.host_table(44100, 882, "chroma")) == 74


def test_reference_error_cases(L):
    with pytest.raises(ValueError):
        L.host_table(8000, 160, "chroma")          # reference: chroma else-branch raises
    with pytest.raises(IndexError):
        L.host_table(4000, 400, "mel")             # reference: fancy store beyond num_fft raises IndexError
    with pytest.raises(IndexError):
        O.mel_filterbank(4000, 200)


def test_counts(L):
    lib = L.lib()
    for n, w, s in [(128164, 800, 400), (16000, 800, 800), (799, 800, 400), (800, 800, 400), (1199, 800, 400),
                    (1200, 800, 400), (2646000, 882, 441), (16300, 800, 400), (16000, 800, 300), (16000, 800, 200)]:
        assert lib.b200aa_num_frames(n, w, s) == O.frame_count(n, w, s)
        x = np.zeros(n, dtype=np.int16)
        if n > 2 * w:
            assert lib.b200aa_spectrogram_rows(n, w, s) == O.spectrogram(x, 16000, w, s)[0].shape[0]
            assert lib.b200aa_chromagram_rows(n, w, s) == int((n - s - w) / s) + 1
    assert lib.b200aa_mid_windows(319, 40) == 8 and lib.b200aa_mid_windows(143999, 40) == 3600


def _first_cuda_call_fails(L):
    """One entry point of each kernel family's own .cu, with arguments that pass its checks: (name, call, the start of the
    CUDA call its failure names).  Fake device pointers are never dereferenced: each call stops at its first CUDA call."""
    lib, dev = L.lib(), ctypes.c_void_p(1 << 20)
    clip = np.array([(0, 1, 1, 1)], dtype=[("offset", "<i8"), ("n_frames", "<i8"), ("format", "<i4"), ("channels", "<i4")])
    off, idx, one = np.array([0, 1], np.int64), np.zeros(1, np.int64), np.ones(1, np.int64)
    node, roots, values = np.array([[-1, 0, 0, 0]], np.int32), np.zeros(1, np.int32), np.full((1, 2), 0.5)
    h = ctypes.c_void_p()

    def ptr(a):
        return ctypes.c_void_p(a.ctypes.data)
    return [
        ("mid.cu", lambda: lib.b200aa_frame_counts(dev, 1, 800, 400, 40, dev, dev, None), "frame_counts_kernel: "),
        ("pcm.cu", lambda: lib.b200aa_decode_pcm(dev, 16, ptr(clip), 1, L.DTYPE_I16, dev, 1, 1, None), "cudaMallocAsync("),
        ("beat.cu", lambda: lib.b200aa_beat_extraction(dev, 1, 68, 10, 10, None, 0.05, dev, None), "cudaMallocAsync("),
        ("knn.cu", lambda: lib.b200aa_knn_classify(dev, dev, 1, 1, 1, 1, dev, L.DTYPE_F32, 1, 1, dev, dev, None),
         "cudaMallocAsync("),
        ("hmm.cu", lambda: lib.b200aa_hmm_statistics(dev, L.DTYPE_F32, 1, 1, 1, ptr(one), 1, ptr(off), ptr(idx), dev, None),
         "cudaMallocAsync("),
        ("trees.cu", lambda: lib.b200aa_trees_create(ctypes.byref(h), ptr(node), 1, ptr(roots), 1, ptr(values), 1, 2, 1, 0,
                                                     None, 0), "cudaGetDevice("),
    ]


def test_error_state_is_shared_by_every_file(L):
    """b200aa_last_cuda_error() and b200aa_launch_count() live in b200aa.cu and report the entry points of every .cu: each
    call runs in a thread of its own, whose error text starts empty, and must leave the text of its own failed CUDA call."""
    import threading
    import torch
    if torch.cuda.device_count() != 0:
        pytest.skip("on a GPU host these calls would run")
    lib = L.lib()
    for name, call, what in _first_cuda_call_fails(L):
        got = {}

        def run():
            before = lib.b200aa_launch_count()
            got["rc"] = call()
            got["launches"] = lib.b200aa_launch_count() - before
            got["err"] = lib.b200aa_last_cuda_error().decode()
        t = threading.Thread(target=run)
        t.start()
        t.join()
        assert got["rc"] == L.ERR_CUDA, (name, got)
        assert got["err"].startswith(what), (name, got["err"])
        assert got["launches"] == (1 if what.endswith("_kernel: ") else 0), (name, got)


def test_python_mirror_names():
    from pyaudioanalysis_b200 import ShortTermFeatures as S
    assert S.feature_names(True) == O.feature_names(True)
    assert S.feature_names(False) == O.feature_names(False)
    from pyaudioanalysis_b200.batch import mid_ratios
    assert mid_ratios(16000, 16000, 800, 400) == O.mid_ratios(16000, 16000, 800, 400) == (39, 40)
    assert mid_ratios(1.0 * 16000, 0.1 * 16000, 0.05 * 16000, 0.05 * 16000) == O.mid_ratios(16000.0, 1600.0, 800.0, 800.0)


def test_no_cpu_fallback():
    """The product path must refuse CPU tensors instead of computing on the host."""
    import torch
    import pyaudioanalysis_b200 as pkg
    with pytest.raises(TypeError):
        pkg.feature_extraction_batch(torch.zeros(2, 16000, dtype=torch.int16), 16000, 800, 400)
    src = "".join(open(os.path.join(ROOT, "pyaudioanalysis_b200", f)).read()
                  for f in os.listdir(os.path.join(ROOT, "pyaudioanalysis_b200")) if f.endswith(".py"))
    assert "oracle" not in src, "product code must never import the oracle"
