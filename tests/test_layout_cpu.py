"""CPU: Layout (csrc/entry.h), the rule every entry point's scratch is laid out by: regions in order from a starting
offset, each padded to a multiple of 256 bytes.  A region that took fewer bytes than it was given would let a kernel write
past its allocation; one that took more would change the scratch sizes the slicing and refusal rules are computed from.
Thumbnails' argmax parts when only the similarity matrix is asked for, and the forests' optional weights, are laid out as
zero-length regions and must take no bytes."""
import subprocess

import numpy as np
import pytest

from tests import host_exe


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return host_exe.build(tmp_path_factory, "layout_host.cu")


def layout(exe, at, sizes):
    res = subprocess.run([exe, str(at)] + [str(s) for s in sizes], capture_output=True, text=True)
    assert res.returncode == 0, res
    offsets, total = res.stdout.split("\n")[:2]
    return [int(v) for v in offsets.split()], int(total)


def padded(b):
    return (b + 255) // 256 * 256


def check(exe, at, sizes):
    offsets, total = layout(exe, at, sizes)
    assert len(offsets) == len(sizes)
    assert total == at + sum(padded(s) for s in sizes), (at, sizes, total)
    ends = [o + s for o, s in zip(offsets, sizes)]
    for i, (o, s) in enumerate(zip(offsets, sizes)):
        assert o % 256 == 0, (at, sizes, offsets)
        assert o == (at if i == 0 else offsets[i - 1] + padded(sizes[i - 1])), (at, sizes, offsets)
        assert i == 0 or o >= ends[i - 1], (at, sizes, offsets)            # no overlap with the region before
        assert o + s <= total, (at, sizes, offsets, total)
    return offsets, total


@pytest.mark.parametrize("sizes", [[1], [255, 256, 257], [4, 8, 4096, 3, 1 << 20], [16, 1, 1, 1],
                                   [32 * 4, 2 * 8, 256 * 1000 + 1]], ids=["one", "edges", "mixed", "small", "large"])
def test_offsets_ascend_padded_and_disjoint(exe, sizes):
    check(exe, 0, sizes)


@pytest.mark.parametrize("at", [0, 256, 512, 1 << 20])
def test_starting_offset_is_honoured(exe, at):
    offsets, total = check(exe, at, [100, 300, 8])
    assert offsets == [at, at + 256, at + 768] and total == at + 1024


def test_zero_length_region_takes_no_bytes(exe):
    assert check(exe, 0, [0, 0, 0]) == ([0, 0, 0], 0)
    assert check(exe, 512, [0]) == ([512], 512)
    offsets, total = check(exe, 0, [8, 0, 8, 0])
    assert offsets == [0, 256, 256, 512] and total == 512
    # the same layout with and without the zero-length regions ends at the same byte
    assert check(exe, 256, [40, 0, 1000, 0, 0, 7])[1] == check(exe, 256, [40, 1000, 7])[1]


def test_random_layouts(exe):
    rng = np.random.default_rng(13)
    for _ in range(50):
        n = int(rng.integers(1, 12))
        sizes = [int(v) if rng.random() > 0.2 else 0 for v in rng.integers(1, 1 << 22, n)]
        check(exe, 256 * int(rng.integers(0, 64)), sizes)
