"""CPU: the work-slot ring of a plan (csrc/slots.h) with fake events that remember which launch recorded them.

A slot is in flight from a launch's acquire until its done.  No slot in flight is handed out again, and every reuse of
a slot makes the new launch's stream wait on the record of the launch that used the slot last.  Under the rule the ring
had before (the next slot round-robin, whatever holds it) scenario (b) fails: the 65th acquisition after the held launch
gets its slot again and waits on the record of the launch before it.

(a) one thread, 1 000 launches round-robin over 4 streams;
(b) one launch held between acquire and done while 200 others acquire and finish: none of them gets its slot;
(c) 64 launches held: a 65th, from another thread, blocks until one of them is done, then gets that slot;
(d) 8 threads with seeded random hold times (some of a millisecond, as a descheduled thread would hold its slot).
"""
import json
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    path = str(tmp_path_factory.mktemp("slots") / "slots_host")
    res = subprocess.run(["g++", "-O2", "-std=c++17", "-pthread", "-o", path, os.path.join(ROOT, "tests", "slots_host.cpp")],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    return path


def run(exe, scenario):
    out = subprocess.run([exe, scenario], capture_output=True, text=True, timeout=120)
    r = json.loads(out.stdout)
    assert out.returncode == 0 and r["shared"] == 0 and r["bad_wait"] == 0, r
    return r


def test_round_robin_one_thread(exe):
    r = run(exe, "a")
    assert r["launches"] == 1000 and r["reuses"] == 1000 - 64 and r["wraps"] == 1000 // 64, r


def test_held_slot_is_not_handed_out(exe):
    r = run(exe, "b")
    assert r["launches"] == 1 + 200 + 64, r
    assert r["held_slot_given"] == 0 and r["held_slot_reused_after"] == 1, r


def test_full_ring_blocks_until_done(exe):
    r = run(exe, "c")
    assert r["blocked"] and r["got_freed_slot"], r


def test_threads_with_random_holds(exe):
    r = run(exe, "d")
    assert r["launches"] == 8 * 3000 and r["wraps"] > 100, r
