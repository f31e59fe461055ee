"""Compile-time variants of libb200aa.so for A/B runs on the GPU (the default library is untouched):

    python scripts/build_variants.py p2x8       # one
    python scripts/build_variants.py            # all
    python scripts/ab_run.py default p2x8       # on the GPU

Variants land in pyaudioanalysis_b200/variants/libb200aa_<name>.so and are selected per process with B200AA_LIB.
"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pyaudioanalysis_b200 import build as B   # noqa: E402

VARIANTS = {
    # pair kernel: CTAs per SM x warps per CTA (default 1 x 24, the 800-sample window gets 20 by its shared memory)
    "p2x8": ["-DB200AA_PAIR_MINBLOCKS=2", "-DB200AA_PAIR_MAXWARPS=8"],
    "p1x20": ["-DB200AA_PAIR_MAXWARPS=20"],
    "p1x16": ["-DB200AA_PAIR_MAXWARPS=16"],
    # solo kernel, feature layout (default 1 x 24)
    "s2x8": ["-DB200AA_SOLO_MINBLOCKS=2", "-DB200AA_SOLO_MAXWARPS=8"],
    "s1x20": ["-DB200AA_SOLO_MAXWARPS=20"],
    "s1x16": ["-DB200AA_SOLO_MAXWARPS=16"],
    # CTA kernel at 64 registers / 4 CTAs per SM
    "mb4": ["-DB200AA_FAST_MINBLOCKS=4"],
    # reference point for bisecting: IEEE MUFU wrappers
    "noftz": ["-DB200AA_NO_FTZ_MUFU"],
}


def build(name, verbose=False):
    out_dir = os.path.join(B.HERE, "variants")
    os.makedirs(out_dir, exist_ok=True)
    out = os.path.join(out_dir, "libb200aa_%s.so" % name)
    flags = [f for f in B.NVCC_FLAGS if not f.startswith("--use_fast_math")]
    cmd = [B._nvcc()] + flags + VARIANTS[name] + (["-Xptxas", "-v"] if verbose else []) + \
          ["-o", out] + [os.path.join(B.CSRC, s) for s in B.SOURCES]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError("nvcc failed building variant " + name)
    if verbose:
        sys.stderr.write(res.stderr)
    return out


if __name__ == "__main__":
    names = [a for a in sys.argv[1:] if not a.startswith("-")] or list(VARIANTS)
    for n in names:
        print(build(n, verbose="-v" in sys.argv))
