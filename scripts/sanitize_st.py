"""Small driver for compute-sanitizer: every kernel family once on tiny inputs (pair / CTA / generic feature kernels incl.
the large-window form, rows, mid-term pooling, the WAV decode, the chunked host pipeline)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import pyaudioanalysis_b200 as pkg
from oracle import st_oracle as O

pkg.ShortTermFeatures.PRINT_SPECTROGRAM_SHAPE = False
clips = torch.from_numpy(np.stack([O.synth_clip(i, 24000, 16000) for i in range(6)])).cuda()
from pyaudioanalysis_b200._lib import Plan
out = pkg.feature_extraction_batch(clips, 16000, 800, 400)                       # pair kernel, shared halves
for w, s_ in ((800, 200), (800, 800), (800, 333), (1024, 512), (512, 128), (960, 480), (640, 320), (480, 240), (320, 160)):
    pkg.feature_extraction_batch(clips, 16000, w, s_)                             # pair kernel: independent frames, other shapes
pkg.feature_extraction_batch(clips.float() * 0.5, 16000, 800, 400)               # float input
pkg.feature_extraction_batch(clips[:, :1200], 16000, 800, 400)                   # two frames: a single pair
pkg.feature_extraction_batch(clips[:, :1199], 16000, 800, 400)                   # one frame: odd tail
pc = Plan(16000, 800, 400).prefer_kernel(1)
pkg.feature_extraction_batch(clips, 16000, 800, 400, plan=pc)                    # CTA kernel, RUNS + TMA
lens = torch.tensor([24000, 800, 12345, 23999, 20000, 4000], dtype=torch.int64, device="cuda")
pkg.feature_extraction_batch(clips, 16000, 800, 400, lengths=lens)               # ragged (pair kernel)
pkg.feature_extraction_batch(clips, 16000, 800, 400, lengths=lens, plan=pc)      # ragged (CTA kernel)
pkg.feature_extraction_batch(clips[:, 3:23003].contiguous(), 16000, 800, 400)    # same kernel, other lengths
pkg.feature_extraction_batch(clips, 16000, 800, 200)                              # 75 % overlap: no Zs aliasing
pkg.feature_extraction_batch(clips, 16000, 800, 800)                              # no overlap
c44 = torch.from_numpy(np.stack([O.synth_clip(9 + i, 30000, 44100) for i in range(3)])).cuda()
pkg.feature_extraction_batch(c44, 44100, 882, 441)                                # R = 21, odd hop
pkg.feature_extraction_batch(clips, 16000, 640, 160)                              # 20x16 (Cooley-Tukey 16-point codelet)
pkg.feature_extraction_batch(clips, 16000, 320, 160)                              # 16x10
pkg.feature_extraction_batch(clips, 16000, 2048, 1024)                            # generic kernel
pkg.feature_extraction_batch(clips, 16000, 22050, 1950)                           # generic kernel, large-window (global scratch) form
pkg.feature_extraction_batch(clips, 16000, 400, 160)                              # 20x10 rectangular, run staging
pkg.feature_extraction_batch(clips, 16000, 480, 240)                              # 20x12
pkg.feature_extraction_batch(clips, 16000, 600, 150)                              # 20x15, no runs
pkg.spectrogram_batch(clips, 16000, 400, 160)
pkg.spectrogram_batch(clips, 16000, 800, 400)
pkg.chromagram_batch(clips, 16000, 800, 400)
pkg.spectrogram_batch(c44, 44100, 882, 441)
pkg.mid_feature_extraction_batch(clips, 16000, 8000, 4000, 800, 400)
x = clips[0].cpu().numpy()
pkg.ShortTermFeatures.chromagram(x[:16300], 16000, 800, 400)                      # clipped last frame (generic launch)
from pyaudioanalysis_b200.hostpipe import HostPipeline
# steal-half scheduler with more pair steps than warps and stealing forced by tiny claims (B200AA_PAIR_STEAL=1,2 in the
# environment makes every warp's range change hands): 40 clips x 10 s
if os.environ.get("B200AA_SANITIZE_STEAL"):
    big = torch.from_numpy(np.stack([O.synth_clip(40 + i, 160000, 16000) for i in range(40)])).cuda()
    lens_b = torch.randint(800, 160001, (40,), dtype=torch.int64, device="cuda")
    pkg.feature_extraction_batch(big, 16000, 800, 400, lengths=lens_b)
    pkg.feature_extraction_batch(big[:, :132300].contiguous(), 44100, 882, 441)
from pyaudioanalysis_b200.consumers import normalize_windows_batch
normalize_windows_batch(torch.randn(2, 136, 9, device="cuda"), np.zeros(136), np.ones(136))      # consumers: normalise + transpose
import tempfile
from tests import wavgen
with tempfile.TemporaryDirectory() as d:                                         # WAV decode: all 12 flavours, one launch
    paths = []
    for k, (name, ch) in enumerate(wavgen.FLAVOURS):
        paths.append(os.path.join(d, "%02d.wav" % k))
        wavgen.write(paths[-1], 16000, wavgen.signal(name, ch, 1000 + 3 * k, k), name)
    pkg.audioio.stage([pkg.MidTermFeatures._open_clip(p) for p in paths])
hp = HostPipeline(16000, 800, 400, 24000, max_clips=6, device=0, bind_numa=False)
hp.h_in[:] = clips.cpu().numpy()
hp.run()
torch.cuda.synchronize()
print("sanitize driver done", tuple(out.shape))
