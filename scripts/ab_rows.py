import sys, os, json, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pyaudioanalysis_b200 as pkg
from pyaudioanalysis_b200.batch import clip_stats
g = torch.Generator(device="cuda"); g.manual_seed(3)
c3 = torch.empty((64, 2646000), dtype=torch.int16, device="cuda")
for i in range(0, 64, 8):
    c3[i:i+8] = (3000.0 * torch.randn((8, 2646000), generator=g, device="cuda")).round().clamp(-32768, 32767).to(torch.int16)
n3 = clip_stats(c3); o = torch.empty((64, 5999, 441), device="cuda")
def t(fn, reps=10):
    for _ in range(3): fn()
    torch.cuda.synchronize(); e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps): fn()
    e1.record(); torch.cuda.synchronize(); return e0.elapsed_time(e1) / reps
print(json.dumps({"lib": os.environ.get("B200AA_LIB", "default"), "spectrogram_ms": t(lambda: pkg.spectrogram_batch(c3, 44100, 882, 441, norm=n3, out=o)), "chromagram_ms": t(lambda: pkg.chromagram_batch(c3, 44100, 882, 441, norm=n3))}))
