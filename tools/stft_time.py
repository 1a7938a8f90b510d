"""Times the fused STFT->linear+mel kernel alone (device-resident, CUDA events) on BASELINE config #5's clip shape and
prints algorithmic GB/s against the measured HBM peak."""
import json, os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deepvoice3_pytorch_b200 import audio

nb, n = 256, 220500
wav = (0.1 * torch.randn(nb, n, device="cuda")).clamp_(-1, 1)
frames = audio.num_frames(n)
for _ in range(3):
    audio.stft_mel_batch(wav)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
iters = 20
e0.record()
for _ in range(iters):
    lin, mel = audio.stft_mel_batch(wav)
e1.record(); torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / iters
b = 4.0 * nb * (n + frames * 513 + frames * 80)
pk = json.load(open(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json"))) if os.path.exists(
    os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")) else {}
print("stft_mel: %.3f ms / %d clips  -> %.0f clips/s, %.1f GB/s algorithmic, %.0f clk/frame/SM" % (
    ms, nb, nb / ms * 1e3, b / ms / 1e6, ms * 1e-3 * 1.98e9 * 132 / (nb * frames)))
