"""A small fake VCTK-Corpus tree and the host restatements the VCTK preprocessing tests compare against."""
import os

import numpy as np
from scipy.io import wavfile

SR_IN = 48000

# speaker -> [(stem, seconds, label (start, end) in seconds or None, wav format)]; p226_003 has no wav, p315 no txt,
# p301_002's label cut lies past the end of its audio (an empty segment: no row, its index is not reused)
LAYOUT = {
    "225": [("p225_001", 1.2, (0.25, 0.95), "int16"), ("p225_002", 0.9, None, "int16"),
            ("p225_003", 1.4, (0.30, 1.10), "int16")],
    "226": [("p226_001", 1.0, None, "float32"), ("p226_002", 0.8, None, "native"), ("p226_003", 1.0, None, None)],
    "301": [("p301_001", 1.1, None, "int16"), ("p301_002", 0.7, (2.0, 2.5), "int16"),
            ("p301_003", 1.3, (0.20, 1.00), "int16"), ("p301_004", 0.6, None, "int16")],
}
TEXTS = {"p225_001": "Please call Stella.", "p226_002": "Ça va, Zoë? naïve café.", "p301_004": "Ask her to bring these."}


def clip(seed, seconds, sr=SR_IN):
    """Silent head and tail (quiet noise), a voiced middle: decaying harmonics plus noise."""
    rng = np.random.RandomState(seed)
    n = int(seconds * sr)
    t = np.arange(n) / sr
    x = 1e-4 * rng.randn(n)
    a, b = int(0.2 * n), int(0.75 * n)
    f0 = 110 + 20 * (seed % 7)
    mid = sum(np.sin(2 * np.pi * k * f0 * t[a:b]) / k for k in range(1, 6))
    x[a:b] += 0.3 * mid * np.exp(-np.linspace(0, 2, b - a)) + 0.02 * rng.randn(b - a)
    return x


def write_tree(root, seed=0):
    """-> the (stem, speaker index) pairs that have a wav, in the reference's order."""
    pairs = []
    for si, (spk, utts) in enumerate(sorted(LAYOUT.items(), key=lambda kv: int(kv[0]))):
        for d in ("txt", "wav48", "lab"):
            os.makedirs(os.path.join(root, d, "p" + spk), exist_ok=True)
        for ui, (stem, seconds, lab, fmt) in enumerate(utts):
            text = TEXTS.get(stem, "Utterance %s of speaker %s." % (stem[-3:], spk))
            with open(os.path.join(root, "txt", "p" + spk, stem + ".txt"), "wb") as f:
                f.write((text + "\n").encode("utf-8"))
            if fmt is None:
                continue
            sr = 22050 if fmt == "native" else SR_IN
            x = clip(seed + 10 * si + ui, seconds, sr)
            path = os.path.join(root, "wav48", "p" + spk, stem + ".wav")
            wavfile.write(path, sr, x.astype(np.float32) if fmt == "float32" else (x * 32767).astype(np.int16))
            if lab is not None:
                b, e = (int(round(v * 1e7)) for v in lab)
                with open(os.path.join(root, "lab", "p" + spk, stem + ".lab"), "w") as f:
                    f.write("0 %d pau\n%d %d h\n%d %d iy\n%d %d pau\n" % (b, b, (b + e) // 2, (b + e) // 2, e, e,
                                                                         e + 2000000))
            pairs.append((stem, si))
    os.makedirs(os.path.join(root, "wav48", "p315"), exist_ok=True)          # VCTK 0.80: p315 has no transcripts
    wavfile.write(os.path.join(root, "wav48", "p315", "p315_001.wav"), SR_IN, (clip(99, 0.5) * 32767).astype(np.int16))
    return pairs


def trim_margin(y, top_db):
    """Smallest distance in dB of any frame of ``audio.trim_bounds_reference`` from its threshold."""
    y = np.asarray(y, dtype=np.float64)
    L = len(y)
    padded = np.pad(y, 1024, mode="reflect")
    mse = np.array([np.mean(padded[512 * f: 512 * f + 2048] ** 2) for f in range(L // 512 + 1)])
    db = 10 * np.log10(np.maximum(1e-10, mse)) - 10 * np.log10(np.maximum(1e-10, mse.max()))
    return float(np.abs(db + top_db).min())


def cut_segment(x, cut):
    """x[b:e] of vctk.py:65 -> (offset, length, top_db)."""
    n = len(x)
    if cut is None:
        return 0, n, 15
    b, e = min(cut[0], n), min(max(cut[1], 0), n)
    return b, max(0, e - b), 25
