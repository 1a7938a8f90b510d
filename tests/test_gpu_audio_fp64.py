"""GPU: every audio kernel elementwise against the fp64 oracles, within the derived bounds of tests/audio_bounds.py
(its header has the error model).  For each output tensor the largest error-to-bound ratio must be <= 1; run with -s to
see them.  Output buffers are filled with NaN first, so every element must be written; every clip row is filled past
its length with loud garbage, so a kernel that reads a sample at or past ``len`` fails.

Entry points: dv3_stft_mel, dv3_stft_mel_targets with dv3_peak_abs_batched, dv3_stft_mel_geom (the nine frames of
test_gpu_stft_geometry.py and 1024 / 256 called directly), dv3_stft_complex_geom with and without the magnitude
projection and dv3_istft_geom (the same frames), dv3_spec_to_amp, dv3_deemphasis."""
import ctypes

import numpy as np
import pytest
import torch

import audio_bounds as AB
from oracle import audio_oracle as A
from test_gpu_stft_geometry import GEOMS, IDS, frame

pytestmark = pytest.mark.gpu

KINDS = ("noise", "tone", "dc", "nyquist", "impulse", "silent_middle", "quiet", "full")


def _vp(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _nan(*shape):
    return torch.full(shape, float("nan"), device="cuda")


def _signal(kind, n, N, rng):
    t = np.arange(n)
    if kind == "noise":
        x = 0.3 * rng.randn(n)
    elif kind == "tone":                                   # on the centre of bin N/16 + 3
        x = 0.5 * np.cos(2 * np.pi * (N // 16 + 3) * t / N + 0.3)
    elif kind == "dc":
        x = np.full(n, 0.4)
    elif kind == "nyquist":
        x = 0.4 * (-1.0) ** t
    elif kind == "impulse":
        x = np.zeros(n); x[n // 3] = 0.8
    elif kind == "silent_middle":                          # the -100 dB floor in the middle of the clip
        x = 0.3 * rng.randn(n) * ((t < n // 4) | (t > 3 * n // 4))
    elif kind == "quiet":                                  # peak ~1e-4: a large rescale
        x = 1e-4 * np.tanh(rng.randn(n)) + 2e-5 * np.cos(2 * np.pi * 5 * t / N)
    else:                                                  # full scale
        x = np.sign(rng.randn(n)) * (1.0 - 2.0 ** -15)
    return np.clip(x, -1.0, 1.0 - 2.0 ** -15)


def _batch(lens, N, pitch, int16, seed=0):
    """(B, pitch) rows: clip c of lens[c] samples of kind KINDS[c % 8], then loud garbage to the end of the row."""
    rng = np.random.RandomState(seed)
    if int16:
        wav = rng.choice(np.array([-32768, 32767], np.int16), size=(len(lens), pitch))
    else:
        wav = rng.uniform(-0.9, 0.9, size=(len(lens), pitch)).astype(np.float32)
    for c, n in enumerate(lens):
        x = _signal(KINDS[c % len(KINDS)], n, N, rng)
        wav[c, :n] = np.round(x * 32768).astype(np.int16) if int16 else x.astype(np.float32)
    return wav


def _n_for_frames(F, N, R):
    n = (F - 1) * R - (N - 2 * R)
    assert n >= 1 and A.num_frames(n, N, R) == F
    return n


class Worst(dict):
    def add(self, key, r):
        self[key] = max(self.get(key, 0.0), r)

    def report(self, title):
        print("\n%s: largest error / bound" % title)
        for k in sorted(self):
            print("  %-44s %.3g" % (k, self[k]))
        bad = {k: v for k, v in self.items() if not v <= 1.0}
        assert not bad, bad


def _check_forward(worst, tag, kernel, lin, mel, wav, lens, int16, gain, N, R, basis, start, length, lead=0, ds=1,
                   peak=None):
    """lin (B, T_lin, K), mel (B, T_mel, n_mels) numpy outputs in the (lead, ds) layout."""
    Bm = basis.cpu().numpy()
    st, ln = start.cpu().numpy(), length.cpu().numpy()
    for c, n in enumerate(lens):
        x, pk = AB.kernel_samples(wav[c], n, int16, gain)
        if peak is not None:
            assert peak[c] == pk, (c, peak[c], pk)                        # peak_abs: exact
        fw = AB.Forward(x, N, R, kernel)
        nf = fw.T
        rows = lead + np.arange(nf)
        ref, lo, hi = AB.linear_db(fw)
        worst.add("%s linear" % tag, AB.interval_ratio(lin[c, rows], ref, lo, hi))
        keep = np.ones(lin.shape[1], bool); keep[rows] = False
        assert not np.isnan(lin[c]).any() and not lin[c, keep].any(), (tag, c)
        mref, mlo, mhi = AB.mel_db(fw, Bm, st, ln)
        sel = rows % ds == 0
        worst.add("%s mel" % tag, AB.interval_ratio(mel[c, rows[sel] // ds], mref[sel], mlo[sel], mhi[sel]))
        mkeep = np.ones(mel.shape[1], bool); mkeep[rows[sel] // ds] = False
        assert not np.isnan(mel[c]).any() and not mel[c, mkeep].any(), (tag, c)
        assert mel.shape[1] == -(-lin.shape[1] // ds)


LENS_1024 = [1, 255, 256, 257, 768, 1024, 1025] + [_n_for_frames(F, 1024, 256) for F in (63, 64, 65, 128, 129)]


def test_stft_mel_1024_every_staging_path_and_dense_filterbank():
    """dv3_stft_mel (fp32, lead 0, ds 1): row pitch a multiple of 4 samples (bulk and 16-byte staging) and odd (4-byte
    staging); the presets' packed filterbank and a dense 24 x 513 one (the plain loop)."""
    from deepvoice3_pytorch_b200 import audio
    from deepvoice3_pytorch_b200._lib import lib
    worst = Worst()
    basis, start, length = audio._device_basis(torch.device("cuda"))
    rng = np.random.RandomState(7)
    dense = torch.from_numpy((rng.rand(24, 513).astype(np.float32) + 0.1) / 513.0).cuda()
    dstart, dlen = torch.zeros(24, dtype=torch.int32).cuda(), torch.full((24,), 513, dtype=torch.int32).cuda()
    for pitch in (max(LENS_1024) + 4 * 64, max(LENS_1024) + 4 * 64 + 1):
        wav = _batch(LENS_1024, 1024, pitch, False, seed=pitch)
        wd, ld = torch.from_numpy(wav).cuda(), torch.tensor(LENS_1024, dtype=torch.int32).cuda()
        T = audio.num_frames(pitch)
        for name, (bs, s, l) in (("packed", (basis, start, length)), ("dense", (dense, dstart, dlen))):
            lin, mel = _nan(len(LENS_1024), T, 513), _nan(len(LENS_1024), T, bs.shape[0])
            lib.call("dv3_stft_mel", _vp(wd), _vp(ld), _vp(bs), _vp(s), _vp(l), _vp(lin), _vp(mel), len(LENS_1024),
                     pitch, T, bs.shape[0], 0.97, -100.0, 20.0, _st())
            _check_forward(worst, "stft_mel pitch%%4=%d %s" % (pitch % 4, name), "stft1024", lin.cpu().numpy(),
                           mel.cpu().numpy(), wav, LENS_1024, False, None, 1024, 256, bs, s, l)
    worst.report("dv3_stft_mel 1024/256")


def _targets(lib, kernel, wav, lens, int16, rescale, T_lin, r, ds, N, R, basis, start, length, tab=None):
    B, pitch = wav.shape
    wd = torch.from_numpy(wav).cuda()
    ld = torch.tensor(lens, dtype=torch.int32).cuda()
    peak = None
    if rescale:
        peak = _nan(B)
        lib.call("dv3_peak_abs_batched", _vp(wd), int(int16), _vp(ld), pitch, B, _vp(peak), _st())
    K = N // 2 + 1
    lin, mel = _nan(B, T_lin, K), _nan(B, -(-T_lin // ds), basis.shape[0])
    if kernel == "stft1024":
        lib.call("dv3_stft_mel_targets", _vp(wd), int(int16), _vp(ld), _vp(peak), 0.999, _vp(basis), _vp(start),
                 _vp(length), _vp(lin), _vp(mel), B, pitch, T_lin, r, ds, basis.shape[0], 0.97, -100.0, 20.0, _st())
    else:
        lib.call("dv3_stft_mel_geom", _vp(wd), int(int16), _vp(ld), _vp(peak), 0.999, _vp(tab), _vp(basis),
                 _vp(start), _vp(length), _vp(lin), _vp(mel), B, pitch, T_lin, r, ds, basis.shape[0], N, R, 0.97,
                 -100.0, 20.0, _st())
    return lin.cpu().numpy(), mel.cpu().numpy(), None if peak is None else peak.cpu().numpy()


LAYOUTS = [(1, 1), (1, 4), (2, 2), (3, 3), (4, 8)]


@pytest.mark.parametrize("kernel", ["stft1024", "any"])
def test_targets_1024_int16_fp32_rescaling_and_layouts(kernel):
    """dv3_stft_mel_targets and dv3_stft_mel_geom at 1024 / 256: int16 and fp32 rows (pitch a multiple of 8 samples
    and odd), rescaling off and on, every (r, ds) layout."""
    from deepvoice3_pytorch_b200 import audio
    from deepvoice3_pytorch_b200._lib import lib
    worst = Worst()
    dev = torch.device("cuda")
    basis, start, length = audio._device_basis(dev)
    tab = audio._geometry_table(dev, 1024, 256)
    lens = [1, 257, 1025, 5000, 15616, 2000, 3000, 4000]
    T = max(A.num_frames(n) for n in lens)
    for i, (r, ds) in enumerate(LAYOUTS):
        for int16 in (True, False):
            for rescale in (False, True):
                pitch = max(lens) + (8 * 40 if (i + rescale) % 2 else 8 * 40 + 3)
                wav = _batch(lens, 1024, pitch, int16, seed=i)
                T_lin = r + T + ds
                lin, mel, peak = _targets(lib, kernel, wav, lens, int16, rescale, T_lin, r, ds, 1024, 256, basis,
                                          start, length, tab)
                _check_forward(worst, "%s %s%s" % (kernel, "int16" if int16 else "fp32", " rescaled" * rescale),
                               kernel, lin, mel, wav, lens, int16, 0.999 if rescale else None, 1024, 256, basis,
                               start, length, lead=r, ds=ds, peak=peak)
    worst.report("targets at 1024/256, %s" % kernel)


@pytest.mark.parametrize("sr,N,R", GEOMS, ids=IDS)
def test_stft_mel_geom(sr, N, R):
    """dv3_stft_mel_geom: lengths around one hop and one frame and around the frames one CTA stages; fp32 in the
    identity layout, then int16 rescaled in the (3, 3) layout."""
    from deepvoice3_pytorch_b200 import audio
    from deepvoice3_pytorch_b200._lib import lib
    worst = Worst()
    span = 2 * N if N > 2048 else 4096
    F = max(1, min(32, (span - N) // R + 1))                  # stft_any.cu any_frames_per_cta
    lens = [1, R - 1, R, R + 1, N - R, N, N + 1]
    lens += [n for n in ((f - 1) * R - (N - 2 * R) for f in (F - 1, F, F + 1, 2 * F + 1)) if n >= 1]
    with frame(sr, N, R):
        dev = torch.device("cuda")
        basis, start, length = audio._device_basis(dev)
        tab = audio._geometry_table(dev, N, R)
        T = max(A.num_frames(n, N, R) for n in lens)
        for int16, rescale, (r, ds) in ((False, False, (0, 1)), (True, True, (3, 3))):
            wav = _batch(lens, N, max(lens) + 8 * 16, int16, seed=N)
            lin, mel, peak = _targets(lib, "any", wav, lens, int16, rescale, r + T, r, ds, N, R, basis, start,
                                      length, tab)
            _check_forward(worst, "%d/%d %s" % (N, R, "int16 rescaled" if rescale else "fp32"), "any", lin, mel, wav,
                           lens, int16, 0.999 if rescale else None, N, R, basis, start, length, lead=r, ds=ds,
                           peak=peak)
    worst.report("dv3_stft_mel_geom %d/%d" % (N, R))


def _complex(t):
    a = t.cpu().numpy().astype(np.float64)
    return a[..., 0] + 1j * a[..., 1]


def _griffin_lim_step(worst, lib, N, R):
    """stft_complex (plain and projected) and istft on a ragged batch, each against the fp64 reference of its own
    input; the istft also on spectra with non-zero imaginary parts at bins 0 and N/2.  Clip 2 has a silent stretch
    longer than two frames: there X_hat == 0 and the projection must give exactly (mag, 0)."""
    from deepvoice3_pytorch_b200 import audio
    kernel = "any"
    K = N // 2 + 1
    frames = [3 * (N // R), 9, 40]
    ns = [(T - 1) * R - (N - 2 * R) for T in frames]
    pitch = max(ns) + 37
    rng = np.random.RandomState(N)
    wav = rng.uniform(-0.9, 0.9, size=(3, pitch)).astype(np.float32)
    for c, n in enumerate(ns):
        wav[c, :n] = _signal(KINDS[c], n, N, rng) + 0.1 * _signal("tone", n, N, rng)
    wav[2, ns[2] // 3:min(ns[2], ns[2] // 3 + 3 * N)] = 0.0
    wd = torch.from_numpy(wav).cuda()
    nd, fd = torch.tensor(ns, dtype=torch.int32).cuda(), torch.tensor(frames, dtype=torch.int32).cuda()
    Tm = max(frames)
    tab = audio._geometry_table(wd.device, N, R)
    refs = [AB.Forward(wav[c, :ns[c]], N, R, kernel, preemph=None, T=frames[c]) for c in range(3)]
    mags = np.zeros((3, Tm, K), np.float32)
    for c in range(3):
        mags[c, :frames[c]] = (np.abs(refs[c].X) * rng.uniform(0.5, 1.5, refs[c].X.shape)).astype(np.float32)
    mags[1, frames[1] // 2, 7] = 0.0
    silent = [(c, f) for c in range(3) for f in range(frames[c]) if not refs[c].X[f].any()]
    assert len(silent) >= 2 and all(c == 2 for c, _ in silent), silent
    for c, f in silent:
        mags[c, f] = rng.uniform(0.1, 1.0, K)
    md = torch.from_numpy(mags).cuda()
    for mag in (None, md):
        what = "projected" if mag is not None else "plain"
        spec = _nan(3, Tm, K, 2)
        lib.call("dv3_stft_complex_geom", _vp(wd), _vp(nd), pitch, _vp(mag), _vp(spec), _vp(fd), Tm, 3, _vp(tab),
                 N, R, _st())
        got = _complex(spec)
        for c in range(3):
            g = got[c, :frames[c]]
            if mag is None:
                worst.add("stft_complex %s" % kernel, AB.complex_ratio(g, refs[c]))
            else:
                worst.add("stft_complex projected %s" % kernel, AB.projection_ratio(g, refs[c], mags[c, :frames[c]]))
        for c, f in silent:                                      # X_hat == 0: phase 0, or exactly 0 unprojected
            assert np.array_equal(got[c, f], mags[c, f] + 0j if mag is not None else np.zeros(K)), (c, f)
        # the inverse of what the forward kernel wrote, and of a random spectrum with Im X_0, Im X_{N/2} != 0
        rnd = 0.5 * (rng.randn(3, Tm, K) + 1j * rng.randn(3, Tm, K))
        for src_name, src in (("of stft_complex " + what, np.nan_to_num(got)), ("random spectrum", rnd)):
            sd = torch.from_numpy(np.stack([src.real, src.imag], -1).astype(np.float32)).cuda()
            src = _complex(sd)
            y = torch.zeros(3, pitch, device="cuda")
            y[:, -1] = 7.0                                   # past every clip's samples: must stay untouched
            lib.call("dv3_istft_geom", _vp(sd), _vp(y), _vp(nd), pitch, _vp(fd), Tm, 3, _vp(tab), N, R, _st())
            yy = y.cpu().numpy()
            for c in range(3):
                ref, bound = AB.istft(src[c, :frames[c]], N, R, ns[c], kernel)
                worst.add("istft %s %s" % (kernel, src_name), AB.abs_ratio(yy[c, :ns[c]], ref, bound))
                assert not yy[c, ns[c]:-1].any() and yy[c, -1] == 7.0


def test_griffin_lim_step_1024():
    from deepvoice3_pytorch_b200._lib import lib
    worst = Worst()
    _griffin_lim_step(worst, lib, 1024, 256)
    worst.report("Griffin-Lim step 1024/256")


@pytest.mark.parametrize("sr,N,R", GEOMS, ids=IDS)
def test_griffin_lim_step_geom(sr, N, R):
    from deepvoice3_pytorch_b200._lib import lib
    worst = Worst()
    _griffin_lim_step(worst, lib, N, R)
    worst.report("Griffin-Lim step %d/%d" % (N, R))


def test_spec_to_amp_and_deemphasis():
    from deepvoice3_pytorch_b200._lib import lib
    worst = Worst()
    rng = np.random.RandomState(3)
    s = np.concatenate([rng.uniform(-0.1, 1.1, 20000), np.linspace(0, 1, 4097), [0.0, 1.0, 0.5]]).astype(np.float32)
    sd = torch.from_numpy(s).cuda()
    for power in (1.0, 1.4, 1.5):
        amp = _nan(s.size)
        lib.call("dv3_spec_to_amp", _vp(sd), _vp(amp), s.size, -100.0, 20.0, power, _st())
        ref, bound = AB.spec_to_amp(s, power=power)
        worst.add("spec_to_amp power %g" % power, AB.abs_ratio(amp.cpu().numpy(), ref, bound))
    n = 5000
    x = np.stack([0.5 * rng.randn(n), 0.9 * np.sign(rng.randn(n)), np.full(n, 0.3)]).astype(np.float32)
    xd = torch.from_numpy(x).cuda()
    y = _nan(3, n)
    lib.call("dv3_deemphasis", _vp(xd), _vp(y), 3, n, n, 0.97, _st())
    yy = y.cpu().numpy()
    for c in range(3):
        ref, bound = AB.deemphasis(x[c])
        worst.add("deemphasis", AB.abs_ratio(yy[c], ref, bound))
    worst.report("spec_to_amp, deemphasis")
